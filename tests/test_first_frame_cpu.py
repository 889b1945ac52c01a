"""CPU: the first-frame-conditioned motion models (use_first_frame_condition, use_first_frame_condition_concat).

  - the oracle reproduces the fixtures the unmodified reference wrote (tests/golden/make_golden_first_frame.py);
  - the host code of UNet3DConditionModel / AnimationPipeline, with every kernel launch replaced by tests/ops_emulator.py, reproduces them
    (mini UNet and 2-step pipeline, both modes, shared CFG prefix on and off, CUDA-graph bookkeeping and the eager loop);
  - every combination the reference cannot sample raises, naming both options.
Tolerances are the engine's own (tests/test_engine_gpu.py): fp32 rel-L2 <= 1e-4, bf16 rel-L2 <= 3e-2, video max-abs <= 2e-3 (fp32) /
PSNR >= 30 dB (bf16).
"""
import json
import os

import pytest
import torch

from tests import ops_emulator
from tests.cfgs_first_frame import PIPE_CASES, UNET_CASES

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
DTYPES = [(torch.float32, 1e-4), (torch.bfloat16, 3e-2)]


@pytest.fixture
def emulated(monkeypatch):
    ops_emulator.install(monkeypatch)
    torch.set_num_threads(8)


# ------------------------------------------------------------------------------------------------ oracle vs the reference's fixtures
@pytest.mark.parametrize("name", list(UNET_CASES))
def test_oracle_unet_reproduces_reference_fixture(name):
    from tests import oracle_first_frame
    from tests.cfgs_first_frame import ff_oracle_cfg, unet_case_inputs
    from tests.engine_helpers import golden, stats
    from tests.first_frame_helpers import make_ff_unet
    mode, fps, b, cfg = UNET_CASES[name]
    _, sd = make_ff_unet(mode, fps, device=None)
    inp = unet_case_inputs(name)
    kw = dict(use_first_frame_condition=True) if mode == "ff" else dict(use_first_frame_condition_concat=True,
                                                                         reference_images_latent=inp["first"])
    out = oracle_first_frame.unet3d_forward(sd, ff_oracle_cfg(mode, fps), inp["sample"], inp["timestep"], inp["ctx"], fps_tensor=inp.get("fps"),
                                  flow_control=inp.get("flow"), **kw)
    s = stats(out, torch.from_numpy(golden("first_frame_unet.npz")["out_" + name]))
    assert s["maxabs"] < 5e-5 and s["rel_l2"] < 2e-5, s


@pytest.mark.parametrize("name", list(PIPE_CASES))
def test_oracle_pipeline_reproduces_reference_fixture(name):
    from followyourclick_b200.synth import synth_clip_inputs
    from oracle import ref_vae
    from tests import oracle_first_frame
    from tests.cfgs import MINI_VAE, SCHED_V
    from tests.cfgs_first_frame import PIPE_F, PIPE_HW, PIPE_STEPS, ff_oracle_cfg, pipe_case_oracle_kwargs
    from tests.engine_helpers import golden, make_vae, stats
    from tests.first_frame_helpers import make_ff_unet
    mode, fps, gs, vs = PIPE_CASES[name]
    _, usd = make_ff_unet(mode, fps, device=None)
    _, vsd = make_vae(device=None)
    ci = synth_clip_inputs(1, PIPE_F, PIPE_HW, PIPE_HW)
    text = ci["text_embeddings"] if gs > 1.0 else ci["text_embeddings"][1:2]
    lat = oracle_first_frame.denoise(usd, ff_oracle_cfg(mode, fps), SCHED_V, ci["latents"], text,
                               PIPE_STEPS, gs, **pipe_case_oracle_kwargs(name, ci))
    g = golden("first_frame_pipeline.npz")
    assert stats(lat, torch.from_numpy(g["final_latents_" + name]))["maxabs"] < 1e-5
    video = ref_vae.decode_latents(vsd, MINI_VAE, lat)
    assert stats(video, torch.from_numpy(g["video_" + name]))["maxabs"] < 2e-3


def test_reference_refusals_are_recorded():
    pins = json.load(open(os.path.join(GOLD, "first_frame_pins.json")))
    assert set(pins["reference_refuses"]) == {"ff+fps (CFG)", "ff+camera (CFG)", "ff+mask_concat", "ffc+mask_concat", "ffc+video_scale"}


# ------------------------------------------------------------------------------------------------ host code under the kernel emulator
@pytest.mark.parametrize("name", list(UNET_CASES))
@pytest.mark.parametrize("dtype,tol", DTYPES)
def test_unet_host_logic_vs_reference_fixture(emulated, name, dtype, tol):
    from tests.first_frame_helpers import run_ff_unet_case
    s = run_ff_unet_case(name, dtype, device="cpu")
    assert s["finite"] and s["rel_l2"] < tol, s
    if UNET_CASES[name][3]:                  # CFG-shaped: the shared prefix computes the same thing
        s2 = run_ff_unet_case(name, dtype, device="cpu", share=True)
        assert s2["finite"] and s2["rel_l2"] < tol, s2


@pytest.mark.parametrize("name", ["ff", "ffc"])
def test_unet_public_forward_host_logic(emulated, name):
    from tests.first_frame_helpers import run_ff_unet_case
    s = run_ff_unet_case(name, torch.float32, device="cpu", via_forward=True)
    assert s["finite"] and s["rel_l2"] < 1e-4, s


@pytest.mark.parametrize("name", list(PIPE_CASES))
@pytest.mark.parametrize("graph,share", [(True, True), (False, False)])
def test_pipeline_host_logic_vs_reference_fixture(emulated, monkeypatch, name, graph, share):
    from followyourclick_b200.pipeline_animation import _GraphedUNetStep
    from tests.first_frame_helpers import run_ff_pipeline_case
    monkeypatch.setattr(_GraphedUNetStep, "capture", False)       # the graph branch's bookkeeping, replayed by re-running the forward
    r = run_ff_pipeline_case(name, torch.float32, device="cpu", graph=graph, share=share)
    assert r["finite"] and r["shape"] == (1, 3, 4, 64, 64) and r["video_maxabs"] < 2e-3 and r["latent_rel_l2"] < 1e-4, r
    r = run_ff_pipeline_case(name, torch.bfloat16, device="cpu", graph=graph, share=share)
    assert r["finite"] and r["psnr"] > 30.0, r


def test_first_frame_prologue_contract_emulated(emulated):
    """frame 0 of the caller's latents is replaced in place, the concat repeats the first-image latents on every frame"""
    from followyourclick_b200 import ops
    g = torch.Generator().manual_seed(3)
    lat, first = torch.randn(2, 4, 3, 2, 5, generator=g), torch.randn(2, 4, 2, 5, generator=g)
    keep = lat.clone()
    x = ops.build_unet_input_first(lat, first, 2, torch.float32, ops.FIRST_CONCAT | ops.FIRST_FRAME, c_pad=16)
    assert torch.equal(lat[:, :, 0], first) and torch.equal(lat[:, :, 1:], keep[:, :, 1:])
    assert torch.equal(x[:2, ..., :4], lat.permute(0, 2, 3, 4, 1)) and torch.equal(x[2:], x[:2])
    assert torch.equal(x[:2, ..., 4:8], first.permute(0, 2, 3, 1)[:, None].expand(2, 3, 2, 5, 4)) and not x[..., 8:].any()


# ------------------------------------------------------------------------------------------------ refused combinations
REFUSED = {
    "ff+fps (CFG)": (dict(use_first_frame_condition=True, use_fps_condition=True, unet_batch=2), ("use_first_frame_condition", "use_fps_condition")),
    "ff+camera (CFG)": (dict(use_first_frame_condition=True, use_camera_motion_condition=True, unet_batch=2),
                        ("use_first_frame_condition", "use_camera_motion_condition")),
    "ff+mask_concat": (dict(use_first_frame_condition=True, use_first_frame_mask_condition_concat=True),
                       ("use_first_frame_condition", "use_first_frame_mask_condition_concat")),
    "ffc+mask_concat": (dict(use_first_frame_condition_concat=True, use_first_frame_mask_condition_concat=True),
                        ("use_first_frame_condition_concat", "use_first_frame_mask_condition_concat")),
    "ffc+video_scale": (dict(use_first_frame_condition_concat=True, video_scale=0.7), ("use_first_frame_condition_concat", "video_scale")),
}


@pytest.mark.parametrize("case", list(REFUSED))
def test_refused_combination_raises_naming_both_options(case):
    from followyourclick_b200.pipeline_animation import check_first_frame_options
    kw, names = REFUSED[case]
    with pytest.raises(ValueError) as e:
        check_first_frame_options(first_image_latents=torch.zeros(1, 4, 8, 8), **kw)
    assert all(n in str(e.value) for n in names), str(e.value)


def test_sampled_combinations_pass_the_check():
    from followyourclick_b200.pipeline_animation import check_first_frame_options
    z = torch.zeros(1, 4, 8, 8)
    check_first_frame_options(use_first_frame_condition=True, first_image_latents=z, video_scale=0.7, unet_batch=2)
    check_first_frame_options(use_first_frame_condition=True, first_image_latents=z, use_fps_condition=True, use_camera_motion_condition=True,
                              unet_batch=1)
    check_first_frame_options(use_first_frame_condition_concat=True, first_image_latents=z, use_fps_condition=True,
                              use_camera_motion_condition=True, unet_batch=2)
    check_first_frame_options(use_first_frame_condition=True, use_first_frame_condition_concat=True, first_image_latents=z, unet_batch=2)
    with pytest.raises(ValueError, match="first_image_latents"):
        check_first_frame_options(use_first_frame_condition_concat=True)


def test_pipeline_call_refuses_before_sampling(emulated):
    """__call__ raises for a refused pair before any work (the engine UNet's own batch check is tested below)"""
    from tests.first_frame_helpers import make_ff_pipeline
    pipe, ci = make_ff_pipeline("ffc", torch.float32, device="cpu")
    with pytest.raises(ValueError, match="video_scale"):
        pipe("p", video_length=4, height=64, width=64, num_inference_steps=2, guidance_scale=8.0, latents=ci["latents"].clone(),
             use_first_frame_condition_concat=True, first_image_latents=ci["first_image_latents"], video_scale=0.7)
    assert pipe.text_encoder.calls == 0


def test_unet_refuses_first_frame_condition_with_fps_at_batch_2(emulated):
    from tests.first_frame_helpers import make_ff_unet
    unet, _ = make_ff_unet("ff", True, device="cpu")
    x = torch.zeros(2, 4, 4, 8, 8)
    with pytest.raises(ValueError, match="use_first_frame_condition.*use_fps_condition"):
        unet(x, 501, torch.zeros(2, 77, 768), use_first_frame_condition=True, use_fps_condition=True, fps_tensor=torch.tensor([2, 2]),
             flow_control=torch.tensor([4, 4]))
