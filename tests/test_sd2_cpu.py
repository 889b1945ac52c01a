"""CPU: SD-2.x-based motion models (linear transformer projections, upcast attention, per-level heads of head dim 64, 1024-wide text
context) - the oracle against the unmodified reference's SD-2 fixtures, the engine's key contract and checkpoint loading, and the engine's
host logic with every kernel launch emulated (tests/ops_emulator.py), including which attention entry points the bf16 mode routes to.

Tolerances are those of the SD-1.5 host-logic tests (tests/test_host_emulated_cpu.py): fp32 rel-L2 <= 1e-4, bf16 rel-L2 <= 3e-2, pipeline
video max-abs <= 2e-3 (fp32) / PSNR >= 30 dB (bf16).
"""
import json
import os

import pytest
import torch

from tests import ops_emulator
from tests.cfgs_sd2 import MINI_SD2, MINI_SD2_2D, mini_sd2_oracle_cfg, oracle_state_dict, sd2_inputs
from tests.sd2_helpers import (make_sd2_unet, run_sd2_pipeline_case, run_sd2_unet2d_case, run_sd2_unet_case, sd2_keys, sd2_pins)

DTYPES = [(torch.float32, 1e-4), (torch.bfloat16, 3e-2)]

# the unet/config.json of an SD-2.1 base, at the mini width of MINI_SD2_2D (the full model: 320 / 640 / 1280 / 1280, heads 5 / 10 / 20 / 20)
SD21_CONFIG = {"_class_name": "UNet2DConditionModel", "_diffusers_version": "0.10.0.dev0", "act_fn": "silu", "attention_head_dim": [2, 4, 8, 8],
               "block_out_channels": [128, 256, 512, 512], "center_input_sample": False, "cross_attention_dim": 1024,
               "down_block_types": ["CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "CrossAttnDownBlock2D", "DownBlock2D"],
               "downsample_padding": 1, "dual_cross_attention": False, "flip_sin_to_cos": True, "freq_shift": 0, "in_channels": 4,
               "layers_per_block": 1, "mid_block_scale_factor": 1, "norm_eps": 1e-05, "norm_num_groups": 32, "num_class_embeds": None,
               "only_cross_attention": False, "out_channels": 4, "resnet_time_scale_shift": "default", "sample_size": 16,
               "up_block_types": ["UpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D", "CrossAttnUpBlock2D"], "upcast_attention": True,
               "use_linear_projection": True}
# unet_additional_kwargs of configs/training/org_config_files/training_14M_448x256_w_multi_scale_w_fps_sd_v2.1.yaml
SD21_MOTION_KWARGS = dict(use_motion_module=True, motion_module_resolutions=[1, 2, 4, 8], unet_use_cross_frame_attention=False,
                          unet_use_temporal_attention=False, use_linear_projection=True, use_inflated_groupnorm=True,
                          motion_module_mid_block=True, use_fps_condition=True, motion_module_type="Vanilla",
                          motion_module_kwargs=dict(num_attention_heads=8, num_transformer_block=1,
                                                    attention_block_types=["Temporal_Self", "Temporal_Self"], temporal_position_encoding=True,
                                                    temporal_position_encoding_max_len=32, temporal_attention_dim_div=1, zero_initialize=True))


def _oracle_sd(keys):
    from followyourclick_b200.synth import synth_state_dict
    from followyourclick_b200.unet import sinusoidal_pe
    sd = synth_state_dict(dict(keys))
    for k, s in keys.items():
        if k.endswith(".pos_encoder.pe"):
            sd[k] = sinusoidal_pe(s[1], s[2])
    return sd


# ------------------------------------------------------------------------------------------------ (a) oracle vs the reference fixtures
def test_sd2_oracle_vs_reference_fixtures():
    import numpy as np
    from followyourclick_b200.synth import synth_clip_inputs
    from oracle import ref_pipeline, ref_unet, ref_vae
    from tests.cfgs import MINI_VAE, SCHED_V
    from tests.cfgs_sd2 import SD2_CTX_DIM
    from tests.engine_helpers import golden
    pins = sd2_pins()
    torch.set_num_threads(8)
    sd = oracle_state_dict(_oracle_sd(sd2_keys("unet3d")))
    inp = sd2_inputs()
    out = ref_unet.unet3d_forward(sd, mini_sd2_oracle_cfg(), inp["sample"], inp["timestep"], inp["ctx"], fps_tensor=inp["fps"],
                                  flow_control=inp["flow"])
    ref = torch.from_numpy(golden("unet_sd2.npz")["out"])
    assert float((out - ref).abs().max()) <= 4 * pins["unet_sd2"] + 1e-5
    g = golden("unet2d_sd2.npz")
    out2 = ref_unet.unet3d_forward(oracle_state_dict(_oracle_sd(sd2_keys("unet2d"))), mini_sd2_oracle_cfg(two_d=True), torch.from_numpy(g["x"]).unsqueeze(2),
                                   torch.tensor(501), torch.from_numpy(g["ctx"])).squeeze(2)
    assert float((out2 - torch.from_numpy(g["out"])).abs().max()) <= 4 * pins["unet2d_sd2"] + 1e-5
    p = golden("pipeline_sd2.npz")
    ci = synth_clip_inputs(1, 4, 16, 16, seed=4321, ctx_dim=SD2_CTX_DIM)
    lat = ref_pipeline.denoise(sd, mini_sd2_oracle_cfg(), SCHED_V, ci["latents"], ci["text_embeddings"], int(p["steps"]), float(p["guidance"]),
                               fps_tensor=torch.tensor([3]), flow_control=torch.tensor([5]))
    assert float((lat - torch.from_numpy(p["final_latents"])).abs().max()) < 1e-4
    vsd = _oracle_sd({k: tuple(s) for k, s in json.load(open(os.path.join(os.path.dirname(__file__), "golden", "vae_keys.json"))).items()})
    video = ref_vae.decode_latents(vsd, MINI_VAE, lat)
    assert float((video - torch.from_numpy(p["video"])).abs().max()) <= 4 * pins["pipeline_sd2"] + 1e-5
    assert all(v < 1e-4 for v in pins.values()) and np.isfinite(list(pins.values())).all()


# ------------------------------------------------------------------------------------------------ (b) key contract
def test_sd2_key_contract_equals_reference():
    from followyourclick_b200 import UNet2DConditionModel, UNet3DConditionModel
    m = UNet3DConditionModel(**MINI_SD2)
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == sd2_keys("unet3d")
    assert m._p("down_blocks.0.attentions.0.proj_in.weight").shape == (128, 128)           # Linear, not a 1x1 conv
    m2 = UNet2DConditionModel(**MINI_SD2_2D)
    assert {k: tuple(v.shape) for k, v in m2.state_dict().items()} == sd2_keys("unet2d")


# ------------------------------------------------------------------------------------------------ (c) loading an SD-2.1-layout unet/ folder
def test_from_pretrained_2d_loads_an_sd21_unet_folder(tmp_path, capsys):
    from followyourclick_b200 import UNet2DConditionModel, UNet3DConditionModel
    from tests.engine_helpers import load_synth
    src = UNet2DConditionModel(**MINI_SD2_2D)
    sd = load_synth(src)
    folder = tmp_path / "stable-diffusion-2-1" / "unet"
    folder.mkdir(parents=True)
    (folder / "config.json").write_text(json.dumps(SD21_CONFIG))
    torch.save(sd, folder / "diffusion_pytorch_model.bin")
    capsys.readouterr()
    m = UNet3DConditionModel.from_pretrained_2d(str(tmp_path / "stable-diffusion-2-1"), subfolder="unet",
                                                unet_additional_kwargs=SD21_MOTION_KWARGS)
    printed = capsys.readouterr().out
    assert "### unexpected keys: 0;" in printed, printed
    msd = m.state_dict()
    missing = set(msd) - set(sd)
    # only what the 2-D checkpoint cannot have is new: the motion modules and the fps / motion-strength embeddings
    assert missing and all(".motion_modules." in k or k.startswith(("fps_embedding.", "motion_embedding.")) for k in missing), missing
    assert all(torch.equal(msd[k], v) for k, v in sd.items())
    assert m._heads == (2, 4, 8, 8) and m.config["cross_attention_dim"] == 1024 and m.config["upcast_attention"]
    m2 = UNet2DConditionModel.from_pretrained(str(folder))
    assert all(torch.equal(m2.state_dict()[k], v) for k, v in sd.items())


# ------------------------------------------------------------------------------------------------ (d) host logic, kernels emulated
@pytest.fixture
def emulated(monkeypatch):
    ops_emulator.install(monkeypatch)
    torch.set_num_threads(8)
    yield monkeypatch


@pytest.mark.parametrize("dtype,tol", DTYPES)
def test_sd2_unet_host_logic_vs_reference_golden_and_d64_routes(emulated, dtype, tol):
    """bf16 mode must run the level-0 self-attention (16 x 16 = 256 tokens) on the head-dim-64 wgmma entry point with the fused [q | k | v]
    projection unpadded, and every cross-attention on the resident-context entry point with D = 64; strict fp32 on neither."""
    from followyourclick_b200 import ops
    calls = {"self": [], "cross": []}
    self_tc, cross_tc = ops.self_attention_tc, ops.cross_attention_tc

    def self_spy(qk, q_col0, k_col0, vt, heads, D, scale):
        calls["self"].append((D, qk.shape[-1] == 3 * heads * D, k_col0 == heads * D))
        return self_tc(qk, q_col0, k_col0, vt, heads, D, scale)

    def cross_spy(q, k, vt, heads, D, *a, **kw):
        calls["cross"].append((D, k.shape[-1] == heads * ops.cross_dkp(D)))
        return cross_tc(q, k, vt, heads, D, *a, **kw)
    emulated.setattr(ops, "self_attention_tc", self_spy)
    emulated.setattr(ops, "cross_attention_tc", cross_spy)
    s = run_sd2_unet_case(dtype, device="cpu")
    assert s["finite"] and s["rel_l2"] < tol, s
    if dtype == torch.bfloat16:
        assert calls["self"] == [(64, True, True)] * 3, calls      # down 0 (one layer) + up 3 (two layers): the 256-token level
        assert calls["cross"] == [(64, True)] * 10, calls          # every transformer block: 3 down + mid + 6 up
    else:
        assert calls == {"self": [], "cross": []}, calls


@pytest.mark.parametrize("dtype,tol", DTYPES)
def test_sd2_unet2d_host_logic_vs_reference_golden(emulated, dtype, tol):
    s = run_sd2_unet2d_case(dtype, device="cpu")
    assert s["finite"] and s["rel_l2"] < tol, s


def test_sd2_pipeline_host_logic_vs_reference_golden(emulated):
    r = run_sd2_pipeline_case(torch.float32, device="cpu", graph=False)
    assert r["finite"] and r["shape"] == (1, 3, 4, 128, 128) and r["video_maxabs"] < 2e-3, r
    r = run_sd2_pipeline_case(torch.bfloat16, device="cpu", graph=False)
    assert r["finite"] and r["psnr"] > 30.0, r


def test_sd2_context_hoisting_packs_every_block_for_the_d64_cross_attention(emulated):
    """prepare_context with the 1024-wide text context: every block's K/V packed for the tensor-core cross-attention (head stride 64), and
    the hoisted context gives the per-forward result bit for bit."""
    from followyourclick_b200 import ops
    unet, _ = make_sd2_unet(torch.bfloat16, "cpu")
    inp = sd2_inputs()
    ctx = unet.prepare_context(inp["ctx"])
    assert len(ctx.kx) == len(unet._transformer_prefixes()) == 10 and not ctx.kv
    for p, (kvp, vt) in ctx.kx.items():
        C = unet._p(p + ".transformer_blocks.0.attn2.to_q.weight").shape[0]
        assert kvp.shape == (2, ops.CROSS_LK, 2 * C) and vt.shape == (2, C, ops.CROSS_LK)
    x = ops.ncfhw_to_nfhwc(inp["sample"].contiguous(), torch.bfloat16)
    kw = dict(fps_tensor=inp["fps"], flow_control=inp["flow"], use_fps_condition=True)
    a = unet.forward_nfhwc(x, inp["timestep"], inp["ctx"], **kw)
    b = unet.forward_nfhwc(x, inp["timestep"], None, context=ctx, **kw)
    assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------ (e) what is still not built
@pytest.mark.parametrize("over,name", [(dict(use_temporal_conv=True), "use_temporal_conv"), (dict(use_pseudo_conv3d=True), "use_pseudo_conv3d"),
                                       (dict(use_text_encoder_2=True), "use_text_encoder_2"),
                                       (dict(motion_module_kwargs=dict(MINI_SD2["motion_module_kwargs"], use_rope_postion_encoding=True)),
                                        "use_rope_postion_encoding"),
                                       (dict(unet_use_temporal_attention=True), "unet_use_temporal_attention")])
def test_unbuilt_options_still_raise(over, name):
    from followyourclick_b200 import UNet3DConditionModel
    with pytest.raises(NotImplementedError, match=name):
        UNet3DConditionModel(**dict(MINI_SD2, **over))
