"""GPU: the first-frame-conditioned motion models (use_first_frame_condition, use_first_frame_condition_concat) on the engine.

  - the step prologue (fyc_build_unet_input_first) and the per-image time-embedding table (fyc_first_frame_temb_rows) element by element,
    bit-exact against their fyc.h contracts, including the in-place write of frame 0;
  - mini UNets and 2-step pipelines against the unmodified reference's fixtures (tests/golden/make_golden_first_frame.py) at the
    tolerances of tests/test_engine_gpu.py / tests/test_fp16_gpu.py: UNet rel-L2 fp32 <= 1e-4, bf16 <= 3e-2, fp16 <= 1e-2; video max-abs
    fp32 <= 2e-3, PSNR >= 30 dB bf16 / fp16;
  - CUDA-graph replay bit-identical to the kernel-by-kernel loop; the shared CFG prefix against the duplicated batch;
  - full width at cfg2 (64x64 latents, 16 frames): one UNet forward per mode against the fp32 oracle run on the device (bf16 output
    rel-L2 <= 2e-2, DESIGN.md section 2), and one 25-step clip per mode (video PSNR >= 35 dB, final latent rel-L2 <= 0.05).
"""
import pytest
import torch

from tests.cfgs_first_frame import PIPE_CASES, UNET_CASES

pytestmark = pytest.mark.gpu

UNET_TOL = [(torch.float32, 1e-4), (torch.bfloat16, 3e-2), (torch.float16, 1e-2)]


@pytest.fixture(autouse=True)
def _impl(cuda):
    from followyourclick_b200 import ops
    ops.set_impl("auto")
    yield
    ops.set_impl("auto")


# ------------------------------------------------------------------------------------------------ kernels vs their contracts
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("mode", [1, 2, 3])
@pytest.mark.parametrize("dup,c_pad", [(1, None), (2, 16)])
def test_prologue_bit_exact(dtype, mode, dup, c_pad):
    from followyourclick_b200 import ops
    g = torch.Generator().manual_seed(100 + mode)
    b, f, h, w = 2, 5, 6, 10
    lat = torch.randn(b, 4, f, h, w, generator=g)
    first = torch.randn(b, 4, h, w, generator=g)
    lat_d, first_d = lat.cuda(), first.cuda()
    out = ops.build_unet_input_first(lat_d, first_d, dup, dtype, mode, c_pad=c_pad)
    torch.cuda.synchronize()
    # the contract, restated
    want_lat = lat.clone()
    if mode & ops.FIRST_FRAME:
        want_lat[:, :, 0] = first
    cin = 8 if mode & ops.FIRST_CONCAT else 4
    cp = cin if c_pad is None else c_pad
    x = torch.zeros(b, f, h, w, cp)
    x[..., :4] = want_lat.permute(0, 2, 3, 4, 1)
    if mode & ops.FIRST_CONCAT:
        x[..., 4:8] = first.permute(0, 2, 3, 1)[:, None]
    want = torch.cat([x] * dup).to(dtype)
    assert out.shape == want.shape and torch.equal(out.cpu(), want)
    assert torch.equal(lat_d.cpu(), want_lat)                  # frame 0 written in place (mode 2 / 3), nothing else touched


def test_first_frame_temb_rows_bit_exact():
    from followyourclick_b200 import ops
    B, F, N = 3, 7, 1000
    t = torch.randn(B + 1, N, generator=torch.Generator().manual_seed(5))
    out = ops.first_frame_temb_rows(t.cuda(), B, F).cpu()
    for bi in range(B):
        for f in range(F):
            assert torch.equal(out[bi * F + f], t[B if f == 0 else bi])


# ------------------------------------------------------------------------------------------------ mini models vs the reference fixtures
@pytest.mark.parametrize("name", list(UNET_CASES))
@pytest.mark.parametrize("dtype,tol", UNET_TOL)
def test_unet_matches_reference_fixture(name, dtype, tol):
    from tests.first_frame_helpers import run_ff_unet_case
    s = run_ff_unet_case(name, dtype)
    assert s["finite"] and s["rel_l2"] < tol, s


@pytest.mark.parametrize("name", ["ff", "ffc"])
@pytest.mark.parametrize("dtype,tol", UNET_TOL)
def test_unet_public_forward_matches_reference_fixture(name, dtype, tol):
    from tests.first_frame_helpers import run_ff_unet_case
    s = run_ff_unet_case(name, dtype, via_forward=True)
    assert s["finite"] and s["rel_l2"] < tol, s


@pytest.mark.parametrize("name", [n for n, c in UNET_CASES.items() if c[3]])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_shared_prefix_vs_duplicated_batch(name, dtype):
    """cfg_dup = 2 on one copy of the input (the first ResnetBlock3D reads the per-image time-embedding rows of the first half) vs the
    duplicated batch, and vs the fixture"""
    from tests.engine_helpers import stats
    from tests.first_frame_helpers import UNET_CASES as _C, ff_unet_forward, make_ff_unet
    mode, fps, b, cfg = _C[name]
    unet, _ = make_ff_unet(mode, fps, dtype)
    full = ff_unet_forward(unet, name, "cuda")
    shared = ff_unet_forward(unet, name, "cuda", share=True)
    s = stats(shared, full)
    assert s["finite"] and s["rel_l2"] < (1e-6 if dtype == torch.float32 else 2e-3), s


@pytest.mark.parametrize("name", list(PIPE_CASES))
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
def test_pipeline_matches_reference_fixture(name, dtype):
    from tests.first_frame_helpers import run_ff_pipeline_case
    r = run_ff_pipeline_case(name, dtype)
    assert r["finite"] and r["shape"] == (1, 3, 4, 64, 64), r
    if dtype == torch.float32:
        assert r["video_maxabs"] < 2e-3 and r["latent_rel_l2"] < 1e-4, r
    else:
        assert r["psnr"] > 30.0, r


@pytest.mark.parametrize("name", list(PIPE_CASES))
def test_graph_replay_bit_identical_to_eager(name):
    from tests.first_frame_helpers import ff_pipeline_call, make_ff_pipeline
    pipe, ci = make_ff_pipeline(name, torch.bfloat16)
    outs = []
    for graph in (True, False):
        pipe.use_cuda_graph = graph
        outs.append(ff_pipeline_call(pipe, ci, name))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])


@pytest.mark.parametrize("name", ["ff", "ffc"])
def test_pipeline_shared_prefix_off_matches_fixture(name):
    from tests.first_frame_helpers import run_ff_pipeline_case
    for dtype in (torch.float32, torch.bfloat16):
        r = run_ff_pipeline_case(name, dtype, share=False)
        assert r["finite"] and (r["video_maxabs"] < 2e-3 if dtype == torch.float32 else r["psnr"] > 30.0), r


# ------------------------------------------------------------------------------------------------ full width, cfg2
_full = {}


def _full_unet(mode):
    """full-width UNet3D of the mode (tests/cfgs_first_frame.py at the shipped widths), deterministic on-device weights"""
    if mode not in _full:
        import bench
        from followyourclick_b200 import UNet3DConditionModel
        from followyourclick_b200.synth import synth_on_device_
        kw = dict(bench.unet_kwargs(False), use_first_frame_mask_condition_concat=False, use_fps_condition=(mode == "ffc"))
        if mode == "ffc":
            kw["use_first_frame_condition_concat"] = True
        _full.clear()
        torch.cuda.empty_cache()
        unet = UNet3DConditionModel(**kw).to("cuda")
        synth_on_device_(unet, seed=0)
        _full[mode] = unet
    return _full[mode]


@pytest.fixture
def strict_torch(cuda):
    old = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield cuda
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old


def _rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _mode_kw(mode, first, fps):
    if mode == "ff":
        return dict(use_first_frame_condition=True)
    return dict(use_first_frame_condition_concat=True, reference_images_latent=first, use_fps_condition=True, fps_tensor=fps,
                flow_control=fps + 2)


@pytest.mark.parametrize("mode", ["ff", "ffc"])
def test_unet_full_width_cfg2_bf16_vs_fp32_oracle(strict_torch, mode):
    from oracle import ref_unet
    from tests import oracle_first_frame
    unet = _full_unet(mode)
    g = torch.Generator().manual_seed(11)
    sample = torch.randn(1, 4, 16, 64, 64, generator=g).cuda()
    first = torch.randn(1, 4, 64, 64, generator=g).cuda()
    sample[:, :, 0] = first
    sample, first = torch.cat([sample] * 2), torch.cat([first] * 2)               # the CFG batch the reference feeds
    ctx = torch.randn(2, 77, 768, generator=g).cuda()
    fps = torch.tensor([2, 2], device="cuda")
    kw = _mode_kw(mode, first, fps)
    cfg = dict(ref_unet.default_unet_config(), use_first_frame_mask_condition_concat=False, use_first_frame_condition_concat=(mode == "ffc"),
               use_fps_condition=(mode == "ffc"))
    okw = {k: v for k, v in kw.items() if k != "use_fps_condition"}
    with torch.no_grad():
        ref = oracle_first_frame.unet3d_forward({k: v.detach() for k, v in unet.state_dict().items()}, cfg, sample, torch.tensor(501), ctx, **okw).cpu()
    torch.cuda.empty_cache()
    unet.to(torch.bfloat16)
    try:
        out = unet(sample, torch.tensor(501), ctx, **kw).sample
    finally:
        unet.to(torch.float32)
    r = _rel(out, ref)
    assert bool(torch.isfinite(out).all()) and r <= 2e-2, r


@pytest.mark.parametrize("mode", ["ff", "ffc"])
def test_pipeline_cfg2_25_steps_bf16_vs_fp32_oracle(strict_torch, mode):
    import bench
    from followyourclick_b200 import AnimationPipeline, AutoencoderKL, DDIMScheduler
    from followyourclick_b200.synth import synth_clip_inputs, synth_on_device_
    from oracle import ref_unet, ref_vae
    from oracle.ref_ddim import default_scheduler_config
    from tests import oracle_first_frame
    unet = _full_unet(mode)
    vae = AutoencoderKL(**bench.vae_kwargs(False)).to("cuda")
    synth_on_device_(vae, seed=1)
    F, h, w, steps, gs = 16, 64, 64, 25, 8.0
    ci = {k: v.cuda() for k, v in synth_clip_inputs(1, F, h, w, seed=1234).items()}
    fps = dict(fps_tensor=torch.tensor([2]), flow_control=torch.tensor([4])) if mode == "ffc" else {}
    cfg = dict(ref_unet.default_unet_config(), use_first_frame_mask_condition_concat=False, use_first_frame_condition_concat=(mode == "ffc"),
               use_fps_condition=(mode == "ffc"))
    with torch.no_grad():
        lat_ref = oracle_first_frame.denoise({k: v.detach() for k, v in unet.state_dict().items()}, cfg, default_scheduler_config(),
                                             ci["latents"], ci["text_embeddings"], steps, gs, first_image_latents=ci["first_image_latents"],
                                             use_first_frame_condition=(mode == "ff"), **fps)
        video_ref = ref_vae.decode_latents({k: v.detach() for k, v in vae.state_dict().items()}, ref_vae.default_vae_config(), lat_ref).cpu()
    torch.cuda.empty_cache()
    unet.to(torch.bfloat16)
    vae.to(torch.bfloat16)
    try:
        pipe = AnimationPipeline(vae=vae, text_encoder=bench._TextEnc(ci["text_embeddings"]), tokenizer=bench._Tok(), unet=unet,
                                 scheduler=DDIMScheduler(**bench.SCHED))
        pipe.set_progress_bar_config(disable=True)
        mkw = dict(use_first_frame_condition=True) if mode == "ff" else dict(use_first_frame_condition_concat=True, use_fps_condition=True)
        lat = pipe.denoise(ci["latents"], ci["text_embeddings"], steps, gs, first_image_latents=ci["first_image_latents"], **fps, **mkw)
        video = pipe.decode_latents_device(lat).cpu()
    finally:
        unet.to(torch.float32)
    mse = float(((video.double() - video_ref.double()) ** 2).mean())
    psnr = float(10 * torch.log10(torch.tensor(1.0 / max(mse, 1e-20))))
    rl = _rel(lat, lat_ref)
    assert bool(torch.isfinite(video).all()) and psnr >= 35.0 and rl <= 0.05, (psnr, rl)
