"""GPU: SD-2.x-based motion models on the engine.

  (a) the head-dim-64 wgmma kernels against torch fp32 on the same bf16 operands, at the SD-2 shapes of a 64 x 64 x 16-frame forward with
      B = 2 (32 images): self-attention L = 4096 / 1024 / 256 with 5 / 10 / 20 heads; cross-attention against 77 text keys, with and
      without a 4- or 16-token second context, one context per clip (kv_batch_div = 16).  Bounds: rel-L2 <= 4e-3, worst (token, head) row
      rel-L2 <= 1.5e-2, max-abs <= 2^-7 max|ref|.  The output is NaN-prefilled and wider than the heads: only the heads' columns may change;
  (b) the mini SD-2 model (tests/cfgs_sd2.py MINI_SD2) against the unmodified reference's fixtures: UNet3D (strict fp32 rel-L2 <= 1e-4, bf16
      <= 3e-2), UNet2D, the 2-step pipeline (fp32 video max-abs <= 2e-3, bf16 PSNR >= 30 dB) - the SD-1.5 mini-model tolerances;
  (c) full-size parity: SD-2 width (320 / 640 / 1280 / 1280, heads 5 / 10 / 20 / 20, 1024-wide context, linear projections, inflated
      GroupNorm, mid-block motion module), one UNet forward at 64 x 64 x 16 frames, B = 2, against the fp32 oracle run on the GPU (TF32 off):
      strict fp32 rel-L2 <= 5e-5 at every tap, bf16 <= 2e-2 at the output and <= 3e-2 at every tap.  Figures go to FYC_PARITY_JSON.
"""
import time

import pytest
import torch

from tests.test_full_parity_gpu import err, record

pytestmark = pytest.mark.gpu

NB = 32                       # 2 clips x 16 frames
REL, ROW, MAXABS = 4e-3, 1.5e-2, 2.0 ** -7


def rnd(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).bfloat16().cuda()


def mha_fp32(q, k, v, heads, scale, chunk=4):
    """softmax(scale q k^T) v in fp32 per head, q [B, Lq, heads D], k / v [B, Lk, heads D] (batch entries in chunks: bounded scores)"""
    B, Lq, C = q.shape
    D = C // heads
    outs = []
    for i in range(0, B, chunk):
        qh = q[i:i + chunk].float().view(-1, Lq, heads, D).transpose(1, 2)
        kh = k[i:i + chunk].float().view(qh.shape[0], -1, heads, D).transpose(1, 2)
        vh = v[i:i + chunk].float().view(qh.shape[0], -1, heads, D).transpose(1, 2)
        outs.append((torch.softmax(qh @ kh.transpose(-1, -2) * scale, dim=-1) @ vh).transpose(1, 2).reshape(qh.shape[0], Lq, C))
    return torch.cat(outs)


def check(out, ref, heads, what):
    D = ref.shape[-1] // heads
    e = err(out.float().reshape(-1, heads, D), ref.reshape(-1, heads, D))
    record(f"sd2_kernels/{what}", e)
    assert e["finite"] and e["rel_l2"] <= REL and e["worst_row"] <= ROW and e["maxabs"] <= MAXABS * e["ref_absmax"], (what, e)
    return e


@pytest.mark.parametrize("L,heads", [(4096, 5), (1024, 10), (256, 20)])
def test_self_attention_d64(strict, L, heads):
    """fyc_self_attention_tc with D = 64: q / k straight from the fused, unpadded [q | k | v] projection (heads 64 columns apart)."""
    from followyourclick_b200 import ops
    from followyourclick_b200._lib import check as fyc_check, lib, ptr, stream_ptr
    D, C = 64, heads * 64
    assert ops.self_attention_tc_ok(torch.bfloat16, L, D)
    qkv = rnd((NB, L, 3 * C), 1)
    vt = ops.transpose_tokens(qkv, 2 * C, C)
    ld = C + 40                                        # wider than the heads: the extra columns must stay NaN
    out = torch.full((NB, L, ld), float("nan"), dtype=torch.bfloat16, device="cuda")
    fyc_check(lib().fyc_self_attention_tc(ptr(qkv), qkv.stride(1), 0, C, ptr(vt), ptr(out), ld, NB, heads, L, D, float(D ** -0.5),
                                          stream_ptr()))
    torch.cuda.synchronize()
    assert bool(torch.isnan(out[..., C:]).all())
    ref = mha_fp32(qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:], heads, D ** -0.5)
    check(out[..., :C], ref, heads, f"self/L{L}x{heads}")
    # the public wrapper and the mma.sync kernel it replaces on the same operands
    o1 = ops.self_attention_tc(qkv, 0, C, vt, heads, D, D ** -0.5)
    assert torch.equal(o1, out[..., :C])
    o2 = ops.attention(qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:], heads, D ** -0.5)
    assert err(o2, ref)["rel_l2"] <= REL


def _pack(k, v, heads, Lpad):
    NBc, Lk, C = k.shape
    kp = torch.zeros((NBc, Lpad, C), dtype=k.dtype, device=k.device)
    kp[:, :Lk] = k
    vt = torch.zeros((NBc, C, Lpad), dtype=v.dtype, device=v.device)
    vt[:, :, :Lk] = v.transpose(1, 2)
    return kp, vt.contiguous()


@pytest.mark.parametrize("T", [0, 4, 16])
@pytest.mark.parametrize("Lq,heads", [(4096, 5), (1024, 10), (256, 20)])
def test_cross_attention_d64(strict, Lq, heads, T):
    """fyc_cross_attention_tc with D = 64 (DKP = DV = 64): 77 text keys (+ T image keys), one packed context per clip for its 16 frames."""
    from followyourclick_b200 import ops
    D, C, div, Lk = 64, heads * 64, 16, 77
    assert ops.cross_attention_tc_ok(torch.bfloat16, D, Lk, T) and ops.cross_dkp(D) == 64
    q = rnd((NB, Lq, C), 1)
    kt, vtx = rnd((NB // div, Lk, C), 2), rnd((NB // div, Lk, C), 3)
    kp, vt = _pack(kt, vtx, heads, ops.CROSS_LK)
    k2 = vt2 = ki = vi = None
    a2 = 0.6
    if T:
        ki, vi = rnd((NB // div, T, C), 4), rnd((NB // div, T, C), 5)
        k2, vt2 = _pack(ki, vi, heads, ops.CROSS_LK2)
    ld = C + 40
    buf = torch.full((NB, Lq, ld), float("nan"), dtype=torch.bfloat16, device="cuda")
    out = buf[..., :C]
    ops.cross_attention_tc(q, kp, vt, heads, D, D ** -0.5, Lk, out, k2=k2, vt2=vt2, Lk2=T, alpha2=a2, kv_batch_div=div)
    torch.cuda.synchronize()
    assert bool(torch.isnan(buf[..., C:]).all())
    rep = lambda t: t.repeat_interleave(div, 0)
    ref = mha_fp32(q, rep(kt), rep(vtx), heads, D ** -0.5)
    if T:
        ref = ref + a2 * mha_fp32(q, rep(ki), rep(vi), heads, D ** -0.5)
    check(out, ref, heads, f"cross/L{Lq}x{heads}+{T}")
    old = ops.attention(q, kt, vtx, heads, D ** -0.5, kv_batch_div=div, k2=ki, v2=vi, alpha2=a2)
    assert err(old, ref)["rel_l2"] <= REL


@pytest.fixture(scope="module")
def strict(cuda):
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    torch.set_float32_matmul_precision("highest")
    return cuda


# ------------------------------------------------------------------------------------------------ (b) mini model vs the reference fixtures
@pytest.mark.parametrize("dtype,tol", [(torch.float32, 1e-4), (torch.bfloat16, 3e-2)])
def test_sd2_mini_unet_and_unet2d_vs_reference_fixtures(strict, dtype, tol):
    from tests.sd2_helpers import run_sd2_unet2d_case, run_sd2_unet_case
    s = run_sd2_unet_case(dtype)
    record(f"sd2_mini/unet3d/{dtype}", s)
    assert s["finite"] and s["rel_l2"] < tol, s
    s = run_sd2_unet2d_case(dtype)
    record(f"sd2_mini/unet2d/{dtype}", s)
    assert s["finite"] and s["rel_l2"] < tol, s


def test_sd2_mini_pipeline_vs_reference_fixture(strict):
    from tests.sd2_helpers import run_sd2_pipeline_case
    r = run_sd2_pipeline_case(torch.float32)
    record("sd2_mini/pipeline/f32", r)
    assert r["finite"] and r["shape"] == (1, 3, 4, 128, 128) and r["video_maxabs"] < 2e-3, r
    r = run_sd2_pipeline_case(torch.bfloat16)
    record("sd2_mini/pipeline/bf16", r)
    assert r["finite"] and r["psnr"] > 30.0, r


# ------------------------------------------------------------------------------------------------ (c) full-size parity
def sd2_full_kwargs():
    """an SD-2.1 base (unet/config.json) with the unet_additional_kwargs of training_14M_448x256_w_multi_scale_w_fps_sd_v2.1.yaml"""
    mm = dict(num_attention_heads=8, num_transformer_block=1, attention_block_types=("Temporal_Self", "Temporal_Self"),
              temporal_position_encoding=True, temporal_position_encoding_max_len=32, temporal_attention_dim_div=1)
    return dict(sample_size=96, in_channels=4, out_channels=4, block_out_channels=(320, 640, 1280, 1280), layers_per_block=2,
                attention_head_dim=[5, 10, 20, 20], cross_attention_dim=1024, use_linear_projection=True, upcast_attention=True,
                use_motion_module=True, motion_module_resolutions=(1, 2, 4, 8), unet_use_cross_frame_attention=False,
                unet_use_temporal_attention=False, use_inflated_groupnorm=True, motion_module_mid_block=True, use_fps_condition=True,
                motion_module_type="Vanilla", motion_module_kwargs=mm)


def sd2_full_oracle_cfg():
    from oracle import ref_unet
    kw = sd2_full_kwargs()
    return ref_unet.default_unet_config(attention_head_dim=kw["attention_head_dim"], cross_attention_dim=1024,
                                        use_inflated_groupnorm=True, motion_module_mid_block=True, motion_module_kwargs=kw["motion_module_kwargs"],
                                        use_first_frame_mask_condition_concat=False, use_fps_condition=True)


def test_sd2_unet_forward_full_width(strict):
    from followyourclick_b200 import UNet3DConditionModel
    from followyourclick_b200.synth import synth_on_device_
    from oracle import ref_unet
    from tests.cfgs_sd2 import oracle_state_dict
    dev = strict
    unet = UNet3DConditionModel(**sd2_full_kwargs()).to(dev)
    synth_on_device_(unet, seed=5)
    g = torch.Generator().manual_seed(19)
    F, h, w = 16, 64, 64
    x, ctx = torch.randn(2, 4, F, h, w, generator=g).to(dev), torch.randn(2, 77, 1024, generator=g).to(dev)
    t, fps, flow = torch.tensor(501, device=dev), torch.tensor([3, 3], device=dev), torch.tensor([5, 5], device=dev)
    taps = {}
    t0 = time.time()
    with torch.no_grad():
        ref = ref_unet.unet3d_forward(oracle_state_dict({k: v.detach() for k, v in unet.state_dict().items()}), sd2_full_oracle_cfg(), x, t, ctx,
                                      fps_tensor=fps, flow_control=flow, taps=taps)
    ref = ref.cpu()
    ref_taps = {k: v.permute(0, 2, 3, 4, 1).reshape(-1, v.shape[3], v.shape[4], v.shape[1]).cpu() for k, v in taps.items()}
    del taps
    torch.cuda.empty_cache()
    record("sd2_unet_forward/64x64x16/oracle_seconds", round(time.time() - t0, 2))
    for dtype in (torch.float32, torch.bfloat16):
        unet.to(dtype)
        unet._taps = {}
        try:
            out = unet(x, t, encoder_hidden_states=ctx, use_fps_condition=True, fps_tensor=fps, flow_control=flow).sample
            torch.cuda.synchronize()
            etaps = unet._taps
        finally:
            unet._taps = None
        res = {k: err(etaps[k], ref_taps[k]) for k in ref_taps}
        res["out"] = err(out.cpu().permute(0, 2, 3, 4, 1), ref.permute(0, 2, 3, 4, 1))
        name = "f32" if dtype == torch.float32 else "bf16"
        record(f"sd2_unet_forward/64x64x16/{name}", res)
        assert all(v["finite"] for v in res.values())
        worst = max((v["rel_l2"], k) for k, v in res.items())
        if dtype == torch.float32:
            assert worst[0] <= 5e-5, worst
        else:
            assert res["out"]["rel_l2"] <= 2e-2, res["out"]
            assert worst[0] <= 3e-2, worst
