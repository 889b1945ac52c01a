"""The opt-in fp16 tensor-core mode on the GPU.

Kernel families: every 16-bit kernel the engine runs - the wgmma GEMM in each launch mode (plain, ragged into a window, aliasing
residual, batched, two-segment K, fp32 output, GEGLU, LayerNorm fold with row bias, W-resident), the 3x3 convolutions (stride 1, stride 2
in both padding modes, the four-phase upsampler, the N = 16 head), the wgmma self-attention (D = 40 / 64 / 80) and cross-attention with
IP key counts T = 0 / 4 / 16, the mma.sync attention, temporal attention at F = 16 and 32, GroupNorm / LayerNorm / LayerNorm statistics,
the elementwise and layout kernels and the CUDA-core fallbacks.  Each case builds its inputs once in fp32, runs in bf16 and in fp16
(twice: the outputs must be bit-identical) and compares both with torch fp32 on the unrounded inputs.  The fp16 rel-L2 must be at most
1/4 of the bf16 rel-L2 (the significands predict 1/8); the ratios are written to the JSON record.

Models: the mini models against the reference fixtures in tests/golden/ (fp16 error below the bf16 error), and at full width the cfg2
UNet forward per tap and the 25-step cfg2 pipeline against the fp32 oracle (tests/test_full_parity_gpu.py helpers), with every value
finite and the largest |value| of every tap recorded: fp16 ends at 65504.
"""
import json
import os
import sys
import tempfile

import pytest
import torch
import torch.nn.functional as Fn

from tests.fp16_helpers import literal_fp16_to

pytestmark = pytest.mark.gpu

OUT = os.environ.get("FYC_FP16_JSON") or os.path.join(tempfile.gettempdir(), "fyc_fp16.json")
RATIO = 0.25            # fp16 rel-L2 <= RATIO * bf16 rel-L2


def record(key, value):
    d = {}
    if os.path.exists(OUT):
        try:
            d = json.load(open(OUT))
        except Exception:
            d = {}
    d[key] = value
    os.makedirs(os.path.dirname(os.path.abspath(OUT)), exist_ok=True)
    json.dump(d, open(OUT, "w"), indent=1, sort_keys=True)
    print(f"[fp16] {key}: {json.dumps(value)}", file=sys.stderr, flush=True)


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / (b.norm() + 1e-30))


def rnd(shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).cuda()


@pytest.fixture(autouse=True)
def _impl(cuda):
    from followyourclick_b200 import ops
    ops.set_impl("auto")
    yield
    ops.set_impl("auto")


@pytest.fixture
def tc_only(cuda):
    """pin the tensor-core route: with impl "tc" a GEMM / convolution the wgmma kernel cannot take raises instead of falling back to the
    CUDA-core kernels"""
    from followyourclick_b200 import ops
    ops.set_impl("tc")
    yield


def compare(name, run, ref, ratio=RATIO):
    """run(dtype) -> output tensor (or tuple); ref: fp32 reference (or tuple).  bf16 once, fp16 twice (bit-identical).  An output the
    bf16 run stores in bf16 must come out of the fp16 run in fp16; fp32 outputs (fp32-out epilogue, layout to fp32) stay fp32."""
    def flat(o):
        return [t for t in (o if isinstance(o, (tuple, list)) else (o,))]
    ob = flat(run(torch.bfloat16))
    eb = [rel(a, r) for a, r in zip(ob, flat(ref))]
    o1, o2 = flat(run(torch.float16)), flat(run(torch.float16))
    torch.cuda.synchronize()
    for a, b, c in zip(o1, o2, ob):
        assert a.dtype == (torch.float16 if c.dtype == torch.bfloat16 else torch.float32) and c.dtype in (torch.bfloat16, torch.float32), \
            (name, a.dtype, c.dtype)
        assert torch.equal(a, b), f"{name}: two fp16 runs differ"
        assert bool(torch.isfinite(a.float()).all()), name
    e16 = [rel(a, r) for a, r in zip(o1, flat(ref))]
    res = dict(bf16=eb, fp16=e16, ratio=[f / b if b > 0 else 0.0 for f, b in zip(e16, eb)])
    record(f"kernels/{name}", res)
    for f, b in zip(e16, eb):
        assert f <= ratio * b or f < 1e-6, (name, res)
    return res


# ---------------------------------------------------------------------------------------------------------------- GEMM
@pytest.mark.parametrize("M,N,K", [(128 * 3 + 1, 320, 320), (128 * 3 - 1, 320, 320), (128 * 9 - 30, 320, 512), (128 * 16, 720, 640),
                                   (128 * 5 + 1, 48, 256), (4096 + 64, 1280, 1280), (2000, 960, 320), (32768, 320, 320)])
def test_gemm_ragged_window_bias_residual(M, N, K, tc_only):
    from followyourclick_b200 import ops
    A, W, bias, R = rnd((M, K), 1), rnd((N, K), 2, K ** -0.5), rnd((N,), 3), rnd((M, N), 4)

    def run(dt):
        big = torch.full((M + 5, N + 48), -777.0, dtype=dt, device="cuda")
        win = big[3:3 + M, 16:16 + N]
        ops.gemm(A.to(dt), W.to(dt), bias=bias, residual=R.to(dt), out=win)
        inner = torch.zeros_like(big, dtype=torch.bool)
        inner[3:3 + M, 16:16 + N] = True
        assert bool((big[~inner] == -777.0).all())
        return win.clone()
    compare(f"gemm_window[{M}x{N}x{K}]", run, A @ W.t() + bias + R)


def test_gemm_residual_aliasing_output(tc_only):
    from followyourclick_b200 import ops
    M, N, K = 4096, 640, 640
    A, W, R = rnd((M, K), 1), rnd((N, K), 2, K ** -0.5), rnd((M, N), 3)

    def run(dt):
        r = R.to(dt)
        ops.gemm(A.to(dt), W.to(dt), residual=r, out=r)
        return r
    compare("gemm_residual_alias", run, A @ W.t() + R)


def test_gemm_batched_f32_out_rowbias_two_segment(tc_only):
    from followyourclick_b200 import ops
    B, M, N, K = 3, 640, 256, 320
    A, W = rnd((B, M, K), 1), rnd((B, N, K), 2, K ** -0.5)
    compare("gemm_batched", lambda dt: ops.gemm(A.to(dt), W.to(dt)), A @ W.transpose(1, 2))
    M, N, K = 2048, 640, 320
    A, W, rb = rnd((M, K), 3), rnd((N, K), 4, K ** -0.5), rnd((M // 256, N), 5)
    compare("gemm_f32_out_rowbias", lambda dt: ops.gemm(A.to(dt), W.to(dt), rowbias=rb, rows_per_group=256, out_f32=True),
            A @ W.t() + rb.repeat_interleave(256, dim=0))
    M, N, K1, K2 = 4096, 640, 640, 320
    A1, A2, W = rnd((M, K1), 6), rnd((M, K2), 7), rnd((N, K1 + K2), 8, (K1 + K2) ** -0.5)
    compare("gemm_two_segment", lambda dt: ops.gemm(A1.to(dt), W.to(dt), A2=A2.to(dt)), torch.cat([A1, A2], 1) @ W.t())


@pytest.mark.parametrize("M,C", [(4096, 320), (1024, 1280)])
def test_gemm_geglu_and_layernorm_fold(M, C, tc_only):
    from followyourclick_b200 import ops
    from followyourclick_b200.modeling import geglu_interleave
    x = rnd((M, C), 1) * 1.3 + rnd((M, 1), 2) * 4.0                    # per-row offsets: the folded mean subtraction matters
    w, b = rnd((8 * C, C), 3, C ** -0.5), 0.05 * rnd((8 * C,), 4)
    gamma, beta = 1 + 0.1 * rnd((C,), 5), 0.05 * rnd((C,), 6)
    wi, bi = geglu_interleave(w, b)
    h = x @ w.t() + b
    a, g = h.chunk(2, dim=-1)
    compare(f"gemm_geglu[{M}x{C}]", lambda dt: ops.gemm(x.to(dt), wi.to(dt).contiguous(), bias=bi, geglu=True), a * Fn.gelu(g))

    def run_ln_geglu(dt):
        wp, cb = ops.ln_fold_weight(w, gamma, dt), (w @ beta + b).contiguous()
        wpi, cbi = geglu_interleave(wp.float(), cb)
        xd = x.to(dt)
        return ops.gemm(xd, wpi.to(dt).contiguous(), bias=cbi.contiguous(), geglu=True, ln=ops.layernorm_stats(xd))
    h = Fn.layer_norm(x, (C,), gamma, beta, 1e-5) @ w.t() + b
    a, g = h.chunk(2, dim=-1)
    compare(f"gemm_geglu_lnfold[{M}x{C}]", run_ln_geglu, a * Fn.gelu(g))
    N, rpg = 3 * C, 256
    w2, rb = rnd((N, C), 7, C ** -0.5), rnd((M // rpg, N), 8)

    def run_ln_rb(dt):
        xd = x.to(dt)
        return ops.gemm(xd, ops.ln_fold_weight(w2, gamma, dt), bias=(w2 @ beta).contiguous(), rowbias=rb, rows_per_group=rpg,
                        ln=ops.layernorm_stats(xd))
    compare(f"gemm_lnfold_rowbias[{M}x{C}]", run_ln_rb, Fn.layer_norm(x, (C,), gamma, beta, 1e-5) @ w2.t() + rb.repeat_interleave(rpg, 0))


def test_gemm_cuda_core_fallbacks():
    """shapes the tensor-core path does not take: small M (gemv), N % 16 != 0 (SIMT GEMM)"""
    from followyourclick_b200 import ops
    A, W, bias = rnd((2, 1280), 1), rnd((1280, 1280), 2, 1280 ** -0.5), rnd((1280,), 3)
    compare("gemv_small_m", lambda dt: ops.gemm(A.to(dt), W.to(dt), bias=bias), A @ W.t() + bias)
    A, W = rnd((300, 72), 4), rnd((40, 72), 5, 72 ** -0.5)
    compare("gemm_simt", lambda dt: ops.gemm(A.to(dt), W.to(dt)), A @ W.t())


# ---------------------------------------------------------------------------------------------------------------- convolution
def _conv_ref(x, w, bias=None, stride=1, pad_mode=0, up=1):
    xc = x.permute(0, 3, 1, 2)
    if up == 2:
        xc = Fn.interpolate(xc, scale_factor=2, mode="nearest")
    if pad_mode == 1:
        y = Fn.conv2d(Fn.pad(xc, (0, 1, 0, 1)), w, bias, stride=stride)
    else:
        y = Fn.conv2d(xc, w, bias, stride=stride, padding=1)
    return y.permute(0, 2, 3, 1)


def _packed(w, dt):
    return w.permute(0, 2, 3, 1).to(dt).contiguous()          # [Cout, Cin, 3, 3] -> [Cout, 3, 3, Cin]


@pytest.mark.parametrize("NB,H,W,Cin,Cout", [(2, 64, 64, 320, 320), (8, 32, 32, 640, 640), (4, 16, 16, 1280, 1280), (4, 8, 12, 64, 48)])
def test_conv3x3_stride1_bias_residual_rowbias(NB, H, W, Cin, Cout, tc_only):
    from followyourclick_b200 import ops
    x, w, b = rnd((NB, H, W, Cin), 1), rnd((Cout, Cin, 3, 3), 2, (9 * Cin) ** -0.5), rnd((Cout,), 3)
    R, rb = rnd((NB, H, W, Cout), 4), rnd((NB // 2, Cout), 5)
    ref = _conv_ref(x, w, b) + R + rb.repeat_interleave(2, 0)[:, None, None, :]
    compare(f"conv3x3[{NB}x{H}x{W}x{Cin}->{Cout}]",
            lambda dt: ops.conv3x3(x.to(dt), _packed(w, dt), bias=b, residual=R.to(dt), rowbias=rb, images_per_group=2), ref)


@pytest.mark.parametrize("pad_mode", [0, 1])
@pytest.mark.parametrize("NB,H,W,Cin,Cout", [(4, 64, 64, 320, 320), (2, 32, 32, 640, 640), (2, 16, 16, 128, 160)])
def test_conv3x3_stride2(NB, H, W, Cin, Cout, pad_mode, tc_only):
    from followyourclick_b200 import ops
    x, w, b = rnd((NB, H, W, Cin), 1), rnd((Cout, Cin, 3, 3), 2, (9 * Cin) ** -0.5), rnd((Cout,), 3)
    compare(f"conv3x3_s2_pad{pad_mode}[{NB}x{H}x{W}x{Cin}]", lambda dt: ops.conv3x3(x.to(dt), _packed(w, dt), bias=b, stride=2, pad_mode=pad_mode),
            _conv_ref(x, w, b, stride=2, pad_mode=pad_mode))


@pytest.mark.parametrize("NB,H,W,Cin,Cout", [(4, 8, 8, 1280, 1280), (4, 16, 16, 1280, 1280), (2, 32, 32, 640, 640)])
def test_conv3x3_upsample_four_phases(NB, H, W, Cin, Cout, tc_only):
    from followyourclick_b200 import ops
    from followyourclick_b200.modeling import upsample_phase_weights
    x, w, b = rnd((NB, H, W, Cin), 1), rnd((Cout, Cin, 3, 3), 2, (9 * Cin) ** -0.5), rnd((Cout,), 3)
    wph = upsample_phase_weights(w)

    def run(dt):
        with ops.profile() as p:           # the four-phase wgmma route, not the materialised upsample + 3x3 conv
            y = ops.conv3x3(x.to(dt), _packed(w, dt), bias=b, upsample=2, w_phases=wph.to(dt).contiguous())
        assert set(p.summary) == {"conv_tc_up2"} and y.shape == (NB, 2 * H, 2 * W, Cout), p.summary
        return y
    compare(f"conv3x3_up2[{NB}x{H}x{W}x{Cin}]", run, _conv_ref(x, w, b, up=2))


def test_conv3x3_heads_n16_and_small_n():
    """the 4 / 3-channel output heads zero-padded to N = 16 (fp32 out) on the tensor cores, and the Cout <= 4 CUDA-core kernel"""
    from followyourclick_b200 import ops
    x, w, b = rnd((16, 64, 64, 320), 1), rnd((16, 320, 3, 3), 2, (9 * 320) ** -0.5), rnd((16,), 3)
    compare("conv3x3_head16_f32out", lambda dt: ops.conv3x3(x.to(dt), _packed(w, dt), bias=b, out_f32=True, impl=ops.L.IMPL_TC),
            _conv_ref(x, w, b))
    w4 = w[:4].contiguous()
    compare("conv3x3_small_n", lambda dt: ops.conv3x3(x.to(dt), _packed(w4, dt), bias=b[:4].contiguous()), _conv_ref(x, w4, b[:4]))


# ---------------------------------------------------------------------------------------------------------------- attention
def _mha(q, k, v, heads, scale):
    B, Lq, C = q.shape
    d = C // heads
    qh, kh, vh = (t.reshape(t.shape[0], t.shape[1], heads, d).transpose(1, 2) for t in (q, k, v))
    return ((qh @ kh.transpose(-1, -2)) * scale).softmax(-1).matmul(vh).transpose(1, 2).reshape(B, Lq, C)


@pytest.mark.parametrize("D,heads,L", [(40, 8, 4096), (64, 5, 1024), (80, 8, 1024)])
def test_self_attention_wgmma(D, heads, L):
    from followyourclick_b200 import ops
    NB, C = 2, heads * D
    q, k, v = rnd((NB, L, C), 1), rnd((NB, L, C), 2), rnd((NB, L, C), 3)
    sc = D ** -0.5
    ref = _mha(q, k, v, heads, sc)

    def run(dt):
        vt = ops.transpose_tokens(v.to(dt).contiguous(), 0, C)
        if D == 80:
            qkv = torch.cat([q, k, v], -1).to(dt).contiguous()
            assert ops.self_attention_tc80_ok(dt, L, D)
            return ops.self_attention_tc_d80(qkv, 0, C, vt, heads, sc)
        assert ops.self_attention_tc_ok(dt, L, D)
        if D == 64:
            return ops.self_attention_tc(torch.cat([q, k, v], -1).to(dt).contiguous(), 0, C, vt, heads, D, sc)
        qk = torch.zeros((NB, L, 2, heads, 64), device="cuda")
        qk[:, :, 0, :, :D], qk[:, :, 1, :, :D] = q.view(NB, L, heads, D), k.view(NB, L, heads, D)
        return ops.self_attention_tc(qk.view(NB, L, 2 * heads * 64).to(dt), 0, heads * 64, vt, heads, D, sc)
    compare(f"self_attention_tc[D{D}x{heads}x{L}]", run, ref)


@pytest.mark.parametrize("T", [0, 4, 16])
@pytest.mark.parametrize("D,heads,Lq", [(40, 8, 4096), (64, 10, 1024), (80, 8, 1024)])
def test_cross_attention_wgmma_with_ip_keys(D, heads, Lq, T):
    from followyourclick_b200 import ops
    NB, div, Lk, C = 4, 2, 77, heads * D
    NBc, dkp = NB // div, ops.cross_dkp(D)
    q, kt, vt_, ki, vi = rnd((NB, Lq, C), 1), rnd((NBc, Lk, C), 2), rnd((NBc, Lk, C), 3), rnd((NBc, max(T, 1), C), 4), rnd((NBc, max(T, 1), C), 5)
    sc, a1, a2 = D ** -0.5, 1.0, 0.7
    rep = lambda t: t.repeat_interleave(div, 0)
    ref = a1 * _mha(q, rep(kt), rep(vt_), heads, sc)
    if T:
        ref = ref + a2 * _mha(q, rep(ki), rep(vi), heads, sc)

    def pack_k(k, rows):
        p = torch.zeros((NBc, rows, heads, dkp), device="cuda")
        p[:, :k.shape[1], :, :D] = k.view(NBc, k.shape[1], heads, D)
        return p.view(NBc, rows, heads * dkp)

    def pack_vt(v, rows):
        p = torch.zeros((NBc, C, rows), device="cuda")
        p[:, :, :v.shape[1]] = v.transpose(1, 2)
        return p

    def run(dt):
        assert ops.cross_attention_tc_ok(dt, D, Lk, T)
        out = torch.empty((NB, Lq, C), dtype=dt, device="cuda")
        extra = dict(k2=pack_k(ki, 16).to(dt), vt2=pack_vt(vi, 16).to(dt), Lk2=T, alpha2=a2) if T else {}
        return ops.cross_attention_tc(q.to(dt), pack_k(kt, 80).to(dt), pack_vt(vt_, 80).to(dt), heads, D, sc, Lk, out, out_alpha=a1,
                                      kv_batch_div=div, **extra)
    compare(f"cross_attention_tc[D{D}x{heads}x{Lq}+T{T}]", run, ref)


@pytest.mark.parametrize("heads,D,Lq,Lk,T", [(8, 160, 256, 77, 16), (8, 40, 1024, 1024, 0), (4, 80, 100, 77, 4), (2, 160, 64, 64, 0)])
def test_attention_mma_sync(heads, D, Lq, Lk, T):
    from followyourclick_b200 import ops
    B, C = 4, heads * D
    q, k, v = rnd((B, Lq, C), 1), rnd((B, Lk, C), 2), rnd((B, Lk, C), 3)
    k2, v2 = rnd((B, max(T, 1), C), 4), rnd((B, max(T, 1), C), 5)
    sc = D ** -0.5
    ref = _mha(q, k, v, heads, sc) + (0.5 * _mha(q, k2, v2, heads, sc) if T else 0)

    def run(dt):
        extra = dict(k2=k2.to(dt), v2=v2.to(dt), alpha2=0.5) if T else {}
        return ops.attention(q.to(dt), k.to(dt), v.to(dt), heads, sc, impl=ops.L.IMPL_TC, **extra)
    compare(f"attention_mma[{heads}x{D}x{Lq}x{Lk}+{T}]", run, ref)


@pytest.mark.parametrize("F", [16, 32])
@pytest.mark.parametrize("D,heads,HW", [(40, 8, 4096), (80, 8, 1024), (160, 8, 64)])
def test_temporal_attention(F, D, heads, HW):
    from followyourclick_b200 import ops
    B, C = 2, heads * D
    qkv = rnd((B, F, HW, 3 * C), 1)
    sc = D ** -0.5
    t = qkv.permute(0, 2, 1, 3).reshape(B * HW, F, 3 * C)
    ref = _mha(t[..., :C], t[..., C:2 * C], t[..., 2 * C:], heads, sc).reshape(B, HW, F, C).permute(0, 2, 1, 3)
    compare(f"temporal_attention[F{F}xD{D}xHW{HW}]", lambda dt: ops.temporal_attention(qkv.to(dt), heads, sc), ref)


# ---------------------------------------------------------------------------------------------------------------- norms, elementwise
@pytest.mark.parametrize("NB,R,C,G,stat,silu", [(2, 16 * 4096, 320, 32, 2, True), (32, 4096, 320, 32, 32, False), (2, 16 * 64, 1280, 32, 2, True),
                                                 (4, 64, 40, 8, 4, True)])
def test_groupnorm(NB, R, C, G, stat, silu):
    from followyourclick_b200 import ops
    x, g, b = rnd((NB, R, C), 1) * 2 + 0.5, 1 + 0.1 * rnd((C,), 2), 0.1 * rnd((C,), 3)
    ref = Fn.group_norm(x.permute(0, 2, 1), G, g, b, 1e-6).permute(0, 2, 1)
    ref = Fn.silu(ref) if silu else ref
    compare(f"groupnorm[{NB}x{R}x{C}]", lambda dt: ops.groupnorm(x.to(dt), g, b, G, 1e-6, silu=silu, stat_batches=stat), ref)


def test_groupnorm_two_sources():
    from followyourclick_b200 import ops
    NB, R, C1, C2, G = 2, 1024, 1280, 640, 32
    x1, x2 = rnd((NB, R, C1), 1), rnd((NB, R, C2), 2) * 3
    g, b = 1 + 0.1 * rnd((C1 + C2,), 3), 0.1 * rnd((C1 + C2,), 4)
    ref = Fn.silu(Fn.group_norm(torch.cat([x1, x2], -1).permute(0, 2, 1), G, g, b, 1e-5).permute(0, 2, 1))
    compare("groupnorm_concat", lambda dt: ops.groupnorm(x1.to(dt), g, b, G, 1e-5, silu=True, stat_batches=NB, x2=x2.to(dt)), ref)


@pytest.mark.parametrize("M,C", [(32768, 320), (8192, 640), (2048, 1280), (4096, 768), (4096, 160)])
def test_layernorm_with_pe_and_stats(M, C):
    from followyourclick_b200 import ops
    x, g, b = rnd((M, C), 1) * 1.5 + rnd((M, 1), 2) * 3, 1 + 0.1 * rnd((C,), 3), 0.1 * rnd((C,), 4)
    F, rpf = 16, M // 16 if M % 16 == 0 else 1
    pe = 0.1 * rnd((F, C), 5)
    rows = torch.arange(M, device="cuda")
    ref = Fn.layer_norm(x, (C,), g, b, 1e-5) + pe[(rows // rpf) % F]
    compare(f"layernorm_pe[{M}x{C}]", lambda dt: ops.layernorm(x.to(dt), g, b, pe=pe, rows_per_frame=rpf, frames=F), ref)

    def stats(dt):
        xd = x.to(dt)
        assert torch.equal(ops.layernorm_stats(xd), ops.layernorm_stats(xd))
        return ops.layernorm_stats(xd)
    eb, e16 = rel(stats(torch.bfloat16), torch.rsqrt(x.var(1, unbiased=False) + 1e-5)), rel(stats(torch.float16), torch.rsqrt(x.var(1, unbiased=False) + 1e-5))
    record(f"kernels/layernorm_stats[{M}x{C}]", dict(bf16=eb, fp16=e16))
    assert e16 <= RATIO * eb, (e16, eb)


def test_elementwise_and_layout_kernels():
    from followyourclick_b200 import ops
    x = rnd((4096, 640), 1) * 3
    compare("silu", lambda dt: ops.silu(x.to(dt)), Fn.silu(x))
    compare("gelu", lambda dt: ops.gelu(x.to(dt)), Fn.gelu(x))
    s = rnd((64, 4096), 2) * 4
    compare("softmax_rows", lambda dt: ops.softmax_rows(s, dt), s.softmax(-1))
    lat = rnd((2, 4, 16, 64, 64), 3)
    compare("ncfhw_to_nfhwc", lambda dt: ops.ncfhw_to_nfhwc(lat, dt, scale=1 / 0.18215), lat.permute(0, 2, 3, 4, 1) / 0.18215)
    compare("nfhwc_to_ncfhw", lambda dt: ops.nfhwc_to_ncfhw(lat.permute(0, 2, 3, 4, 1).contiguous().to(dt)), lat)
    mask, first = (rnd((1, 1, 1, 64, 64), 4) > 0).float(), rnd((1, 4, 64, 64), 5)
    build = lambda dt: ops.build_unet_input(lat[:1].contiguous(), mask, first, 2, dt, c_pad=16)
    compare("build_unet_input", build, build(torch.float32))          # a pure layout op: its fp32 instantiation is exact
    img = rnd((16, 64, 64, 3), 6)
    compare("frames_finalize", lambda dt: ops.frames_finalize(img.to(dt), 1, 16),
            (img.reshape(1, 16, 64, 64, 3).permute(0, 4, 1, 2, 3) / 2 + 0.5).clamp(0, 1))
    up = rnd((4, 16, 16, 320), 7)
    compare("upsample_concat", lambda dt: (ops.upsample_nearest2x(up.to(dt)), ops.concat_channels(up.to(dt), up.to(dt))),
            (up.repeat_interleave(2, 1).repeat_interleave(2, 2), torch.cat([up, up], -1)))


# ---------------------------------------------------------------------------------------------------------------- mini models
@pytest.fixture
def fp16_models(monkeypatch):
    literal_fp16_to(monkeypatch)
    yield


# fp16 tolerances: the bf16 ones of tests/test_engine_gpu.py (rel-L2 3e-2) scaled by the 8x finer rounding, with head-room
@pytest.mark.parametrize("variant", ["base", "ip", "cam"])
def test_mini_unet_vs_reference_fixture(fp16_models, variant):
    from tests.engine_helpers import run_unet_case
    s16, sb = run_unet_case(variant, torch.float16), run_unet_case(variant, torch.bfloat16)
    record(f"mini/unet_{variant}", dict(fp16=s16, bf16=sb))
    assert s16["finite"] and s16["rel_l2"] < 1e-2 and s16["rel_l2"] < sb["rel_l2"], (s16, sb)


def test_mini_sd2_unet_and_vae_vs_reference_fixture(fp16_models):
    from tests.engine_helpers import run_vae_case
    from tests.sd2_helpers import run_sd2_unet_case
    s16, sb = run_sd2_unet_case(torch.float16), run_sd2_unet_case(torch.bfloat16)
    v16, vb = run_vae_case(torch.float16), run_vae_case(torch.bfloat16)
    record("mini/sd2_unet_vae", dict(sd2_fp16=s16, sd2_bf16=sb, vae_fp16=v16, vae_bf16=vb))
    assert s16["finite"] and s16["rel_l2"] < 1e-2 and s16["rel_l2"] < sb["rel_l2"], (s16, sb)
    assert v16["finite"] and v16["rel_l2"] < 1e-2 and v16["rel_l2"] < vb["rel_l2"], (v16, vb)


def test_mini_pipeline_2_steps_vs_oracle(fp16_models):
    from tests.engine_helpers import run_pipeline_case
    r16, rb = run_pipeline_case(torch.float16, steps=2), run_pipeline_case(torch.bfloat16, steps=2)
    record("mini/pipeline_2steps", dict(fp16=r16, bf16=rb))
    assert r16["finite"] and r16["video_maxabs"] < 0.05 and r16["video_maxabs"] < rb["video_maxabs"] and r16["psnr"] > rb["psnr"], (r16, rb)


def test_pipeline_set_compute_dtype_runs_fp16_kernels(monkeypatch):
    """AnimationPipeline.set_compute_dtype(torch.float16) is the one call a launcher needs: every activation is then fp16"""
    from followyourclick_b200 import ops
    from tests.engine_helpers import make_pipeline, pipeline_call
    pipe, ci, _, _ = make_pipeline(torch.bfloat16)
    pipe.set_compute_dtype(torch.float16)
    seen = set()
    conv = ops.conv3x3
    monkeypatch.setattr(ops, "conv3x3", lambda x, *a, **kw: (seen.add(x.dtype), conv(x, *a, **kw))[1])
    pipe.use_cuda_graph = False
    video = pipeline_call(pipe, ci, 4, 8, 8, 2, 8.0)
    assert seen == {torch.float16} and bool(torch.isfinite(video).all())


@pytest.mark.parametrize("case", ["tok_t4", "img_t16", "res_t4"])
def test_ip_attn_processor_fp16_vs_reference_processor(case, monkeypatch):
    """IPAttnProcessor.set_compute_dtype(torch.float16) against the unmodified reference processor's output (the fixture of
    tests/test_engine_gpu.py): the projections and the fused two-context attention run with fp16 operands, error below bf16's"""
    from followyourclick_b200 import ops
    from followyourclick_b200.ip_adapter import IPAttnProcessor
    from tests.engine_helpers import run_ip_attn_processor_case
    mode = {}
    init = IPAttnProcessor.__init__

    def init_in_mode(self, *a, **kw):
        init(self, *a, **kw)
        self.set_compute_dtype(mode["dt"])
    monkeypatch.setattr(IPAttnProcessor, "__init__", init_in_mode)
    seen = set()
    gemm = ops.gemm
    monkeypatch.setattr(ops, "gemm", lambda A, *a, **kw: (seen.add(A.dtype), gemm(A, *a, **kw))[1])
    res = {}
    for dt, name in ((torch.bfloat16, "bf16"), (torch.float16, "fp16")):
        mode["dt"] = dt
        seen.clear()
        res[name] = run_ip_attn_processor_case(case, dt)
        assert seen == {dt}, (name, seen)
    record(f"ip_attn_processor/{case}", res)
    assert res["fp16"]["finite"] and res["fp16"]["rel_l2"] < 1.5e-2 / 4 and res["fp16"]["rel_l2"] < res["bf16"]["rel_l2"], res


def test_layernorm_stats_aug_mean_split():
    """fyc_layernorm_stats' optional aug row [m_hi, m_hi, m_lo, m_lo, 0, 0, 0, 0] in the storage dtype: m_hi + m_lo carries the row
    mean to 2^-17 relative in bf16; in fp16 to 2^-22 relative while m_lo is normal (|mean| >= 2^-3) and to 2^-25 absolute below, which
    is at least as exact as bf16 for |mean| >= 2^-8"""
    from followyourclick_b200 import _lib, ops
    M, C = 4096, 320
    scale = torch.logspace(-6, 2, M, device="cuda")[:, None]             # row means from ~1e-6 to ~100, both signs
    sign = torch.where(torch.arange(M, device="cuda") % 2 == 0, 1.0, -1.0)[:, None]
    x32 = sign * scale * (1 + 0.5 * rnd((M, C), 1))
    res = {}
    for dt, name in ((torch.bfloat16, "bf16"), (torch.float16, "fp16")):
        x = x32.to(dt)
        rstd = torch.empty(M, device="cuda")
        aug = torch.full((M, 8), 7.0, dtype=dt, device="cuda")
        _lib.check(_lib.lib().fyc_layernorm_stats(x.data_ptr(), rstd.data_ptr(), aug.data_ptr(), M, C, 1e-5, _lib.dtype_code(dt),
                                                   _lib.stream_ptr()))
        torch.cuda.synchronize()
        assert torch.equal(rstd, ops.layernorm_stats(x))
        a = aug.double()
        assert torch.equal(a[:, 0], a[:, 1]) and torch.equal(a[:, 2], a[:, 3]) and bool((a[:, 4:] == 0).all())
        mean = x.double().mean(dim=1)
        err = (a[:, 0] + a[:, 2] - mean).abs()
        slack = 2e-6 * x.double().abs().mean(dim=1)                       # the kernel's own fp32 row sum
        bound = (2.0 ** -17 * mean.abs() if dt == torch.bfloat16 else torch.maximum(2.0 ** -22 * mean.abs(), torch.tensor(2.0 ** -25)))
        res[name] = dict(max_excess=float((err - bound - slack).max()), worst_rel=float((err / mean.abs()).max()))
        assert bool((err <= bound + slack).all()), (name, res[name])
        res[name + "_err"] = err
    big = x32.double().mean(dim=1).abs() >= 2.0 ** -8
    e16, eb = res.pop("fp16_err"), res.pop("bf16_err")
    record("kernels/layernorm_stats_aug", res)
    assert float(e16[big].max()) <= float(eb[big].max()), res


# ---------------------------------------------------------------------------------------------------------------- full size
class ActivationWatch:
    """Records, for every 16-bit activation a GEMM / convolution / GroupNorm / attention call stores (GEGLU outputs, the residual stream,
    every VAE decoder block), whether it is finite and its largest |value|: the range check of the fp16 mode, taken on the stored
    tensors themselves and not on a clamped result."""
    NAMES = ("gemm", "conv3x3", "groupnorm", "layernorm", "self_attention_tc", "self_attention_tc_d80", "cross_attention_tc", "attention",
             "temporal_attention")

    def __init__(self, monkeypatch):
        from followyourclick_b200 import ops
        self.calls = []
        for n in self.NAMES:
            fn = getattr(ops, n)

            def spy(*a, _fn=fn, _n=n, **kw):
                y = _fn(*a, **kw)
                if self.on and y.dtype == torch.float16:
                    self.calls.append((_n, float(y.float().abs().amax()), bool(torch.isfinite(y).all())))
                return y
            monkeypatch.setattr(ops, n, spy)
        self.on = False

    def summary(self, last=None):
        c = self.calls[-last:] if last else self.calls
        return dict(calls=len(c), absmax=max(x[1] for x in c), all_finite=all(x[2] for x in c),
                    absmax_by_op={n: max((x[1] for x in c if x[0] == n), default=0.0) for n in self.NAMES})


def test_frames_finalize_fp16_reports_overflow_instead_of_clipping():
    """an inf or NaN that reached the decoder output must reach the video: the fp16 instantiation turns it into NaN (fminf / fmaxf would
    have clipped it to 0 or 1); finite values are finalised exactly as in bf16 / fp32"""
    from followyourclick_b200 import ops
    x = rnd((4, 8, 8, 3), 1) * 1.5
    x[0, 0, 0] = torch.tensor([float("inf"), float("-inf"), float("nan")])
    x[1, 2, 3, 0] = 65504.0
    v16 = ops.frames_finalize(x.half(), 1, 4)
    ref = (x.half().float().reshape(1, 4, 8, 8, 3).permute(0, 4, 1, 2, 3) / 2 + 0.5).clamp(0, 1)
    bad = ~torch.isfinite(x.reshape(1, 4, 8, 8, 3).permute(0, 4, 1, 2, 3))
    assert int(bad.sum()) == 3 and bool(torch.isnan(v16[bad]).all())
    assert torch.equal(v16[~bad], ref[~bad]) and bool((v16[~bad] >= 0).all() and (v16[~bad] <= 1).all())
    assert float(v16[0, 0, 1, 2, 3]) == 1.0                  # 65504 is finite: clamped like any other bright pixel


def test_full_width_unet_cfg2_taps_fp16(cuda, monkeypatch):
    """cfg2 (64x64x16f, B = 2) full-width UNet forward, bf16 and fp16 engine against the fp32 oracle at every tap; every stored fp16
    activation of the forward (residual stream, GEGLU outputs, attention outputs) finite, largest |value| recorded"""
    from tests import test_full_parity_gpu as P
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    unet, _ = P.full_models(cuda)
    inp = P.unet_case_inputs(16, 64, 64, cuda)
    ref_out, ref_taps = P._oracle_unet(unet, inp)
    torch.cuda.empty_cache()
    watch = ActivationWatch(monkeypatch)
    res = {}
    try:
        for dt, name in ((torch.bfloat16, "bf16"), (torch.float16, "fp16")):
            unet.set_compute_dtype(dt)
            unet._taps = {}
            watch.on = dt == torch.float16
            try:
                out = unet(inp["sample"], inp["t"], encoder_hidden_states=inp["ctx"], use_fps_condition=True, fps_tensor=inp["fps"],
                           flow_control=inp["flow"]).sample
                torch.cuda.synchronize()
                taps = unet._taps
            finally:
                unet._taps = None
                watch.on = False
            r = {k: dict(P.err(taps[k], ref_taps[k]), engine_absmax=float(taps[k].abs().max())) for k in ref_taps}
            r["out"] = P.err(out.cpu().permute(0, 2, 3, 4, 1), ref_out.permute(0, 2, 3, 4, 1))
            res[name] = r
    finally:
        unet.set_compute_dtype(torch.float32)
    res["fp16_activations"] = watch.summary()
    record("full/unet_cfg2_taps", res)
    for name in ("bf16", "fp16"):
        assert all(v["finite"] for v in res[name].values()), name
    act = res["fp16_activations"]
    assert act["calls"] > 500 and act["all_finite"] and act["absmax"] < 65504, act
    assert res["fp16"]["out"]["rel_l2"] <= P.TOL["unet_bf16_out"] and res["fp16"]["out"]["rel_l2"] < res["bf16"]["out"]["rel_l2"], res["fp16"]["out"]
    assert max(v["rel_l2"] for v in res["fp16"].values()) <= P.TOL["unet_bf16_tap"]


def test_full_width_vae_decode_16_frames_512_fp16(cuda, monkeypatch):
    """the KL-f8 decoder at the bench size (16 latents 64x64 -> 512x512) in bf16 and fp16 against the fp32 oracle, on the UNCLAMPED
    decoder output; every stored fp16 activation (the late 512x512 / 128-channel blocks included) finite, largest |value| recorded"""
    from oracle import ref_vae
    from tests import test_full_parity_gpu as P
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    _, vae = P.full_models(cuda)
    z = torch.randn(16, 4, 64, 64, generator=torch.Generator().manual_seed(5)).to(cuda)
    with torch.no_grad():
        sd = P.oracle_sd(vae)
        ref = torch.cat([ref_vae.vae_decode(sd, ref_vae.default_vae_config(), z[i:i + 1]).cpu() for i in range(16)])
    torch.cuda.empty_cache()
    watch = ActivationWatch(monkeypatch)
    res = {}
    try:
        for dt, name in ((torch.bfloat16, "bf16"), (torch.float16, "fp16")):
            vae.set_compute_dtype(dt)
            watch.on = dt == torch.float16
            out = vae.decode(z).sample
            torch.cuda.synchronize()
            watch.on = False
            res[name] = dict(P.err(out.cpu().permute(0, 2, 3, 1), ref.permute(0, 2, 3, 1)), out_absmax=float(out.abs().max()))
    finally:
        vae.set_compute_dtype(torch.float32)
    n_late = 12                                              # the last up block's resnets + norm_out + conv_out
    res["fp16_activations"], res["fp16_activations_late_blocks"] = watch.summary(), watch.summary(last=n_late)
    record("full/vae_decode_16x512", res)
    assert res["bf16"]["finite"] and res["fp16"]["finite"], res
    assert res["fp16_activations"]["all_finite"] and res["fp16_activations"]["absmax"] < 65504, res["fp16_activations"]
    assert res["fp16"]["rel_l2"] <= P.TOL["vae_bf16"] and res["fp16"]["rel_l2"] < res["bf16"]["rel_l2"], res


def test_full_width_pipeline_cfg2_25_steps_fp16(cuda):
    """the headline configuration (64x64x16f, 25 DDIM steps, CFG 8) in bf16 and fp16 against the fp32 oracle loop on the device.  The
    finiteness checks are on the final latents and on the decoder's unclamped output, which frames_finalize would clip."""
    from oracle import ref_pipeline, ref_unet, ref_vae
    from oracle.ref_ddim import default_scheduler_config
    from followyourclick_b200 import ops
    from tests import test_full_parity_gpu as P
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    unet, vae = P.full_models(cuda)
    F, h, w, steps, gs = 16, 64, 64, 25, 8.0
    ci = P.clip_inputs(F, h, w, cuda)
    fps, flow = torch.tensor([2]), torch.tensor([4])
    with torch.no_grad():
        lat_ref = ref_pipeline.denoise(P.oracle_sd(unet), ref_unet.default_unet_config(), default_scheduler_config(), ci["latents"],
                                       ci["text_embeddings"], steps, gs, first_image_latents=ci["first_image_latents"],
                                       first_images_mask=ci["first_images_mask"], fps_tensor=fps, flow_control=flow)
        video_ref = ref_vae.decode_latents(P.oracle_sd(vae), ref_vae.default_vae_config(), lat_ref).cpu()
    torch.cuda.empty_cache()
    out = {}
    try:
        for dt, name in ((torch.bfloat16, "bf16"), (torch.float16, "fp16")):
            pipe = P._pipeline(unet, vae, ci["text_embeddings"])
            pipe.set_compute_dtype(dt)
            lat = pipe.denoise(ci["latents"], ci["text_embeddings"], steps, gs, first_image_latents=ci["first_image_latents"],
                               first_images_mask=ci["first_images_mask"], use_first_frame_mask_condition_concat=True, fps_tensor=fps,
                               flow_control=flow, use_fps_condition=True)
            video = pipe.decode_latents_device(lat).cpu()
            frames = vae.decode_nhwc(ops.ncfhw_to_nfhwc(lat.contiguous(), dt, scale=1 / 0.18215).view(F, h, w, 4))
            out[name] = dict(final_latent_rel_l2=P.rel(lat, lat_ref), video_psnr_db=P._psnr(video, video_ref),
                             video_maxabs=float((video - video_ref).abs().max()), latents_finite=bool(torch.isfinite(lat).all()),
                             latents_absmax=float(lat.abs().max()), frames_finite=bool(torch.isfinite(frames).all()),
                             frames_absmax=float(frames.float().abs().max()), video_finite=bool(torch.isfinite(video).all()))
    finally:
        unet.set_compute_dtype(torch.float32)
        vae.set_compute_dtype(torch.float32)
    record("full/pipeline_cfg2_25steps", out)
    r = out["fp16"]
    assert r["latents_finite"] and r["frames_finite"] and r["video_finite"], out
    assert r["video_psnr_db"] >= out["bf16"]["video_psnr_db"] and r["video_psnr_db"] >= P.TOL["pipe_bf16_psnr_db"], out
