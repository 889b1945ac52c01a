"""Tensor-core GEMM / convolution epilogue (GPU): the output half-tiles are staged in shared memory and written by TMA stores clipped at
the output tensor's extent, and the residual is TMA-loaded into the same buffer.  These cases check what that changes: ragged M and N,
outputs that are row / column slices of a wider buffer (canary fill around the written region must stay untouched), a residual that
aliases the output, fp32 output, GEGLU and the LayerNorm fold with row bias, every convolution patch geometry, and the stride-2 and
four-phase upsampler outputs.  Each case is compared with torch fp32 and run twice for bit-identical results.
"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

BF16_TOL = 1.5e-2          # bf16 storage, fp32 accumulation (tests/test_kernels_gpu.py)
F32_OUT_TOL = 4e-3         # bf16 operands, fp32 output
CANARY = -777.0


def rel(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / (b.norm() + 1e-12))


def rnd(shape, seed, dtype=torch.float32, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale).to(dtype).cuda()


@pytest.fixture(autouse=True)
def _tc(cuda):
    from followyourclick_b200 import ops
    ops.set_impl("tc")
    yield
    ops.set_impl("auto")


def framed(M, N, dtype, top=3, left=16, bottom=2, right=32):
    """a canary-filled buffer and its [M, N] window at a non-zero row offset and column offset (ldo > N)"""
    big = torch.full((top + M + bottom, left + N + right), CANARY, dtype=dtype, device="cuda")
    return big, big[top:top + M, left:left + N]


def check_frame(big, M, N, top=3, left=16):
    inner = torch.zeros_like(big, dtype=torch.bool)
    inner[top:top + M, left:left + N] = True
    assert bool((big[~inner] == CANARY).all()), "a store touched memory outside the output window"


@pytest.mark.parametrize("M,N,K", [(128 * 3 + 1, 320, 320), (128 * 3 - 1, 320, 320), (128 * 9 - 30, 320, 512), (128 * 16, 720, 640),
                                   (128 * 5 + 1, 48, 256), (4096 + 64, 1280, 1280), (2000, 960, 320)])
def test_gemm_window_residual(M, N, K):
    """ragged M / N into a row-and-column slice of a wider buffer, with bias and residual"""
    from followyourclick_b200 import ops
    dt = torch.bfloat16
    A, W = rnd((M, K), 1, dt), rnd((N, K), 2, dt, K ** -0.5)
    bias, R = rnd((N,), 3), rnd((M, N), 4, dt)
    ref = A.float() @ W.float().t() + bias + R.float()
    outs = []
    for _ in range(2):
        big, win = framed(M, N, dt)
        o = ops.gemm(A, W, bias=bias, residual=R, out=win)
        assert o.data_ptr() == win.data_ptr()
        check_frame(big, M, N)
        assert rel(win, ref) < BF16_TOL, rel(win, ref)
        outs.append(win.clone())
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("M,N,K", [(128 * 7 + 5, 320, 320), (4096, 640, 640), (300, 1280, 1280)])
def test_gemm_residual_aliases_output(M, N, K):
    """out += A W^T + bias in place (the transformer's proj_out / attention-out pattern)"""
    from followyourclick_b200 import ops
    dt = torch.bfloat16
    A, W, bias = rnd((M, K), 1, dt), rnd((N, K), 2, dt, K ** -0.5), rnd((N,), 3)
    R0 = rnd((M, N), 4, dt)
    ref = A.float() @ W.float().t() + bias + R0.float()
    outs = []
    for _ in range(2):
        R = R0.clone()
        o = ops.gemm(A, W, bias=bias, residual=R, out=R)
        assert o.data_ptr() == R.data_ptr() and rel(R, ref) < BF16_TOL, rel(R, ref)
        outs.append(R)
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("M,N,K", [(1000, 256, 256), (128 * 4 + 3, 512, 128), (640, 16, 320)])
def test_gemm_f32_out(M, N, K):
    """fp32 output (BN capped at 128) with bias, row bias and an fp32 residual, into a framed window"""
    from followyourclick_b200 import ops
    dt = torch.bfloat16
    rpg = 64
    A, W = rnd((M, K), 1, dt), rnd((N, K), 2, dt, K ** -0.5)
    bias, rb, R = rnd((N,), 3), rnd(((M + rpg - 1) // rpg, N), 4), rnd((M, N), 5)
    ref = A.float() @ W.float().t() + bias + rb.repeat_interleave(rpg, dim=0)[:M] + R
    outs = []
    for _ in range(2):
        big, win = framed(M, N, torch.float32)
        ops.gemm(A, W, bias=bias, rowbias=rb, rows_per_group=rpg, residual=R, out_f32=True, out=win)
        check_frame(big, M, N)
        assert rel(win, ref) < F32_OUT_TOL, rel(win, ref)
        outs.append(win.clone())
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("M,C", [(128 * 3 + 1, 320), (128 * 21, 640)])
def test_gemm_geglu_ln_fold(M, C):
    """LayerNorm-folded GEGLU (the feed-forward's first projection) on a ragged M, into a framed window"""
    from followyourclick_b200 import ops
    from followyourclick_b200.modeling import geglu_interleave
    dt = torch.bfloat16
    x = (rnd((M, C), 1) * 1.3 + rnd((M, 1), 2)).to(dt)
    w, b = rnd((8 * C, C), 3, torch.float32, C ** -0.5), 0.05 * rnd((8 * C,), 4)
    gamma, beta = 1 + 0.1 * rnd((C,), 5), 0.05 * rnd((C,), 6)
    wp, cb = ops.ln_fold_weight(w, gamma, dt), (w @ beta + b).contiguous()
    wi, cbi = geglu_interleave(wp.float(), cb)
    wi, cbi = wi.to(dt).contiguous(), cbi.contiguous()
    h = F.layer_norm(x.float(), (C,), gamma, beta, 1e-5) @ w.t() + b
    a, g = h.chunk(2, dim=-1)
    ref = a * F.gelu(g)
    outs = []
    for _ in range(2):
        big, win = framed(M, 4 * C, dt)
        ops.gemm(x, wi, bias=cbi, geglu=True, ln=ops.layernorm_stats(x), out=win)
        check_frame(big, M, 4 * C)
        assert rel(win, ref) < 8e-3, rel(win, ref)
        outs.append(win.clone())
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("M,N,K,rpg", [(128 * 6, 960, 320, 128), (128 * 16, 320, 320, 256)])
def test_gemm_ln_fold_rowbias(M, N, K, rpg):
    """LayerNorm fold with a per-group row bias (the temporal q/k/v projection with its position table)"""
    from followyourclick_b200 import ops
    dt = torch.bfloat16
    x = (rnd((M, K), 1) * 1.7 + rnd((M, 1), 2) * 3.0).to(dt)
    w = rnd((N, K), 3, torch.float32, K ** -0.5)
    gamma, beta, bias = 1 + 0.1 * rnd((K,), 4), 0.05 * rnd((K,), 5), 0.05 * rnd((N,), 6)
    wp, cb = ops.ln_fold_weight(w, gamma, dt), (w @ beta + bias).contiguous()
    rb = rnd((M // rpg, N), 7)
    ref = F.layer_norm(x.float(), (K,), gamma, beta, 1e-5) @ w.t() + bias + rb.repeat_interleave(rpg, dim=0)
    outs = []
    for _ in range(2):
        big, win = framed(M, N, dt)
        ops.gemm(x, wp, bias=cb, rowbias=rb, rows_per_group=rpg, ln=ops.layernorm_stats(x), out=win)
        check_frame(big, M, N)
        assert rel(win, ref) < 6e-3, rel(win, ref)
        outs.append(win.clone())
    assert torch.equal(outs[0], outs[1])


def _conv_ref(x, w, bias, stride=1, pad_mode=0):
    xf = x.float().permute(0, 3, 1, 2)
    wf = w.float().permute(0, 3, 1, 2)
    if pad_mode == 1:
        y = F.conv2d(F.pad(xf, (0, 1, 0, 1)), wf, bias, stride=stride)
    else:
        y = F.conv2d(xf, wf, bias, stride=stride, padding=1)
    return y.permute(0, 2, 3, 1)


# every pick_patch geometry the models use: 64-wide (64 x 2 patch), 32 (32 x 4), 16 (16 x 8), 8 x 8 x 2 images, and the VAE's
# 128-wide rows; plus Cout values with ragged BN choices
@pytest.mark.parametrize("NB,H,W,Cin,Cout", [(1, 64, 64, 64, 320), (2, 32, 32, 64, 640), (2, 16, 16, 128, 1280), (4, 8, 8, 128, 1280),
                                             (1, 8, 256, 64, 128), (1, 128, 128, 32, 48)])
def test_conv_patch_geometries(NB, H, W, Cin, Cout):
    from followyourclick_b200 import ops
    dt = torch.bfloat16
    x, w = rnd((NB, H, W, Cin), 1, dt), rnd((Cout, 3, 3, Cin), 2, dt, (9 * Cin) ** -0.5)
    bias, R = rnd((Cout,), 3), rnd((NB, H, W, Cout), 4, dt)
    ref = _conv_ref(x, w, bias) + R.float()
    o1 = ops.conv3x3(x, w, bias=bias, residual=R)
    assert rel(o1, ref) < BF16_TOL, rel(o1, ref)
    assert torch.equal(o1, ops.conv3x3(x, w, bias=bias, residual=R))


def test_conv_f32_head():
    """the N = 16 fp32-out output head"""
    from followyourclick_b200 import ops
    dt = torch.bfloat16
    x, w = rnd((2, 32, 32, 320), 1, dt), rnd((16, 3, 3, 320), 2, dt, (9 * 320) ** -0.5)
    bias = rnd((16,), 3)
    o = ops.conv3x3(x, w, bias=bias, out_f32=True)
    assert o.dtype == torch.float32 and rel(o, _conv_ref(x, w, bias)) < F32_OUT_TOL
    assert torch.equal(o, ops.conv3x3(x, w, bias=bias, out_f32=True))


@pytest.mark.parametrize("pad_mode", [0, 1])
@pytest.mark.parametrize("NB,H,W,C", [(2, 16, 16, 64), (1, 64, 64, 128), (2, 32, 32, 320)])
def test_conv_stride2(NB, H, W, C, pad_mode):
    from followyourclick_b200 import ops
    dt = torch.bfloat16
    x, w, bias = rnd((NB, H, W, C), 1, dt), rnd((C, 3, 3, C), 2, dt, (9 * C) ** -0.5), rnd((C,), 3)
    o = ops.conv3x3(x, w, bias=bias, stride=2, pad_mode=pad_mode)
    ref = _conv_ref(x, w, bias, stride=2, pad_mode=pad_mode)
    assert o.shape == ref.shape and rel(o, ref) < BF16_TOL, rel(o, ref)
    assert torch.equal(o, ops.conv3x3(x, w, bias=bias, stride=2, pad_mode=pad_mode))


@pytest.mark.parametrize("NB,H,W,Cin,Cout", [(2, 8, 8, 64, 64), (1, 16, 32, 64, 48), (1, 4, 128, 32, 32), (4, 16, 16, 128, 1280)])
def test_conv_upsample_phases(NB, H, W, Cin, Cout):
    from followyourclick_b200 import ops
    from followyourclick_b200.modeling import upsample_phase_weights
    dt = torch.bfloat16
    x = rnd((NB, H, W, Cin), 1, dt)
    w = rnd((Cout, Cin, 3, 3), 2, torch.float32, (9 * Cin) ** -0.5)
    bias = rnd((Cout,), 3)
    wp = w.permute(0, 2, 3, 1).to(dt).contiguous()
    wph = upsample_phase_weights(w).to(dt).contiguous()
    o = ops.conv3x3(x, wp, bias=bias, upsample=2, w_phases=wph)
    ref = F.conv2d(F.interpolate(x.float().permute(0, 3, 1, 2), scale_factor=2.0, mode="nearest"), w.to(dt).float(), bias,
                   padding=1).permute(0, 2, 3, 1)
    assert o.shape == ref.shape and rel(o, ref) < BF16_TOL, rel(o, ref)
    assert torch.equal(o, ops.conv3x3(x, wp, bias=bias, upsample=2, w_phases=wph))
