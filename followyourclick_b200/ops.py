"""Tensor-level wrappers over the C ABI: PyTorch tensors in, PyTorch tensors out.

PyTorch is used for device memory (caching allocator), streams and nothing else: every FLOP below is executed by
a kernel of libfyc_sm90a.so.  All tensors must be CUDA, contiguous in the last dimension; activations are either
all fp32 (strict parity mode) or all bf16 / all fp16 (tensor-core mode).
"""
import ctypes as C
import os

import torch

from . import _lib as L
from ._lib import check, dtype_code, lib, ptr, stream_ptr

_impl = L.IMPL_AUTO
_prof_shapes = False   # per-shape family names in the profile (diagnostics)
_prof = None      # list of (family, algorithmic_flops, algorithmic_bytes, start_event, end_event) while profiling
_pad_flops = 0.0  # FLOPs of the last profile that multiplied zero padding (q/k heads 40 -> 64, 9 -> 16 channel stem, 4 -> 16 channel head)


def note_padding(flops):
    """called by the models where they hand a zero-padded operand to a tensor-core kernel: bench.py reports executed and useful FLOPs"""
    global _pad_flops
    if _prof is not None:
        _pad_flops += float(flops)


def padded_flops():
    return _pad_flops


class profile:
    """Context manager: record a CUDA-event pair around every C-ABI call (bench.py's live per-kernel timing)."""

    def __enter__(self):
        global _prof, _pad_flops
        _prof = []
        _pad_flops = 0.0
        self.records = _prof
        return self

    def __exit__(self, *a):
        global _prof
        _prof = None
        torch.cuda.synchronize()
        self.summary = {}
        for fam, fl, by, e0, e1 in self.records:
            d = self.summary.setdefault(fam, dict(ms=0.0, flops=0.0, bytes=0.0, launches=0))
            d["ms"] += e0.elapsed_time(e1); d["flops"] += fl; d["bytes"] += by; d["launches"] += 1
        return False


class _rec:
    def __init__(self, fam, flops=0.0, nbytes=0.0):
        self.a = (fam, float(flops), float(nbytes))

    def __enter__(self):
        if _prof is not None:
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e1 = torch.cuda.Event(enable_timing=True)
            self.e0.record()
        return self

    def __exit__(self, *a):
        if _prof is not None:
            self.e1.record()
            _prof.append(self.a + (self.e0, self.e1))
        return False


def set_impl(name):
    """'auto' (tensor-core kernels where eligible), 'simt' (CUDA-core kernels only) or 'tc' (fail if not eligible)."""
    global _impl
    _impl = {"auto": L.IMPL_AUTO, "simt": L.IMPL_SIMT, "tc": L.IMPL_TC}[name]


def get_impl():
    return {L.IMPL_AUTO: "auto", L.IMPL_SIMT: "simt", L.IMPL_TC: "tc"}[_impl]


def _cuda(t, name):
    if t is None:
        return
    if not t.is_cuda:
        raise L.FycError(f"{name}: tensor must live on a CUDA device (the engine has no CPU path)")
    if t.stride(-1) != 1:
        raise L.FycError(f"{name}: last dimension must be contiguous")


def require_cuda(t, what):
    """The engine has no CPU path: every model entry point calls this on its input."""
    if not t.is_cuda:
        raise RuntimeError(f"{what} runs only on CUDA (H100); the CPU path is the reference/oracle")


def _f32vec(t, name):
    if t is not None and (t.dtype != torch.float32 or not t.is_contiguous()):
        raise L.FycError(f"{name}: expected a contiguous fp32 tensor")


HALF_DTYPES = (torch.bfloat16, torch.float16)     # the 16-bit storage formats of the tensor-core mode
COMPUTE_DTYPES = (torch.float32,) + HALF_DTYPES    # what set_compute_dtype accepts


def check_compute_dtype(dtype):
    """the argument check every set_compute_dtype shares: ValueError unless dtype is fp32, bf16 or fp16"""
    if dtype not in COMPUTE_DTYPES:
        raise ValueError(f"unsupported compute dtype {dtype}: expected torch.float32, torch.bfloat16 or torch.float16")


def tc_available():
    """does this device run the tensor-core kernels?  The one hardware query under every route rule below (the CPU tests' kernel
    emulator answers it with True and keeps the rules themselves)."""
    return lib().fyc_tcgen05_available() == 1


def _tc_open(dtype, impl):
    """the tensor-core routes are open to a call: 16-bit operands, neither the global setting nor the call's ``impl`` is IMPL_SIMT,
    and the device runs the tensor-core kernels"""
    return _impl != L.IMPL_SIMT and impl != L.IMPL_SIMT and dtype in HALF_DTYPES and tc_available()


def tc_ok(dtype, M, impl=None):
    return M >= 64 and _tc_open(dtype, impl)


use_ln_fold = os.environ.get("FYC_LN_FOLD", "1") != "0"          # A/B switch: LayerNorm folded into the consuming GEMM's epilogue


def ln_fold_ok(dtype, M, C, impl=None):
    """can a LayerNorm over C channels feeding a GEMM on M rows be folded into that GEMM (fyc.h FYC_EPI_LNFOLD: tensor-core path only)?"""
    return use_ln_fold and C % 8 == 0 and C <= 2048 and tc_ok(dtype, M, impl)


def layernorm_stats(x, eps=1e-5):
    """x [..., C] -> rstd fp32 [rows]: the statistics pass of a LayerNorm whose scale / shift AND mean subtraction live in the consuming
    GEMM's weights (gamma-scaled, row-centred: fyc.h FYC_EPI_LNFOLD) - one read of x, no normalised copy."""
    _cuda(x, "layernorm_stats.x")
    assert x.is_contiguous()
    Cc = x.shape[-1]
    M = x.numel() // Cc
    rstd = torch.empty((M,), dtype=torch.float32, device=x.device)
    fam = f"layernorm_stats[{M}x{Cc}]" if _prof_shapes else "layernorm_stats"
    with _rec(fam, 0, x.numel() * x.element_size()):
        check(lib().fyc_layernorm_stats(ptr(x), ptr(rstd), None, M, Cc, float(eps), dtype_code(x.dtype), stream_ptr()))
    return rstd


# significand bits after the point and the smallest normal exponent of each 16-bit format
_ULP_BITS = {torch.bfloat16: (7, -126), torch.float16: (10, -14)}


def _balance_rows(w, dtype, iters=12):
    """w: fp32 tensor holding `dtype`-representable values [N, K] (dtype bf16 or fp16) -> the same with a handful of elements per row moved
    by ONE ulp of `dtype` so that every row sums to ~0 (<= a few 1e-6 instead of ~sqrt(K) * ulp * |w|).  Each step picks, per row, the
    element whose ulp is closest to the remaining row sum and steps it against the sum's sign; a one-ulp step of a representable value is
    always representable (below the smallest normal exponent the ulp is the subnormal spacing)."""
    frac, emin = _ULP_BITS[dtype]
    w = w.clone()
    rows = torch.arange(w.shape[0], device=w.device)
    inf = torch.tensor(float("inf"), device=w.device)
    for _ in range(iters):
        r = w.sum(dim=1)
        ulp = torch.exp2(torch.floor(torch.log2(w.abs().clamp_min(1e-30))).clamp_min(emin) - frac)
        ulp = torch.where(w == 0, inf, ulp)
        target = r.abs()[:, None]
        score = torch.where(ulp <= 1.5 * target, (target - ulp).abs(), inf)
        idx = score.argmin(dim=1)
        good = torch.isfinite(score[rows, idx])
        step = torch.where(good, ulp[rows, idx] * torch.sign(r), torch.zeros_like(r))
        w[rows, idx] -= torch.where(torch.isfinite(step), step, torch.zeros_like(step))
    return w


def ln_fold_weight(w, gamma, dtype):
    """[N, K] fp32 weight, [K] LayerNorm gain -> the LN-folded GEMM operand: gamma-scaled, every row centred (the mean of LN's input then
    cancels inside the product: x W"^T = x W'^T - mean colsum), rounded ONCE to the compute dtype; in bf16 / fp16 the rounded rows are
    re-balanced to sum to zero (_balance_rows): the leftover row sum is what a large row mean would multiply - with it the fold is
    as accurate as LN -> bf16 -> GEMM for row means of 100 sigma, without it only for means below ~2 sigma (tests/test_kernels_gpu.py)."""
    wp = w.float() * gamma.float()[None, :]
    wc = (wp - wp.mean(dim=1, keepdim=True)).to(dtype)
    if dtype in HALF_DTYPES:
        wc = _balance_rows(wc.float(), dtype).to(dtype)
    return wc.contiguous()


use_dual_source = os.environ.get("FYC_DUAL_SOURCE", "1") != "0"  # A/B switch: skip-concat read in place (two-source GroupNorm / shortcut GEMM)


def gemm(A, W, bias=None, residual=None, rowbias=None, rows_per_group=0, alpha=1.0, geglu=False, out_f32=False,
         out=None, impl=None, ln=None, A2=None):
    """out[M, N] = alpha * A[M, K] @ W[N, K]^T (+bias) (+rowbias[m // rows_per_group]) (+residual); GEGLU halves N.
    A may be 2-D [M, K] or batched 3-D [B, M, K] with W [B, N, K] (one launch per batch on the tensor-core path).
    ``ln`` = rstd [M] from layernorm_stats: A is the RAW input of a LayerNorm, W = ln_fold_weight(...) (gamma-scaled, row-centred),
    ``bias`` carries the beta term - out = rstd * (A W^T) + bias (fyc.h FYC_EPI_LNFOLD).
    ``A2`` [M, K2]: the K dimension is the concatenation [A | A2] read in place."""
    _cuda(A, "gemm.A"); _cuda(W, "gemm.W"); _cuda(residual, "gemm.residual"); _cuda(A2, "gemm.A2")
    _f32vec(bias, "gemm.bias"); _f32vec(rowbias, "gemm.rowbias")
    impl = _impl if impl is None else impl
    K1 = 0
    if A2 is not None:
        # A = [A | A2] along K without the concatenation ever being written (fyc.h A2): tensor-core path with K1 % 64 == 0, else concatenate
        assert A.dim() == 2 and A2.dim() == 2 and A2.shape[0] == A.shape[0] and A2.dtype == A.dtype
        if tc_ok(A.dtype, A.shape[0], impl) and A.shape[1] % 64 == 0 and A2.shape[1] % 8 == 0 and use_dual_source:
            K1 = A.shape[1]
        else:
            A, A2 = concat_channels(A.contiguous(), A2.contiguous()), None
    if ln is not None:
        _f32vec(ln, "gemm.ln_rstd")
        assert A2 is None and A.dim() == 2 and ln.shape == (A.shape[0],)
    batched = A.dim() == 3
    if batched:
        Bn, M, K = A.shape
        N = W.shape[1]
        sA, sW, lda, ldw = A.stride(0), W.stride(0), A.stride(1), W.stride(1)
    else:
        Bn, (M, K), N = 1, A.shape, W.shape[0]
        sA = sW = 0
        lda, ldw = A.stride(0), W.stride(0)
    if K1:
        K = K1 + A2.shape[1]
    assert W.shape[-1] == K and W.dtype == A.dtype
    fused_geglu = geglu and tc_ok(A.dtype, M, impl)
    n_out = N // 2 if fused_geglu else N
    if geglu and not fused_geglu and out is not None and not out.is_contiguous():
        # fyc_geglu writes packed [M, N / 2] rows: a wider row stride would put rows in the wrong place and write outside the view
        raise L.FycError("gemm: the unfused GEGLU epilogue (CUDA-core path) writes a contiguous output; got row stride "
                         f"{out.stride(-2)} for {N // 2} columns")
    odt = torch.float32 if out_f32 else A.dtype
    if out is None or (geglu and not fused_geglu):
        o = torch.empty((Bn, M, n_out) if batched else (M, n_out), dtype=odt, device=A.device)
    else:
        o = out
    epi = (L.EPI_BIAS if bias is not None else 0) | (L.EPI_RESIDUAL if residual is not None else 0) | \
          (L.EPI_ROWBIAS if rowbias is not None else 0) | (L.EPI_GEGLU if fused_geglu else 0) | (L.EPI_OUT_F32 if out_f32 else 0) | \
          (L.EPI_LNFOLD if ln is not None else 0)
    a = L.GemmArgs(ptr(A), ptr(W), ptr(o), ptr(bias), ptr(residual), ptr(rowbias), M, N, K, lda, ldw,
                   o.stride(-2), residual.stride(-2) if residual is not None else 0, Bn, sA, sW,
                   o.stride(0) if batched else 0, rows_per_group, float(alpha), dtype_code(A.dtype), epi, impl,
                   ptr(A2) if K1 else None, A2.stride(0) if K1 else 0, K1, ptr(ln))
    fam = "gemm_tc" if (tc_ok(A.dtype, M, impl) and N % 16 == 0 and K % 8 == 0) else "gemm_simt"
    if _prof_shapes:
        fam += f"[{Bn}x{M}x{N}x{K}{'g' if fused_geglu else ''}{'r' if residual is not None else ''}{'L' if ln is not None else ''}]"
    with _rec(fam, 2.0 * Bn * M * N * K, A.element_size() * Bn * (M * K + N * K + M * n_out)):
        check(lib().fyc_gemm(C.byref(a), stream_ptr()))
    if geglu and not fused_geglu:
        assert not batched
        g = out if out is not None else torch.empty((M, N // 2), dtype=A.dtype, device=A.device)
        check(lib().fyc_geglu(ptr(o), ptr(g), M, N // 2, dtype_code(A.dtype), stream_ptr()))
        return g
    return o


use_up2_phases = os.environ.get("FYC_UP2_PHASES", "1") != "0"    # A/B switch for the four-phase upsample convolution
use_tc_head = os.environ.get("FYC_TC_HEAD", "1") != "0"          # A/B switch: 3- / 4-channel output convs zero-padded to N = 16 on the tensor cores


def up2_phases_ok(dtype, pixels, residual, rowbias, out_f32, impl=None):
    """the host side of the four-phase upsampler route for a conv over ``pixels`` low-res pixels (``residual`` / ``rowbias``: the call's
    operands or None): a bias-only epilogue with a 16-bit output on the tensor cores.  The C query fyc_conv3x3_up2_eligible decides
    the rest (the patch geometry)."""
    return use_up2_phases and residual is None and rowbias is None and not out_f32 and tc_ok(dtype, pixels, impl)


def conv3x3(x, w, bias=None, residual=None, rowbias=None, images_per_group=0, stride=1, upsample=1, out_f32=False, impl=None,
            pad_mode=0, w_phases=None):
    """x [NB, H, W, Cin] (NHWC), w [Cout, 3, 3, Cin] -> [NB, Ho, Wo, Cout]; pad 1 (pad_mode 1: stride-2 conv with the padding on
    the bottom / right only - diffusers Downsample2D(padding=0), used by the VAE encoder).  upsample=2 with ``w_phases``
    ([4, Cout, 2, 2, Cin], modeling.upsample_phase_weights): nearest-x2 + conv as four 2x2-tap convs on the low-res image."""
    _cuda(x, "conv.x"); _cuda(w, "conv.w"); _cuda(residual, "conv.residual"); _cuda(w_phases, "conv.w_phases")
    _f32vec(bias, "conv.bias")
    ld_rb = 0
    if rowbias is not None:        # [groups, Cout] fp32, rows possibly strided (a column block of a wider table: fyc.h ld_rowbias)
        if rowbias.dtype != torch.float32 or rowbias.dim() != 2 or rowbias.stride(1) != 1 or rowbias.shape[1] != w.shape[0]:
            raise L.FycError("conv.rowbias: expected fp32 [groups, Cout] with unit column stride")
        _cuda(rowbias, "conv.rowbias")
        ld_rb = rowbias.stride(0) if rowbias.shape[0] > 1 else rowbias.shape[1]
    assert x.is_contiguous() and w.is_contiguous() and x.dtype == w.dtype
    impl = _impl if impl is None else impl
    NB, H, W_, Cin = x.shape
    Cout = w.shape[0]
    if upsample == 2 and w_phases is not None and up2_phases_ok(x.dtype, NB * H * W_, residual, rowbias, out_f32, impl):
        assert w_phases.is_contiguous() and w_phases.dtype == x.dtype and tuple(w_phases.shape) == (4, Cout, 2, 2, Cin)
        out = torch.empty((NB, 2 * H, 2 * W_, Cout), dtype=x.dtype, device=x.device)
        a = L.ConvArgs(ptr(x), ptr(w), ptr(out), ptr(bias), None, None, NB, H, W_, Cin, Cout, 1, 2, 0, dtype_code(x.dtype),
                       L.EPI_BIAS if bias is not None else 0, impl, None, 0, 0, ptr(w_phases), 0)
        if lib().fyc_conv3x3_up2_eligible(C.byref(a)) == 1:
            fam = "conv_tc_up2" + (f"[{NB}x{H}x{W_} {Cin}->{Cout}]" if _prof_shapes else "")
            # executed work: 4 phases x 4 taps on the low-res grid (the reference's upsample + 3x3 conv is 36 MACs per input pixel)
            with _rec(fam, 2.0 * NB * H * W_ * Cout * 16 * Cin, x.element_size() * (x.numel() + w_phases.numel() + out.numel())):
                check(lib().fyc_conv3x3(C.byref(a), stream_ptr()))
            return out
    if upsample == 2 and tc_ok(x.dtype, NB * H * W_, impl):
        x = upsample_nearest2x(x)            # the tensor-core path reads unit-stride boxes: materialise the upsample
        NB, H, W_, Cin = x.shape
        upsample = 1
    Ho = (H * upsample + 2 - 3) // stride + 1
    Wo = (W_ * upsample + 2 - 3) // stride + 1
    out = torch.empty((NB, Ho, Wo, Cout), dtype=torch.float32 if out_f32 else x.dtype, device=x.device)
    if residual is not None:
        assert residual.is_contiguous() and residual.shape == out.shape
    epi = (L.EPI_BIAS if bias is not None else 0) | (L.EPI_RESIDUAL if residual is not None else 0) | \
          (L.EPI_ROWBIAS if rowbias is not None else 0) | (L.EPI_OUT_F32 if out_f32 else 0)
    a = L.ConvArgs(ptr(x), ptr(w), ptr(out), ptr(bias), ptr(residual), ptr(rowbias), NB, H, W_, Cin, Cout, stride,
                   upsample, images_per_group, dtype_code(x.dtype), epi, impl, None, 0, pad_mode, None, ld_rb)
    nbytes = lib().fyc_conv3x3_workspace_bytes(C.byref(a))
    ws = None
    if nbytes:
        ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
        a.workspace, a.workspace_bytes = ptr(ws), nbytes
    # the label names the kernel fyc_conv3x3 runs: channel counts alone do not decide it (a 5 x 9 grid has no 128-pixel patch)
    fam = "conv_tc" if lib().fyc_conv3x3_tc_route(C.byref(a)) == 1 else "conv_simt"
    if _prof_shapes:
        fam += f"[{NB}x{Ho}x{Wo} {Cin}->{Cout} s{stride}]"
    with _rec(fam, 2.0 * NB * Ho * Wo * Cout * 9 * Cin, x.element_size() * (x.numel() + w.numel() + out.numel())):
        check(lib().fyc_conv3x3(C.byref(a), stream_ptr()))
    return out


def groupnorm(x, gamma, beta, groups, eps, silu=False, stat_batches=None, x2=None, out=None):
    """x [..., C] contiguous; statistics per (stat batch, group) where x is viewed as [stat_batches, R, C].
    ``x2`` [..., C2]: normalise the channel concatenation [x | x2] (gamma / beta of C + C2 channels) reading both tensors in place
    (fyc_groupnorm_concat: the up blocks' skip concatenation is never written); returns [..., C + C2]."""
    _cuda(x, "groupnorm.x"); _f32vec(gamma, "groupnorm.gamma"); _f32vec(beta, "groupnorm.beta"); _cuda(x2, "groupnorm.x2")
    assert x.is_contiguous()
    C1 = x.shape[-1]
    vec = 8 if x.dtype in HALF_DTYPES else 4
    if x2 is not None and not (use_dual_source and C1 % vec == 0 and x2.shape[-1] % vec == 0):
        x, x2 = concat_channels(x, x2.contiguous()), None
        C1 = x.shape[-1]
    Cc = C1 + (x2.shape[-1] if x2 is not None else 0)
    NB = x.shape[0] if stat_batches is None else stat_batches
    R = x.numel() // (NB * C1)
    if out is None:
        out = torch.empty(x.shape[:-1] + (Cc,), dtype=x.dtype, device=x.device)
    assert out.is_contiguous() and tuple(out.shape) == tuple(x.shape[:-1]) + (Cc,) and out.dtype == x.dtype
    nbytes = lib().fyc_groupnorm_workspace_bytes(NB, Cc, groups)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
    fam = f"groupnorm[{NB}x{R}x{Cc}]" if _prof_shapes else "groupnorm"
    with _rec(fam, 0, 3 * out.numel() * x.element_size()):
        if x2 is None:
            check(lib().fyc_groupnorm(ptr(x), ptr(gamma), ptr(beta), ptr(out), NB, R, Cc, groups, float(eps), int(silu),
                                      dtype_code(x.dtype), ptr(ws), nbytes, stream_ptr()))
        else:
            assert x2.is_contiguous() and x2.shape[:-1] == x.shape[:-1] and x2.dtype == x.dtype
            check(lib().fyc_groupnorm_concat(ptr(x), C1, ptr(x2), x2.shape[-1], ptr(gamma), ptr(beta), ptr(out), NB, R, groups, float(eps),
                                             int(silu), dtype_code(x.dtype), ptr(ws), nbytes, stream_ptr()))
    return out


def layernorm(x, gamma, beta, eps=1e-5, pe=None, rows_per_frame=0, frames=0):
    _cuda(x, "layernorm.x"); _f32vec(gamma, "layernorm.gamma"); _f32vec(beta, "layernorm.beta"); _f32vec(pe, "layernorm.pe")
    assert x.is_contiguous()
    Cc = x.shape[-1]
    out = torch.empty_like(x)
    fam = f"layernorm[{x.numel() // Cc}x{Cc}]" if _prof_shapes else "layernorm"
    with _rec(fam, 0, 2 * x.numel() * x.element_size()):
        check(lib().fyc_layernorm(ptr(x), ptr(gamma), ptr(beta), ptr(out), x.numel() // Cc, Cc, float(eps), ptr(pe),
                                  rows_per_frame, frames, dtype_code(x.dtype), stream_ptr()))
    return out


def attention(q, k, v, heads, scale, out=None, out_alpha=1.0, accumulate=False, kv_batch_div=1, impl=None, k2=None, v2=None, alpha2=1.0):
    """q [B, Lq, >=heads*D] / k, v [B', Lk, ...] are (possibly strided) views; head h occupies columns [h*D, (h+1)*D).
    Returns out [B, Lq, heads*D].  B' = B / kv_batch_div.  With ``k2`` / ``v2`` [B', Lk2, ...] (the IP-Adapter's image keys):
    out = out_alpha * softmax(scale q k^T) v + alpha2 * softmax(scale q k2^T) v2 in ONE launch (fyc.h: second context)."""
    for t, n in ((q, "q"), (k, "k"), (v, "v"), (k2, "k2"), (v2, "v2")):
        _cuda(t, "attention." + n)
    B, Lq, _ = q.shape
    Lk = k.shape[1]
    if out is None:
        assert not accumulate
        assert q.shape[2] % heads == 0
        out = torch.empty((B, Lq, q.shape[2]), dtype=q.dtype, device=q.device)
    D = out.shape[2] // heads
    a = L.AttnArgs(ptr(q), ptr(k), ptr(v), ptr(out), B, heads, Lq, Lk, D, q.stride(1), k.stride(1), v.stride(1),
                   out.stride(1), q.stride(0), k.stride(0), v.stride(0), out.stride(0), kv_batch_div, float(scale),
                   float(out_alpha), int(accumulate), dtype_code(q.dtype), _impl if impl is None else impl,
                   ptr(k2), ptr(v2), 0, 0, 0, 0, 0, float(alpha2))
    Lk2 = 0
    if k2 is not None:
        assert v2 is not None and k2.shape[0] == k.shape[0] and v2.shape[:2] == k2.shape[:2]
        Lk2 = k2.shape[1]
        a.Lk2, a.ldk2, a.ldv2, a.bsk2, a.bsv2 = Lk2, k2.stride(1), v2.stride(1), k2.stride(0), v2.stride(0)
    with _rec(f"attention[{B}x{heads}x{Lq}x{Lk}{'+' + str(Lk2) if Lk2 else ''}x{D}]" if _prof_shapes else "attention", 4.0 * B * heads * Lq * (Lk + Lk2) * D,
              q.element_size() * (2 * B * Lq * heads * D + 2 * (B // kv_batch_div) * (Lk + Lk2) * heads * D)):
        check(lib().fyc_attention(C.byref(a), stream_ptr()))
    return out


def transpose_tokens(x, col0, C):
    """x [NB, L, ld] (bf16 / fp16) -> columns [col0, col0+C) transposed per batch entry: [NB, C, L]."""
    assert x.dtype in HALF_DTYPES and x.dim() == 3 and x.stride(2) == 1 and x.stride(0) == x.shape[1] * x.stride(1)
    NB, L, _ = x.shape
    out = torch.empty((NB, C, L), dtype=x.dtype, device=x.device)
    with _rec("transpose", 0, 2 * NB * L * C * 2):
        check(lib().fyc_transpose_tokens(ptr(x), ptr(out), NB, L, C, x.stride(1), col0, stream_ptr()))
    return out


def _tc_entry(name, t):
    """the wgmma attention entry point for t's 16-bit dtype: `name` (bf16) or `name`_f16 (fp16)"""
    if t.dtype not in HALF_DTYPES:
        raise L.FycError(f"{name}: 16-bit operands required (got {t.dtype})")
    return getattr(lib(), name + "_f16" if t.dtype == torch.float16 else name)


def self_attention_tc_ok(dtype, L, D, impl=None):
    return D in (40, 64) and L % 128 == 0 and _tc_open(dtype, impl)


def self_attention_tc(qk, q_col0, k_col0, vt, heads, D, scale):
    """tensor-core self-attention: qk [NB, L, ld] with 64-wide q/k heads (D = 40: zero-padded, D = 64: the fused projection as is),
    vt [NB, heads*D, L] -> [NB, L, heads*D]."""
    NB, L, _ = qk.shape
    out = torch.empty((NB, L, heads * D), dtype=qk.dtype, device=qk.device)
    with _rec("attention_tc", 4.0 * NB * heads * L * L * D, qk.element_size() * (4 * NB * L * heads * D)):
        check(_tc_entry("fyc_self_attention_tc", qk)(ptr(qk), qk.stride(1), q_col0, k_col0, ptr(vt), ptr(out), out.stride(1), NB, heads, L, D,
                                          float(scale), stream_ptr()))
    return out


use_attn_d80 = os.environ.get("FYC_ATTN_D80", "1") != "0"        # A/B switch: head-dim-80 self-attention on the wgmma kernel (else the mma.sync kernel)


def self_attention_tc80_ok(dtype, L, D, impl=None):
    return use_attn_d80 and D == 80 and L % 256 == 0 and _tc_open(dtype, impl)


def self_attention_tc_d80(qkv, q_col0, k_col0, vt, heads, scale):
    """tensor-core self-attention for head dim 80: qkv [NB, L, ld] with UNPADDED 80-wide q / k heads (the fused projection as is), vt
    [NB, heads * 80, L] -> [NB, L, heads * 80]."""
    NB, L, _ = qkv.shape
    D = 80
    out = torch.empty((NB, L, heads * D), dtype=qkv.dtype, device=qkv.device)
    with _rec(f"attention_tc80[{NB}x{heads}x{L}]" if _prof_shapes else "attention_tc", 4.0 * NB * heads * L * L * D, qkv.element_size() * (4 * NB * L * heads * D)):
        check(_tc_entry("fyc_self_attention_tc_d80", qkv)(ptr(qkv), qkv.stride(1), q_col0, k_col0, ptr(vt), ptr(out), out.stride(1), NB, heads, L,
                                              float(scale), stream_ptr()))
    return out


use_cross_tc = os.environ.get("FYC_CROSS_TC", "1") != "0"        # A/B switch: text / image cross-attention on the wgmma kernel (else the mma.sync kernel)
CROSS_LK, CROSS_LK2 = 80, 16                                      # padded key counts of the resident-context kernel


def cross_attention_tc_ok(dtype, D, Lk, Lk2, impl=None):
    return use_cross_tc and D in (40, 64, 80) and 1 <= Lk <= CROSS_LK and 0 <= Lk2 <= CROSS_LK2 and _tc_open(dtype, impl)


def cross_dkp(D):
    """column stride between the heads of the packed context keys: 64 (zero-padded heads) for D = 40, D itself for D = 64 / 80"""
    return 64 if D == 40 else D


def cross_attention_tc(q, k, vt, heads, D, scale, Lk, out, k2=None, vt2=None, Lk2=0, out_alpha=1.0, alpha2=1.0, kv_batch_div=1):
    """tensor-core cross-attention with a resident short context (fyc.h fyc_cross_attention_tc).  q [NB, Lq, >= heads D]; k [NBc, 80, ...] (a view is
    fine: its row stride is passed), vt [NBc, heads D, 80]; k2 [NBc, 16, ...], vt2 [NBc, heads D, 16]; out [NB, Lq, heads D] is written."""
    for t, nme in ((q, "q"), (k, "k"), (vt, "vt"), (k2, "k2"), (vt2, "vt2"), (out, "out")):
        _cuda(t, "cross_attention_tc." + nme)
    NB, Lq, _ = q.shape
    assert k.shape[1] == CROSS_LK and vt.is_contiguous() and tuple(vt.shape[1:]) == (heads * D, CROSS_LK) and k.stride(0) == CROSS_LK * k.stride(1)
    if k2 is not None:
        assert k2.shape[1] == CROSS_LK2 and vt2.is_contiguous() and tuple(vt2.shape[1:]) == (heads * D, CROSS_LK2) and k2.stride(0) == CROSS_LK2 * k2.stride(1)
    assert q.stride(0) == Lq * q.stride(1) and out.stride(0) == Lq * out.stride(1) and k.shape[0] * kv_batch_div == NB
    with _rec(f"cross_attention_tc[{NB}x{heads}x{Lq}x{Lk}+{Lk2}x{D}]" if _prof_shapes else "cross_attention_tc", 4.0 * NB * heads * Lq * (Lk + Lk2) * D,
              q.element_size() * 2 * NB * Lq * heads * D):
        check(_tc_entry("fyc_cross_attention_tc", q)(ptr(q), q.stride(1), 0, ptr(k), k.stride(1), ptr(vt), ptr(k2), k2.stride(1) if k2 is not None else 0,
                                           ptr(vt2), ptr(out), out.stride(1), NB, heads, Lq, D, Lk, Lk2, kv_batch_div, float(scale), float(out_alpha),
                                           float(alpha2), stream_ptr()))
    return out


def temporal_attention(qkv, heads, scale):
    """qkv [B, F, HW, 3C] -> [B, F, HW, C]; softmax over the F frames of each (clip, pixel, head)."""
    _cuda(qkv, "temporal_attention.qkv")
    assert qkv.is_contiguous()
    B, F, HW, C3 = qkv.shape
    Cc = C3 // 3
    out = torch.empty((B, F, HW, Cc), dtype=qkv.dtype, device=qkv.device)
    with _rec(f"temporal_attention[{B}x{F}x{HW}x{heads}x{Cc // heads}]" if _prof_shapes else "temporal_attention", 4.0 * B * HW * heads * F * F * (Cc // heads), (qkv.numel() + out.numel()) * qkv.element_size()):
        check(lib().fyc_temporal_attention(ptr(qkv), ptr(out), B, F, HW, heads, Cc // heads, float(scale),
                                           dtype_code(qkv.dtype), stream_ptr()))
    return out


def softmax_rows(scores, out_dtype):
    assert scores.dtype == torch.float32 and scores.is_contiguous()
    Lk = scores.shape[-1]
    out = torch.empty(scores.shape, dtype=out_dtype, device=scores.device)
    check(lib().fyc_softmax_rows(ptr(scores), ptr(out), scores.numel() // Lk, Lk, dtype_code(out_dtype), stream_ptr()))
    return out


def timestep_embed(t, freqs, flip_sin_to_cos):
    assert t.dtype == torch.int64 and t.is_cuda and freqs.dtype == torch.float32
    n, dim = t.numel(), 2 * freqs.numel()
    out = torch.empty((n, dim), dtype=torch.float32, device=t.device)
    check(lib().fyc_timestep_embed(ptr(t), ptr(freqs), ptr(out), n, dim, int(flip_sin_to_cos), stream_ptr()))
    return out


def silu(x):
    _cuda(x, "silu.x")
    out = torch.empty_like(x)
    check(lib().fyc_silu(ptr(x), ptr(out), x.numel(), dtype_code(x.dtype), stream_ptr()))
    return out


def gelu(x):
    _cuda(x, "gelu.x")
    assert x.is_contiguous()
    out = torch.empty_like(x)
    check(lib().fyc_gelu(ptr(x), ptr(out), x.numel(), dtype_code(x.dtype), stream_ptr()))
    return out


def upsample_nearest2x(x):
    assert x.is_contiguous()
    NB, H, W_, Cc = x.shape
    out = torch.empty((NB, 2 * H, 2 * W_, Cc), dtype=x.dtype, device=x.device)
    check(lib().fyc_upsample_nearest2x(ptr(x), ptr(out), NB, H, W_, Cc, dtype_code(x.dtype), stream_ptr()))
    return out


def concat_channels(a, b):
    assert a.is_contiguous() and b.is_contiguous() and a.shape[:-1] == b.shape[:-1] and a.dtype == b.dtype
    C1, C2 = a.shape[-1], b.shape[-1]
    out = torch.empty(a.shape[:-1] + (C1 + C2,), dtype=a.dtype, device=a.device)
    check(lib().fyc_concat_channels(ptr(a), ptr(b), ptr(out), a.numel() // C1, C1, C2, dtype_code(a.dtype), stream_ptr()))
    return out


def ncfhw_to_nfhwc(x, dtype, scale=1.0):
    """fp32 (b, c, f, h, w) * scale -> dtype [b, f, h, w, c]."""
    assert x.dtype == torch.float32 and x.is_contiguous() and x.is_cuda
    b, c, f, h, w = x.shape
    out = torch.empty((b, f, h, w, c), dtype=dtype, device=x.device)
    check(lib().fyc_ncfhw_to_nfhwc(ptr(x), ptr(out), b, c, f, h * w, float(scale), dtype_code(dtype), stream_ptr()))
    return out


def _channel_sliced(x):
    """x [..., C] that is either contiguous or a leading-channel slice x_full[..., :C] of a contiguous tensor -> channel stride."""
    assert x.stride(-1) == 1
    ld = x.stride(-2)
    # strides of the enclosing contiguous [.., ld] tensor
    want, acc = [1], ld
    for n in reversed(x.shape[:-1]):
        want.insert(0, acc)
        acc *= n
    ok = all(n == 1 or st == wt for n, st, wt in zip(x.shape, x.stride(), want))
    assert ld >= x.shape[-1] and ok, "expected a contiguous tensor or a [..., :C] slice of one"
    return ld


def nfhwc_to_ncfhw(x):
    """dtype [b, f, h, w, c] (or its [..., :c] slice of a wider channels-last tensor) -> fp32 (b, c, f, h, w)."""
    ld = _channel_sliced(x)
    b, f, h, w, c = x.shape
    out = torch.empty((b, c, f, h, w), dtype=torch.float32, device=x.device)
    check(lib().fyc_nfhwc_to_ncfhw(ptr(x), ptr(out), b, c, f, h * w, ld, dtype_code(x.dtype), stream_ptr()))
    return out


def build_unet_input(latents, mask, first, dup, dtype, c_pad=None, out=None):
    """latents (b,4,f,h,w) fp32, mask (b,1,1,h,w) fp32 | None, first (b,4,h,w) fp32 | None -> [dup*b, f, h, w, 9|4]."""
    assert latents.dtype == torch.float32 and latents.is_contiguous() and latents.is_cuda
    b, c, f, h, w = latents.shape
    assert c == 4
    cin = 9 if first is not None else 4
    c_pad = cin if c_pad is None else c_pad
    if out is None:
        out = torch.empty((dup * b, f, h, w, c_pad), dtype=dtype, device=latents.device)
    assert out.shape == (dup * b, f, h, w, c_pad) and out.dtype == dtype and out.is_contiguous()
    check(lib().fyc_build_unet_input(ptr(latents), ptr(mask), ptr(first), ptr(out), b, f, h * w, dup, c_pad, dtype_code(dtype), stream_ptr()))
    return out


FIRST_CONCAT, FIRST_FRAME = 1, 2      # fyc.h FYC_FIRST_*: bits of build_unet_input_first's mode


def build_unet_input_first(latents, first, dup, dtype, mode, c_pad=None, out=None):
    """Step prologue of the first-frame-conditioned models (fyc.h fyc_build_unet_input_first): latents (b,4,f,h,w) fp32, first (b,4,h,w)
    fp32 -> [dup*b, f, h, w, 8 | 4].  ``mode`` & FIRST_CONCAT: [latents | first on every frame]; ``mode`` & FIRST_FRAME: frame 0 of
    ``latents`` is overwritten with ``first`` in place first (the caller's persistent latents, read by the DDIM step that follows)."""
    assert latents.dtype == torch.float32 and latents.is_contiguous() and latents.is_cuda
    b, c, f, h, w = latents.shape
    assert c == 4 and first is not None and first.dtype == torch.float32 and first.is_contiguous() and tuple(first.shape) == (b, 4, h, w)
    assert mode in (FIRST_CONCAT, FIRST_FRAME, FIRST_CONCAT | FIRST_FRAME)
    cin = 8 if mode & FIRST_CONCAT else 4
    c_pad = cin if c_pad is None else c_pad
    if out is None:
        out = torch.empty((dup * b, f, h, w, c_pad), dtype=dtype, device=latents.device)
    assert out.shape == (dup * b, f, h, w, c_pad) and out.dtype == dtype and out.is_contiguous()
    check(lib().fyc_build_unet_input_first(ptr(latents), ptr(first), ptr(out), b, f, h * w, dup, mode, c_pad, dtype_code(dtype), stream_ptr()))
    return out


def first_frame_temb_rows(temb, B, F):
    """temb [B + 1, N] fp32 (t = 0 row last) -> [B * F, N]: row b F + f = temb[B] for f == 0, else temb[b] (fyc.h
    fyc_first_frame_temb_rows; the per-image row bias of every conv1 under use_first_frame_condition)."""
    assert temb.dtype == torch.float32 and temb.is_contiguous() and temb.is_cuda and temb.shape[0] == B + 1
    N = temb.shape[1]
    out = torch.empty((B * F, N), dtype=torch.float32, device=temb.device)
    check(lib().fyc_first_frame_temb_rows(ptr(temb), ptr(out), B, F, N, stream_ptr()))
    return out


def cfg_ddim_step(pred, sample, coefs, noise=None, out=None, single=None, video_scale=0.0):
    """pred fp32 [2, ...] (uncond, cond) if coefs.cfg_pair else [1, ...]; sample fp32; returns prev sample.
    ``single`` (same shape as sample): the per-frame prediction of the video_scale > 0 branch (pipeline_animation.py:738-761)."""
    assert pred.dtype == torch.float32 and sample.dtype == torch.float32 and pred.is_contiguous() and sample.is_contiguous()
    out = torch.empty_like(sample) if out is None else out
    if single is not None:
        assert single.dtype == torch.float32 and single.is_contiguous() and single.numel() == sample.numel() and pred.numel() == 2 * sample.numel()
        check(lib().fyc_cfg_video_ddim_step(ptr(pred), ptr(single), float(video_scale), ptr(sample), ptr(noise), ptr(out), sample.numel(),
                                            C.byref(coefs), stream_ptr()))
        return out
    check(lib().fyc_cfg_ddim_step(ptr(pred), ptr(sample), ptr(noise), ptr(out), sample.numel(), C.byref(coefs), stream_ptr()))
    return out


def frames_finalize(x, b, f):
    """x [b*f, H, W, 3] (or the [..., :3] slice of a wider channels-last tensor) -> video (b, 3, f, H, W) fp32 =
    (x / 2 + 0.5).clamp(0, 1)."""
    ld = _channel_sliced(x)
    _, H, W_, c = x.shape
    assert c == 3
    out = torch.empty((b, 3, f, H, W_), dtype=torch.float32, device=x.device)
    check(lib().fyc_frames_finalize(ptr(x), ptr(out), b, f, H * W_, ld, dtype_code(x.dtype), stream_ptr()))
    return out


def video_grid_shape(b, F, H, W, nrow, padding=2):
    pad = 0 if b == 1 else padding
    xmaps = min(nrow, b)
    ymaps = (b + xmaps - 1) // xmaps
    return F, (H + pad) * ymaps + pad, (W + pad) * xmaps + pad, 3


def video_grid_u8(video, nrow=6, padding=2, rescale=False):
    """video (b, 3, F, H, W) fp32 on device -> uint8 [F, Hg, Wg, 3]: per-frame make_grid tiling + trunc(x * 255) (util.py:18-27)."""
    assert video.dtype == torch.float32 and video.is_contiguous() and video.dim() == 5 and video.shape[1] == 3
    require_cuda(video, "video_grid_u8")
    b, _, F, H, W_ = video.shape
    out = torch.empty(video_grid_shape(b, F, H, W_, nrow, padding), dtype=torch.uint8, device=video.device)
    check(lib().fyc_video_grid_u8(ptr(video), ptr(out), b, F, H, W_, nrow, padding, int(bool(rescale)), stream_ptr()))
    return out
