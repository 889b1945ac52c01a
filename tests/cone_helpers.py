"""Dependency-cone and per-element bound checks of the kernel entry points (pure torch: runs on the CPU and on the GPU).

A case is one call of a public ``ops`` function on operands held inside larger allocations.  Three checks run on it:

* surround - the operands sit inside NaN-filled memory (rows wider than the view where the entry point takes a leading dimension,
  guard bands before and after where it takes a contiguous tensor) and every output the call allocates is prefilled with NaN inside a
  NaN frame.  The same call with zero-filled surroundings must give a finite output bit-identical to the first, and the frames must
  still hold NaN bit for bit: nothing outside an operand reaches the result, every output element is written, nothing outside the
  output is;
* cone - one operand element set to NaN: the set of NaN outputs must be the set of NaN outputs of the fp64 reference on the same
  seeded operands (the mathematical dependency cone), and every other element must be bit-identical to the unseeded run;
* bound - every output element against the fp64 reference of the fyc.h contract on the exact operands the kernel received:
  |out - ref| <= u_o |ref| + C_BOUND * named_terms + floor, where u_o is the unit roundoff of the output type and the named terms
  (``mag64``) scale with the operand magnitudes of each operation.

Views never extend past their allocation and every pointer stays 16-byte aligned: the poison is ordinary data in valid memory.
"""
import contextlib
import math
from dataclasses import dataclass, field

import torch
import torch.nn.functional as F

from followyourclick_b200 import ops

C_BOUND = 4.0                 # the one constant every named term is multiplied by
GUARD = 64                    # guard-band elements before and after a contiguous operand (128 / 256 bytes: alignment kept)
U = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11, torch.float32: 2.0 ** -24}
TINY = {torch.bfloat16: 2.0 ** -133, torch.float16: 2.0 ** -24, torch.float32: 2.0 ** -149}   # smallest subnormal
ACC = 2.0 ** -23              # fp32 accumulation, per term of a K-long sum
EXP_U = 2.0 ** -20            # ex2.approx and the fp32 softmax normaliser
GELU_EPS = 1.3e-6             # absolute error of gelu_erf_fast (common.cuh), plus 2^-23 |x| of fp32 rounding
GELU_DMAX = 1.13              # max |gelu'(x)|


# ---- operands in poisoned memory -------------------------------------------------------------------------------------------

def _strides(shape, ld):
    st, acc = [], 1
    for i, n in enumerate(reversed(shape)):
        st.insert(0, acc)
        acc *= (ld if (i == 0 and ld is not None) else n)
    return tuple(st)


def embedded(shape, dtype, fill, ld=None, guard=GUARD, device="cpu", values=None):
    """a tensor view of ``shape`` inside a larger ``fill``-filled allocation: rows ld >= shape[-1] elements apart (the remaining
    columns are ``fill``) and ``guard`` elements of ``fill`` before and after.  Returns (view, buffer)."""
    shape = tuple(int(s) for s in shape)
    assert ld is None or (ld >= shape[-1] and ld % 8 == 0)
    st = _strides(shape, ld)
    extent = 1 + sum((n - 1) * s for n, s in zip(shape, st))
    buf = torch.full((guard + extent + guard,), fill, dtype=dtype, device=device)
    view = buf.as_strided(shape, st, guard)
    if values is not None:
        view.copy_(values)
    return view, buf


def _inside_mask(view, buf):
    m = torch.zeros(buf.shape, dtype=torch.bool, device=buf.device)
    m.as_strided(view.shape, view.stride(), view.storage_offset() - buf.storage_offset()).fill_(True)
    return m


def _bits(t):
    return t.view({2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


class _FramedTorch:
    """stands in for ``torch`` inside followyourclick_b200.ops: every floating-point output the wrapper allocates is NaN-prefilled
    inside a NaN frame (integer workspaces stay plain allocations)."""

    def __init__(self, alloc):
        self._alloc = alloc

    def __getattr__(self, n):
        return getattr(torch, n)

    def empty(self, *shape, dtype=None, device=None, **kw):
        if len(shape) == 1 and isinstance(shape[0], (tuple, list, torch.Size)):
            shape = tuple(shape[0])
        if dtype is None or not dtype.is_floating_point:
            return torch.empty(shape, dtype=dtype, device=device, **kw)
        return self._alloc(shape, dtype)

    def empty_like(self, t, **kw):
        return self._alloc(tuple(t.shape), kw.get("dtype", t.dtype))


@contextlib.contextmanager
def framed_outputs(alloc):
    real = ops.torch
    ops.torch = _FramedTorch(alloc)
    try:
        yield
    finally:
        ops.torch = real


# ---- cases ----------------------------------------------------------------------------------------------------------------

@dataclass
class Case:
    name: str
    op: str                               # key of REF / MAG
    operands: dict                        # name -> clean tensor in its storage dtype (contiguous)
    call: object                          # (operand views, alloc) -> output tensor
    params: dict = field(default_factory=dict)
    lds: dict = field(default_factory=dict)   # name -> row stride of the embedded view (None: contiguous with guard bands)
    seeds: list = field(default_factory=list)  # (operand name, index)
    widen: object = None                  # (seed, expected NaN mask) -> mask: a cone wider than the mathematics, stated in fyc.h
    out_dtype: object = None
    device: str = "cpu"
    exact: bool = False                   # data movement: the output must equal the reference bit for bit


def run(case, fill, operands=None):
    """one call with the operands embedded in ``fill``; returns (output copy, [frame intact per output allocation])"""
    operands = case.operands if operands is None else operands
    views = {n: embedded(t.shape, t.dtype, fill, ld=case.lds.get(n), device=case.device, values=t)[0] for n, t in operands.items()}
    allocs = []

    def alloc(shape, dtype, ld=None, init=None):
        v, b = embedded(shape, dtype, float("nan"), ld=ld, device=case.device, values=init)
        allocs.append((v, b))
        return v
    with framed_outputs(alloc):
        out = case.call(views, alloc)
    out = out.clone()
    nan_bits = {}
    frames = []
    for v, b in allocs:
        if b.dtype not in nan_bits:
            nan_bits[b.dtype] = _bits(torch.full((1,), float("nan"), dtype=b.dtype, device=b.device))
        outside = ~_inside_mask(v, b)
        frames.append(bool((_bits(b)[outside] == nan_bits[b.dtype]).all()))
    return out, frames


def _f64(ops_in):
    return {n: t.double() for n, t in ops_in.items()}


def ref64(case, operands=None, elems=None):
    return _blocked(REF[case.op], case, case.operands if operands is None else operands, elems)


def mag64(case, elems=None):
    return _blocked(MAG[case.op], case, case.operands, elems)


def check_surround(out_nan, out_zero, frames_nan, frames_zero):
    fin = torch.isfinite(out_nan.float())
    same = _bits(out_nan) == _bits(out_zero)
    r = dict(finite=bool(fin.all()), identical=bool(same.all()), frames=frames_nan + frames_zero)
    if not r["finite"]:
        r["first_nonfinite"] = tuple(int(i) for i in (~fin).nonzero()[0])
    if not r["identical"]:
        i = tuple(int(j) for j in (~same).nonzero()[0])
        r["first_diff"] = (i, float(out_nan[i]), float(out_zero[i]))
    r["ok"] = r["finite"] and r["identical"] and all(r["frames"])
    return r


def check_cone(out_seed, out_clean, expected):
    got = torch.isnan(out_seed.float())
    wrong = got != expected
    keep = ~expected
    changed = keep & (_bits(out_seed) != _bits(out_clean))
    r = dict(cone=int(expected.sum()), nan=int(got.sum()), wrong=int(wrong.sum()), changed_outside=int(changed.sum()))
    if r["wrong"]:
        i = tuple(int(j) for j in wrong.nonzero()[0])
        r["first_wrong"] = (i, "NaN" if bool(got[i]) else "finite", "expected NaN" if bool(expected[i]) else "expected finite")
    if r["changed_outside"]:
        i = tuple(int(j) for j in changed.nonzero()[0])
        r["first_changed"] = (i, float(out_seed[i]), float(out_clean[i]))
    r["ok"] = r["wrong"] == 0 and r["changed_outside"] == 0
    return r


def bound(ref, mag, out_dtype, c=C_BOUND, exact=False):
    return (0 if exact else U[out_dtype] * ref.abs()) + c * mag + 4 * TINY[out_dtype]


def check_bound(out, ref, mag, out_dtype, c=C_BOUND, exact=False):
    err = (out.double() - ref).abs()
    b = bound(ref, mag, out_dtype, c, exact)
    ratio = err / b
    ratio = torch.where(torch.isnan(ratio), torch.full_like(ratio, float("inf")), ratio)
    i = tuple(int(j) for j in (ratio == ratio.max()).nonzero()[0])
    r = dict(ratio=float(ratio.max()), worst=i, ref=float(ref[i]), out=float(out[i]), bound=float(b[i]))
    r["ok"] = r["ratio"] <= 1.0
    return r


def run_checks(case, seeds=None):
    """all three checks; returns {"surround": .., "cones": [..], "bound": ..}"""
    out_nan, fr_nan = run(case, float("nan"))
    out_zero, fr_zero = run(case, 0.0)
    res = dict(surround=check_surround(out_nan, out_zero, fr_nan, fr_zero), cones=[])
    for name, idx in (case.seeds if seeds is None else seeds):
        seeded = dict(case.operands)
        t = seeded[name].clone()
        t[idx] = float("nan")
        seeded[name] = t
        out_s, _ = run(case, float("nan"), seeded)
        expected = torch.isnan(ref64(case, seeded))
        if case.widen is not None:
            expected = case.widen((name, idx), expected)
        r = check_cone(out_s, out_nan, expected)
        r["seed"] = (name, idx)
        res["cones"].append(r)
    res["bound"] = check_bound(out_zero, ref64(case), mag64(case), case.out_dtype, exact=case.exact)
    return res


# ---- fp64 references of the fyc.h contracts and their named error terms ------------------------------------------------------

def _gelu64(g):
    return 0.5 * g * (1 + torch.erf(g / math.sqrt(2.0)))


def _rowbias_rows(rb, rows, rpg):
    return rb[torch.arange(rows, device=rb.device) // rpg]


def _gemm_pre(o, alpha=1.0, rows_per_group=0, geglu=False, absval=False):
    f = torch.abs if absval else (lambda t: t)
    A = torch.cat([o["A"], o["A2"]], dim=-1) if "A2" in o else o["A"]
    y = abs(alpha) * (f(A) @ f(o["W"]).transpose(-1, -2)) if absval else alpha * (A @ o["W"].transpose(-1, -2))
    if "ln" in o:
        y = f(o["ln"])[:, None] * y
    if "bias" in o:
        y = y + f(o["bias"])
    if "rowbias" in o:
        y = y + f(_rowbias_rows(o["rowbias"], y.shape[-2], rows_per_group))
    return y


def _geglu_split(y):
    M, N = y.shape
    t = y.reshape(M, N // 256, 2, 128)
    return t[:, :, 0].reshape(M, N // 2), t[:, :, 1].reshape(M, N // 2)


def gemm_ref(o, alpha=1.0, rows_per_group=0, geglu=False, **_):
    y = _gemm_pre(o, alpha, rows_per_group)
    if geglu:
        a, g = _geglu_split(y)
        return a * _gelu64(g)
    return y + o["residual"] if "residual" in o else y


def gemm_mag(o, alpha=1.0, rows_per_group=0, geglu=False, **_):
    K = o["W"].shape[-1]
    m = K * ACC * _gemm_pre(o, alpha, rows_per_group, absval=True)
    if geglu:
        a, g = _geglu_split(_gemm_pre(o, alpha, rows_per_group))
        ma, mg = _geglu_split(m)
        return _gelu64(g).abs() * ma + a.abs() * GELU_DMAX * mg + a.abs() * (GELU_EPS + ACC * g.abs())
    return m + (K * ACC * o["residual"].abs() if "residual" in o else 0)


def _nchw(x):
    return x.permute(0, 3, 1, 2)


def _conv64(x, w, stride=1, upsample=1, pad_mode=0):
    """3x3 conv as im2col + matmul (NaN reaches exactly the outputs whose window holds it): x NHWC, w [Cout, 3, 3, Cin] -> NHWC"""
    xc = _nchw(x)
    if upsample == 2:
        xc = xc.repeat_interleave(2, 2).repeat_interleave(2, 3)
    xc = F.pad(xc, (0, 1, 0, 1) if pad_mode == 1 else (1, 1, 1, 1))
    NB, Cin, Hp, Wp = xc.shape
    Ho, Wo = (Hp - 3) // stride + 1, (Wp - 3) // stride + 1
    cols = F.unfold(xc, 3, stride=stride)                              # [NB, Cin*9, L], (c, kh, kw) order
    wm = w.permute(0, 3, 1, 2).reshape(w.shape[0], -1)
    return (wm @ cols).reshape(NB, -1, Ho, Wo).permute(0, 2, 3, 1)


def _phases64(x, wph):
    """fyc.h w_phases: phase (py, px), tap (a, b) reads source pixel (oh + a - 1 + py, ow + b - 1 + px)"""
    NB, H, W, Cin = x.shape
    Cout = wph.shape[1]
    xp = F.pad(_nchw(x), (1, 1, 1, 1))
    out = torch.zeros(NB, 2 * H, 2 * W, Cout, dtype=x.dtype, device=x.device)
    for py in range(2):
        for px in range(2):
            patch = xp[:, :, py:py + H + 1, px:px + W + 1]
            cols = F.unfold(patch, 2)                                  # [NB, Cin*4, H*W], (c, a, b) order
            wm = wph[2 * py + px].permute(0, 3, 1, 2).reshape(Cout, -1)
            out[:, py::2, px::2] = (wm @ cols).reshape(NB, Cout, H, W).permute(0, 2, 3, 1)
    return out


def _conv_pre(o, stride=1, upsample=1, pad_mode=0, images_per_group=1, absval=False, **_):
    f = torch.abs if absval else (lambda t: t)
    if "w_phases" in o:
        y = _phases64(f(o["x"]), f(o["w_phases"]))
    else:
        y = _conv64(f(o["x"]), f(o["w"]), stride, upsample, pad_mode)
    if "bias" in o:
        y = y + f(o["bias"])
    if "rowbias" in o:
        y = y + f(o["rowbias"])[torch.arange(y.shape[0], device=y.device) // images_per_group][:, None, None, :]
    if "residual" in o:
        y = y + f(o["residual"])
    return y


def conv_ref(o, **p):
    return _conv_pre(o, **p)


def conv_mag(o, **p):
    k_eff = 4 * o["x"].shape[-1] if "w_phases" in o else 9 * o["x"].shape[-1]
    return k_eff * ACC * _conv_pre(o, absval=True, **p)


def _gn(x, gamma, beta, groups, eps, stat_batches, silu):
    """x [..., C] viewed as [stat_batches, R, C] -> (y, |x - mean| rstd, n)"""
    shape, C = x.shape, x.shape[-1]
    t = x.reshape(stat_batches, -1, groups, C // groups)
    mean = t.mean(dim=(1, 3), keepdim=True)
    var = ((t - mean) ** 2).mean(dim=(1, 3), keepdim=True)
    z = ((t - mean) * torch.rsqrt(var + eps)).reshape(shape)
    y = z * gamma + beta
    return (y * torch.sigmoid(y) if silu else y), z.abs(), t.shape[1] * t.shape[3]


def _norm_mag(z, n, gamma, beta, y):
    # fp32 statistics: mean and variance of n terms carry ~sqrt(n) 2^-23 relative error; it reaches the output through
    # (x - mean) rstd gamma (the mean's error: sigma rstd = 1) - plus exp.approx of the SiLU
    return ((z + 1) * gamma.abs() + beta.abs()) * (math.sqrt(n) + 2) * ACC + EXP_U * y.abs()


def groupnorm_ref(o, groups, eps, stat_batches, silu=False, **_):
    x = torch.cat([o["x"], o["x2"]], dim=-1) if "x2" in o else o["x"]
    return _gn(x, o["gamma"], o["beta"], groups, eps, stat_batches, silu)[0]


def groupnorm_mag(o, groups, eps, stat_batches, silu=False, **_):
    x = torch.cat([o["x"], o["x2"]], dim=-1) if "x2" in o else o["x"]
    y, z, n = _gn(x, o["gamma"], o["beta"], groups, eps, stat_batches, silu)
    return _norm_mag(z, n, o["gamma"], o["beta"], y)


def _ln(o, eps, rows_per_frame=0, frames=0):
    x = o["x"]
    mean = x.mean(dim=-1, keepdim=True)
    z = (x - mean) * torch.rsqrt(((x - mean) ** 2).mean(dim=-1, keepdim=True) + eps)
    y = z * o["gamma"] + o["beta"]
    if "pe" in o:
        y = y + o["pe"][(torch.arange(x.shape[0], device=x.device) // rows_per_frame) % frames]
    return y, z.abs()


def layernorm_ref(o, eps, **p):
    return _ln(o, eps, **p)[0]


def layernorm_mag(o, eps, **p):
    y, z = _ln(o, eps, **p)
    m = _norm_mag(z, o["x"].shape[-1], o["gamma"], o["beta"], y)
    return m + (ACC * o["pe"].abs()[(torch.arange(y.shape[0], device=y.device) // p["rows_per_frame"]) % p["frames"]] if "pe" in o else 0)


def lnstats_ref(o, eps, **_):
    x = o["x"]
    return torch.rsqrt(((x - x.mean(dim=-1, keepdim=True)) ** 2).mean(dim=-1) + eps)


def lnstats_mag(o, eps, **_):
    return lnstats_ref(o, eps) * (math.sqrt(o["x"].shape[-1]) + 2) * ACC


def _heads(t, heads, D, stride):
    """[N, L, >= ...] -> [N, heads, L, D] taking head h from columns [h * stride, + D)"""
    N, L = t.shape[:2]
    return torch.stack([t[:, :, h * stride:h * stride + D] for h in range(heads)], dim=1)


def _softmax_pv(q, k, v, scale, u_s, absterm):
    """q [N, h, Lq, D], k / v [N, h, Lk, D] -> (out, named error term): (u_s + 2^-20) sum_j p_j |v_j| + sum_j p_j ds_j (|v_j| + |o|),
    ds_j = D 2^-23 scale sum_d |q_d k_jd| the fp32 error of a score"""
    s = scale * (q @ k.transpose(-1, -2))
    p = torch.softmax(s, dim=-1)
    o = p @ v
    if not absterm:
        return o, None
    ds = q.shape[-1] * ACC * abs(scale) * (q.abs() @ k.abs().transpose(-1, -2))
    pv = p @ v.abs()
    pd = p * ds
    return o, (u_s + EXP_U) * pv + pd @ v.abs() + pd.sum(-1, keepdim=True) * o.abs()


def _merge(t):
    N, h, L, D = t.shape
    return t.transpose(1, 2).reshape(N, L, h * D)


def _attn(o, heads, D, scale, kv_batch_div=1, out_alpha=1.0, alpha2=1.0, accumulate=False, u_s=0.0, absterm=False, **_):
    rep = lambda t: t.repeat_interleave(kv_batch_div, 0)
    q = _heads(o["q"], heads, D, D)
    y, m = _softmax_pv(q, rep(_heads(o["k"], heads, D, D)), rep(_heads(o["v"], heads, D, D)), scale, u_s, absterm)
    y, m = out_alpha * y, (abs(out_alpha) * m if absterm else None)
    if "k2" in o:
        y2, m2 = _softmax_pv(q, rep(_heads(o["k2"], heads, D, D)), rep(_heads(o["v2"], heads, D, D)), scale, u_s, absterm)
        y = y + alpha2 * y2
        m = m + abs(alpha2) * m2 if absterm else None
    y = _merge(y)
    if accumulate:
        y = y + o["out0"]
    return y, (_merge(m) if absterm else None)


def attention_ref(o, **p):
    return _attn(o, **p)[0]


def attention_mag(o, **p):
    return _attn(o, absterm=True, **p)[1]


def _cross_tc(o, heads, D, scale, Lk, Lk2=0, kv_batch_div=1, out_alpha=1.0, alpha2=1.0, u_s=0.0, absterm=False, **_):
    """fyc_cross_attention_tc: packed keys (head stride DKP), V^T with the keys contiguous, keys >= Lk / Lk2 are padding"""
    dkp = 64 if D == 40 else D
    rep = lambda t: t.repeat_interleave(kv_batch_div, 0)
    q = _heads(o["q"], heads, D, D)

    def one(k, vt, L):
        kh = _heads(k[:, :L], heads, D, dkp)
        vh = vt[:, :, :L].reshape(vt.shape[0], heads, D, L).transpose(-1, -2)
        return _softmax_pv(q, rep(kh), rep(vh), scale, u_s, absterm)
    y, m = one(o["k"], o["vt"], Lk)
    y, m = out_alpha * y, (abs(out_alpha) * m if absterm else None)
    if Lk2:
        y2, m2 = one(o["k2"], o["vt2"], Lk2)
        y = y + alpha2 * y2
        m = m + abs(alpha2) * m2 if absterm else None
    return _merge(y), (_merge(m) if absterm else None)


def cross_tc_ref(o, **p):
    return _cross_tc(o, **p)[0]


def cross_tc_mag(o, **p):
    return _cross_tc(o, absterm=True, **p)[1]


def _self_tc(o, heads, D, scale, q_col0, k_col0, hstride, u_s=0.0, absterm=False, q_rows=None, **_):
    """``q_rows`` (lo, hi): only the outputs of query rows lo..hi - 1 (every key still attends)"""
    qk = o["qk"]
    qr = qk if q_rows is None else qk[:, q_rows[0]:q_rows[1]]
    q, k = _heads(qr[:, :, q_col0:], heads, D, hstride), _heads(qk[:, :, k_col0:], heads, D, hstride)
    vt = o["vt"]
    v = vt.reshape(vt.shape[0], heads, D, -1).transpose(-1, -2)
    y, m = _softmax_pv(q, k, v, scale, u_s, absterm)
    return _merge(y), (_merge(m) if absterm else None)


def self_tc_ref(o, **p):
    return _self_tc(o, **p)[0]


def self_tc_mag(o, **p):
    return _self_tc(o, absterm=True, **p)[1]


def _temporal(o, heads, scale, u_s=0.0, absterm=False, **_):
    qkv = o["qkv"]
    B, Fr, HW, C3 = qkv.shape
    C = C3 // 3
    D = C // heads
    t = qkv.permute(0, 2, 1, 3).reshape(B * HW, Fr, C3)                # (b p) f c
    y, m = _softmax_pv(_heads(t, heads, D, D), _heads(t[:, :, C:], heads, D, D), _heads(t[:, :, 2 * C:], heads, D, D), scale, u_s, absterm)
    back = lambda r: _merge(r).reshape(B, HW, Fr, C).permute(0, 2, 1, 3)
    return back(y), (back(m) if absterm else None)


def temporal_ref(o, **p):
    return _temporal(o, **p)[0]


def temporal_mag(o, **p):
    return _temporal(o, absterm=True, **p)[1]


def transpose_ref(o, col0, C, **_):
    return o["x"][:, :, col0:col0 + C].transpose(1, 2)


def transpose_mag(o, col0, C, **_):
    return torch.zeros_like(transpose_ref(o, col0, C))


def softmax_ref(o, **_):
    return torch.softmax(o["s"], dim=-1)


def softmax_mag(o, **_):
    p = softmax_ref(o)
    return (o["s"].shape[-1] * ACC / 2 + EXP_U) * p


REF = dict(gemm=gemm_ref, conv=conv_ref, groupnorm=groupnorm_ref, layernorm=layernorm_ref, lnstats=lnstats_ref, attention=attention_ref,
           cross_tc=cross_tc_ref, self_tc=self_tc_ref, temporal=temporal_ref, transpose=transpose_ref, softmax=softmax_ref)
MAG = dict(gemm=gemm_mag, conv=conv_mag, groupnorm=groupnorm_mag, layernorm=layernorm_mag, lnstats=lnstats_mag, attention=attention_mag,
           cross_tc=cross_tc_mag, self_tc=self_tc_mag, temporal=temporal_mag, transpose=transpose_mag, softmax=softmax_mag)


# ---- the references in blocks of output rows ----------------------------------------------------------------------------------
# A block's largest fp64 intermediate (attention scores, a conv's im2col matrix, a GEMM's pre-activation) holds about CHUNK_ELEMS
# elements (256 MB); the few such tensors alive at once keep a case within ~4 GB of device memory at any shape.  Output rows are
# independent in every chunked operation, so the blocks concatenate to the unchunked result.

CHUNK_ELEMS = 1 << 25


def _blocks(n, per_row, align, elems):
    step = max(align, (elems // max(per_row, 1)) // align * align)
    return [(lo, min(lo + step, n)) for lo in range(0, n, step)]


def _rows(t, axis, lo, hi):
    return t.narrow(axis % t.dim(), lo, hi - lo)


def _group_rows(t, lo, hi, per):
    """rows of a per-group table (row bias) that serve items lo..hi - 1, ``per`` items a group, lo a multiple of ``per``"""
    return t[lo // per:-(-hi // per)]


def _split_gemm(o, p, elems):
    A = o["A"]
    M = A.shape[-2]
    rpg = p.get("rows_per_group", 0) if "rowbias" in o else 0
    per_row = (o["W"].shape[-2] + A.shape[-1]) * (A.shape[0] if A.dim() == 3 else 1)
    out = []
    for lo, hi in _blocks(M, per_row, max(rpg, 1), elems):
        b = {n: (_rows(t, -2, lo, hi) if n in ("A", "A2", "residual") else t) for n, t in o.items()}
        if "ln" in o:
            b["ln"] = o["ln"][lo:hi]
        if rpg:
            b["rowbias"] = _group_rows(o["rowbias"], lo, hi, rpg)
        out.append((b, p))
    return -2, out


def _split_conv(o, p, elems):
    NB, H, W, Cin = o["x"].shape
    ipg = p.get("images_per_group", 1)
    up = p.get("upsample", 1)
    Cout = o["w_phases"].shape[1] if "w_phases" in o else o["w"].shape[0]
    per_img = H * W * up * up * (9 * Cin + Cout)
    out = []
    for lo, hi in _blocks(NB, per_img, ipg if "rowbias" in o else 1, elems):
        b = {n: (t[lo:hi] if n in ("x", "residual") else t) for n, t in o.items()}
        if "rowbias" in o:
            b["rowbias"] = _group_rows(o["rowbias"], lo, hi, ipg)
        out.append((b, p))
    return 0, out


def _split_query(key_rows):
    """attention over query rows (operand "q", axis 1) against every key: the block holds rows x (batch heads keys) scores"""
    def split(o, p, elems):
        q = o["q"]
        per_row = q.shape[0] * p["heads"] * key_rows(o, p)
        out = []
        for lo, hi in _blocks(q.shape[1], per_row, 1, elems):
            out.append(({n: (t[:, lo:hi] if n in ("q", "out0") else t) for n, t in o.items()}, p))
        return 1, out
    return split


def _split_self_tc(o, p, elems):
    NB, L = o["qk"].shape[:2]
    return 1, [(o, dict(p, q_rows=(lo, hi))) for lo, hi in _blocks(L, NB * p["heads"] * L, 1, elems)]


SPLIT = dict(gemm=_split_gemm, conv=_split_conv, self_tc=_split_self_tc,
             attention=_split_query(lambda o, p: o["k"].shape[1] + (o["k2"].shape[1] if "k2" in o else 0)),
             cross_tc=_split_query(lambda o, p: p["Lk"] + p.get("Lk2", 0)))


def _blocked(fn, case, operands, elems=None):
    """fn (a REF or MAG entry) on the fp64 operands, one block of output rows at a time"""
    split = SPLIT.get(case.op)
    if split is None:
        return fn(_f64(operands), **case.params)
    axis, blocks = split(operands, case.params, CHUNK_ELEMS if elems is None else elems)
    if len(blocks) == 1:
        return fn(_f64(operands), **case.params)
    return torch.cat([fn(_f64(b), **p) for b, p in blocks], dim=axis)


# ---- case builders (shared by the GPU test and its CPU self-test) -----------------------------------------------------------------

PAD = 16                      # extra columns of an operand row where the entry point takes a leading dimension


def rnd(shape, seed, dtype, device, scale=1.0, offset=0.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * scale + offset).to(dtype).to(device)


def _seeds(cands, operands):
    """keep the candidate seeds whose index lies inside the operand, without duplicates"""
    out = []
    for name, idx in cands:
        if name not in operands:
            continue
        shp = operands[name].shape
        idx = tuple(int(i) for i in idx)
        if len(idx) == len(shp) and all(0 <= i < n for i, n in zip(idx, shp)) and (name, idx) not in out:
            out.append((name, idx))
    return out


def gemm_case(dtype, M, N, K, device, bias=True, residual=False, rpg=0, alpha=1.0, out_f32=False, impl=None, K2=0, ln=False,
              geglu=False, batch=0, name=None):
    """one ops.gemm call; every operand row (A, W, A2, residual, out) wider than its view.  ``geglu``: N = 2 Hd with the weight rows in
    the fyc.h 128-column granule interleave; ``ln``: A is the raw LayerNorm input, W the packed W'' and ``ln`` the rstd operand"""
    from followyourclick_b200 import _lib
    odt = torch.float32 if out_f32 else dtype
    n_out = N // 2 if geglu else N
    lead = (batch,) if batch else ()
    o = dict(A=rnd(lead + (M, K), 1, dtype, device, offset=0.0))
    if ln:
        o["A"] = (rnd((M, K), 1, torch.float32, "cpu", 1.3) + rnd((M, 1), 2, torch.float32, "cpu", 1.5)).to(dtype).to(device)
        w = rnd((N, K), 3, torch.float32, "cpu", K ** -0.5)
        gamma = 1 + 0.1 * rnd((K,), 4, torch.float32, "cpu")
        o["W"] = ops.ln_fold_weight(w, gamma, dtype).to(device)
        x = o["A"].float()
        o["ln"] = torch.rsqrt(x.var(dim=1, unbiased=False) + 1e-5).contiguous()
    else:
        o["W"] = rnd(lead + (N, K + K2), 3, dtype, device, (K + K2) ** -0.5)
    if K2:
        o["A2"] = rnd((M, K2), 5, dtype, device)
    if bias:
        o["bias"] = rnd((N,), 6, torch.float32, device, 0.5)
    if rpg:
        o["rowbias"] = rnd((-(-M // rpg), N), 7, torch.float32, device, 0.5)
    if residual:
        o["residual"] = rnd((M, n_out), 8, odt, device)
    lds = dict(A=K + PAD, W=K + K2 + PAD, A2=K2 + PAD, residual=n_out + PAD)
    lds = {k: v for k, v in lds.items() if k in o}
    impl_code = {None: None, "simt": _lib.IMPL_SIMT}[impl]

    # the unfused GEGLU (CUDA-core path) writes packed rows: its output view is contiguous inside guard bands
    fused = geglu and ops.tc_ok(dtype, M, impl_code)
    ldo = None if geglu and not fused else n_out + PAD

    def call(v, alloc):
        out = alloc(lead + (M, n_out), odt, ld=ldo)
        return ops.gemm(v["A"], v["W"], bias=v.get("bias"), residual=v.get("residual"), rowbias=v.get("rowbias"), rows_per_group=rpg,
                        alpha=alpha, geglu=geglu, out_f32=out_f32, out=out, impl=impl_code, ln=v.get("ln"), A2=v.get("A2"))
    b = (batch - 1,) if batch else ()
    z = (0,) if batch else ()
    seeds = _seeds([("A", z + (0, 0)), ("A", b + (M - 1, K - 1)), ("A", z + (127, K // 2)), ("A", b + (128, 0)), ("A", z + ((M - 1) // 128 * 128, 1)),
                    ("W", z + (0, 0)), ("W", b + (N - 1, K + K2 - 1)), ("W", z + (63, 3)), ("W", b + (64, 63)), ("W", z + (N // 2, 64)),
                    ("A2", (M - 1, K2 - 1)), ("A2", (0, 0)), ("bias", (N - 1,)), ("bias", (0,)), ("rowbias", ((M - 1) // max(rpg, 1), N - 1)),
                    ("rowbias", (0, 5)), ("residual", (M - 1, n_out - 1)), ("residual", (128, 64)), ("ln", (M - 1,)), ("ln", (128,))], o)
    return Case(name or f"gemm_{M}x{N}x{K}", "gemm", o, call, dict(alpha=alpha, rows_per_group=rpg, geglu=geglu), lds, seeds,
                out_dtype=odt, device=device)


def conv_case(dtype, NB, H, W, Cin, Cout, device, stride=1, up=1, pad_mode=0, bias=True, residual=False, ipg=0, out_f32=False,
              phases=False, impl=None, name=None):
    """one ops.conv3x3 call on NHWC images with guard bands; ``ipg``: the row bias is a column block of a wider [groups, 3 Cout] table
    (fyc.h ld_rowbias) whose other columns are poison"""
    from followyourclick_b200 import _lib
    from followyourclick_b200.modeling import upsample_phase_weights
    odt = torch.float32 if out_f32 else dtype
    o = dict(x=rnd((NB, H, W, Cin), 1, dtype, device))
    w = rnd((Cout, Cin, 3, 3), 2, torch.float32, "cpu", (9 * Cin) ** -0.5)
    o["w"] = w.permute(0, 2, 3, 1).to(dtype).contiguous().to(device)
    if phases:
        o["w_phases"] = upsample_phase_weights(w).to(dtype).contiguous().to(device)
    if bias:
        o["bias"] = rnd((Cout,), 3, torch.float32, device, 0.5)
    if ipg:
        o["rowbias"] = rnd((NB // ipg, Cout), 4, torch.float32, device, 0.5)
    Ho, Wo = (H * up + 2 - 3) // stride + 1, (W * up + 2 - 3) // stride + 1
    if pad_mode == 1:
        Ho, Wo = H // 2, W // 2
    if residual:
        o["residual"] = rnd((NB, Ho, Wo, Cout), 5, odt, device)
    lds = dict(rowbias=3 * Cout) if ipg else {}
    impl_code = {None: None, "simt": _lib.IMPL_SIMT}[impl]

    def call(v, alloc):
        return ops.conv3x3(v["x"], v["w"], bias=v.get("bias"), residual=v.get("residual"), rowbias=v.get("rowbias"), images_per_group=ipg,
                           stride=stride, upsample=up, out_f32=out_f32, impl=impl_code, pad_mode=pad_mode, w_phases=v.get("w_phases"))
    # weight seeds sit on taps that never meet the zero padding: a NaN weight times a padding zero is NaN where the padding is
    # multiplied (tensor-map zero fill) and absent where it is skipped (CUDA-core bounds checks) - both are the contract
    wname = "w_phases" if phases else "w"
    wl, w0 = ((3, Cout - 1, 0, 0, Cin - 1), (0, 0, 1, 1, 0)) if phases else ((Cout - 1, 1, 1, Cin - 1), (0, 1, 1, 0))
    seeds = _seeds([("x", (0, 0, 0, 0)), ("x", (0, H - 1, W - 1, Cin - 1)), ("x", (NB - 1, H - 1, 0, 3)), ("x", (NB - 1, 0, W - 1, Cin // 2)),
                    ("x", (min(1, NB - 1), 0, W // 2, 1)), ("x", (0, H // 2, 0, 2)), ("x", (0, H - 1, W // 2, 5)),
                    (wname, wl), (wname, w0), ("bias", (Cout - 1,)), ("rowbias", (NB // max(ipg, 1) - 1, Cout - 1)),
                    ("rowbias", (0, 0)), ("residual", (NB - 1, Ho - 1, Wo - 1, Cout - 1)), ("residual", (0, 0, Wo - 1, 0))], o)
    return Case(name or f"conv_{NB}x{H}x{W}_{Cin}to{Cout}", "conv", o, call,
                dict(stride=stride, upsample=up, pad_mode=pad_mode, images_per_group=max(ipg, 1)), lds, seeds, out_dtype=odt, device=device)


def groupnorm_case(dtype, NB, R, C, G, stat, device, silu=False, C2=0, name=None):
    """ops.groupnorm (two sources when C2: the channel concatenation read in place); inputs offset by 1.5 sigma"""
    o = dict(x=rnd((NB, R, C), 1, dtype, device, 2.0, 3.0))
    if C2:
        o["x2"] = rnd((NB, R, C2), 2, dtype, device, 1.5, 0.3)
    o["gamma"] = 1 + 0.1 * rnd((C + C2,), 3, torch.float32, device)
    o["beta"] = 0.1 * rnd((C + C2,), 4, torch.float32, device)

    def call(v, alloc):
        return ops.groupnorm(v["x"], v["gamma"], v["beta"], G, 1e-5, silu=silu, stat_batches=stat, x2=v.get("x2"))
    per = NB // stat
    seam = C - 1
    seeds = _seeds([("x", (0, 0, 0)), ("x", (NB - 1, R - 1, C - 1)), ("x", (per - 1, R - 1, seam)), ("x", (per, 0, 1)),
                    ("x2", (0, 0, 0)), ("x2", (NB - 1, R - 1, C2 - 1)), ("gamma", (C + C2 - 1,)), ("beta", (0,))], o)
    return Case(name or f"groupnorm_{NB}x{R}x{C}+{C2}", "groupnorm", o, call, dict(groups=G, eps=1e-5, stat_batches=stat, silu=silu), {},
                seeds, out_dtype=dtype, device=device)


def layernorm_case(dtype, M, C, device, pe=False, stats_only=False, name=None):
    """ops.layernorm (+ the position table of frame (row / rows_per_frame) % frames) or ops.layernorm_stats"""
    rpf, frames = 16, 4
    o = dict(x=(rnd((M, C), 1, torch.float32, "cpu", 1.5) + rnd((M, 1), 2, torch.float32, "cpu", 1.5)).to(dtype).to(device))
    if not stats_only:
        o["gamma"] = 1 + 0.1 * rnd((C,), 3, torch.float32, device)
        o["beta"] = 0.1 * rnd((C,), 4, torch.float32, device)
    if pe:
        o["pe"] = rnd((24, C), 5, torch.float32, device)

    def call(v, alloc):
        if stats_only:
            return ops.layernorm_stats(v["x"])
        return ops.layernorm(v["x"], v["gamma"], v["beta"], pe=v.get("pe"), rows_per_frame=rpf if pe else 0, frames=frames if pe else 0)
    seeds = _seeds([("x", (0, 0)), ("x", (M - 1, C - 1)), ("x", (M // 2, 7)), ("gamma", (C - 1,)), ("beta", (0,)), ("pe", (frames - 1, C - 1)),
                    ("pe", (1, 0))], o)
    p = dict(eps=1e-5) if stats_only else dict(eps=1e-5, rows_per_frame=rpf, frames=frames) if pe else dict(eps=1e-5)
    return Case(name or f"layernorm_{M}x{C}", "lnstats" if stats_only else "layernorm", o, call, p, {}, seeds,
                out_dtype=torch.float32 if stats_only else dtype, device=device)


LAYOUTS = ("gaussian", "ascending", "late_peak", "flat")
SPAN = 30.0                   # logit range of the ascending and late-peak layouts


def layout_qk(layout, N, L, heads, D, scale):
    """self-attention q, k [N, L, heads, D] fp32 (cpu) whose scores have a given structure:
    gaussian  - independent N(0, 1) entries;
    ascending - every row's score rises with the key index (0 .. ~SPAN): each key tile raises the running max of the online softmax;
    late_peak - key L - 2, in the last key tile, exceeds every other score of every row by ~SPAN;
    flat      - every key row is the same: a row's scores are all equal, the normaliser sums over every tile."""
    q, k = rnd((N, L, heads, D), 1, torch.float32, "cpu"), rnd((N, L, heads, D), 2, torch.float32, "cpu")
    if layout == "ascending":
        # q0 in [3, 4) per row and head, q1.. zero: s = scale q0 k0, k0 a ramp that reaches SPAN at q0 = 4
        q = torch.cat([3 + rnd((N, L, heads, 1), 3, torch.float32, "cpu").abs().clamp(max=0.99), torch.zeros(N, L, heads, D - 1)], dim=-1)
        k[..., 0] = torch.linspace(0, SPAN / (4 * scale), L)[None, :, None]
    elif layout == "late_peak":
        q, k = 0.5 * q, 0.5 * k
        q[..., 0], k[..., 0] = 4.0, 0.0
        k[:, L - 2, :, 0] = SPAN / (4 * scale)
    elif layout == "flat":
        k = k[:, :1].expand(N, L, heads, D).contiguous()
    else:
        assert layout == "gaussian", layout
    return q, k


def attention_case(dtype, heads, D, B, Lq, Lk, div, device, T=0, accumulate=False, impl=None, layout="gaussian", name=None):
    """ops.attention on strided q / k / v views (rows wider than the heads), context n / div, optional fused second context of T keys,
    or the accumulate form (out = out0 + out_alpha softmax(..) v, out0 a finite prefill); ``layout``: a score structure of layout_qk
    (self-attention shapes: Lq = Lk, div = 1)"""
    from followyourclick_b200 import _lib
    C, Bc = heads * D, B // div
    o = dict(q=rnd((B, Lq, C), 1, dtype, device), k=rnd((Bc, Lk, C), 2, dtype, device), v=rnd((Bc, Lk, C), 3, dtype, device))
    if layout != "gaussian":
        assert Lq == Lk and div == 1
        q, k = layout_qk(layout, B, Lq, heads, D, D ** -0.5)
        o["q"], o["k"] = q.reshape(B, Lq, C).to(dtype).to(device), k.reshape(B, Lk, C).to(dtype).to(device)
    if T:
        o["k2"], o["v2"] = rnd((Bc, T, C), 4, dtype, device), rnd((Bc, T, C), 5, dtype, device)
    if accumulate:
        o["out0"] = rnd((B, Lq, C), 6, dtype, device)
    a1, a2 = (0.7 if accumulate else 1.0), 0.6
    lds = {n: C + PAD for n in ("q", "k", "v", "k2", "v2")}
    impl_code = {None: None, "simt": _lib.IMPL_SIMT}[impl]

    def call(v, alloc):
        out = alloc((B, Lq, C), dtype, ld=C + PAD, init=v.get("out0"))
        return ops.attention(v["q"], v["k"], v["v"], heads, D ** -0.5, out=out, out_alpha=a1, accumulate=accumulate, kv_batch_div=div,
                             impl=impl_code, k2=v.get("k2"), v2=v.get("v2"), alpha2=a2)
    seeds = _seeds([("q", (0, 0, 0)), ("q", (B - 1, Lq - 1, C - 1)), ("q", (1, 64, D)), ("k", (Bc - 1, Lk - 1, C - 1)), ("k", (0, 0, 0)),
                    ("k", (0, 63, D - 1)), ("k", (Bc - 1, 64, 1)), ("v", (Bc - 1, Lk - 1, C - 1)), ("v", (0, 0, D)), ("v", (0, 64, 0)),
                    ("k2", (Bc - 1, T - 1, C - 1)), ("v2", (0, 0, 0)), ("out0", (B - 1, Lq - 1, C - 1))], o)
    return Case(name or f"attention_{heads}x{D}_{Lq}x{Lk}", "attention", o, call,
                dict(heads=heads, D=D, scale=D ** -0.5, kv_batch_div=div, out_alpha=a1, alpha2=a2, accumulate=accumulate, u_s=U[dtype]),
                lds, seeds, out_dtype=dtype, device=device)


def cross_tc_case(dtype, heads, D, NB, Lq, Lk, T, div, device, name=None):
    """ops.cross_attention_tc: unpadded q heads in rows wider than the heads, context keys packed per fyc.h (head stride 64 for D = 40
    with columns D..63 zero, rows Lk..79 zero; V^T columns Lk..79 zero - those zeros are part of the operand), out rows wider too"""
    dkp = ops.cross_dkp(D)
    C, NBc = heads * D, NB // div
    o = dict(q=rnd((NB, Lq, C), 1, dtype, device))

    def pack(L, Lpad, s):
        k, v = rnd((NBc, L, C), s, dtype, "cpu"), rnd((NBc, L, C), s + 1, dtype, "cpu")
        kp = torch.zeros((NBc, Lpad, heads * dkp), dtype=dtype)
        kp.view(NBc, Lpad, heads, dkp)[:, :L, :, :D] = k.view(NBc, L, heads, D)
        vt = torch.zeros((NBc, C, Lpad), dtype=dtype)
        vt[:, :, :L] = v.transpose(1, 2)
        return kp.to(device), vt.to(device)
    o["k"], o["vt"] = pack(Lk, ops.CROSS_LK, 2)
    if T:
        o["k2"], o["vt2"] = pack(T, ops.CROSS_LK2, 4)
    lds = dict(q=C + PAD, k=heads * dkp + PAD, k2=heads * dkp + PAD)
    scale, a1, a2 = D ** -0.5, 1.0, 0.6

    def call(v, alloc):
        out = alloc((NB, Lq, C), dtype, ld=C + PAD)
        return ops.cross_attention_tc(v["q"], v["k"], v["vt"], heads, D, scale, Lk, out, k2=v.get("k2"), vt2=v.get("vt2"), Lk2=T,
                                      out_alpha=a1, alpha2=a2, kv_batch_div=div)

    last = (heads - 1) * dkp
    seeds = _seeds([("q", (0, 0, 0)), ("q", (NB - 1, Lq - 1, C - 1)), ("q", (0, 5, D)), ("q", (NB - 1, 130, C - D)), ("q", (0, 64, D - 1)),
                    ("k", (NBc - 1, Lk - 1, last + D - 1)), ("k", (0, 0, 0)), ("vt", (NBc - 1, C - 1, Lk - 1)), ("vt", (0, 0, 0)),
                    ("k2", (NBc - 1, T - 1, last + D - 1)), ("vt2", (0, 0, T - 1))], o)
    return Case(name or f"cross_tc_{heads}x{D}_{Lq}x{Lk}+{T}", "cross_tc", o, call,
                dict(heads=heads, D=D, scale=scale, Lk=Lk, Lk2=T, kv_batch_div=div, out_alpha=a1, alpha2=a2, u_s=U[dtype]), lds, seeds,
                out_dtype=dtype, device=device)


def self_tc_case(dtype, D, NB, L, heads, device, wide_out=True, layout="gaussian", name=None):
    """fyc_self_attention_tc (D 40 / 64: 64-wide q / k heads, D = 40 columns 40..63 zero) or fyc_self_attention_tc_d80 (unpadded heads of
    the fused projection: the operand is the [q | k] part, the v block of the row is poison the kernel must not read).  ``wide_out``:
    output rows wider than the heads - a row stride ops does not expose, so the entry point is called directly.  ``layout``: the score
    structure of layout_qk."""
    from followyourclick_b200 import _lib
    C = heads * D
    hs = 80 if D == 80 else 64
    if layout == "gaussian":
        q, k = rnd((NB, L, heads, D), 1, dtype, "cpu"), rnd((NB, L, heads, D), 2, dtype, "cpu")
    else:
        q, k = (t.to(dtype) for t in layout_qk(layout, NB, L, heads, D, D ** -0.5))
    qk = torch.zeros((NB, L, 2, heads, hs), dtype=dtype)
    qk[:, :, 0, :, :D], qk[:, :, 1, :, :D] = q, k
    o = dict(qk=qk.reshape(NB, L, 2 * heads * hs).to(device), vt=rnd((NB, C, L), 3, dtype, device))
    k_col0 = heads * hs
    lds = dict(qk=3 * C if D == 80 else 2 * heads * hs + 64)
    scale = D ** -0.5

    def call(v, alloc):
        qkv, vt = v["qk"], v["vt"]
        if not wide_out:
            if D == 80:
                return ops.self_attention_tc_d80(qkv, 0, k_col0, vt, heads, scale)
            return ops.self_attention_tc(qkv, 0, k_col0, vt, heads, D, scale)
        out = alloc((NB, L, C), dtype, ld=C + PAD)
        if D == 80:
            fn = ops._tc_entry("fyc_self_attention_tc_d80", qkv)
            _lib.check(fn(_lib.ptr(qkv), qkv.stride(1), 0, k_col0, _lib.ptr(vt), _lib.ptr(out), out.stride(1), NB, heads, L, float(scale),
                          _lib.stream_ptr()))
        else:
            fn = ops._tc_entry("fyc_self_attention_tc", qkv)
            _lib.check(fn(_lib.ptr(qkv), qkv.stride(1), 0, k_col0, _lib.ptr(vt), _lib.ptr(out), out.stride(1), NB, heads, L, D, float(scale),
                          _lib.stream_ptr()))
        return out
    seeds = _seeds([("qk", (0, 0, 0)), ("qk", (NB - 1, L - 1, k_col0 + (heads - 1) * hs + D - 1)), ("qk", (0, 127, (heads - 1) * hs + D - 1)),
                    ("qk", (NB - 1, 128, k_col0)), ("qk", (0, 63, k_col0 + hs + 1)), ("vt", (NB - 1, C - 1, L - 1)), ("vt", (0, 0, 63)),
                    ("vt", (0, D, 64))], o)
    return Case(name or f"self_tc_{heads}x{D}_{L}", "self_tc", o, call,
                dict(heads=heads, D=D, scale=scale, q_col0=0, k_col0=k_col0, hstride=hs, u_s=U[dtype]), lds, seeds, out_dtype=dtype,
                device=device)


def temporal_case(dtype, B, Fr, HW, heads, D, device, name=None):
    C = heads * D
    o = dict(qkv=rnd((B, Fr, HW, 3 * C), 1, dtype, device))

    def call(v, alloc):
        return ops.temporal_attention(v["qkv"], heads, D ** -0.5)
    seeds = _seeds([("qkv", (B - 1, Fr - 1, HW - 1, 3 * C - 1)), ("qkv", (B - 1, Fr - 1, HW - 1, 2 * C - 1)), ("qkv", (0, 0, 0, 0)),
                    ("qkv", (0, Fr - 1, HW - 1, C - 1)), ("qkv", (B - 1, 0, 0, 2 * C))], o)
    return Case(name or f"temporal_{Fr}x{HW}_{heads}x{D}", "temporal", o, call, dict(heads=heads, scale=D ** -0.5, u_s=U[dtype]), {}, seeds,
                out_dtype=dtype, device=device)


def transpose_case(dtype, NB, L, C, col0, device, name=None):
    o = dict(x=rnd((NB, L, col0 + C + 8), 1, dtype, device))

    def call(v, alloc):
        return ops.transpose_tokens(v["x"], col0, C)
    seeds = _seeds([("x", (0, 0, col0)), ("x", (NB - 1, L - 1, col0 + C - 1)), ("x", (0, 64, col0 + 64)), ("x", (0, 1, 0))], o)
    return Case(name or f"transpose_{L}x{C}", "transpose", o, call, dict(col0=col0, C=C), dict(x=col0 + C + 8 + PAD), seeds,
                out_dtype=dtype, device=device, exact=True)


def softmax_case(out_dtype, rows, L, device, name=None):
    o = dict(s=rnd((rows, L), 1, torch.float32, device, 4.0))

    def call(v, alloc):
        return ops.softmax_rows(v["s"], out_dtype)
    seeds = _seeds([("s", (0, 0)), ("s", (rows - 1, L - 1)), ("s", (rows // 2, 127))], o)
    return Case(name or f"softmax_{rows}x{L}", "softmax", o, call, {}, {}, seeds, out_dtype=out_dtype, device=device)
