"""TEST INFRASTRUCTURE: a plain-PyTorch emulation of every ``followyourclick_b200.ops`` entry point.

Purpose: this container has no GPU, and the product has no CPU path (by contract).  To check the *host logic* of the drop-in
classes on CPU - weight packing (fused q/k/v, 64-padded heads, GEGLU interleave, phase-summed upsampler filters, 16-channel
padded heads), the ClipContext hoisting, the Resampler, the pipeline plumbing - the CPU tests swap ``ops`` for this module's
functions, which restate each kernel's *documented contract* (include/fyc.h) with torch ops in fp32 and round to the storage
dtype exactly once, like the kernels do.  The host code under test is the product's own; only the kernel launches are replaced.
The route rules that pick a kernel (ops.tc_ok, ops.self_attention_tc_ok, ...) are the product's too: the emulator answers only
the hardware query under them, ops.tc_available, with True.  Nothing in ``followyourclick_b200/`` imports this file, and it is
never used on a GPU box (the ``-m gpu`` tests call the real library through the C ABI).
"""
import inspect
import math

import torch
import torch.nn.functional as F

from followyourclick_b200 import _lib, ops


def _store(y, dtype):
    return y.to(dtype)


def tc_available():
    """the tensor cores are reported available, so the route rules of ops send 16-bit calls down the tensor-core paths and the host
    code's packing / layout branches for them are the ones exercised"""
    return True


def require_cuda(t, what):
    return None


def layernorm_stats(x, eps=1e-5):
    C = x.shape[-1]
    t = x.float().reshape(-1, C)
    mean = t.mean(dim=1)
    return torch.rsqrt(((t - mean[:, None]) ** 2).mean(dim=1) + eps).contiguous()


def gemm(A, W, bias=None, residual=None, rowbias=None, rows_per_group=0, alpha=1.0, geglu=False, out_f32=False, out=None, impl=None, ln=None, A2=None):
    if ln is not None:          # fyc.h FYC_EPI_LNFOLD: row-centred weights, the epilogue scales the accumulator by rstd
        assert A2 is None and alpha == 1.0 and residual is None and not out_f32 and ops.tc_ok(A.dtype, A.shape[0], impl)
    if A2 is not None:          # fyc.h A2: the K dimension is the concatenation [A | A2]
        A = torch.cat([A, A2], dim=-1)
    y = alpha * (A.float() @ W.float().transpose(-1, -2))
    if ln is not None:
        y = ln[:, None] * y
    if bias is not None:
        y = y + bias
    if rowbias is not None:
        idx = torch.arange(y.shape[-2]) // rows_per_group
        y = y + rowbias[idx]
    if residual is not None:
        y = y + residual.float()
    if geglu:
        M, N = y.shape
        t = y.view(M, N // 256, 2, 128)
        y = (t[:, :, 0] * F.gelu(t[:, :, 1])).reshape(M, N // 2)
    y = _store(y, torch.float32 if out_f32 else A.dtype)
    if out is not None:
        out.copy_(y)
        return out
    return y


def _phase_conv(x, w_phases, bias):
    """the four 2x2-tap convolutions of fyc.h `w_phases`, written interleaved"""
    NB, H, W_, Cin = x.shape
    Cout = w_phases.shape[1]
    xp = F.pad(x.float().permute(0, 3, 1, 2), (1, 1, 1, 1))
    out = torch.zeros(NB, Cout, 2 * H, 2 * W_)
    for py in range(2):
        for px in range(2):
            acc = 0
            for a in range(2):
                for b in range(2):
                    dy, dx = a - 1 + py, b - 1 + px
                    acc = acc + torch.einsum("nchw,oc->nohw", xp[:, :, 1 + dy:1 + dy + H, 1 + dx:1 + dx + W_], w_phases[2 * py + px, :, a, b, :].float())
            out[:, :, py::2, px::2] = acc
    if bias is not None:
        out = out + bias[None, :, None, None]
    return out.permute(0, 2, 3, 1)


def conv3x3(x, w, bias=None, residual=None, rowbias=None, images_per_group=0, stride=1, upsample=1, out_f32=False, impl=None,
            pad_mode=0, w_phases=None):
    assert x.is_contiguous() and w.is_contiguous() and x.dtype == w.dtype
    NB, H, W_, Cin = x.shape
    if upsample == 2 and w_phases is not None and ops.up2_phases_ok(x.dtype, NB * H * W_, residual, rowbias, out_f32, impl):
        assert tuple(w_phases.shape) == (4, w.shape[0], 2, 2, Cin) and w_phases.dtype == x.dtype
        return _store(_phase_conv(x, w_phases, bias), x.dtype).contiguous()
    xr = x.float().permute(0, 3, 1, 2)
    if upsample == 2:
        xr = F.interpolate(xr, scale_factor=2.0, mode="nearest")
    wr = w.float().permute(0, 3, 1, 2)
    if pad_mode == 1:
        y = F.conv2d(F.pad(xr, (0, 1, 0, 1)), wr, bias, stride=2)
    else:
        y = F.conv2d(xr, wr, bias, stride=stride, padding=1)
    if rowbias is not None:
        y = y + rowbias[torch.arange(NB) // images_per_group][:, :, None, None]
    y = y.permute(0, 2, 3, 1)
    if residual is not None:
        assert residual.shape == y.shape
        y = y + residual.float()
    return _store(y, torch.float32 if out_f32 else x.dtype).contiguous()


def groupnorm(x, gamma, beta, groups, eps, silu=False, stat_batches=None, x2=None, out=None):
    if out is not None:
        out.copy_(groupnorm(x, gamma, beta, groups, eps, silu=silu, stat_batches=stat_batches, x2=x2))
        return out
    if x2 is not None:          # fyc_groupnorm_concat
        x = torch.cat([x, x2], dim=-1)
    C = x.shape[-1]
    NB = x.shape[0] if stat_batches is None else stat_batches
    t = x.float().reshape(NB, -1, C).permute(0, 2, 1)
    y = F.group_norm(t, groups, gamma, beta, eps)
    if silu:
        y = F.silu(y)
    return _store(y.permute(0, 2, 1).reshape(x.shape), x.dtype).contiguous()


def layernorm(x, gamma, beta, eps=1e-5, pe=None, rows_per_frame=0, frames=0):
    C = x.shape[-1]
    y = F.layer_norm(x.float(), (C,), gamma, beta, eps)
    if pe is not None:
        rows = torch.arange(y.numel() // C)
        y = (y.view(-1, C) + pe[(rows // rows_per_frame) % frames]).view(x.shape)
    return _store(y, x.dtype)


def _mha(q, k, v, heads, D, scale, kv_batch_div):
    B, Lq = q.shape[:2]
    qh = q[..., :heads * D].float().reshape(B, Lq, heads, D).transpose(1, 2)
    kh = k[..., :heads * D].float().reshape(k.shape[0], -1, heads, D).transpose(1, 2).repeat_interleave(kv_batch_div, 0)
    vh = v[..., :heads * D].float().reshape(v.shape[0], -1, heads, D).transpose(1, 2).repeat_interleave(kv_batch_div, 0)
    p = torch.softmax(qh @ kh.transpose(-1, -2) * scale, dim=-1)
    return (p @ vh).transpose(1, 2).reshape(B, Lq, heads * D)


def attention(q, k, v, heads, scale, out=None, out_alpha=1.0, accumulate=False, kv_batch_div=1, impl=None, k2=None, v2=None, alpha2=1.0):
    def both(D):        # fyc.h second context: out_alpha * softmax(q k^T) v + alpha2 * softmax(q k2^T) v2
        y = out_alpha * _mha(q, k, v, heads, D, scale, kv_batch_div)
        return y if k2 is None else y + alpha2 * _mha(q, k2, v2, heads, D, scale, kv_batch_div)
    if out is None:
        assert not accumulate and q.shape[2] % heads == 0
        D = q.shape[2] // heads
        return _store(both(D), q.dtype)
    D = out.shape[2] // heads
    y = both(D)
    out.copy_(_store((out.float() + y) if accumulate else y, out.dtype))
    return out


def transpose_tokens(x, col0, C):
    return x[:, :, col0:col0 + C].transpose(1, 2).contiguous()


def self_attention_tc(qk, q_col0, k_col0, vt, heads, D, scale):
    NB, L, _ = qk.shape
    q = qk[:, :, q_col0:q_col0 + heads * 64].float().reshape(NB, L, heads, 64).transpose(1, 2)
    k = qk[:, :, k_col0:k_col0 + heads * 64].float().reshape(NB, L, heads, 64).transpose(1, 2)
    v = vt.float().reshape(NB, heads, D, L).transpose(2, 3)
    p = torch.softmax(q @ k.transpose(-1, -2) * scale, dim=-1)
    return _store((p @ v).transpose(1, 2).reshape(NB, L, heads * D), qk.dtype)


def self_attention_tc_d80(qkv, q_col0, k_col0, vt, heads, scale):
    NB, L, _ = qkv.shape
    D = 80
    q = qkv[:, :, q_col0:q_col0 + heads * D].float().reshape(NB, L, heads, D).transpose(1, 2)
    k = qkv[:, :, k_col0:k_col0 + heads * D].float().reshape(NB, L, heads, D).transpose(1, 2)
    v = vt.float().reshape(NB, heads, D, L).transpose(2, 3)
    p = torch.softmax(q @ k.transpose(-1, -2) * scale, dim=-1)
    return _store((p @ v).transpose(1, 2).reshape(NB, L, heads * D), qkv.dtype)


def cross_attention_tc(q, k, vt, heads, D, scale, Lk, out, k2=None, vt2=None, Lk2=0, out_alpha=1.0, alpha2=1.0, kv_batch_div=1):
    """fyc_cross_attention_tc: packed context keys (head stride 64 | 80), V^T with the keys contiguous; keys >= Lk / Lk2 are padding"""
    NB, Lq, _ = q.shape
    dkp = ops.cross_dkp(D)

    def one(kk, vv, L):
        qh = q[..., :heads * D].float().reshape(NB, Lq, heads, D).transpose(1, 2)
        kh = kk.float()[:, :L].reshape(kk.shape[0], L, -1)[..., :heads * dkp].reshape(kk.shape[0], L, heads, dkp)[..., :D].transpose(1, 2)
        vh = vv.float().reshape(vv.shape[0], heads, D, -1)[..., :L].transpose(2, 3)
        kh, vh = kh.repeat_interleave(kv_batch_div, 0), vh.repeat_interleave(kv_batch_div, 0)
        return (torch.softmax(qh @ kh.transpose(-1, -2) * scale, dim=-1) @ vh).transpose(1, 2).reshape(NB, Lq, heads * D)
    y = out_alpha * one(k, vt, Lk)
    if k2 is not None:
        y = y + alpha2 * one(k2, vt2, Lk2)
    out.copy_(_store(y, out.dtype))
    return out


def temporal_attention(qkv, heads, scale):
    B, Fr, HW, C3 = qkv.shape
    C = C3 // 3
    D = C // heads
    t = qkv.float().permute(0, 2, 1, 3).reshape(B * HW, Fr, 3, heads, D)
    q, k, v = (t[:, :, i].transpose(1, 2) for i in range(3))            # [B HW, heads, F, D]
    p = torch.softmax(q @ k.transpose(-1, -2) * scale, dim=-1)
    o = (p @ v).transpose(1, 2).reshape(B, HW, Fr, C).permute(0, 2, 1, 3)
    return _store(o, qkv.dtype).contiguous()


def softmax_rows(scores, out_dtype):
    return _store(torch.softmax(scores.float(), dim=-1), out_dtype)


def timestep_embed(t, freqs, flip_sin_to_cos):
    ang = t[:, None].float() * freqs[None, :]
    s, c = torch.sin(ang), torch.cos(ang)
    return torch.cat([c, s] if flip_sin_to_cos else [s, c], dim=-1)


def silu(x):
    return _store(F.silu(x.float()), x.dtype)


def gelu(x):
    return _store(F.gelu(x.float()), x.dtype)


def upsample_nearest2x(x):
    return x.repeat_interleave(2, 1).repeat_interleave(2, 2).contiguous()


def concat_channels(a, b):
    return torch.cat([a, b], dim=-1).contiguous()


def ncfhw_to_nfhwc(x, dtype, scale=1.0):
    return _store((x * scale).permute(0, 2, 3, 4, 1), dtype).contiguous()


def nfhwc_to_ncfhw(x):
    ops._channel_sliced(x)            # the product's own view check (contiguous, or a [..., :C] slice of a wider channels-last tensor)
    return x.float().permute(0, 4, 1, 2, 3).contiguous()


def build_unet_input(latents, mask, first, dup, dtype, c_pad=None, out=None):
    b, c, f, h, w = latents.shape
    cin = 9 if first is not None else 4
    c_pad = cin if c_pad is None else c_pad
    x = torch.zeros(b, f, h, w, c_pad)
    x[..., :4] = latents.permute(0, 2, 3, 4, 1)
    if first is not None:
        if mask is not None:
            x[..., 4] = mask.reshape(b, 1, h, w).clamp(0, 1)
        else:
            x[:, 0, :, :, 4] = 1.0
        x[:, 0, :, :, 5:9] = first.permute(0, 2, 3, 1)
    x = _store(torch.cat([x] * dup, dim=0), dtype)
    if out is not None:
        out.copy_(x)
        return out
    return x


def build_unet_input_first(latents, first, dup, dtype, mode, c_pad=None, out=None):
    b, c, f, h, w = latents.shape
    cin = 8 if mode & ops.FIRST_CONCAT else 4
    c_pad = cin if c_pad is None else c_pad
    if mode & ops.FIRST_FRAME:
        latents[:, :, 0] = first                      # in place: the DDIM step that follows reads the replaced frame
    x = torch.zeros(b, f, h, w, c_pad)
    x[..., :4] = latents.permute(0, 2, 3, 4, 1)
    if mode & ops.FIRST_CONCAT:
        x[..., 4:8] = first.permute(0, 2, 3, 1)[:, None]
    x = _store(torch.cat([x] * dup, dim=0), dtype)
    if out is not None:
        out.copy_(x)
        return out
    return x


def first_frame_temb_rows(temb, B, F):
    idx = torch.tensor([B if f == 0 else bi for bi in range(B) for f in range(F)])
    return temb[idx].contiguous()


def cfg_ddim_step(pred, sample, coefs, noise=None, out=None, single=None, video_scale=0.0):
    c = coefs
    n = sample.numel()
    p = pred.reshape(-1)
    if single is not None:
        sg = single.reshape(-1)
        m = sg + video_scale * (p[:n] - sg) + c.guidance * (p[n:2 * n] - p[:n])
    else:
        m = p[:n] + c.guidance * (p[n:2 * n] - p[:n]) if c.cfg_pair else p[:n]
    x = sample.reshape(-1)
    if c.prediction_type == _lib.PRED["epsilon"]:
        x0, eps = (x - c.sqrt_beta_t * m) / c.sqrt_alpha_t, m
    elif c.prediction_type == _lib.PRED["sample"]:
        x0, eps = m, m
    else:
        x0, eps = c.sqrt_alpha_t * x - c.sqrt_beta_t * m, c.sqrt_alpha_t * m + c.sqrt_beta_t * x
    if c.clip_sample:
        x0 = x0.clamp(-1, 1)
    r = c.sqrt_alpha_prev * x0 + c.dir_coef * eps
    if noise is not None:
        r = r + c.noise_coef * noise.reshape(-1)
    r = r.view(sample.shape)
    if out is not None:
        out.copy_(r)
        return out
    return r


def frames_finalize(x, b, f):
    ops._channel_sliced(x)
    _, H, W_, c = x.shape
    assert c == 3
    return (x.float().reshape(b, f, H, W_, 3).permute(0, 4, 1, 2, 3) / 2 + 0.5).clamp(0, 1).contiguous()


def video_grid_u8(video, nrow=6, padding=2, rescale=False):
    import numpy as np
    from oracle import ref_util
    return torch.from_numpy(np.stack(ref_util.video_frames_uint8(video, rescale=rescale, n_rows=nrow)))


_NAMES = ["tc_available", "require_cuda", "layernorm_stats", "gemm", "conv3x3", "groupnorm", "layernorm", "attention", "transpose_tokens",
          "self_attention_tc", "self_attention_tc_d80", "cross_attention_tc", "temporal_attention", "softmax_rows", "timestep_embed", "silu", "gelu",
          "upsample_nearest2x", "concat_channels", "ncfhw_to_nfhwc", "nfhwc_to_ncfhw", "build_unet_input", "build_unet_input_first",
          "first_frame_temb_rows", "cfg_ddim_step", "frames_finalize", "video_grid_u8"]


def _library_callers():
    """the public functions of ops whose own code calls into the library: they name ``lib`` (a query or launch) or ``check`` (the status
    of a launch, also of those made through a private helper such as ops._tc_entry)"""
    return {n for n, f in vars(ops).items() if inspect.isfunction(f) and f.__module__ == ops.__name__ and not n.startswith("_")
            and {"lib", "check"} & set(f.__code__.co_names)}


def install(monkeypatch):
    """Replace the hardware query ops.tc_available (answered True), ops.require_cuda and every kernel-launching function of
    followyourclick_b200.ops for the duration of a test.  The route rules (ops.tc_ok, ops.self_attention_tc_ok, ...) stay the product's."""
    missing = _library_callers() - set(_NAMES)
    assert not missing, f"ops functions that call the library have no emulation here: {sorted(missing)}"
    g = globals()
    for n in _NAMES:
        assert hasattr(ops, n), n
        monkeypatch.setattr(ops, n, g[n])
