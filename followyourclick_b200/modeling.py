"""Host-side object model shared by the drop-in classes.

The reference classes derive from diffusers 0.11.1 ``ModelMixin`` / ``ConfigMixin`` (diffusers/modeling_utils.py,
configuration_utils.py).  The engine keeps their *observable surface* - ``.config`` (attribute + mapping access),
``.dtype`` / ``.device`` / ``.to()``, ``state_dict()`` / ``load_state_dict()`` with the reference key names,
``enable_xformers_memory_efficient_attention()`` - on top of a generic parameter tree whose forward pass is the CUDA
engine, not nn.Module composition.
"""
from collections import OrderedDict

import torch
from torch import nn

from . import ops


class FrozenDict(OrderedDict):
    """Read-only mapping with attribute access (mirror of diffusers.configuration_utils.FrozenDict)."""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        for k, v in self.items():
            object.__setattr__(self, k, v)
        object.__setattr__(self, "_frozen", True)

    def __setitem__(self, k, v):
        if getattr(self, "_frozen", False):
            raise TypeError("FrozenDict is immutable")
        super().__setitem__(k, v)

    def __setattr__(self, k, v):
        if getattr(self, "_frozen", False):
            raise TypeError("FrozenDict is immutable")
        super().__setattr__(k, v)


class _Node(nn.Module):
    """Anonymous container; children named after the dotted key components ('0', 'resnets', 'to_q', ...)."""


class ParamTreeModel(nn.Module):
    """nn.Module whose parameters/buffers are created from a flat {dotted key: shape} spec.

    ``state_dict()`` therefore has exactly the spec's keys (= the reference's key contract, SURVEY App. E), and
    ``load_state_dict`` works as for any module.  Sub-classes implement the forward pass with followyourclick_b200.ops
    on *packed* copies of the weights (bf16/fp32, conv filters re-laid out as [Cout, 3, 3, Cin], q/k/v fused ...),
    built lazily by ``_packed()`` and invalidated whenever the parameters may have changed.
    """

    _BUFFER_SUFFIXES = (".pe",)

    def _build_tree(self, spec, buffers=None):
        buffers = buffers or {}
        for key, shape in spec.items():
            parts = key.split(".")
            node = self
            for p in parts[:-1]:
                nxt = node._modules.get(p)
                if nxt is None:
                    nxt = _Node()
                    node.add_module(p, nxt)
                node = nxt
            if key in buffers:
                node.register_buffer(parts[-1], buffers[key].clone(), persistent=True)
            else:
                node.register_parameter(parts[-1], nn.Parameter(torch.zeros(tuple(shape)), requires_grad=False))
        self._pack_cache = {}
        self._flat = None
        self._pack_version = 0
        self._compute_dtype = torch.float32
        self._xformers_semantics = False

    # ---- reference-surface helpers -------------------------------------------------------------------------
    @property
    def dtype(self):
        return self._compute_dtype

    @property
    def device(self):
        return next(self.parameters()).device

    def _invalidate(self):
        self._pack_cache = {}
        self._flat = None
        self._pack_version += 1

    def load_state_dict(self, state_dict, strict=True, **kw):
        r = super().load_state_dict(state_dict, strict=strict, **kw)
        self._invalidate()
        return r

    def to(self, *args, **kwargs):
        """Moves master weights; a floating dtype selects the *compute* dtype (fp32 strict / bf16 tensor-core;
        fp16 maps to bf16, the engine's 16-bit format) - master weights stay fp32 so re-packing is lossless."""
        dtype = kwargs.pop("dtype", None)
        rest = []
        for a in args:
            if isinstance(a, torch.dtype):
                dtype = a
            else:
                rest.append(a)
        if dtype is not None:
            if dtype in (torch.float16, torch.bfloat16):
                self._compute_dtype = torch.bfloat16
            elif dtype == torch.float32:
                self._compute_dtype = torch.float32
            else:
                raise ValueError(f"unsupported compute dtype {dtype}")
        if rest or kwargs:
            super().to(*rest, **kwargs)
        self._invalidate()
        return self

    def set_compute_dtype(self, dtype):
        """Select the compute dtype directly: torch.float32 (strict fp32, CUDA cores), torch.bfloat16 (the default tensor-core mode) or
        torch.float16 (the tensor-core mode in IEEE half: the precision of the reference's torch.autocast("cuda"); activations must stay
        below 65504).  `.to(torch.float16)` / `.half()` keep selecting bf16; this is the one way to run in fp16."""
        ops.check_compute_dtype(dtype)
        self._compute_dtype = dtype
        self._invalidate()
        return self

    def cuda(self, device=None):
        super().cuda(device)
        self._invalidate()
        return self

    def half(self):
        return self.to(torch.float16)

    def bfloat16(self):
        return self.to(torch.bfloat16)

    def float(self):
        return self.to(torch.float32)

    def enable_xformers_memory_efficient_attention(self, *a, **kw):
        """scripts/inference.py:157 calls this and asserts success.  The engine's fused attention never materialises
        scores, so there is nothing to switch on - except the one numerical difference between the reference's two
        attention paths: with xformers the IP cross-attention logits are scaled by d^-1/2, without it by the IP scale
        (reference quirk, animatediff/models/attention.py:43).  This flag selects the xformers semantics."""
        self._xformers_semantics = True

    def disable_xformers_memory_efficient_attention(self):
        self._xformers_semantics = False

    def set_use_memory_efficient_attention_xformers(self, valid=True):
        self._xformers_semantics = bool(valid)

    def enable_gradient_checkpointing(self):
        pass

    def requires_grad_(self, flag=False):
        return self

    # ---- packing helpers -----------------------------------------------------------------------------------
    def _flat_params(self):
        if self._flat is None:
            self._flat = self.state_dict(keep_vars=True)
        return self._flat

    def _p(self, key):
        """master (fp32) tensor for a dotted key"""
        return self._flat_params()[key]

    def _has(self, key):
        return key in self._flat_params()

    def _cached(self, name, fn):
        c = self._pack_cache
        if name not in c:
            c[name] = fn()
        return c[name]

    def _w(self, key):
        """weight in compute dtype, contiguous"""
        return self._cached(("w", key), lambda: self._p(key).detach().to(self._compute_dtype).contiguous())

    def _f(self, key):
        """fp32 vector (bias / norm gamma / beta)"""
        return self._cached(("f", key), lambda: self._p(key).detach().float().contiguous())

    def _conv_w(self, key):
        """[Cout, Cin, 3, 3] -> [Cout, 3, 3, Cin] in compute dtype"""
        return self._cached(("c", key), lambda: self._p(key).detach().permute(0, 2, 3, 1).to(self._compute_dtype).contiguous())

    def _conv_w_up2(self, key):
        """phase-summed filter of an upsampler conv, [4, Cout, 2, 2, Cin] (16-bit tensor-core mode only, else None)"""
        if self._compute_dtype not in ops.HALF_DTYPES:
            return None
        return self._cached(("up2", key), lambda: upsample_phase_weights(self._p(key).detach().float()).to(self._compute_dtype).contiguous())

    def _conv_head(self, name, pixels):
        """(filter [N, 3, 3, Cin], bias [N], true Cout) of a 3- / 4-channel output convolution.  In tensor-core mode the output
        channels are zero-padded to N = 16 so the head is a tensor-core implicit GEMM (its N must be a multiple of 16) instead of a
        CUDA-core kernel; consumers read the first Cout of the 16 channels (fyc_nfhwc_to_ncfhw / fyc_frames_finalize `ldc`)."""
        cout = self._p(name + ".weight").shape[0]
        if not (ops.use_tc_head and cout < 16 and ops.tc_ok(self._compute_dtype, pixels)):
            return self._conv_w(name + ".weight"), self._f(name + ".bias"), cout

        def make():
            w = self._conv_w(name + ".weight")
            wp = torch.zeros((16,) + tuple(w.shape[1:]), dtype=w.dtype, device=w.device)
            wp[:cout] = w
            bp = torch.zeros(16, dtype=torch.float32, device=w.device)
            bp[:cout] = self._f(name + ".bias")
            return wp, bp
        wp, bp = self._cached(("head16", name), make)
        return wp, bp, cout

    def _w1x1(self, key):
        """1x1 conv weight [Cout, Cin, 1, 1] -> [Cout, Cin]"""
        return self._cached(("1", key), lambda: self._p(key).detach().flatten(1).to(self._compute_dtype).contiguous())


def geglu_interleave(w, b):
    """Re-order the rows of the GEGLU projection (diffusers/models/attention.py:800-821: [a | gate] halves) into
    256-row tiles [a_t(128) | gate_t(128)] so one GEMM tile holds matching a/gate columns (fyc.h FYC_EPI_GEGLU)."""
    hd = w.shape[0] // 2
    assert hd % 128 == 0, hd
    a, g = w[:hd].reshape(hd // 128, 128, -1), w[hd:].reshape(hd // 128, 128, -1)
    wi = torch.cat([a, g], dim=1).reshape(2 * hd, -1)
    ba, bg = b[:hd].reshape(hd // 128, 128), b[hd:].reshape(hd // 128, 128)
    return wi.contiguous(), torch.cat([ba, bg], dim=1).reshape(2 * hd).contiguous()


def upsample_phase_weights(w):
    """[Cout, Cin, 3, 3] fp32 -> [4, Cout, 2, 2, Cin]: nearest-x2 upsampling followed by a zero-padded 3x3 convolution
    (animatediff/models/resnet.py:155-168, diffusers/models/resnet.py:128-139) restated per output parity.  Output pixel
    (2*oh + py, 2*ow + px) reads upsampled rows 2*oh + py + kh - 1, i.e. source rows {oh-1, oh, oh} for py = 0 and {oh, oh, oh+1}
    for py = 1, so the three filter rows collapse to two taps: py = 0 -> (oh-1: w[0]; oh: w[1]+w[2]), py = 1 -> (oh: w[0]+w[1];
    oh+1: w[2]); columns alike.  Phase index 2*py + px, tap (a, b) reads source pixel (oh + a - 1 + py, ow + b - 1 + px).
    The sums are taken in fp32 before the single rounding to the compute dtype."""
    rows = (((0,), (1, 2)), ((0, 1), (2,)))
    Cout, Cin = w.shape[:2]
    out = torch.zeros(4, Cout, 2, 2, Cin, dtype=torch.float32, device=w.device)
    for py in range(2):
        for px in range(2):
            for a in range(2):
                for b in range(2):
                    acc = 0
                    for kh in rows[py][a]:
                        for kw in rows[px][b]:
                            acc = acc + w[:, :, kh, kw]
                    out[2 * py + px, :, a, b, :] = acc
    return out
