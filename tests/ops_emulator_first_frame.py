"""tests/ops_emulator.py plus the first-frame condition kernels: torch restatements of the fyc.h contracts of
fyc_build_unet_input_first and fyc_first_frame_temb_rows, for the CPU tests of the host code."""
import torch

from followyourclick_b200 import ops
from tests import ops_emulator
from tests.ops_emulator import _store


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


def install(monkeypatch):
    """ops_emulator.install, then the two first-frame kernels"""
    ops_emulator.install(monkeypatch)
    for n in ("build_unet_input_first", "first_frame_temb_rows"):
        assert hasattr(ops, n), n
        monkeypatch.setattr(ops, n, globals()[n])
