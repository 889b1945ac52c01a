"""The kernel plans that shipped resolutions and frame counts select, restated from the rules that pick them (pure Python).

A kernel's tile plan depends on the latent grid, the frame count and the batch, not only on the layer.  The table below lists the
resolutions the engine is run at; ``levels`` derives every UNet level's grid and what each rule selects there:

* conv patch geometry: ``pick_patch`` (csrc/gemm_tc.cu) tiles 128 output pixels as bw x bh x bn - bw the largest power of two <= 128
  dividing Wo, then bh the largest dividing Ho with bw bh <= 128, bn = 128 / (bw bh) images, which must divide NB; otherwise the
  convolution runs on the CUDA-core kernel.  Stride-2 convolutions tile their output grid, the four-phase upsampler its low-resolution
  input grid; an upsampler whose low-resolution grid has no patch materialises the upsample and tiles the high-resolution grid;
* self-attention route (ops.self_attention_tc_ok / self_attention_tc80_ok): the wgmma kernel for D = 40 / 64 when L % 128 == 0 and for
  D = 80 when L % 256 == 0 (128-key tiles), else the mma.sync kernel (64-key tiles).

tests/test_kernel_plans_gpu.py runs the kernels at these plans; tests/test_kernel_plans_cpu.py checks that they cover every patch
geometry.
"""
from dataclasses import dataclass

CHANNELS = (320, 640, 1280, 1280)      # UNet width per level (SD-1.5 and SD-2.x)


@dataclass(frozen=True)
class Resolution:
    name: str
    h: int                # latent grid (pixels / 8)
    w: int
    frames: int
    head_dim: int = 0     # 0: SD-1.5 (8 heads, D = C / 8); else SD-2.x (D fixed, C / D heads)

    @property
    def nb(self):
        return 2 * self.frames           # the CFG pair of one clip: images per UNet call; a clip's frames share a time embedding


RESOLUTIONS = (
    Resolution("256x256", 32, 32, 16),
    Resolution("384x384", 48, 48, 16),
    Resolution("320x576", 40, 72, 16),
    Resolution("512x256", 64, 32, 16),
    Resolution("768x768_F32", 96, 96, 32),
    Resolution("384x384_sd2", 48, 48, 16, head_dim=64),
)
BY_NAME = {r.name: r for r in RESOLUTIONS}


def pick_patch(NB, Ho, Wo):
    """csrc/gemm_tc.cu pick_patch: (bw, bh, bn) or None (no tensor-core plan)"""
    w = 1
    while w < 128 and Wo % (2 * w) == 0:
        w *= 2
    h = 1
    while w * h < 128 and Ho % (2 * h) == 0:
        h *= 2
    n = 128 // (w * h)
    return (w, h, n) if NB % n == 0 else None


def conv_plan(kind, NB, h, w):
    """(route, patch) of a 3x3 conv on an h x w input grid of NB images.  kind "s1"; "s2" (stride 2, padding 1: the patch tiles the
    h/2 x w/2 output grid of an even grid); "up2" (nearest x2 + conv: the four-phase kernel tiles the low-resolution grid; without a
    patch there the upsample is materialised and the 2h x 2w grid is tiled).  route: "tc", "tc_up2", "upsample_tc" or "simt" /
    "upsample_simt" (no patch: the CUDA-core kernel)."""
    if kind == "s1":
        p = pick_patch(NB, h, w)
    elif kind == "s2":
        p = pick_patch(NB, h // 2, w // 2) if h % 2 == 0 and w % 2 == 0 else None
    else:
        assert kind == "up2", kind
        p = pick_patch(NB, h, w)
        if p:
            return "tc_up2", p
        p = pick_patch(NB, 2 * h, 2 * w)
        return ("upsample_tc" if p else "upsample_simt"), p
    return ("tc" if p else "simt"), p


def attention_route(L, D):
    """(route, key tiles): "wgmma" (fyc_self_attention_tc), "wgmma_d80" (fyc_self_attention_tc_d80) or "mma" (fyc_attention)"""
    if D in (40, 64) and L % 128 == 0:
        return "wgmma", L // 128
    if D == 80 and L % 256 == 0:
        return "wgmma_d80", L // 128
    return "mma", -(-L // 64)


@dataclass(frozen=True)
class Level:
    res: str
    level: int
    h: int
    w: int
    channels: int
    nb: int
    frames: int
    patch: object             # stride-1 3x3 conv on this grid
    down_patch: object        # stride-2 conv from this grid to the next level (None: odd grid or no patch; not at the last level)
    up_patch: object          # four-phase upsampler on this (low-resolution) grid up to the level above (levels 1..3)
    up_materialised: object   # the patch of the materialised upsample when up_patch is None
    heads: int
    head_dim: int
    attn_route: str
    key_tiles: int

    @property
    def rows(self):
        return self.nb * self.h * self.w


def levels(res):
    out, h, w = [], res.h, res.w
    for lv, C in enumerate(CHANNELS):
        D = res.head_dim or C // 8
        last = lv == len(CHANNELS) - 1
        down = None if last else conv_plan("s2", res.nb, h, w)[1]
        up_route, up_p = conv_plan("up2", res.nb, h, w) if lv > 0 else (None, None)
        up, up_mat = (up_p, None) if up_route == "tc_up2" else (None, up_p)
        route, tiles = attention_route(h * w, D)
        out.append(Level(res.name, lv, h, w, C, res.nb, res.frames, pick_patch(res.nb, h, w), down, up, up_mat, C // D, D, route, tiles))
        h, w = -(-h // 2), -(-w // 2)        # stride 2, padding 1
    return out


def all_levels():
    return [lv for r in RESOLUTIONS for lv in levels(r)]


def level(name, lv):
    return levels(BY_NAME[name])[lv]


# bn = 16 needs a 4 x 2 grid (bw 4, bh 2), which no listed resolution produces: one synthetic grid for every conv kind
SYNTHETIC_BN16 = dict(h=2, w=4, nb=32)
