"""Test configuration of the SD-2.x-based motion model ("mini" = the reference architecture at reduced width / depth), and the state-dict
adapter its oracle needs.

The mini model keeps the unet_additional_kwargs of configs/training/org_config_files/training_14M_448x256_w_multi_scale_w_fps_sd_v2.1.yaml on
the SD-2.1 unet/config.json settings (use_linear_projection, upcast_attention, per-level attention_head_dim, 1024-wide text context),
with v-prediction.  The per-level head counts keep SD-2.x's spatial head dim 64 at every level; 4 temporal heads give temporal head dims
32 / 64 / 128 (the temporal kernels take any multiple of 8 up to 160).  It is deliberately not one of tests/cfgs.MINI_UNET_VARIANTS: it has
its own fixtures (tests/golden/make_golden_sd2.py) and tests.
"""
import re

import torch

from oracle.ref_unet import default_unet_config

SD2_CTX_DIM = 1024
_MM_SD2 = dict(num_attention_heads=4, num_transformer_block=1, attention_block_types=("Temporal_Self", "Temporal_Self"),
               temporal_position_encoding=True, temporal_position_encoding_max_len=32, temporal_attention_dim_div=1,
               zero_initialize=True)
MINI_SD2 = dict(sample_size=16, in_channels=4, out_channels=4, block_out_channels=(128, 256, 512, 512), layers_per_block=1,
                attention_head_dim=[2, 4, 8, 8], cross_attention_dim=SD2_CTX_DIM, norm_num_groups=32, use_linear_projection=True,
                upcast_attention=True, use_motion_module=True, motion_module_resolutions=(1, 2, 4, 8), unet_use_cross_frame_attention=False,
                unet_use_temporal_attention=False, use_inflated_groupnorm=True, motion_module_mid_block=True, use_fps_condition=True,
                motion_module_type="Vanilla", motion_module_kwargs=dict(_MM_SD2))
# the 2-D base of the same width (a SD-2.1-layout unet/config.json at mini size)
MINI_SD2_2D = dict(sample_size=16, in_channels=4, out_channels=4, block_out_channels=(128, 256, 512, 512), layers_per_block=1,
                   attention_head_dim=[2, 4, 8, 8], cross_attention_dim=SD2_CTX_DIM, norm_num_groups=32, use_linear_projection=True,
                   upcast_attention=True)


def mini_sd2_oracle_cfg(two_d=False):
    mm = {k: v for k, v in _MM_SD2.items() if k != "zero_initialize"}
    kw = MINI_SD2_2D if two_d else MINI_SD2
    return default_unet_config(block_out_channels=kw["block_out_channels"], layers_per_block=1, attention_head_dim=kw["attention_head_dim"],
                               cross_attention_dim=SD2_CTX_DIM, use_motion_module=not two_d, use_inflated_groupnorm=not two_d,
                               motion_module_mid_block=not two_d, motion_module_kwargs=mm, use_first_frame_mask_condition_concat=False,
                               use_fps_condition=not two_d)


def sd2_inputs(b=2, f=4, h=16, w=16, seed=41):
    g = torch.Generator().manual_seed(seed)
    return dict(sample=torch.randn(b, 4, f, h, w, generator=g), timestep=torch.tensor(501), ctx=torch.randn(b, 77, SD2_CTX_DIM, generator=g),
                fps=torch.tensor([3] * b), flow=torch.tensor([5] * b))


_SPATIAL_PROJ = re.compile(r"\.attentions\.\d+\.proj_(in|out)\.weight$")


def oracle_state_dict(sd):
    """An SD-2.x state dict in the form the fp32 oracle (oracle/ref_unet.transformer_3d) reads.  With use_linear_projection the
    Transformer3DModel's proj_in / proj_out are Linear (C, C) layers applied to the tokens (animatediff/models/attention.py:179-215,
    270-295); the oracle applies them as 1x1 convolutions, which is the same per-token product y = W x + b.  The Linear weight [C, C] is
    that convolution's [C, C, 1, 1] filter; nothing else differs."""
    return {k: (v.reshape(*v.shape, 1, 1) if v.dim() == 2 and _SPATIAL_PROJ.search(k) else v) for k, v in sd.items()}
