"""Mini configurations of the first-frame-conditioned motion models (configs/training/org_config_files/training_w_first_frame.yaml:
use_first_frame_condition; training_w_first_frame_concat.yaml and the 14M concat configs: use_first_frame_condition_concat).

Same widths / heads as the shipped mini UNet of tests/cfgs.py, with the mask-concat stem replaced by the mode's own: a 4-channel conv_in
for the first-frame condition, an 8-channel one for the concat.  ``fps``: the fps / motion embeddings on (a combination the reference
samples with the concat mode, and with the first-frame condition only at a UNet batch of 1).
"""
import torch

from oracle.ref_unet import default_unet_config
from tests.cfgs import mini_unet_ref_kwargs

MODES = ("ff", "ffc")            # use_first_frame_condition, use_first_frame_condition_concat
F_, H_, W_ = 4, 16, 16            # UNet-forward fixtures: frames, latent height / width
PIPE_F, PIPE_HW, PIPE_STEPS, PIPE_GS, PIPE_VS = 4, 8, 2, 8.0, 0.7


def ff_ref_kwargs(mode, fps=False):
    """constructor kwargs accepted by the reference UNet3DConditionModel and by ours"""
    kw = dict(mini_unet_ref_kwargs("base"), use_first_frame_mask_condition_concat=False, use_fps_condition=fps)
    if mode == "ffc":
        kw["use_first_frame_condition_concat"] = True
    return kw


def ff_oracle_cfg(mode, fps=False):
    kw = ff_ref_kwargs(mode, fps)
    mm = {k: v for k, v in kw["motion_module_kwargs"].items() if k != "zero_initialize"}
    return default_unet_config(block_out_channels=kw["block_out_channels"], layers_per_block=kw["layers_per_block"],
                               attention_head_dim=kw["attention_head_dim"], motion_module_kwargs=mm,
                               use_first_frame_mask_condition_concat=False, use_first_frame_condition_concat=(mode == "ffc"),
                               use_fps_condition=fps)


# UNet-forward cases of tests/golden/first_frame_unet.npz: name -> (mode, fps model, batch, CFG-shaped: the two halves of the batch
# carry the same latents (and first-image latents) as the reference's torch.cat([latents] * 2) does, so the shared CFG prefix applies)
UNET_CASES = {
    "ff": ("ff", False, 2, False),
    "ff_cfg": ("ff", False, 2, True),
    "ff_fps_b1": ("ff", True, 1, False),       # the fps embedding broadcasts onto the 2-row emb at a batch of 1
    "ffc": ("ffc", True, 2, False),
    "ffc_cfg": ("ffc", True, 2, True),
}


def unet_case_inputs(name, seed=31):
    """sample (b, 4, F, H, W), timestep, ctx (b, 77, 768), first (b, 4, H, W) and fps / flow for case ``name``."""
    mode, fps, b, cfg = UNET_CASES[name]
    g = torch.Generator().manual_seed(seed)
    nb = 1 if cfg else b
    sample = torch.randn(nb, 4, F_, H_, W_, generator=g)
    first = torch.randn(nb, 4, H_, W_, generator=g)
    if cfg:
        sample, first = torch.cat([sample] * 2), torch.cat([first] * 2)
    if mode == "ff":                # the pipeline hands the UNet latents whose frame 0 IS the first-image latents (:691-692)
        sample[:, :, 0] = first
    d = dict(sample=sample, first=first, timestep=torch.tensor(501), ctx=torch.randn(b, 77, 768, generator=g))
    if fps:
        d["fps"], d["flow"] = torch.tensor([2] * b), torch.tensor([4] * b)
    return d


# 2-step pipeline cases of tests/golden/first_frame_pipeline.npz: name -> (mode, fps model, guidance, video_scale)
PIPE_CASES = {
    "ff": ("ff", False, PIPE_GS, 0.0),
    "ffc": ("ffc", True, PIPE_GS, 0.0),
    "ff_vs": ("ff", False, PIPE_GS, PIPE_VS),
    "ff_fps_nocfg": ("ff", True, 1.0, 0.0),
}


def pipe_case_kwargs(name, ci):
    """reference-pipeline / engine-pipeline kwargs of case ``name`` on the clip inputs ``ci`` (followyourclick_b200.synth.synth_clip_inputs)"""
    mode, fps, gs, vs = PIPE_CASES[name]
    kw = dict(first_image_latents=ci["first_image_latents"], video_scale=vs)
    kw["use_first_frame_condition" if mode == "ff" else "use_first_frame_condition_concat"] = True
    if fps:
        kw.update(use_fps_condition=True, fps_tensor=torch.tensor([2]), flow_control=torch.tensor([4]))
    return kw


def pipe_case_oracle_kwargs(name, ci):
    mode, fps, gs, vs = PIPE_CASES[name]
    okw = dict(first_image_latents=ci["first_image_latents"], video_scale=vs, use_first_frame_condition=(mode == "ff"))
    if fps:
        okw.update(fps_tensor=torch.tensor([2]), flow_control=torch.tensor([4]))
    return okw
