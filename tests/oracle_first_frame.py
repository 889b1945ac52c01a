"""Oracle of the first-frame-conditioned motion models: fp32 restatement of the reference's two image-to-video modes, built on the
primitives of oracle/ref_unet.py and oracle/ref_pipeline.py (which it leaves as they are).

  use_first_frame_condition        pipeline_animation.py:691-692 (frame 0 of the latents replaced before every step, in the tensor the
                                   step then reads); unet.py:523-524 (a zero timestep appended: emb has B + 1 rows); resnet.py:304-320
                                   (every ResnetBlock3D adds the t = 0 row to frame 0 and the clip's row to frames 1..).  The B-row
                                   camera / fps / motion embeddings are added to the (B + 1)-row emb as the reference does: a broadcast
                                   that only runs for B == 1.
  use_first_frame_condition_concat pipeline_animation.py:717-719 (the CFG-duplicated first-image latents handed to the UNet);
                                   unet.py:578-590 (concatenated on every frame, conv_in output halved) - ref_unet.unet3d_forward already
                                   restates the UNet side.

TEST INFRASTRUCTURE: imported by the tests and by tests/golden/make_golden_first_frame.py only.
"""
import torch
import torch.nn.functional as F

from oracle import ref_unet as R
from oracle.ref_ddim import DDIMOracle, cfg_combine
from oracle.ref_pipeline import build_unet_input


def resnet_block_3d(sd, p, x, emb, cfg):
    """animatediff/models/resnet.py:296-342 with the first-frame branch of :304-320 (emb has one row more than x has clips)."""
    g, eps, pf = cfg["norm_num_groups"], cfg["norm_eps"], cfg["use_inflated_groupnorm"]
    h = F.silu(R.group_norm_5d(sd, p + ".norm1", x, g, eps, pf))
    h = R.conv2d_per_frame(sd, p + ".conv1", h)
    t = F.linear(F.silu(emb), sd[p + ".time_emb_proj.weight"], sd[p + ".time_emb_proj.bias"])
    bz = h.shape[0]
    assert t.shape[0] == bz + 1
    z = torch.zeros_like(h)
    z[:, :, 0] = z[:, :, 0] + t[bz:].repeat(bz, 1)[:, :, None, None]          # frame 0: the t = 0 row
    z[:, :, 1:] = z[:, :, 1:] + t[:bz, :, None, None, None]                   # frames 1..: the clip's row
    h = F.silu(R.group_norm_5d(sd, p + ".norm2", h + z, g, eps, pf))
    h = R.conv2d_per_frame(sd, p + ".conv2", h)
    if (p + ".conv_shortcut.weight") in sd:
        x = R.conv2d_per_frame(sd, p + ".conv_shortcut", x, padding=0)
    return x + h


def unet3d_forward(sd, cfg, sample, timestep, encoder_hidden_states, fps_tensor=None, flow_control=None,
                   reference_images_clip_feat=None, camera_movement_type_tensor=None, use_first_frame_condition_concat=False,
                   reference_images_latent=None, use_first_frame_condition=False):
    """animatediff/models/unet.py:422-672 with ``use_first_frame_condition``; without it, oracle/ref_unet.unet3d_forward."""
    kw = dict(fps_tensor=fps_tensor, flow_control=flow_control, reference_images_clip_feat=reference_images_clip_feat,
              camera_movement_type_tensor=camera_movement_type_tensor, use_first_frame_condition_concat=use_first_frame_condition_concat,
              reference_images_latent=reference_images_latent)
    if not use_first_frame_condition:
        return R.unet3d_forward(sd, cfg, sample, timestep, encoder_hidden_states, **kw)
    sd = {k: v.float() for k, v in sd.items()}
    sample = sample.float()
    B = sample.shape[0]
    boc = cfg["block_out_channels"]
    n_lvl = len(boc)

    def as_vec(v):
        v = torch.as_tensor(v).to(sample.device)
        return (v[None] if v.dim() == 0 else v).expand(B)

    def sinus(v):
        return R.timestep_sinusoid(v, boc[0], cfg["flip_sin_to_cos"], cfg["freq_shift"])

    ts = as_vec(timestep)
    ts = torch.cat([ts, torch.zeros(1, dtype=ts.dtype, device=ts.device)])                 # unet.py:523-524
    emb = R.timestep_mlp(sd, "time_embedding", sinus(ts))
    if cfg["use_camera_motion_condition"] and camera_movement_type_tensor is not None:      # :537-542 (B rows onto B + 1)
        emb = emb + R.timestep_mlp(sd, "camera_motion_embedding", sinus(as_vec(camera_movement_type_tensor)))
    if cfg["use_fps_condition"] and fps_tensor is not None:                                  # :545-558
        emb = emb + R.timestep_mlp(sd, "fps_embedding", sinus(as_vec(fps_tensor)))
        emb = emb + R.timestep_mlp(sd, "motion_embedding", sinus(as_vec(flow_control)))
    if use_first_frame_condition_concat and reference_images_latent is not None:            # :578-583
        first = reference_images_latent.float().unsqueeze(2).repeat(1, 1, sample.shape[2], 1, 1)
        sample = torch.cat((sample, first), dim=1)
    x = R.conv2d_per_frame(sd, "conv_in", sample)                                           # :586
    if use_first_frame_condition_concat:
        x = x / 2                                                                           # :589-590
    ctx = encoder_hidden_states.float()
    if cfg["use_ip_cross_attention"] and reference_images_clip_feat is not None:
        ctx = torch.cat([ctx, R.image_proj(sd, reference_images_clip_feat.float(), cfg)], dim=1)   # :592-594

    def maybe_motion(p, x, res_index, decoder):
        on = cfg["use_motion_module"] and (2 ** res_index) in cfg["motion_module_resolutions"]
        if not decoder and cfg["motion_module_decoder_only"]:
            on = False
        return R.motion_module(sd, p, x, cfg) if on else x

    skips = [x]
    for i in range(n_lvl):                                                                  # down, :601-626
        p = f"down_blocks.{i}"
        for j in range(cfg["layers_per_block"]):
            x = resnet_block_3d(sd, f"{p}.resnets.{j}", x, emb, cfg)
            if i < n_lvl - 1:
                x = R.transformer_3d(sd, f"{p}.attentions.{j}", x, ctx, R._heads(cfg, i), cfg)
            x = maybe_motion(f"{p}.motion_modules.{j}", x, i, decoder=False)
            skips.append(x)
        if i < n_lvl - 1:
            x = R.conv2d_per_frame(sd, f"{p}.downsamplers.0.conv", x, stride=2)
            skips.append(x)
    x = resnet_block_3d(sd, "mid_block.resnets.0", x, emb, cfg)                             # unet_blocks.py:342-360
    x = R.transformer_3d(sd, "mid_block.attentions.0", x, ctx, R._heads(cfg, n_lvl - 1), cfg)
    if cfg["use_motion_module"] and cfg["motion_module_mid_block"]:
        x = R.motion_module(sd, "mid_block.motion_modules.0", x, cfg)
    x = resnet_block_3d(sd, "mid_block.resnets.1", x, emb, cfg)
    for i in range(n_lvl):                                                                  # up, :636-660
        p = f"up_blocks.{i}"
        lvl = n_lvl - 1 - i
        for j in range(cfg["layers_per_block"] + 1):
            x = torch.cat([x, skips.pop()], dim=1)
            x = resnet_block_3d(sd, f"{p}.resnets.{j}", x, emb, cfg)
            if i > 0:
                x = R.transformer_3d(sd, f"{p}.attentions.{j}", x, ctx, R._heads(cfg, lvl), cfg)
            x = maybe_motion(f"{p}.motion_modules.{j}", x, lvl, decoder=True)
        if i < n_lvl - 1:
            x = R.upsample_3d(sd, f"{p}.upsamplers.0", x)
    x = F.silu(R.group_norm_5d(sd, "conv_norm_out", x, cfg["norm_num_groups"], cfg["norm_eps"], cfg["use_inflated_groupnorm"]))
    return R.conv2d_per_frame(sd, "conv_out", x)                                            # :665-667


def denoise(unet_sd, unet_cfg, sched_cfg, latents, text_embeddings, num_inference_steps, guidance_scale, first_image_latents=None,
            fps_tensor=None, flow_control=None, camera_movement_type=None, video_scale=0, use_first_frame_condition=False):
    """pipeline_animation.py:686-773 for the first-frame models: returns final latents (b, 4, f, h, w).  guidance_scale > 1: CFG on
    (text_embeddings [uncond; cond]), else one UNet batch and no combine.  unet_cfg["use_first_frame_condition_concat"]: the UNet gets the
    (CFG-duplicated) first-image latents (:717-719); ``use_first_frame_condition``: frame 0 replaced before every step (:691-692)."""
    sched = DDIMOracle(sched_cfg)
    latents = latents.float().clone()
    ffc = unet_cfg["use_first_frame_condition_concat"]
    cfg_on = guidance_scale > 1.0
    dup = lambda v: None if v is None else (torch.cat([torch.as_tensor(v).reshape(-1)] * 2) if cfg_on else torch.as_tensor(v).reshape(-1))
    for t in sched.set_timesteps(num_inference_steps):
        if use_first_frame_condition:
            latents[:, :, 0] = first_image_latents                                          # :691-692
        x = build_unet_input(latents, None, None, False)                                    # torch.cat([latents] * 2), :709
        if not cfg_on:
            x = x[:x.shape[0] // 2]
        ref_lat = None
        if ffc:
            ref_lat = torch.cat([first_image_latents] * 2) if cfg_on else first_image_latents  # :717-719
        pred = unet3d_forward(unet_sd, unet_cfg, x, t, text_embeddings, fps_tensor=dup(fps_tensor), flow_control=dup(flow_control),
                              camera_movement_type_tensor=dup(camera_movement_type), use_first_frame_condition_concat=ffc,
                              reference_images_latent=ref_lat, use_first_frame_condition=use_first_frame_condition)
        if video_scale > 0:                                                                  # :738-761 (per-frame forward: no first-frame flags)
            b, f = latents.shape[0], latents.shape[2]
            xs = x.permute(0, 2, 1, 3, 4).reshape(-1, x.shape[1], x.shape[3], x.shape[4]).unsqueeze(2).chunk(2, dim=0)[0]
            ts = torch.cat([text_embeddings] * f, dim=0).chunk(2, dim=0)[0]
            single = R.unet3d_forward(unet_sd, unet_cfg, xs, t, ts)
            single = single.squeeze(2).reshape(b, f, *single.shape[1:2], *single.shape[3:]).permute(0, 2, 1, 3, 4)
            u, c = pred.chunk(2)
            latents = sched.step(single + video_scale * (u - single) + guidance_scale * (c - u), t, latents)
        else:
            latents = sched.step(cfg_combine(pred, guidance_scale) if cfg_on else pred, t, latents)
    return latents
