"""AnimationPipeline: reference call surface (animatediff/pipelines/pipeline_animation.py:42-788), engine loop underneath.

``__call__`` accepts the reference's keyword set (``scripts/inference.py:374-395``) and returns ``.videos`` as a CPU fp32
tensor (b, 3, F, H, W) in [0, 1].  Per DDIM step the engine runs exactly four kinds of work, all libfyc kernels:
  build 9-channel CFG-duplicated input (1 kernel) -> UNet3D forward -> layout to (2b,4,F,h,w) -> fused CFG+DDIM step.
The prompt / image encoders are outside the hot path (their outputs are computed once before the loop, :610-612,
:676-680) and are used as given (any callable with the transformers interface).
"""
import inspect
import os
from collections import OrderedDict
from dataclasses import dataclass
from typing import Union

import numpy as np
import torch

from . import _lib, ops


@dataclass
class AnimationPipelineOutput:
    videos: Union[torch.Tensor, np.ndarray]


class _NullBar:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False

    def update(self, n=1):
        pass


class _GraphedUNetStep:
    """One UNet3D forward (+ layout change of the prediction) captured as a CUDA graph.  Shapes are static per clip
    configuration, so the ~700 kernel launches of a forward are replayed with one call; inputs live in static buffers
    (x: channels-last UNet input, t: timestep, text / fps / flow / camera / clip features)."""

    def __init__(self, unet, x_shape, text, fps, flow, cam, clip, flags, x=None, out_frames=None, cfg_dup=1, hoist=True):
        """``x``: use this (view of another step's) static input instead of allocating one; ``out_frames`` = (b, f): the input is
        b * f single frames (F = 1) whose prediction is returned regrouped as (b, 4, f, h, w) (video_scale branch)."""
        dev = unet.device
        self.version = unet._pack_version
        self.out_frames, self.cfg_dup = out_frames, cfg_dup
        self.x = torch.zeros(x_shape, dtype=unet.dtype, device=dev) if x is None else x
        assert tuple(self.x.shape) == tuple(x_shape)
        self.t = torch.zeros((), dtype=torch.int64, device=dev)
        self.text = text.to(dev).float().contiguous().clone()
        cl = lambda v: None if v is None else v.to(dev).contiguous().clone()
        self.fps, self.flow, self.cam, self.clip = cl(fps), cl(flow), cl(cam), cl(clip)
        self.flags = flags
        # step-invariant conditioning (context tokens, image-prompt tokens, every block's cross-attention K/V): built once per clip
        # into static buffers the captured forward reads (SURVEY 8f row 2); the reference redoes it every step
        self.hoist = hasattr(unet, "prepare_context") and hoist
        self.context = self._context(unet) if self.hoist else None
        self._unet = unet
        if self.capture:
            cur = torch.cuda.current_stream()
            side = torch.cuda.Stream()
            side.wait_stream(cur)
            with torch.cuda.stream(side):           # warm-up outside capture: packs weights, sets kernel attributes
                for _ in range(2):
                    self._run(unet)
            cur.wait_stream(side)
            torch.cuda.synchronize()
            self.graph = torch.cuda.CUDAGraph()
            n0 = _lib.launch_count
            with torch.cuda.graph(self.graph):
                self.pred = self._run(unet)
            self.n_calls = _lib.launch_count - n0      # kernel-launching C-ABI calls replayed by one graph launch
        else:                                          # bookkeeping-only mode of the CPU host-logic tests: replay() re-executes
            self.graph, self.n_calls = None, 0
            self.pred = self._run(unet)

    capture = True         # False: no CUDA graph, replay() re-runs the forward (tests/test_host_emulated_cpu.py walks this class's
                           # buffer / cache / context bookkeeping on CPU with the kernel launches emulated)

    def replay(self):
        if self.graph is not None:
            self.graph.replay()
            _lib.launch_count += self.n_calls
        else:
            self.pred = self._run(self._unet)

    def _context(self, unet):
        return unet.prepare_context(self.text, self.clip, self.flags.get("use_ip_cross_attention", False))

    def _run(self, unet):
        y = unet.forward_nfhwc(self.x, self.t, self.text, fps_tensor=self.fps, flow_control=self.flow,
                               reference_images_clip_feat=self.clip, camera_movement_type_tensor=self.cam, context=self.context,
                               cfg_dup=self.cfg_dup, **self.flags)
        return ops.nfhwc_to_ncfhw(_regroup_frames(y, self.out_frames))

    def load(self, unet, text, fps, flow, cam, clip):
        self.text.copy_(text)
        for name, dst, src in (("fps", self.fps, fps), ("flow", self.flow, flow), ("camera", self.cam, cam), ("clip", self.clip, clip)):
            if (dst is None) != (src is None):
                raise ValueError(f"captured UNet step was built {'with' if dst is not None else 'without'} a `{name}` tensor; "
                                 "this call differs (the graph cache key should have separated them)")
            if dst is not None:
                dst.copy_(src)
        if self.hoist:
            self.context.copy_(self._context(unet))


def _regroup_frames(y, out_frames):
    """[(b f), 1, h, w, c] -> [b, f, h, w, c] (a view: `(b f) c 1 h w -> b c f h w` of pipeline_animation.py:755 is free in
    the channels-last layout)."""
    if out_frames is None:
        return y
    b, f = out_frames
    return y.view(b, f, y.shape[2], y.shape[3], y.shape[4])


@torch.no_grad()
def prepare_first_frame_condition(vae, first_images, first_images_mask, generator=None, vae_scale_factor=8):
    """The per-clip conditioning prep that precedes the loop in the reference driver (scripts/inference.py:355-365):

        first_image_latents = vae.encode(first_images).latent_dist.sample() * 0.18215
        first_images_mask   = clamp(F.interpolate(mask, size=(H / 8, W / 8))[:, None], 0, 1)     # nearest

    first_images (n, 3, H, W) in [-1, 1]; first_images_mask (n, 1, H, W).  Returns the two tensors AnimationPipeline.__call__ takes
    as ``first_image_latents`` / ``first_images_mask`` (SURVEY 8f row 1: with this the whole I2V clip stays on the GPU)."""
    lat = vae.encode(first_images).latent_dist.sample(generator=generator) * 0.18215
    h, w = first_images.shape[-2] // vae_scale_factor, first_images.shape[-1] // vae_scale_factor
    mask = first_images_mask.to(device=lat.device, dtype=torch.float32)
    mask = torch.nn.functional.interpolate(mask, size=(h, w))[:, None]           # a (n, 1, h, w) nearest resize: index plumbing, once per clip
    return lat, torch.clamp(mask, 0, 1)


def check_first_frame_options(use_first_frame_condition=False, use_first_frame_condition_concat=False,
                              use_first_frame_mask_condition_concat=False, first_image_latents=None, video_scale=0, unet_batch=1,
                              use_fps_condition=False, use_camera_motion_condition=False):
    """The combinations of the two first-frame condition modes with the other options that the reference pipeline cannot sample
    (pipeline_animation.py:686-773 with unet.py:422-590 and resnet.py:304-320) raise here, each with a message naming both options;
    every other combination is sampled.  ``unet_batch``: rows of the UNet's batch (2 b under classifier-free guidance)."""
    modes = [n for n, on in (("use_first_frame_condition", use_first_frame_condition),
                             ("use_first_frame_condition_concat", use_first_frame_condition_concat)) if on]
    for m in modes:
        if first_image_latents is None:
            raise ValueError(f"{m} needs first_image_latents (the clean first-image latents, (b, 4, h, w))")
        if use_first_frame_mask_condition_concat:
            raise ValueError(f"{m} with use_first_frame_mask_condition_concat: the reference has no UNet input for the pair "
                             "(pipeline_animation.py:691-705 builds the mask-concat input only without use_first_frame_condition; "
                             "with use_first_frame_condition_concat conv_in would get 13 channels)")
    if use_first_frame_condition_concat and video_scale > 0:
        raise ValueError("use_first_frame_condition_concat with video_scale > 0: the reference's per-frame forward passes the 4-channel latents "
                         "without the first-image concat (pipeline_animation.py:738-751), which the 8-channel conv_in rejects")
    if use_first_frame_condition and unet_batch > 1:
        for other, on in (("use_fps_condition", use_fps_condition), ("use_camera_motion_condition", use_camera_motion_condition)):
            if on:
                raise ValueError(f"use_first_frame_condition with {other} at a UNet batch of {unet_batch} (classifier-free guidance doubles it): "
                                 f"the reference adds the {unet_batch}-row {other} embedding to the {unet_batch + 1}-row time embedding of the "
                                 "first-frame condition (unet.py:523-558), which broadcasts only for a batch of 1")


class AnimationPipeline:
    _optional_components = []
    use_cuda_graph = True          # replay one captured UNet forward per DDIM step (set False to launch kernel by kernel)
    hoist_context = True           # build the step-invariant conditioning (ClipContext) once per clip instead of once per step
    last_video_device = None       # the most recent decode's (b, 3, F, H, W) fp32 video, still on the device
    graph_cache_entries = 4        # captured UNet-step graphs kept per pipeline (least recently used shapes are dropped)
    # Shared CFG prefix (UNet3DConditionModel.forward_nfhwc cfg_dup): the uncond / cond halves of the reference's batch are identical
    # until the first cross-attention, so that prefix (incl. the first 64x64 self-attention) is computed once.  Exact arithmetic on the
    # same rows; GPU-verified (tests/test_zz_late_gpu.py, tests/test_full_parity_gpu.py).
    # FYC_SHARED_PREFIX=0 switches it off (A/B).
    share_cfg_prefix = os.environ.get("FYC_SHARED_PREFIX", "1") != "0"

    def __init__(self, vae, text_encoder, tokenizer, unet, scheduler, image_encoder=None, text_encoder_2=None,
                 tokenizer_2=None, ip_adapter=None):
        self.vae, self.text_encoder, self.tokenizer, self.unet, self.scheduler = vae, text_encoder, tokenizer, unet, scheduler
        self.image_encoder, self.text_encoder_2, self.tokenizer_2, self.ip_adapter = image_encoder, text_encoder_2, tokenizer_2, ip_adapter
        self.vae_scale_factor = 2 ** (len(self.vae.config.block_out_channels) - 1)
        self._progress = True

    # ---------------------------------------------------------------- DiffusionPipeline-style plumbing
    def to(self, device=None, dtype=None):
        for m in (self.vae, self.unet, self.text_encoder, self.image_encoder, self.text_encoder_2):
            if m is not None and hasattr(m, "to"):
                m.to(device) if dtype is None else m.to(device, dtype)
        return self

    def set_compute_dtype(self, dtype):
        """Run the engine's models (UNet, VAE, IP-Adapter) in `dtype`: torch.float32, torch.bfloat16 or torch.float16
        (ParamTreeModel.set_compute_dtype).  The text / image encoders are not engine models and keep their own dtype."""
        ops.check_compute_dtype(dtype)
        for m in (self.unet, self.vae, self.ip_adapter):
            if m is not None:
                m.set_compute_dtype(dtype)
        return self

    @property
    def device(self):
        return self.unet.device

    @property
    def _execution_device(self):
        return self.unet.device

    def set_progress_bar_config(self, **kw):
        self._progress = not kw.get("disable", False)

    def progress_bar(self, iterable=None, total=None):
        if not self._progress:
            return _NullBar() if iterable is None else iterable
        try:
            from tqdm.auto import tqdm
        except Exception:       # pragma: no cover
            return _NullBar() if iterable is None else iterable
        return tqdm(iterable, total=total) if iterable is not None else tqdm(total=total)

    def enable_vae_slicing(self):
        self.vae.enable_slicing()

    def disable_vae_slicing(self):
        self.vae.disable_slicing()

    def enable_sequential_cpu_offload(self, gpu_id=0):
        raise NotImplementedError("CPU offload is a memory work-around the 180 GB engine does not need")

    # ---------------------------------------------------------------- prompt encoding (outside the hot path)
    def _encode_prompt(self, prompt, device, num_videos_per_prompt, do_classifier_free_guidance, negative_prompt):
        """pipeline_animation.py:158-245: CLIP text forward for prompt and negative prompt -> cat([uncond, cond])."""
        batch_size = len(prompt) if isinstance(prompt, list) else 1

        def encode(text):
            ti = self.tokenizer(text, padding="max_length", max_length=self.tokenizer.model_max_length, truncation=True,
                                return_tensors="pt")
            mask = None
            cfg = getattr(self.text_encoder, "config", None)
            if cfg is not None and getattr(cfg, "use_attention_mask", False):
                mask = ti.attention_mask.to(device)
            emb = self.text_encoder(ti.input_ids.to(device), attention_mask=mask)[0]
            bs, seq, _ = emb.shape
            return emb.repeat(1, num_videos_per_prompt, 1).view(bs * num_videos_per_prompt, seq, -1)

        text_embeddings = encode(prompt)
        if do_classifier_free_guidance:
            if negative_prompt is None:
                uncond_tokens = [""] * batch_size
            elif isinstance(negative_prompt, str):
                uncond_tokens = [negative_prompt]
            elif batch_size != len(negative_prompt):
                raise ValueError(f"`negative_prompt`: {negative_prompt} has batch size {len(negative_prompt)}, but `prompt`:"
                                 f" {prompt} has batch size {batch_size}.")
            else:
                uncond_tokens = negative_prompt
            text_embeddings = torch.cat([encode(uncond_tokens), text_embeddings])
        return text_embeddings

    def check_inputs(self, prompt, height, width, callback_steps):
        if not isinstance(prompt, str) and not isinstance(prompt, list):
            raise ValueError(f"`prompt` has to be of type `str` or `list` but is {type(prompt)}")
        if height % 8 != 0 or width % 8 != 0:
            raise ValueError(f"`height` and `width` have to be divisible by 8 but are {height} and {width}.")
        if (callback_steps is None) or (callback_steps is not None and (not isinstance(callback_steps, int) or callback_steps <= 0)):
            raise ValueError(f"`callback_steps` has to be a positive integer but is {callback_steps} of type {type(callback_steps)}.")

    def prepare_extra_step_kwargs(self, generator, eta):
        kw = {}
        params = set(inspect.signature(self.scheduler.step).parameters.keys())
        if "eta" in params:
            kw["eta"] = eta
        if "generator" in params:
            kw["generator"] = generator
        return kw

    def prepare_latents(self, batch_size, num_channels_latents, video_length, height, width, dtype, device, generator,
                        latents=None, use_interpolate_noise=False, **unused):
        """pipeline_animation.py:448-537 (init_latents / residual-noise branches are not used by scripts/inference.py)."""
        shape = (batch_size, num_channels_latents, video_length, height // self.vae_scale_factor, width // self.vae_scale_factor)
        if isinstance(generator, list) and len(generator) != batch_size:
            raise ValueError(f"You have passed a list of generators of length {len(generator)}, but requested an effective batch"
                             f" size of {batch_size}. Make sure the batch size matches the length of the generators.")
        if latents is None:
            if isinstance(generator, list):
                latents = torch.cat([torch.randn(shape, generator=g, device=device, dtype=torch.float32) for g in generator], dim=0)
            else:
                latents = torch.randn(shape, generator=generator, device=device, dtype=torch.float32)
                if use_interpolate_noise:
                    latents = latents[:, :, :1].repeat(1, 1, shape[2], 1, 1)
        else:
            if tuple(latents.shape) != shape:
                raise ValueError(f"Unexpected latents shape, got {latents.shape}, expected {shape}")
            latents = latents.to(device=device, dtype=torch.float32)
        return (latents * self.scheduler.init_noise_sigma).contiguous()

    # ---------------------------------------------------------------- decode (hot path, after the loop)
    @torch.no_grad()
    def decode_latents_device(self, latents):
        """latents (b, 4, F, h, w) fp32 on device -> video (b, 3, F, H, W) fp32 on device, (x/2+0.5).clamp(0,1)."""
        b, c, f, h, w = latents.shape
        z = ops.ncfhw_to_nfhwc(latents.to(torch.float32).contiguous(), self.vae.dtype, scale=1 / 0.18215).view(b * f, h, w, c)
        frames = self.vae.decode_nhwc(z)
        self.last_video_device = ops.frames_finalize(frames, b, f)      # kept for callers that continue on the device (gather, uint8 grid, GIF)
        return self.last_video_device

    def decode_latents(self, latents):
        """pipeline_animation.py:400-413: returns a numpy array (b, 3, F, H, W) fp32 (device -> host boundary)."""
        return self.decode_latents_device(latents.to(self.device)).cpu().float().numpy()

    # ---------------------------------------------------------------- the denoising loop
    @torch.no_grad()
    def denoise(self, latents, text_embeddings, num_inference_steps, guidance_scale, first_image_latents=None,
                first_images_mask=None, use_first_frame_mask_condition_concat=False, fps_tensor=None, flow_control=None,
                use_fps_condition=False, use_ip_cross_attention=False, image_clip_feat_pair=None,
                use_camera_motion_condition=False, camera_movement_type=None, eta=0.0, generator=None, callback=None,
                callback_steps=1, progress=False, video_scale=0, use_first_frame_condition=False,
                use_first_frame_condition_concat=False):
        """pipeline_animation.py:686-773 on the engine.  latents fp32 (b,4,F,h,w) on device; returns final latents.
        video_scale > 0 (:738-761): a second forward per step on the clip's frames taken one at a time, combined as
        ``s + video_scale (u - s) + guidance (c - u)`` (SURVEY 8f row 3).
        use_first_frame_condition (:691-692): frame 0 of the latents is replaced by ``first_image_latents`` before every step, so the
        step reads the replaced frame (the last step's output is not replaced); use_first_frame_condition_concat (:717-719): the UNet
        input is [latents | first_image_latents on every frame].  Both go through one prologue kernel (ops.build_unet_input_first)."""
        dev = self.unet.device
        do_cfg = guidance_scale > 1.0
        if video_scale > 0 and not do_cfg:
            raise NotImplementedError("video_scale > 0 without classifier-free guidance (the reference only uses the per-frame "
                                      "prediction inside its CFG combine, pipeline_animation.py:757-761)")
        dup = 2 if do_cfg else 1
        check_first_frame_options(use_first_frame_condition, use_first_frame_condition_concat, use_first_frame_mask_condition_concat,
                                  first_image_latents, video_scale, dup * latents.shape[0], use_fps_condition, use_camera_motion_condition)
        mode = (ops.FIRST_CONCAT if use_first_frame_condition_concat else 0) | (ops.FIRST_FRAME if use_first_frame_condition else 0)
        sched, unet = self.scheduler, self.unet
        sched.set_timesteps(num_inference_steps, device=dev)
        t_host = list(sched._timesteps_host)
        t_dev = sched.timesteps

        def as_dev(v):
            if v is None:
                return None
            v = torch.as_tensor(v).reshape(-1).to(dev)
            return torch.cat([v] * dup) if do_cfg else v

        fps_d, flow_d, cam_d = as_dev(fps_tensor), as_dev(flow_control), as_dev(camera_movement_type)
        mask = first = None
        if use_first_frame_mask_condition_concat:
            first = first_image_latents.to(device=dev, dtype=torch.float32).contiguous()
            if first_images_mask is not None:
                mask = first_images_mask[:, :, 0].to(device=dev, dtype=torch.float32).contiguous()     # :632-635 (frame 0, clamp in-kernel)
        latents = latents.to(device=dev, dtype=torch.float32).contiguous()
        ff_first = None
        if mode:
            ff_first = first_image_latents.to(device=dev, dtype=torch.float32).contiguous()
            if mode & ops.FIRST_FRAME:
                latents = latents.clone()      # the prologue writes frame 0 in place: never into the caller's tensor
        text_embeddings = text_embeddings.to(dev)
        c_pad = unet.input_channel_pad() if hasattr(unet, "input_channel_pad") else None
        bar = self.progress_bar(total=num_inference_steps) if progress else _NullBar()
        flags = dict(use_ip_cross_attention=use_ip_cross_attention, use_camera_motion_condition=use_camera_motion_condition,
                     use_fps_condition=use_fps_condition)
        if mode & ops.FIRST_CONCAT:
            flags["use_first_frame_condition_concat"] = True
        if mode & ops.FIRST_FRAME:
            flags["use_first_frame_condition"] = True

        def prologue(out=None):
            if mode:
                return ops.build_unet_input_first(latents, ff_first, xdup, unet.dtype, mode, c_pad=c_pad, out=out)
            return ops.build_unet_input(latents, mask, first, xdup, unet.dtype, c_pad=c_pad, out=out)
        clip_d = None if image_clip_feat_pair is None else image_clip_feat_pair.to(dev)
        graphed = context = graphed_sf = context_sf = None
        b, _, f, h, w = latents.shape
        text_sf = None
        if video_scale > 0:
            # :743-747 - the text rows for the b*f single frames are the first half of [text] * f, i.e. they ALTERNATE uncond / cond
            # (reference behaviour, kept); the single-frame forward gets no fps / camera / image conditioning (:748-752)
            text_sf = torch.cat([text_embeddings] * f, dim=0).chunk(2, dim=0)[0].contiguous()
            flags_sf = dict(use_ip_cross_attention=False, use_camera_motion_condition=False, use_fps_condition=False)
        # shared CFG prefix: the UNet gets ONE copy of the input and fans out at its first cross-attention (cfg_dup)
        share = 2 if (self.share_cfg_prefix and do_cfg and hasattr(unet, "prepare_context")) else 1
        xdup = dup // share
        if self.use_cuda_graph and hasattr(unet, "forward_nfhwc"):
            cin = c_pad if c_pad is not None else (9 if first is not None else 8 if mode & ops.FIRST_CONCAT else 4)
            # everything the captured forward's control flow depends on: shapes, dtype, flags, WHICH optional inputs exist, and the
            # IP-attention logit-scale semantics (enable_xformers_memory_efficient_attention toggles it without re-packing weights)
            key = (xdup * b, share, self.hoist_context, f, h, w, cin, unet.dtype, tuple(sorted(flags.items())), tuple(text_embeddings.shape),
                   None if clip_d is None else tuple(clip_d.shape), fps_d is None, flow_d is None, cam_d is None,
                   bool(getattr(unet, "_xformers_semantics", False)), mode)
            cache = self.__dict__.setdefault("_graph_cache", OrderedDict())
            graphed = cache.get(key)
            if graphed is not None:
                cache.move_to_end(key)
            if graphed is None or graphed.version != unet._pack_version:
                graphed = cache[key] = _GraphedUNetStep(unet, (xdup * b, f, h, w, cin), text_embeddings, fps_d, flow_d, cam_d, clip_d, flags,
                                                        cfg_dup=share, hoist=self.hoist_context)
            graphed.load(unet, text_embeddings, fps_d, flow_d, cam_d, clip_d)
            while len(cache) > self.graph_cache_entries * 2:       # LRU bound: a graph + its private memory pool per distinct clip shape
                cache.popitem(last=False)                           # (x2: the video_scale branch keeps a second graph per shape)
            if video_scale > 0:
                graphed_sf = cache.get(key + ("sf",))
                if graphed_sf is None or graphed_sf.version != unet._pack_version or graphed_sf.x.data_ptr() != graphed.x.data_ptr():
                    graphed_sf = cache[key + ("sf",)] = _GraphedUNetStep(
                        unet, (b * f, 1, h, w, cin), text_sf, None, None, None, None, flags_sf,
                        x=graphed.x[:b].view(b * f, 1, h, w, cin), out_frames=(b, f), hoist=self.hoist_context)   # the uncond copy's frames: a view
                graphed_sf.load(unet, text_sf, None, None, None, None)
        with bar as pb:
            for i, t in enumerate(t_host):
                if graphed is not None:
                    prologue(out=graphed.x)
                    graphed.t.copy_(t_dev[i])
                    graphed.replay()
                    pred = graphed.pred
                    if graphed_sf is not None:
                        graphed_sf.t.copy_(t_dev[i])
                        graphed_sf.replay()
                        single = graphed_sf.pred
                else:
                    if i == 0 and self.hoist_context and hasattr(unet, "prepare_context"):
                        context = unet.prepare_context(text_embeddings, clip_d, use_ip_cross_attention)
                    x = prologue()
                    y = unet.forward_nfhwc(x, t_dev[i], text_embeddings, fps_tensor=fps_d, flow_control=flow_d,
                                           reference_images_clip_feat=clip_d, camera_movement_type_tensor=cam_d, context=context,
                                           **(dict(flags, cfg_dup=share) if share > 1 else flags))
                    pred = ops.nfhwc_to_ncfhw(y)
                    if video_scale > 0:
                        if i == 0 and self.hoist_context and hasattr(unet, "prepare_context"):
                            context_sf = unet.prepare_context(text_sf, None, False)
                        ys = unet.forward_nfhwc(x[:b].view(b * f, 1, h, w, x.shape[-1]), t_dev[i], text_sf, context=context_sf, **flags_sf)
                        single = ops.nfhwc_to_ncfhw(_regroup_frames(ys, (b, f)))
                latents = sched.step_cfg(pred, t, latents, guidance_scale if do_cfg else 1.0, eta=eta, generator=generator,
                                         single_frame_output=single if video_scale > 0 else None, video_scale=video_scale)
                pb.update()
                if callback is not None and i % callback_steps == 0:
                    callback(i, t, latents)
        return latents

    @torch.no_grad()
    def __call__(self, prompt, video_length, height=None, width=None, num_inference_steps=50, guidance_scale=7.5,
                 negative_prompt=None, num_videos_per_prompt=1, eta=0.0, generator=None, latents=None, output_type="tensor",
                 return_dict=True, callback=None, callback_steps=1, use_first_frame_condition=False,
                 use_first_frame_condition_concat=False, use_first_frame_mask_condition_concat=False,
                 use_first_frame_mask_condition_concat_image_partial_mask=None, first_image_latents=None,
                 use_first_image_as_init_latents=False, video_scale=0, use_ip_cross_attention=False, condition_images=None,
                 use_uncond_images=False, use_camera_motion_condition=False, camera_movement_type=None,
                 use_text_encoder_2=False, use_uncond_text_2=False, use_fps_condition=False, fps_tensor=None,
                 use_interpolate_noise=False, first_images_mask=None, flow_control=None, **kwargs):
        if use_text_encoder_2 or use_first_image_as_init_latents or use_first_frame_mask_condition_concat_image_partial_mask is not None:
            raise NotImplementedError("option outside the scripts/inference.py path (SURVEY 8f)")
        height = height or self.unet.config.sample_size * self.vae_scale_factor
        width = width or self.unet.config.sample_size * self.vae_scale_factor
        self.check_inputs(prompt, height, width, callback_steps)
        batch_size = 1
        if latents is not None:
            batch_size = latents.shape[0]
        if isinstance(prompt, list):
            batch_size = len(prompt)
        device = self._execution_device
        do_cfg = guidance_scale > 1.0
        check_first_frame_options(use_first_frame_condition, use_first_frame_condition_concat, use_first_frame_mask_condition_concat,
                                  first_image_latents, video_scale, (2 if do_cfg else 1) * batch_size * num_videos_per_prompt,
                                  use_fps_condition, use_camera_motion_condition)
        prompt = prompt if isinstance(prompt, list) else [prompt] * batch_size
        if negative_prompt is not None:
            negative_prompt = negative_prompt if isinstance(negative_prompt, list) else [negative_prompt] * batch_size
        text_embeddings = self._encode_prompt(prompt, device, num_videos_per_prompt, do_cfg, negative_prompt)
        latents = self.prepare_latents(batch_size * num_videos_per_prompt, self.unet.in_channels, video_length, height, width,
                                       torch.float32, device, generator, latents, use_interpolate_noise=use_interpolate_noise)
        clip_pair = None
        if use_ip_cross_attention:
            cond, uncond = self.ip_adapter.get_image_clip_feat(input_image=condition_images)       # :676-680
            if use_uncond_images:
                cond = uncond.clone()
            clip_pair = torch.cat([uncond, cond]) if do_cfg else cond
        latents = self.denoise(latents, text_embeddings, num_inference_steps, guidance_scale,
                               first_image_latents=first_image_latents, first_images_mask=first_images_mask,
                               use_first_frame_mask_condition_concat=use_first_frame_mask_condition_concat,
                               fps_tensor=fps_tensor, flow_control=flow_control, use_fps_condition=use_fps_condition,
                               use_ip_cross_attention=use_ip_cross_attention, image_clip_feat_pair=clip_pair,
                               use_camera_motion_condition=use_camera_motion_condition, camera_movement_type=camera_movement_type,
                               eta=eta, generator=generator if not isinstance(generator, list) else None,
                               callback=callback, callback_steps=callback_steps, progress=self._progress, video_scale=video_scale,
                               use_first_frame_condition=use_first_frame_condition,
                               use_first_frame_condition_concat=use_first_frame_condition_concat)
        video = self.decode_latents(latents)
        if output_type == "tensor":
            video = torch.from_numpy(video)
        if not return_dict:
            return video
        return AnimationPipelineOutput(videos=video)
