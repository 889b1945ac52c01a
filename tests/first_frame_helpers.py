"""Helpers of the first-frame-condition tests (CPU emulated and GPU): the mini models of tests/cfgs_first_frame.py through the product
classes, compared with the fixtures of tests/golden/make_golden_first_frame.py."""
import numpy as np
import torch

from followyourclick_b200 import AnimationPipeline, DDIMScheduler, UNet3DConditionModel, ops
from followyourclick_b200.synth import synth_clip_inputs
from tests.cfgs import SCHED_V
from tests.cfgs_first_frame import (PIPE_CASES, PIPE_F, PIPE_HW, PIPE_STEPS, UNET_CASES, ff_ref_kwargs, pipe_case_kwargs,
                                    unet_case_inputs)
from tests.engine_helpers import (FakeTextEncoder, FakeTokenizer, _sync, golden, graph_bookkeeping_on_cpu, load_synth, make_vae,
                                  stats)


def make_ff_unet(mode, fps, dtype=torch.float32, device="cuda"):
    unet = UNet3DConditionModel(**ff_ref_kwargs(mode, fps))
    sd = load_synth(unet)
    if device is not None:
        unet.to(device)
        unet.set_compute_dtype(dtype)         # (.to(torch.float16) would select bf16: the engine's 16-bit default)
    return unet, sd


def mode_bits(mode):
    return ops.FIRST_FRAME if mode == "ff" else ops.FIRST_CONCAT


def ff_unet_forward(unet, name, device, share=False):
    """One UNet forward of case ``name`` through the step prologue (ops.build_unet_input_first) and forward_nfhwc; ``share``: the
    CFG-shaped cases with the shared CFG prefix (one copy of the input, cfg_dup = 2).  Returns the (b, 4, F, H, W) fp32 prediction."""
    mode, fps, b, cfg = UNET_CASES[name]
    inp = unet_case_inputs(name)
    nb = b // 2 if share else b
    assert not share or cfg
    lat = inp["sample"][:nb].contiguous().to(device)
    x = ops.build_unet_input_first(lat, inp["first"][:nb].contiguous().to(device), 1, unet.dtype, mode_bits(mode), c_pad=unet.input_channel_pad())
    mv = lambda t: None if t is None else t.to(device)
    kw = dict(use_first_frame_condition=True) if mode == "ff" else dict(use_first_frame_condition_concat=True)
    y = unet.forward_nfhwc(x, inp["timestep"], mv(inp["ctx"]), fps_tensor=mv(inp.get("fps")), flow_control=mv(inp.get("flow")),
                           use_fps_condition=fps, cfg_dup=2 if share else 1, **kw)
    out = ops.nfhwc_to_ncfhw(y)
    _sync(device)
    return out


def run_ff_unet_case(name, dtype, device="cuda", share=False, via_forward=False):
    """``via_forward``: the public forward(sample, t, ctx, use_first_frame_condition / reference_images_latent) instead of the prologue."""
    mode, fps, b, cfg = UNET_CASES[name]
    unet, _ = make_ff_unet(mode, fps, dtype, device)
    if via_forward:
        inp = unet_case_inputs(name)
        mv = lambda t: None if t is None else t.to(device)
        kw = dict(use_first_frame_condition=True) if mode == "ff" else dict(use_first_frame_condition_concat=True,
                                                                             reference_images_latent=mv(inp["first"]))
        out = unet(mv(inp["sample"]), inp["timestep"], mv(inp["ctx"]), use_fps_condition=fps, fps_tensor=mv(inp.get("fps")),
                   flow_control=mv(inp.get("flow")), **kw).sample
        _sync(device)
    else:
        out = ff_unet_forward(unet, name, device, share)
    return stats(out, torch.from_numpy(golden("first_frame_unet.npz")["out_" + name]))


def make_ff_pipeline(name, dtype, device="cuda"):
    mode, fps, gs, vs = PIPE_CASES[name]
    unet, _ = make_ff_unet(mode, fps, dtype, device)
    vae, _ = make_vae(dtype, device)
    ci = synth_clip_inputs(1, PIPE_F, PIPE_HW, PIPE_HW)
    pipe = AnimationPipeline(vae=vae, text_encoder=FakeTextEncoder(ci["text_embeddings"]), tokenizer=FakeTokenizer(), unet=unet,
                             scheduler=DDIMScheduler(**SCHED_V))
    pipe.set_progress_bar_config(disable=True)
    if device is not None:
        pipe.set_compute_dtype(dtype)
    return pipe, ci


def ff_pipeline_call(pipe, ci, name, **extra):
    """2-step pipeline of case ``name``; returns (video, final latents)"""
    mode, fps, gs, vs = PIPE_CASES[name]
    last = []
    pipe.text_encoder.calls = 0
    video = pipe("p", negative_prompt="n", video_length=PIPE_F, height=PIPE_HW * 8, width=PIPE_HW * 8, num_inference_steps=PIPE_STEPS,
                 guidance_scale=gs, latents=ci["latents"].clone(), callback=lambda i, t, lat: last.append(lat.clone()),
                 **pipe_case_kwargs(name, ci), **extra).videos
    return video, last[-1]


def run_ff_pipeline_case(name, dtype, device="cuda", graph=True, share=True):
    pipe, ci = make_ff_pipeline(name, dtype, device)
    pipe.use_cuda_graph = graph and (str(device).startswith("cuda") or graph_bookkeeping_on_cpu())
    pipe.share_cfg_prefix = share
    video, lat = ff_pipeline_call(pipe, ci, name)
    g = golden("first_frame_pipeline.npz")
    ref = torch.from_numpy(g["video_" + name])
    s = stats(video, ref)
    mse = float(((video.float() - ref) ** 2).mean())
    return dict(video_maxabs=s["maxabs"], psnr=float(10 * np.log10(1.0 / max(mse, 1e-20))), finite=s["finite"], shape=tuple(video.shape),
                latent_rel_l2=stats(lat, torch.from_numpy(g["final_latents_" + name]))["rel_l2"])
