"""Engine runs of the SD-2.x-based mini model (tests/cfgs_sd2.py MINI_SD2 / MINI_SD2_2D) against the fixtures the unmodified reference wrote
(tests/golden/*sd2*, made by tests/golden/make_golden_sd2.py).  Shared by the CPU host-logic tests (kernels emulated) and the GPU tests."""
import json
import os

import numpy as np
import torch

from tests.cfgs import MINI_VAE, SCHED_V
from tests.cfgs_sd2 import MINI_SD2, MINI_SD2_2D, SD2_CTX_DIM, sd2_inputs
from tests.engine_helpers import GOLD, FakeTextEncoder, FakeTokenizer, _sync, golden, load_synth, make_vae, stats


def sd2_keys(which):
    return {k: tuple(s) for k, s in json.load(open(os.path.join(GOLD, "unet_sd2_keys.json")))[which].items()}


def sd2_pins():
    return json.load(open(os.path.join(GOLD, "sd2_pins.json")))["oracle_vs_reference_maxabs"]


def make_sd2_unet(dtype=torch.float32, device="cuda"):
    from followyourclick_b200 import UNet3DConditionModel
    unet = UNet3DConditionModel(**MINI_SD2)
    sd = load_synth(unet)
    if device is not None:
        unet.to(device)
        unet.to(dtype)
    return unet, sd


def run_sd2_unet_case(dtype, device="cuda"):
    unet, _ = make_sd2_unet(dtype, device)
    inp = sd2_inputs()
    mv = lambda t: t.to(device)
    out = unet(mv(inp["sample"]), inp["timestep"], encoder_hidden_states=mv(inp["ctx"]), use_fps_condition=True, fps_tensor=mv(inp["fps"]),
               flow_control=mv(inp["flow"])).sample
    _sync(device)
    return stats(out, torch.from_numpy(golden("unet_sd2.npz")["out"]))


def run_sd2_unet2d_case(dtype, device="cuda"):
    from followyourclick_b200 import UNet2DConditionModel
    m = UNet2DConditionModel(**MINI_SD2_2D)
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == sd2_keys("unet2d")
    load_synth(m)
    m.to(device)
    m.to(dtype)
    g = golden("unet2d_sd2.npz")
    out = m(torch.from_numpy(g["x"]).to(device), torch.tensor(501), encoder_hidden_states=torch.from_numpy(g["ctx"]).to(device)).sample
    _sync(device)
    assert out.shape == (2, 4, 16, 16)
    return stats(out, torch.from_numpy(g["out"]))


def run_sd2_pipeline_case(dtype, device="cuda", graph=True):
    """2-step v-prediction AnimationPipeline (fps condition, 4-channel input, 16 x 16 latents, 1024-wide text embeddings) against the
    reference pipeline's frames."""
    from followyourclick_b200 import AnimationPipeline, DDIMScheduler
    from followyourclick_b200.synth import synth_clip_inputs
    from tests.engine_helpers import graph_bookkeeping_on_cpu
    g = golden("pipeline_sd2.npz")
    F, h, w = 4, 16, 16
    unet, _ = make_sd2_unet(dtype, device)
    vae, _ = make_vae(dtype, device, MINI_VAE)
    ci = synth_clip_inputs(1, F, h, w, seed=4321, ctx_dim=SD2_CTX_DIM)
    pipe = AnimationPipeline(vae=vae, text_encoder=FakeTextEncoder(ci["text_embeddings"]), tokenizer=FakeTokenizer(), unet=unet,
                             scheduler=DDIMScheduler(**SCHED_V))
    pipe.set_progress_bar_config(disable=True)
    pipe.use_cuda_graph = graph and (str(device).startswith("cuda") or graph_bookkeeping_on_cpu())
    video = pipe("p", negative_prompt="n", video_length=F, height=h * 8, width=w * 8, num_inference_steps=int(g["steps"]),
                 guidance_scale=float(g["guidance"]), latents=ci["latents"].clone(), use_fps_condition=True, fps_tensor=torch.tensor([3]),
                 flow_control=torch.tensor([5])).videos
    ref = torch.from_numpy(g["video"])
    s = stats(video, ref)
    mse = float(((video.float().cpu() - ref) ** 2).mean())
    return dict(video_maxabs=s["maxabs"], psnr=float(10 * np.log10(1.0 / max(mse, 1e-20))), finite=s["finite"], shape=tuple(video.shape))
