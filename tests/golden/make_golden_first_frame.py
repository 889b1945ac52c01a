"""Generate the first-frame-condition fixtures from the UNMODIFIED reference (build container only), in files of their own.

Run:  python tests/golden/make_golden_first_frame.py     (needs the reference checkout that make_golden.py imports; a few minutes on 8 cores)

Same procedure as make_golden.py (reference imported with the same shims, deterministic synthetic weights, the oracle pinned against the
reference's outputs with its error recorded) for the two image-to-video modes of tests/cfgs_first_frame.py:
  first_frame_unet.npz       UNet3D forwards per tests/cfgs_first_frame.UNET_CASES (out_<case>);
  first_frame_pipeline.npz   2-step AnimationPipeline runs per PIPE_CASES (video_<case>, final_latents_<case>);
  first_frame_pins.json      oracle-vs-reference errors, and the combinations the reference cannot sample with the exception each raised.
No other fixture is touched.
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import FakeText, FakeTok, import_reference, load_synth, maxabs  # noqa: E402  (also puts the repository root on sys.path)

from followyourclick_b200.synth import synth_clip_inputs  # noqa: E402
from oracle import ref_vae  # noqa: E402
from tests import oracle_first_frame  # noqa: E402
from tests.cfgs import MINI_VAE, SCHED_V, mini_unet_ref_kwargs  # noqa: E402
from tests.cfgs_first_frame import (PIPE_CASES, PIPE_F, PIPE_HW, PIPE_STEPS, UNET_CASES, ff_oracle_cfg, ff_ref_kwargs,  # noqa: E402
                                    pipe_case_kwargs, pipe_case_oracle_kwargs, unet_case_inputs)


def unet_fixtures(UNet, pins):
    outs = {}
    models = {}
    for name, (mode, fps, b, cfg) in UNET_CASES.items():
        if (mode, fps) not in models:
            m = UNet(**ff_ref_kwargs(mode, fps)).eval()
            models[(mode, fps)] = (m, load_synth(m))
        unet, usd = models[(mode, fps)]
        inp = unet_case_inputs(name)
        kw = dict(use_first_frame_condition=True) if mode == "ff" else dict(use_first_frame_condition_concat=True,
                                                                             reference_images_latent=inp["first"])
        okw = dict(use_first_frame_condition=True) if mode == "ff" else dict(use_first_frame_condition_concat=True,
                                                                              reference_images_latent=inp["first"])
        if fps:
            kw.update(use_fps_condition=True, fps_tensor=inp["fps"], flow_control=inp["flow"])
            okw.update(fps_tensor=inp["fps"], flow_control=inp["flow"])
        with torch.no_grad():
            ref = unet(inp["sample"], inp["timestep"], encoder_hidden_states=inp["ctx"], **kw).sample
            orc = oracle_first_frame.unet3d_forward(usd, ff_oracle_cfg(mode, fps), inp["sample"], inp["timestep"], inp["ctx"], **okw)
        err = maxabs(ref, orc)
        print(f"unet[{name}] out {tuple(ref.shape)} |ref|max={float(ref.abs().max()):.3f} oracle-vs-ref maxabs={err:.3e}")
        assert err < 2e-4 * max(1.0, float(ref.abs().max()))
        pins[f"unet_{name}"] = err
        outs["out_" + name] = ref.numpy()
    np.savez_compressed(os.path.join(HERE, "first_frame_unet.npz"), **outs)
    return models


def make_vae(VAE):
    vae = VAE(in_channels=3, out_channels=3, down_block_types=("DownEncoderBlock2D",) * 4,
              up_block_types=("UpDecoderBlock2D",) * 4, block_out_channels=MINI_VAE["block_out_channels"],
              layers_per_block=MINI_VAE["layers_per_block"], latent_channels=4, norm_num_groups=32).eval()
    return vae, load_synth(vae)


class _Text(FakeText):
    """The reference pipeline's ``device`` is that of the first nn.Module among its components, in an order that varies with the string
    hash seed; this text encoder may come first, so it answers too."""
    device = torch.device("cpu")


def run_ref_pipeline(Pipe, DDIM, unet, vae, ci, gs, **kw):
    sched = DDIM(**{k: v for k, v in SCHED_V.items() if k != "set_alpha_to_one"})
    pipe = Pipe(vae=vae, text_encoder=_Text(ci["text_embeddings"]), tokenizer=FakeTok(), unet=unet, scheduler=sched)
    with torch.no_grad():
        return pipe("p", negative_prompt="n", video_length=PIPE_F, height=PIPE_HW * 8, width=PIPE_HW * 8, num_inference_steps=PIPE_STEPS,
                    guidance_scale=gs, latents=ci["latents"].clone(), **kw).videos


def pipeline_fixtures(UNet, Pipe, VAE, DDIM, models, pins):
    vae, vsd = make_vae(VAE)
    ci = synth_clip_inputs(1, PIPE_F, PIPE_HW, PIPE_HW)
    outs = {}
    for name, (mode, fps, gs, vs) in PIPE_CASES.items():
        unet, usd = models[(mode, fps)]
        video = run_ref_pipeline(Pipe, DDIM, unet, vae, ci, gs, **pipe_case_kwargs(name, ci))
        text = ci["text_embeddings"] if gs > 1.0 else ci["text_embeddings"][1:2]
        with torch.no_grad():
            lat = oracle_first_frame.denoise(usd, ff_oracle_cfg(mode, fps), SCHED_V, ci["latents"], text, PIPE_STEPS, gs,
                                             **pipe_case_oracle_kwargs(name, ci))
            orc_video = ref_vae.decode_latents(vsd, MINI_VAE, lat)
        err = maxabs(video, orc_video)
        print(f"pipeline[{name}] video {tuple(video.shape)} oracle-vs-ref maxabs={err:.3e}")
        assert err < 2e-3
        pins[f"pipeline_{name}"] = err
        outs["video_" + name] = video.numpy().astype(np.float32)
        outs["final_latents_" + name] = lat.numpy()
    np.savez_compressed(os.path.join(HERE, "first_frame_pipeline.npz"), **outs)
    return vae, ci


def refused_combinations(UNet, Pipe, DDIM, models, vae, ci):
    """The combinations the reference cannot sample: run each, record the exception (the engine raises for exactly these)."""
    cam = UNet(**dict(ff_ref_kwargs("ff"), use_camera_motion_condition=True)).eval()
    load_synth(cam)
    base = UNet(**mini_unet_ref_kwargs("base")).eval()
    load_synth(base)
    ffc_unet = models[("ffc", True)][0]
    first = dict(first_image_latents=ci["first_image_latents"])
    cases = {
        "ff+fps (CFG)": (models[("ff", True)][0], dict(first, use_first_frame_condition=True, use_fps_condition=True,
                                                       fps_tensor=torch.tensor([2]), flow_control=torch.tensor([4]))),
        "ff+camera (CFG)": (cam, dict(first, use_first_frame_condition=True, use_camera_motion_condition=True,
                                      camera_movement_type=torch.tensor([3]))),
        "ff+mask_concat": (base, dict(first, use_first_frame_condition=True, use_first_frame_mask_condition_concat=True)),
        "ffc+mask_concat": (ffc_unet, dict(first, use_first_frame_condition_concat=True, use_first_frame_mask_condition_concat=True,
                                           use_fps_condition=True, fps_tensor=torch.tensor([2]), flow_control=torch.tensor([4]))),
        "ffc+video_scale": (ffc_unet, dict(first, use_first_frame_condition_concat=True, video_scale=0.7, use_fps_condition=True,
                                           fps_tensor=torch.tensor([2]), flow_control=torch.tensor([4]))),
    }
    out = {}
    for name, (unet, kw) in cases.items():
        try:
            run_ref_pipeline(Pipe, DDIM, unet, vae, ci, 8.0, **kw)
        except Exception as e:          # noqa: BLE001  (whatever the reference raises is what is recorded)
            out[name] = f"{type(e).__name__}: {str(e).splitlines()[0][:160] if str(e) else ''}"
            print(f"refused[{name}]: {out[name]}")
            continue
        raise AssertionError(f"the reference sampled {name}")
    return out


def main():
    torch.manual_seed(0)
    torch.set_num_threads(8)
    UNet, Pipe, VAE, DDIM, _ = import_reference()
    pins = {}
    models = unet_fixtures(UNet, pins)
    vae, ci = pipeline_fixtures(UNet, Pipe, VAE, DDIM, models, pins)
    refused = refused_combinations(UNet, Pipe, DDIM, models, vae, ci)
    with open(os.path.join(HERE, "first_frame_pins.json"), "w") as f:
        json.dump({"oracle_vs_reference_maxabs": pins, "reference_refuses": refused, "torch": torch.__version__,
                   "reference": "mayuelala/FollowYourClick (unmodified)"}, f, indent=1)


if __name__ == "__main__":
    main()
