"""Generate the SD-2.x fixtures from the UNMODIFIED reference (build container only), in files of their own.

Run:  python tests/golden/make_golden_sd2.py        (needs the reference checkout that make_golden.py imports; ~1 min on 8 cores)

Same procedure as make_golden.py (reference imported with the same shims, deterministic synthetic weights, the oracle pinned against
the reference's outputs with its error recorded), for the mini SD-2.x-based motion model of tests/cfgs_sd2.py.
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
from oracle import ref_pipeline, ref_unet, ref_vae  # noqa: E402
from tests.cfgs import MINI_VAE, SCHED_V  # noqa: E402
from tests.cfgs_sd2 import MINI_SD2, MINI_SD2_2D, SD2_CTX_DIM, mini_sd2_oracle_cfg, oracle_state_dict, sd2_inputs  # noqa: E402


def sd2_fixtures(UNet, Pipe, VAE, DDIM):
    """SD-2.x-based motion model (tests/cfgs_sd2.py MINI_SD2: linear transformer projections, upcast attention, per-level heads of head dim 64,
    1024-wide text context, inflated GroupNorm, mid-block motion module, fps condition) through the UNMODIFIED reference: the UNet3D forward,
    its state-dict keys, the 2-D UNet2DConditionModel of the same width and a 2-step v-prediction AnimationPipeline run.  Written to new files
    (unet_sd2.npz, unet_sd2_keys.json, unet2d_sd2.npz, pipeline_sd2.npz, sd2_pins.json); the SD-1.5 fixtures are not touched.  The oracle
    reads the state dicts through tests/cfgs_sd2.oracle_state_dict (Linear proj_in / proj_out as 1x1 convolutions)."""
    from diffusers.models.unet_2d_condition import UNet2DConditionModel as UNet2D
    pins, keys = {}, {}
    ocfg = mini_sd2_oracle_cfg()
    unet = UNet(**MINI_SD2).eval()
    usd = load_synth(unet)
    keys["unet3d"] = {k: list(v.shape) for k, v in usd.items()}
    inp = sd2_inputs()
    with torch.no_grad():
        ref = unet(inp["sample"], inp["timestep"], encoder_hidden_states=inp["ctx"], use_fps_condition=True, fps_tensor=inp["fps"],
                   flow_control=inp["flow"]).sample
        taps = {}
        orc = ref_unet.unet3d_forward(oracle_state_dict(usd), ocfg, inp["sample"], inp["timestep"], inp["ctx"], fps_tensor=inp["fps"], flow_control=inp["flow"],
                                      taps=taps)
    err = maxabs(ref, orc)
    print(f"unet[sd2] out {tuple(ref.shape)} |ref|max={float(ref.abs().max()):.3f} oracle-vs-ref maxabs={err:.3e}")
    assert err < 2e-4 * max(1.0, float(ref.abs().max()))
    pins["unet_sd2"] = err
    np.savez_compressed(os.path.join(HERE, "unet_sd2.npz"), out=ref.numpy(),
                        **{"tap_" + k: v.numpy().astype(np.float16) for k, v in taps.items() if k in ("conv_in", "mid")})

    m = UNet2D(**MINI_SD2_2D).eval()
    sd2d = load_synth(m)
    keys["unet2d"] = {k: list(v.shape) for k, v in sd2d.items()}
    g = torch.Generator().manual_seed(43)
    x, ctx, t = torch.randn(2, 4, 16, 16, generator=g), torch.randn(2, 77, SD2_CTX_DIM, generator=g), torch.tensor(501)
    with torch.no_grad():
        ref2 = m(x, t, encoder_hidden_states=ctx).sample
        orc2 = ref_unet.unet3d_forward(oracle_state_dict(sd2d), mini_sd2_oracle_cfg(two_d=True), x.unsqueeze(2), t, ctx).squeeze(2)
    err = maxabs(ref2, orc2)
    print(f"unet2d[sd2] out {tuple(ref2.shape)} |ref|max={float(ref2.abs().max()):.3f} oracle-vs-ref maxabs={err:.3e}")
    assert err < 2e-4 * max(1.0, float(ref2.abs().max()))
    pins["unet2d_sd2"] = err
    np.savez_compressed(os.path.join(HERE, "unet2d_sd2.npz"), x=x.numpy(), ctx=ctx.numpy(), out=ref2.numpy())
    with open(os.path.join(HERE, "unet_sd2_keys.json"), "w") as f:
        json.dump(keys, f)

    vae = VAE(in_channels=3, out_channels=3, down_block_types=("DownEncoderBlock2D",) * 4,
              up_block_types=("UpDecoderBlock2D",) * 4, block_out_channels=MINI_VAE["block_out_channels"],
              layers_per_block=MINI_VAE["layers_per_block"], latent_channels=4, norm_num_groups=32).eval()
    vsd = load_synth(vae)
    F_, h, w, steps, gs = 4, 16, 16, 2, 7.5
    ci = synth_clip_inputs(1, F_, h, w, seed=4321, ctx_dim=SD2_CTX_DIM)
    sched = DDIM(**{k: v for k, v in SCHED_V.items() if k != "set_alpha_to_one"})
    pipe = Pipe(vae=vae, text_encoder=FakeText(ci["text_embeddings"]), tokenizer=FakeTok(), unet=unet, scheduler=sched)
    with torch.no_grad():
        video = pipe("p", negative_prompt="n", video_length=F_, height=h * 8, width=w * 8, num_inference_steps=steps, guidance_scale=gs,
                     latents=ci["latents"].clone(), use_fps_condition=True, fps_tensor=torch.tensor([3]), flow_control=torch.tensor([5])).videos
        lat = ref_pipeline.denoise(oracle_state_dict(usd), ocfg, SCHED_V, ci["latents"], ci["text_embeddings"], steps, gs, fps_tensor=torch.tensor([3]),
                                   flow_control=torch.tensor([5]))
        orc_video = ref_vae.decode_latents(vsd, MINI_VAE, lat)
    err = maxabs(video, orc_video)
    print(f"pipeline[sd2] video {tuple(video.shape)} oracle-vs-ref maxabs={err:.3e}")
    assert err < 2e-3
    pins["pipeline_sd2"] = err
    np.savez_compressed(os.path.join(HERE, "pipeline_sd2.npz"), video=video.numpy().astype(np.float32), final_latents=lat.numpy(),
                        steps=np.int64(steps), guidance=np.float32(gs))
    with open(os.path.join(HERE, "sd2_pins.json"), "w") as f:
        json.dump({"oracle_vs_reference_maxabs": pins, "torch": torch.__version__,
                   "reference": "mayuelala/FollowYourClick (unmodified)"}, f, indent=1)


def main():
    torch.manual_seed(0)
    torch.set_num_threads(8)
    UNet, Pipe, VAE, DDIM, _ = import_reference()
    sd2_fixtures(UNet, Pipe, VAE, DDIM)


if __name__ == "__main__":
    main()
