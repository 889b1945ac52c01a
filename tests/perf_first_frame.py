"""Time one cfg2 clip per conditioning mode, alternated in one process (GPU only).

    python tests/perf_first_frame.py [--steps 25] [--rounds 3] [--json out.json]

Full-width models with deterministic synthetic weights, 64x64 latents x 16 frames, 25 DDIM steps, CFG 8, bf16, CUDA graph, shared CFG
prefix - the bench.py flagship workload - for:
  mask_concat  the shipped model (use_first_frame_mask_condition_concat + fps / motion condition, 9-channel input),
  ff           use_first_frame_condition (4-channel input, frame 0 replaced in place, B + 1-row time-embedding GEMV + per-image table),
  ffc          use_first_frame_condition_concat (8-channel input, conv_in output halved; fps / motion condition on).
Only the denoising loop is timed (device events around pipe.denoise, after a warm-up clip per mode that captures its graph); the modes
take turns within every round so that drift of the shared machine hits them alike.  Prints one JSON line with the card's name and power
limit beside the times.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def card():
    info = dict(name=torch.cuda.get_device_name(0))
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit"], info["max_sm_clock"] = [v.strip() for v in q.split(",")]
    except Exception as e:         # noqa: BLE001  (reported, not fatal)
        info["power_limit"] = f"unknown ({type(e).__name__})"
    return info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=25)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perf_first_frame.py measures the GPU: no CUDA device")
    import bench
    from followyourclick_b200 import AnimationPipeline, AutoencoderKL, DDIMScheduler, UNet3DConditionModel
    from followyourclick_b200.synth import synth_clip_inputs, synth_on_device_
    dev = "cuda"
    base = bench.unet_kwargs(False)
    kws = {"mask_concat": base,
           "ff": dict(base, use_first_frame_mask_condition_concat=False, use_fps_condition=False),
           "ffc": dict(base, use_first_frame_mask_condition_concat=False, use_first_frame_condition_concat=True)}
    vae = AutoencoderKL(**bench.vae_kwargs(False)).to(dev)
    synth_on_device_(vae, seed=1)
    vae.to(torch.bfloat16)
    F, h, w, gs = 16, 64, 64, 8.0
    ci = {k: v.to(dev) for k, v in synth_clip_inputs(1, F, h, w, seed=1234).items()}
    fps = dict(fps_tensor=torch.tensor([2]), flow_control=torch.tensor([4]), use_fps_condition=True)
    call = {"mask_concat": dict(fps, first_images_mask=ci["first_images_mask"], use_first_frame_mask_condition_concat=True),
            "ff": dict(use_first_frame_condition=True),
            "ffc": dict(fps, use_first_frame_condition_concat=True)}
    pipes = {}
    for mode, kw in kws.items():
        unet = UNet3DConditionModel(**kw).to(dev)
        synth_on_device_(unet, seed=0)
        unet.to(torch.bfloat16)
        pipe = AnimationPipeline(vae=vae, text_encoder=bench._TextEnc(ci["text_embeddings"]), tokenizer=bench._Tok(), unet=unet,
                                 scheduler=DDIMScheduler(**bench.SCHED))
        pipe.set_progress_bar_config(disable=True)
        pipes[mode] = pipe

    def clip(mode):
        return pipes[mode].denoise(ci["latents"], ci["text_embeddings"], a.steps, gs, first_image_latents=ci["first_image_latents"], **call[mode])

    for mode in pipes:                   # warm-up: graph capture, weight packing, kernel attributes
        clip(mode)
    torch.cuda.synchronize()
    ms = {m: [] for m in pipes}
    order = list(pipes)
    for r in range(a.rounds):
        for mode in order[r % len(order):] + order[:r % len(order)]:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            clip(mode)
            e1.record()
            torch.cuda.synchronize()
            ms[mode].append(e0.elapsed_time(e1))
    med = {m: statistics.median(v) for m, v in ms.items()}
    res = dict(card=card(), workload=f"cfg2 64x64x16f, {a.steps} DDIM steps, CFG {gs}, bf16, CUDA graph, denoise loop only",
               rounds=a.rounds, clip_ms_median={m: round(v, 1) for m, v in med.items()},
               clip_ms_all={m: [round(x, 1) for x in v] for m, v in ms.items()},
               step_ms_median={m: round(v / a.steps, 2) for m, v in med.items()},
               vs_mask_concat={m: round(med[m] / med["mask_concat"], 4) for m in med})
    line = json.dumps(res)
    print(line)
    if a.json:
        with open(a.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
