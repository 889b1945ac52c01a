"""Diagnostic (not a test): bf16 against fp16 tensor-core mode at full size (SD-1.5 + motion modules, 1.28 B params).  One cfg2 UNet
forward (64 x 64 x 16 frames, B = 2) and one 25-step cfg2 clip (CUDA graph, hoisted context, decode included) per mode, the two modes
alternated twice in one process, with the per-family CUDA-event breakdown of ops.profile() for the forward.  Reads the card's name,
power limit and clocks before and after.

Usage: python tests/diag_fp16.py [out.json]    (prints one JSON object per measurement and a summary; writes the summary to out.json)
"""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import bench  # noqa: E402
from followyourclick_b200 import AnimationPipeline, AutoencoderKL, DDIMScheduler, UNet3DConditionModel, ops  # noqa: E402
from followyourclick_b200.synth import synth_clip_inputs, synth_on_device_  # noqa: E402

ROUNDS, ITERS = 2, 5
MODES = ((torch.bfloat16, "bf16"), (torch.float16, "fp16"))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm,temperature.gpu", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return dict(device=torch.cuda.get_device_name(0), nvidia_smi=q.stdout.strip())


def main():
    res = {"gpu_before": gpu_info(), "rounds": []}
    unet = UNet3DConditionModel(**bench.unet_kwargs(False)).to("cuda")
    vae = AutoencoderKL(**bench.vae_kwargs(False)).to("cuda")
    synth_on_device_(unet, seed=0)
    synth_on_device_(vae, seed=1)
    F, h, w = 16, 64, 64
    g = torch.Generator(device="cuda").manual_seed(3)
    x32 = torch.randn(2, F, h, w, 9, device="cuda", generator=g)
    ctx = torch.randn(2, 77, 768, device="cuda", generator=g)
    t, fps, flow = torch.tensor(501, device="cuda"), torch.tensor([2, 2], device="cuda"), torch.tensor([4, 4], device="cuda")
    ci = {k: v.to("cuda") for k, v in synth_clip_inputs(1, F, h, w, seed=1234).items()}
    pipe = AnimationPipeline(vae=vae, text_encoder=bench._TextEnc(ci["text_embeddings"]), tokenizer=bench._Tok(), unet=unet,
                             scheduler=DDIMScheduler(**bench.SCHED))
    pipe.set_progress_bar_config(disable=True)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    outs = {}
    for r in range(ROUNDS):
        for dt, name in MODES:
            pipe.set_compute_dtype(dt)
            cp = unet.input_channel_pad()
            x = torch.zeros(2, F, h, w, cp, device="cuda", dtype=dt)
            x[..., :9] = x32.to(dt)
            run = lambda: unet.forward_nfhwc(x, t, ctx, fps_tensor=fps, flow_control=flow, use_fps_condition=True)
            for _ in range(2):
                y = run()
            torch.cuda.synchronize()
            ev0.record()
            for _ in range(ITERS):
                y = run()
            ev1.record()
            torch.cuda.synchronize()
            fwd_ms = ev0.elapsed_time(ev1) / ITERS
            with ops.profile() as p:
                run()
            fam = {k: dict(ms=round(v["ms"], 3), launches=v["launches"]) for k, v in sorted(p.summary.items(), key=lambda kv: -kv[1]["ms"])}
            clip = lambda: pipe.denoise(ci["latents"], ci["text_embeddings"], 25, 8.0, first_image_latents=ci["first_image_latents"],
                                        first_images_mask=ci["first_images_mask"], use_first_frame_mask_condition_concat=True,
                                        fps_tensor=torch.tensor([2]), flow_control=torch.tensor([4]), use_fps_condition=True)
            lat = clip()                                              # warm: graph capture, context packing
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ev0.record()
            lat = clip()
            video = pipe.decode_latents_device(lat)
            ev1.record()
            torch.cuda.synchronize()
            clip_ms, clip_wall = ev0.elapsed_time(ev1), (time.perf_counter() - t0) * 1e3
            outs[name] = (y.float(), video.float())
            row = dict(mode=name, round=r, unet_forward_ms=round(fwd_ms, 2), family_sum_ms=round(sum(v["ms"] for v in fam.values()), 2),
                       clip_25_steps_ms=round(clip_ms, 1), clip_wall_ms=round(clip_wall, 1), latents_finite=bool(torch.isfinite(lat).all()),
                       forward_absmax=float(y.float().abs().max()), families=fam)
            res["rounds"].append(row)
            print(json.dumps(row), flush=True)
    res["gpu_after"] = gpu_info()
    a, b = outs["fp16"], outs["bf16"]
    res["fp16_vs_bf16_forward_rel_l2"] = float((a[0] - b[0]).norm() / b[0].norm())
    res["fp16_vs_bf16_video_maxabs"] = float((a[1] - b[1]).abs().max())
    summ = {}
    for name in ("bf16", "fp16"):
        rows = [x for x in res["rounds"] if x["mode"] == name]
        summ[name] = dict(unet_forward_ms=[x["unet_forward_ms"] for x in rows], clip_25_steps_ms=[x["clip_25_steps_ms"] for x in rows])
        fams = {}
        for x in rows:
            for k, v in x["families"].items():
                fams.setdefault(k, []).append(v["ms"])
        summ[name]["families_ms"] = {k: round(sum(v) / len(v), 3) for k, v in fams.items()}
    summ["family_fp16_over_bf16"] = {k: round(summ["fp16"]["families_ms"].get(k, 0) / v, 3) for k, v in summ["bf16"]["families_ms"].items() if v > 0.05}
    res["summary"] = summ
    s = json.dumps({k: v for k, v in res.items() if k != "rounds"})
    print(s)
    if len(sys.argv) > 1:
        os.makedirs(os.path.dirname(os.path.abspath(sys.argv[1])), exist_ok=True)
        open(sys.argv[1], "w").write(json.dumps(res))


if __name__ == "__main__":
    main()
