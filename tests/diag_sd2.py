"""Diagnostic (not a test): an SD-2.x-based motion model at full size (SD-2.1 widths, heads 5 / 10 / 20 / 20, head dim 64, 1024-wide text
context, linear projections) - one bf16 UNet forward at 64 x 64 x 16 frames, B = 2: wall time, the per-family breakdown of ops.profile(),
and the self- / cross-attention family times on the head-dim-64 wgmma kernels against the mma.sync kernel they replace (the route chosen
by monkeypatching the two *_tc_ok predicates), the two routes alternated in one process.

Usage: python tests/diag_sd2.py [out.json]    (prints one JSON object; also writes it to out.json if given)
"""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from followyourclick_b200 import UNet3DConditionModel, ops  # noqa: E402
from followyourclick_b200.synth import synth_on_device_  # noqa: E402
from tests.test_sd2_gpu import sd2_full_kwargs  # noqa: E402

ROUNDS, ITERS = 2, 5


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return dict(device=torch.cuda.get_device_name(0), nvidia_smi=q.stdout.strip())


def main():
    info = gpu_info()
    unet = UNet3DConditionModel(**sd2_full_kwargs()).to("cuda")
    synth_on_device_(unet, seed=5)
    unet.to(torch.bfloat16)
    F, h, w = 16, 64, 64
    cp = unet.input_channel_pad()
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.zeros(2, F, h, w, cp, device="cuda", dtype=torch.bfloat16)
    x[..., :4] = torch.randn(2, F, h, w, 4, device="cuda", generator=g).bfloat16()
    ctx = torch.randn(2, 77, 1024, device="cuda", generator=g)
    t, fps, flow = torch.tensor(501, device="cuda"), torch.tensor([3, 3], device="cuda"), torch.tensor([5, 5], device="cuda")
    run = lambda: unet.forward_nfhwc(x, t, ctx, fps_tensor=fps, flow_control=flow, use_fps_condition=True)
    tc_self, tc_cross = ops.self_attention_tc_ok, ops.cross_attention_tc_ok

    def route(name):
        if name == "wgmma_d64":
            ops.self_attention_tc_ok, ops.cross_attention_tc_ok = tc_self, tc_cross
        else:            # the route before head dim 64 was instantiated: every D = 64 attention on the mma.sync kernel
            ops.self_attention_tc_ok = lambda dtype, L, D: D != 64 and tc_self(dtype, L, D)
            ops.cross_attention_tc_ok = lambda dtype, D, Lk, Lk2: D != 64 and tc_cross(dtype, D, Lk, Lk2)

    res = {"gpu": info, "shape": "B=2 x 16 frames x 64x64 latents, bf16", "rounds": []}
    outs = {}
    for r in range(ROUNDS):
        for name in ("wgmma_d64", "mma_sync"):
            route(name)
            for _ in range(2):
                y = run()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(ITERS):
                y = run()
            torch.cuda.synchronize()
            ms = (time.perf_counter() - t0) / ITERS * 1e3
            outs[name] = y.float()
            with ops.profile() as p:
                run()
            fam = {k: dict(ms=round(v["ms"], 3), launches=v["launches"]) for k, v in sorted(p.summary.items(), key=lambda kv: -kv[1]["ms"])}
            attn = {k: v["ms"] for k, v in fam.items() if k in ("attention_tc", "cross_attention_tc", "attention")}
            res["rounds"].append(dict(route=name, round=r, forward_ms=round(ms, 2), attention_family_ms=attn,
                                      attention_total_ms=round(sum(attn.values()), 3), families=fam))
            print(json.dumps(res["rounds"][-1]), flush=True)
    route("wgmma_d64")
    a, b = outs["wgmma_d64"], outs["mma_sync"]
    res["routes_rel_l2"] = float((a - b).norm() / b.norm())
    res["gpu_after"] = gpu_info()
    s = json.dumps(res)
    print(s)
    if len(sys.argv) > 1:
        os.makedirs(os.path.dirname(os.path.abspath(sys.argv[1])), exist_ok=True)
        open(sys.argv[1], "w").write(s)


if __name__ == "__main__":
    main()
