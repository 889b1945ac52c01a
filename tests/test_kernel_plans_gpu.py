"""The kernel plans other resolutions and frame counts select, per element against fp64 (tests/cone_helpers.py checks).

tests/test_kernel_cones_gpu.py checks every route at small shapes, which reproduce the tile plans of the 512 x 512 configuration.  The
cases here run the plans tests/plan_shapes.py derives for 256^2, 384^2, 320 x 576, 512 x 256, 768^2 with 32 frames and SD-2.x at 384^2:

* convolutions over 32 images (64 for 768^2) of two clips - a bn = 32 tile spans the time embeddings of both - with residual and row
  bias: each patch geometry bn in {1, 2, 4, 8, 16, 32} for stride 1, stride 2 and the four-phase upsampler on its low-resolution grid
  (plan_shapes.conv_plan picks the plan and the kernels the case expects), and the 5 x 9 level, whose convolution has no patch
  (CUDA-core kernel) and whose upsampler materialises onto the 10 x 18 bn = 32 plan.  Extra
  cone seeds sit on row 0 of image bn / 2 (the warpgroup split) and image bn (the tile boundary), where a NaN lands in the neighbour's
  halo, and on the row bias of the second clip;
* GEMMs at the level-2 / level-3 row counts (4608, 1152, 1440: a ragged last m tile) with the production N / K of q/k/v, the
  LayerNorm-folded GEGLU, FF out and proj - small-M launches where the tile-width model may pick a BN that does not divide N, and
  launches with many tiles per persistent CTA, down to one K block per tile (the staging buffer is rewritten right after its TMA store);
* self-attention at the production sequence lengths of each route (up to 144 key tiles), with Gaussian, ascending, late-peak and flat
  score layouts (cone_helpers.layout_qk).

Each case also asserts, from torch.profiler's CUDA activity, which kernels ran - with their template arguments where the route fixes
them - and that ops.profile() books the call under the family of that kernel.  Per case, plan_ratios.json under pytest's temporary
directory holds the bound ratio, the kernels, the peak device memory and, for a failing case, which check failed and its report.
"""
import json
import re

import pytest
import torch

from tests import cone_helpers as H
from tests import plan_shapes as P

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
# every kernel of the library a case below can launch (checked as names in the profiler's CUDA activity)
KERNELS = ("gemm_tc_kernel", "gemm_simt_kernel", "gemv_small_m_kernel", "space_to_planes_kernel", "upsample2x_kernel", "geglu_kernel",
           "attention_mma_kernel", "attention_mma_shortk_kernel", "attention_simt_kernel", "attention_tc_kernel", "conv3x3_small_n_kernel")
GEMM_TC = r"gemm_tc_kernel<\d+, __nv_bfloat16>"       # BN is the tile-width model's choice
# conv route (plan_shapes.conv_plan) -> (kernel name patterns, ops.profile() family)
CONV_ROUTES = {"tc": ({GEMM_TC}, "conv_tc"), "tc_up2": ({GEMM_TC}, "conv_tc_up2"), "simt": ({r"gemm_simt_kernel<__nv_bfloat16, __nv_bfloat16, \(anonymous namespace\)::ConvAS"}, "conv_simt"),
               "upsample_tc": ({r"upsample2x_kernel<__nv_bfloat16, 8>", GEMM_TC}, "conv_tc")}
SYNTHETIC = dict(P.SYNTHETIC_BN16, frames=16)           # bn = 16: the one grid no listed resolution produces
CONV_PLANS = {}                                          # case id -> (kind, route, patch): tests/test_kernel_plans_cpu.py checks coverage


def _grid(res, lv):
    if res == "synthetic":
        return SYNTHETIC
    v = P.level(res, lv)
    return dict(h=v.h, w=v.w, nb=v.nb, frames=v.frames)


def _conv(kind, g, Cin, Cout):
    """one conv on the input grid g (h, w, nb images of ``frames`` frames per clip): row bias (one row per clip) and residual unless
    upsampling (the upsamplers take a bias only); extra cone seeds on row 0 of images bn / 2 and bn and on the second clip's row bias"""
    route, patch = P.conv_plan(kind, g["nb"], g["h"], g["w"])
    h, w, nb, ipg = g["h"], g["w"], g["nb"], g["frames"]
    bn = patch[2] if patch else 32
    up = kind == "up2"

    def build(d):
        c = H.conv_case(BF, nb, h, w, Cin, Cout, d, stride=2 if kind == "s2" else 1, up=2 if up else 1, phases=up and route == "tc_up2",
                        residual=not up, ipg=0 if up else ipg)
        seeds = [("x", (bn // 2, 0, w // 2, 1)), ("x", (bn, 0, w // 2, 2)), ("x", (min(bn + bn // 2, nb - 1), 0, 0, Cin - 1))]
        if not up:
            seeds.append(("rowbias", (nb // ipg - 1, 7)))       # the second clip: a bn = 32 tile takes it from its second half
        c.seeds = c.seeds + [s for s in H._seeds(seeds, c.operands) if s not in c.seeds]
        return c
    pats, fam = CONV_ROUTES[route]
    if kind == "s2":
        pats = pats | {r"space_to_planes_kernel"}
    return (kind, route, patch), build, pats, {fam}


def _cases():
    c = {}

    def add(family, name, build, kernels, labels):
        c[f"{family}-{name}"] = (family, build, set(kernels), set(labels))

    # ---- convolutions: (kind, resolution, level of the input grid, Cin, Cout); production channels where the fp64 conv is cheap
    convs = [("s1", "256x256", 0, 320, 320), ("s1", "320x576", 0, 320, 320), ("s1", "512x256", 3, 1280, 1280), ("s1", "384x384", 2, 1280, 1280),
             ("s1", "768x768_F32", 3, 1280, 1280), ("s1", "320x576", 1, 640, 640), ("s1", "256x256", 3, 320, 320), ("s1", "synthetic", 0, 320, 320),
             ("s1", "384x384", 3, 1280, 1280), ("s1", "320x576", 2, 1280, 1280),
             ("s1", "320x576", 3, 2560, 1280),           # 5 x 9: no patch, the CUDA-core kernel (the up block's 2560-channel concatenation)
             ("s2", "256x256", 0, 320, 320), ("s2", "384x384", 0, 320, 320), ("s2", "512x256", 2, 1280, 1280), ("s2", "384x384", 1, 320, 320),
             ("s2", "synthetic_4x8", 0, 320, 320), ("s2", "384x384", 2, 1280, 1280),
             ("up2", "256x256", 1, 320, 320), ("up2", "384x384", 1, 320, 320), ("up2", "512x256", 3, 1280, 1280), ("up2", "384x384", 2, 320, 320),
             ("up2", "synthetic", 0, 320, 320), ("up2", "384x384", 3, 1280, 1280),
             ("up2", "320x576", 3, 1280, 1280)]          # 5 x 9: the upsample is materialised onto the 10 x 18 bn = 32 plan
    for kind, res, lv, Cin, Cout in convs:
        g = dict(SYNTHETIC, h=4, w=8) if res == "synthetic_4x8" else _grid(res, lv)
        plan, build, pats, fams = _conv(kind, g, Cin, Cout)
        bn = f"bn{plan[2][2]}" if plan[2] else "nopatch"
        cid = f"conv-{kind}_{plan[1]}_{bn}_{res.split('_')[0]}_{g['h']}x{g['w']}x{g['nb']}_c{Cin}to{Cout}"
        add("conv", cid[len("conv-"):], build, pats, fams)
        CONV_PLANS[cid] = plan
    # ---- GEMMs at the level-2 / 3 row counts: q/k/v (3C), GEGLU (8C, LayerNorm folded), FF out (K = 4C), proj; C = 1280
    C = 1280
    g = ({GEMM_TC}, {"gemm_tc"})
    for M in (P.level("384x384", 2).rows, P.level("384x384", 3).rows, P.level("320x576", 3).rows):
        add("gemm", f"qkv_{M}x{3 * C}x{C}", lambda d, M=M: H.gemm_case(BF, M, 3 * C, C, d, bias=False, residual=True), *g)
        add("gemm", f"geglu_lnfold_{M}x{8 * C}x{C}", lambda d, M=M: H.gemm_case(BF, M, 8 * C, C, d, ln=True, geglu=True), *g)
        add("gemm", f"ff_out_{M}x{C}x{4 * C}", lambda d, M=M: H.gemm_case(BF, M, C, 4 * C, d, residual=True), *g)
        add("gemm", f"proj_{M}x{C}x{C}", lambda d, M=M: H.gemm_case(BF, M, C, C, d, residual=True), *g)
    # one K block per tile and ~10 tiles per CTA on the plain ring (N = 48 rules out the W-resident mode): each tile's epilogue rewrites
    # the staging buffer right after the previous tile's TMA store was issued
    for res in (False, True):
        add("gemm", f"one_kblock_{'residual_' if res else ''}168959x48x64",
            lambda d, res=res: H.gemm_case(BF, 128 * 1320 - 1, 48, 64, d, residual=res), *g)
    # ---- self-attention per route at the production sequence length, four score layouts; the template arguments follow from D
    mma = {40: r"attention_mma_kernel<40, 48, __nv_bfloat16>", 64: r"attention_mma_kernel<64, 64, __nv_bfloat16>",
           80: r"attention_mma_kernel<80, 80, __nv_bfloat16>"}
    tc = {40: r"attention_tc_kernel<1, 3, 48, 40, __nv_bfloat16>", 80: r"attention_tc_kernel<2, 5, 80, 80, __nv_bfloat16>"}
    for layout in H.LAYOUTS:
        a = lambda heads, D, N, L, layout=layout: (lambda d: H.attention_case(BF, heads, D, N, L, L, 1, d, layout=layout))
        s = lambda D, N, L, heads, layout=layout: (lambda d: H.self_tc_case(BF, D, N, L, heads, d, wide_out=False, layout=layout))
        add("attention", f"mma_d40_L2880_{layout}", a(8, 40, 2, 2880), {mma[40]}, {"attention"})        # 320 x 576 level 0: 45 key tiles
        add("attention", f"mma_d80_L720_{layout}", a(8, 80, 2, 720), {mma[80]}, {"attention"})          # 320 x 576 level 1
        add("attention", f"mma_d80_L576_{layout}", a(8, 80, 2, 576), {mma[80]}, {"attention"})          # 384^2 level 1
        add("attention", f"mma_d64_L576_{layout}", a(10, 64, 2, 576), {mma[64]}, {"attention"})         # SD-2.x 384^2 level 1
        add("attention", f"wgmma_d40_L2304_{layout}", s(40, 2, 2304, 8), {tc[40]}, {"attention_tc"})
        add("attention", f"wgmma_d40_L9216_{layout}", s(40, 1, 9216, 8), {tc[40]}, {"attention_tc"})   # 768^2 level 0: 72 key tiles
        add("attention", f"wgmma_d80_L2304_{layout}", s(80, 2, 2304, 8), {tc[80]}, {"attention_tc"})   # 768^2 level 1
    return c


CASES = _cases()


CAPTURES = 3     # profiler sessions per case at most: a session whose activity holds no library kernel is taken again (see _route)


def _route(case):
    """(demangled names of the library kernels that ran, ops.profile() families, profiler sessions) of one call of the case.

    torch.profiler's CUDA activity can come back without the library kernels of a call that ran them (seen on the H100: ops.profile()
    booked the call, its output was right, the activity listed no library kernel).  That is a lost record, not evidence of a route, so
    only a session with no library kernel at all is taken again; any kernel that did get recorded is judged as it is."""
    from torch.profiler import ProfilerActivity, profile

    from followyourclick_b200 import ops
    for n in range(1, CAPTURES + 1):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            with ops.profile() as rec:
                out = H.run(case, 0.0)[0]
            torch.cuda.synchronize()
        names = sorted({e.key for e in prof.key_averages() if any(k in e.key for k in KERNELS)})
        if names:
            break
    return names, set(rec.summary), n, out


def _route_problems(names, patterns, fams, labels):
    """every library kernel that ran matches an expected pattern, every pattern matched a kernel, the families are the expected ones"""
    stray = [n for n in names if not any(re.search(p, n) for p in patterns)]
    missing = [p for p in patterns if not any(re.search(p, n) for n in names)]
    return [] if not stray and not missing and fams == labels else [("route", dict(stray=stray, missing=missing, families=sorted(fams)))]


@pytest.fixture(scope="module")
def ratios(tmp_path_factory):
    r = {}
    yield r
    path = tmp_path_factory.mktemp("plans") / "plan_ratios.json"
    fam = {}
    for cid, v in r.items():
        f = fam.setdefault(CASES[cid][0], dict(cases=0, max_ratio=0.0, max_peak_gb=0.0))
        f["cases"] += 1
        f["max_ratio"] = max(f["max_ratio"], v.get("ratio", float("inf")))
        f["max_peak_gb"] = max(f["max_peak_gb"], v.get("peak_gb", 0.0))
    path.write_text(json.dumps(dict(c=H.C_BOUND, families=fam, cases=r), indent=1, default=str))
    print(f"\nbound ratios (c = {H.C_BOUND}): {json.dumps(fam)} -> {path}")


@pytest.mark.parametrize("cid", list(CASES))
def test_kernel_plan(cuda, cid, ratios):
    from followyourclick_b200 import ops
    ops.set_impl("auto")
    family, build, patterns, labels = CASES[cid]
    rec = ratios.setdefault(cid, {})
    torch.cuda.reset_peak_memory_stats()
    try:
        case = build("cuda")
        names, fams, captures, out_prof = _route(case)
        res = H.run_checks(case)
        # the profiled call computed what an unprofiled one computes: the kernels did run under the profiler
        same = bool((H._bits(out_prof) == H._bits(H.run(case, 0.0)[0])).all())
    except Exception as e:                  # kept in the JSON as the evidence of the failure
        rec["error"] = f"{type(e).__name__}: {e}"[:4000]
        raise
    finally:
        rec["peak_gb"] = torch.cuda.max_memory_allocated() / 2 ** 30
    bad_cones = [c for c in res["cones"] if not c["ok"]]
    problems = _route_problems(names, patterns, fams, labels) + ([] if same else [("route", "the profiled call differs")]) + \
        ([] if res["surround"]["ok"] else [("surround", res["surround"])]) + [("cone", c) for c in bad_cones] + \
        ([] if res["bound"]["ok"] else [("bound", res["bound"])])
    rec.update(ratio=res["bound"]["ratio"], kernels=names, families=sorted(fams), captures=captures, failed=sorted({k for k, _ in problems}))
    if problems:
        rec["report"] = repr(problems)[:4000]
    assert not problems, problems


def test_conv_route_rule_matches_the_plan_table(cuda):
    """plan_shapes.conv_plan (the Python restatement of pick_patch) agrees with the C rule fyc_conv3x3 routes by, on every level of the
    table and on every grid up to 12 x 12 over 1 .. 96 images: the C side is asked through fyc_conv3x3_tc_route and
    fyc_conv3x3_up2_eligible with aligned placeholder pointers (nothing is launched)"""
    import ctypes as C

    from followyourclick_b200 import _lib as L
    ptr, ws = 1 << 20, 1 << 40

    def c_route(kind, nb, h, w, upsample=1, phases=False):
        a = L.ConvArgs(ptr, ptr, ptr, ptr, None, None, nb, h, w, 320, 320, 2 if kind == "s2" else 1, upsample, 0, L.BF16, L.EPI_BIAS,
                       L.IMPL_AUTO, ptr, ws, 0, ptr if phases else None, 0)
        return L.lib().fyc_conv3x3_tc_route(C.byref(a)), L.lib().fyc_conv3x3_up2_eligible(C.byref(a))
    grids = {(v.nb, v.h, v.w) for v in P.all_levels()} | {(nb, h, w) for nb in (1, 2, 4, 8, 16, 32, 64, 96) for h in range(1, 13)
                                                         for w in range(1, 13)}
    wrong = []
    for nb, h, w in sorted(grids):
        for kind in ("s1", "s2", "up2"):
            route, _ = P.conv_plan(kind, nb, h, w)
            if kind == "up2":
                got = "tc_up2" if c_route(kind, nb, h, w, 2, True)[1] else \
                      ("upsample_tc" if c_route("s1", nb, 2 * h, 2 * w)[0] else "upsample_simt")
            else:
                got = "tc" if c_route(kind, nb, h, w)[0] else "simt"
            if got != route:
                wrong.append((kind, nb, h, w, route, got))
    assert not wrong, wrong[:20]
