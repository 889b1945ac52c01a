"""CPU checks of the plan table (tests/plan_shapes.py) that tests/test_kernel_plans_gpu.py runs, and of the blocked fp64 references.

* The conv cases of tests/test_kernel_plans_gpu.py reach every patch geometry bn in {1, 2, 4, 8, 16, 32} for stride 1, stride 2
  (padding 1) and the four-phase upsampler (bn = 16 from the one synthetic 4 x 2 grid), and the levels of the resolution table get the
  plans and routes listed for them.
* ``ref64`` / ``mag64`` evaluated in blocks of output rows equal the single-block evaluation, on the contract emulator (no library is
  needed) at small shapes
  with a block budget small enough to force several blocks (equal up to fp64 rounding: a matmul over fewer rows may order its sums
  differently), and the emulator passes all three checks with that budget.
"""
import pytest
import torch

from tests import cone_helpers as H
from tests import ops_emulator as E
from tests import plan_shapes as P

BF = torch.bfloat16
GEOMETRIES = {1, 2, 4, 8, 16, 32}


def _bn(patches):
    return {p[2] for p in patches if p is not None}


def test_conv_cases_cover_every_patch_geometry():
    """the per-element GPU cases themselves (their plans come from plan_shapes.conv_plan) reach every patch geometry of each conv kind,
    and both routes without a patch; the resolution table reaches them too, bn = 16 from the synthetic grid only"""
    from tests.test_kernel_plans_gpu import CONV_PLANS
    tc_route = dict(s1="tc", s2="tc", up2="tc_up2")
    for kind, route in tc_route.items():
        assert {p[2] for k, r, p in CONV_PLANS.values() if k == kind and r == route} >= GEOMETRIES, kind
    assert {(k, r) for k, r, _ in CONV_PLANS.values()} >= {("s1", "simt"), ("up2", "upsample_tc")}
    lv = P.all_levels()
    s = P.SYNTHETIC_BN16
    syn = P.pick_patch(s["nb"], s["h"], s["w"])
    assert syn == (4, 2, 16)
    assert _bn([v.patch for v in lv]) | {16} >= GEOMETRIES
    assert _bn([v.down_patch for v in lv]) | {16} >= GEOMETRIES            # stride 2 tiles its output grid
    assert _bn([v.up_patch for v in lv]) | {16} >= GEOMETRIES              # the four-phase upsampler tiles its low-resolution grid


@pytest.mark.parametrize("res,lv,patch", [("384x384", 2, (4, 4, 8)), ("256x256", 3, (4, 4, 8)), ("384x384", 3, (2, 2, 32)),
                                          ("320x576", 1, (4, 4, 8)), ("320x576", 2, (2, 2, 32)), ("320x576", 3, None),
                                          ("512x256", 3, (4, 8, 4)), ("768x768_F32", 3, (4, 4, 8))])
def test_patch_geometry_of_the_level(res, lv, patch):
    assert P.level(res, lv).patch == patch


def test_5x9_upsampler_materialises_onto_the_bn32_plan():
    v = P.level("320x576", 3)
    assert (v.h, v.w, v.up_patch, v.up_materialised) == (5, 9, None, (2, 2, 32))


@pytest.mark.parametrize("res,lv,route,tiles", [("320x576", 0, "mma", 45), ("320x576", 1, "mma", 12), ("384x384", 1, "mma", 9),
                                                ("384x384_sd2", 1, "mma", 9), ("768x768_F32", 0, "wgmma", 72),
                                                ("768x768_F32", 1, "wgmma_d80", 18), ("384x384", 0, "wgmma", 18)])
def test_self_attention_route_of_the_level(res, lv, route, tiles):
    v = P.level(res, lv)
    assert (v.attn_route, v.key_tiles) == (route, tiles)


def test_level_row_counts():
    assert [P.level("384x384", i).rows for i in (2, 3)] == [4608, 1152]
    assert P.level("320x576", 3).rows == 1440 and 1440 % 128          # a ragged last m tile


# ---- blocked references ---------------------------------------------------------------------------------------------------------

SMALL = 64          # fp64 elements per block: every case below splits into several blocks

BLOCKED = {
    "gemm_rowbias_residual": (lambda: H.gemm_case(BF, 130, 48, 40, "cpu", residual=True, rpg=4), -2),
    "gemm_lnfold_rowbias": (lambda: H.gemm_case(BF, 256, 32, 24, "cpu", ln=True, rpg=128), -2),
    "gemm_two_segment": (lambda: H.gemm_case(BF, 70, 32, 64, "cpu", K2=24), -2),
    "gemm_geglu": (lambda: H.gemm_case(BF, 66, 512, 24, "cpu", geglu=True), -2),
    "gemm_batched": (lambda: H.gemm_case(BF, 20, 16, 8, "cpu", bias=False, alpha=0.25, out_f32=True, batch=2), -2),
    "conv_rowbias_residual": (lambda: H.conv_case(BF, 8, 4, 4, 8, 16, "cpu", residual=True, ipg=2), 0),
    "conv_stride2": (lambda: H.conv_case(BF, 4, 4, 4, 8, 16, "cpu", stride=2, ipg=2), 0),
    "conv_up2_phases": (lambda: H.conv_case(BF, 3, 4, 8, 8, 16, "cpu", up=2, phases=True), 0),
    "attention_second_context": (lambda: H.attention_case(torch.float32, 2, 8, 2, 6, 5, 1, "cpu", T=3), 1),
    "attention_accumulate": (lambda: H.attention_case(BF, 2, 8, 2, 6, 5, 1, "cpu", accumulate=True), 1),
    "cross_tc_d40": (lambda: H.cross_tc_case(BF, 3, 40, 2, 9, 6, 4, 2, "cpu"), 1),
    "self_tc_d64": (lambda: H.self_tc_case(BF, 64, 1, 16, 2, "cpu", wide_out=False), 1),
    "self_tc_d80_ascending": (lambda: H.self_tc_case(BF, 80, 2, 16, 2, "cpu", wide_out=False, layout="ascending"), 1),
    "attention_late_peak": (lambda: H.attention_case(BF, 2, 8, 2, 70, 70, 1, "cpu", layout="late_peak"), 1),
}


@pytest.fixture
def emulated(monkeypatch):
    E.install(monkeypatch)
    yield


@pytest.mark.parametrize("name", list(BLOCKED))
def test_blocked_reference_equals_single_block(emulated, name):
    case, axis = BLOCKED[name][0](), BLOCKED[name][1]
    split = H.SPLIT[case.op](case.operands, case.params, SMALL)
    assert split[0] == axis and len(split[1]) > 1
    whole = H.ref64(case, elems=1 << 40), H.mag64(case, elems=1 << 40)
    blocked = H.ref64(case, elems=SMALL), H.mag64(case, elems=SMALL)
    for a, b in zip(whole, blocked):
        # the same fp64 sums; a matmul over fewer rows may block its reduction differently, which moves the last bits only
        assert a.shape == b.shape and torch.allclose(a, b, rtol=1e-12, atol=1e-13)
    name0, idx = case.seeds[0]
    seeded = dict(case.operands)
    seeded[name0] = seeded[name0].clone()
    seeded[name0][idx] = float("nan")
    assert torch.equal(torch.isnan(H.ref64(case, seeded, elems=1 << 40)), torch.isnan(H.ref64(case, seeded, elems=SMALL)))


@pytest.mark.parametrize("name", list(BLOCKED))
def test_emulator_passes_with_blocked_references(emulated, monkeypatch, name):
    monkeypatch.setattr(H, "CHUNK_ELEMS", SMALL)
    res = H.run_checks(BLOCKED[name][0]())
    assert res["surround"]["ok"] and all(c["ok"] for c in res["cones"]) and res["bound"]["ok"], res


@pytest.mark.parametrize("layout", H.LAYOUTS)
def test_score_layouts(layout):
    """the operand layouts of the long-key attention cases give the score structure they are named for, with logits spanning ~30"""
    q, k = H.layout_qk(layout, 2, 300, 2, 40, 40 ** -0.5)
    s = 40 ** -0.5 * torch.einsum("nqhd,nkhd->nhqk", q.to(BF).double(), k.to(BF).double())
    if layout == "ascending":
        assert bool((s.diff(dim=-1) >= 0).all()) and float((s[..., -1] - s[..., 0]).min()) > 20
        tile_max = s.unflatten(-1, (-1, 60)).amax(-1)
        assert bool((tile_max.diff(dim=-1) > 0).all())                    # every key tile raises the running max
    elif layout == "late_peak":
        top = s.topk(2, dim=-1)
        assert bool((top.indices[..., 0] >= 256).all()) and float((top.values[..., 0] - top.values[..., 1]).min()) > 25
    elif layout == "flat":
        assert bool((s == s[..., :1]).all())
    else:
        assert float(s.std()) > 0.5
