"""Every kernel route against NaN-poisoned surroundings, single-NaN dependency cones and per-element fp64 bounds (tests/cone_helpers.py).

Relative-L2 comparisons cannot see one wrong element, a wrong head slice of one row, or a read outside an operand that is multiplied by
zero; these checks can.  Per case: (a) surround - operands inside NaN-filled memory, outputs NaN-prefilled inside NaN frames: the
result is finite, bit-identical to the run with zero surroundings, and the frames are untouched; (b) cones - one NaN operand element
makes exactly the outputs NaN that the fp64 reference makes NaN, every other element is bit-identical; (c) values - every element
within u_o |ref| + C_BOUND * (named terms of the operation) of the fp64 reference of the fyc.h contract.  The largest
|out - ref| / bound of every case is written to cone_ratios.json under pytest's temporary directory and printed.

Routes are selected through the public ops functions and their eligibility rules: the shapes below are chosen so that the documented
rule picks the route named in the case id.
"""
import json

import pytest
import torch

from tests import cone_helpers as H

pytestmark = pytest.mark.gpu

HALF = [torch.bfloat16, torch.float16]
ALL = [torch.float32] + HALF
_N = {torch.bfloat16: "bf16", torch.float16: "f16", torch.float32: "f32"}


def _cross_d40_q_atom(seed, expected):
    """fyc.h fyc_cross_attention_tc: "for D = 40 the 64-column q box of head h also holds the first 24 columns of head h + 1, which meet
    the zero key columns 40..63: a NaN in those columns of head h + 1 makes head h's row NaN too" - the one cone the contract widens"""
    name, idx = seed
    if name == "q" and idx[2] >= 40 and idx[2] % 40 < 24:
        h = idx[2] // 40 - 1
        expected = expected.clone()
        expected[idx[0], idx[1], 40 * h:40 * (h + 1)] = True
    return expected


def _widened(build, widen):
    def b(dt, dev):
        case = build(dt, dev)
        case.widen = widen
        return case
    return b


def _cases():
    c = {}

    def add(family, name, dtypes, build):
        for dt in dtypes:
            c[f"{family}-{name}-{_N[dt]}"] = (family, lambda dev, dt=dt: build(dt, dev))
    g = H.gemm_case
    # fyc_gemm: wgmma plain with ragged M / N / K tiles, W-resident (K = 320, m_tiles x n_tiles >= 4 x grid), batched scores, GEGLU,
    # LN fold with row bias, two-segment A2 with a ragged K2, fp32 output, the CUDA-core kernels and the M <= 8 GEMV
    add("gemm", "wgmma_385x720x72", HALF, lambda dt, d: g(dt, 385, 720, 72, d, residual=True, alpha=0.5))
    add("gemm", "wgmma_383x48x328", HALF, lambda dt, d: g(dt, 383, 48, 328, d, residual=True))
    add("gemm", "resident_33919x320x320", HALF, lambda dt, d: g(dt, 128 * 265 - 1, 320, 320, d, residual=True))
    add("gemm", "batched_scores", HALF, lambda dt, d: g(dt, 200, 256, 64, d, bias=False, alpha=0.125, out_f32=True, batch=3))
    add("gemm", "geglu_385x1280x160", HALF, lambda dt, d: g(dt, 385, 1280, 160, d, geglu=True))
    add("gemm", "lnfold_rowbias_512x320x320", HALF, lambda dt, d: g(dt, 512, 320, 320, d, ln=True, rpg=256))
    add("gemm", "two_segment_385x320x320+328", HALF, lambda dt, d: g(dt, 385, 320, 320, d, K2=328, residual=True))
    add("gemm", "out_f32_rowbias_385x320x128", HALF, lambda dt, d: g(dt, 385, 320, 128, d, rpg=128, out_f32=True))
    add("gemm", "simt_100x72x72", ALL, lambda dt, d: g(dt, 100, 72, 72, d, residual=True, rpg=64, impl="simt"))
    add("gemm", "simt_geglu_70x256x40", [torch.float32], lambda dt, d: g(dt, 70, 256, 40, d, geglu=True))
    add("gemm", "gemv_5x1280x320", ALL, lambda dt, d: g(dt, 5, 1280, 320, d, residual=True, alpha=0.5))
    cv = H.conv_case
    # fyc_conv3x3: each stride-1 patch geometry (128 = bw x bh x bn), stride 2 with both paddings, the four-phase and the materialised
    # upsample, the N = 16 head, conv_small_n (Cout <= 4), the CUDA-core kernel; row bias groups of 2 images read from a wider table
    add("conv", "w64_2x4x64", HALF, lambda dt, d: cv(dt, 2, 4, 64, 64, 48, d, residual=True, ipg=1))
    add("conv", "w32_2x8x32", HALF, lambda dt, d: cv(dt, 2, 8, 32, 72, 32, d, ipg=2))
    add("conv", "w16_3x8x16", HALF, lambda dt, d: cv(dt, 3, 8, 16, 64, 64, d, residual=True))
    add("conv", "8x8x2img_4x8x8", HALF, lambda dt, d: cv(dt, 4, 8, 8, 64, 32, d, residual=True, ipg=2))
    add("conv", "vae128_1x2x128", HALF, lambda dt, d: cv(dt, 1, 2, 128, 32, 16, d))
    add("conv", "stride2_pad0", HALF, lambda dt, d: cv(dt, 2, 16, 16, 64, 48, d, stride=2, residual=True, ipg=1))
    add("conv", "stride2_pad1", HALF, lambda dt, d: cv(dt, 2, 16, 16, 64, 48, d, stride=2, pad_mode=1))
    add("conv", "up2_phases", HALF, lambda dt, d: cv(dt, 2, 8, 8, 64, 48, d, up=2, phases=True))
    add("conv", "up2_materialised", HALF, lambda dt, d: cv(dt, 2, 8, 8, 64, 48, d, up=2))
    add("conv", "head16_f32out", HALF, lambda dt, d: cv(dt, 2, 16, 16, 64, 16, d, out_f32=True))
    add("conv", "small_n_cout4", ALL, lambda dt, d: cv(dt, 2, 8, 8, 64, 4, d))
    add("conv", "simt", ALL, lambda dt, d: cv(dt, 2, 8, 8, 16, 24, d, residual=True, ipg=1, impl="simt"))
    # norms: stat batches > 1 (seeds in one leave the others bit-identical), the two-source concatenation with 60-channel groups across
    # the 1280 | 640 seam, LayerNorm with the position table and a ragged row count, the statistics pass of the LN fold
    add("norm", "groupnorm_silu_stat2", ALL, lambda dt, d: H.groupnorm_case(dt, 4, 64, 160, 32, 2, d, silu=True))
    add("norm", "groupnorm_stat4", ALL, lambda dt, d: H.groupnorm_case(dt, 4, 100, 64, 32, 4, d))
    add("norm", "groupnorm_concat_1280+640", ALL, lambda dt, d: H.groupnorm_case(dt, 2, 32, 1280, 32, 2, d, silu=True, C2=640))
    add("norm", "layernorm_pe_131x768", ALL, lambda dt, d: H.layernorm_case(dt, 131, 768, d, pe=True))
    add("norm", "layernorm_131x320", ALL, lambda dt, d: H.layernorm_case(dt, 131, 320, d))
    add("norm", "layernorm_stats_131x320", ALL, lambda dt, d: H.layernorm_case(dt, 131, 320, d, stats_only=True))
    a = H.attention_case
    # fyc_attention: the generic mma.sync kernel (Lk 1, 63, 65, 150), the resident short-context kernel (Lk <= 128, Lq >= 256), the
    # fused and the two-pass second context, the accumulate form, the CUDA-core kernel; head dims 40 / 64 / 80 / 160, kv_batch_div 1 / 2 / 4
    add("attention", "mma_d40_70x65_div2", ALL, lambda dt, d: a(dt, 3, 40, 4, 70, 65, 2, d))
    add("attention", "mma_d64_100x150", HALF, lambda dt, d: a(dt, 2, 64, 2, 100, 150, 1, d))
    add("attention", "mma_d80_33x1_div4", HALF, lambda dt, d: a(dt, 2, 80, 4, 33, 1, 4, d))
    add("attention", "mma_d160_64x63", ALL, lambda dt, d: a(dt, 2, 160, 2, 64, 63, 1, d))
    add("attention", "shortk_d40_300x77_div2", HALF, lambda dt, d: a(dt, 3, 40, 4, 300, 77, 2, d))
    add("attention", "shortk_d80_257x64", HALF, lambda dt, d: a(dt, 2, 80, 2, 257, 64, 1, d))
    add("attention", "shortk_d64_256x4_div4", HALF, lambda dt, d: a(dt, 2, 64, 4, 256, 4, 4, d))
    add("attention", "fused2_d40_300x77+4_div2", HALF, lambda dt, d: a(dt, 3, 40, 4, 300, 77, 2, d, T=4))
    add("attention", "fused2_d160_70x77+16", ALL, lambda dt, d: a(dt, 2, 160, 2, 70, 77, 1, d, T=16))
    add("attention", "twopass_d40_200x150+4_div2", HALF, lambda dt, d: a(dt, 2, 40, 4, 200, 150, 2, d, T=4))
    add("attention", "accumulate_d64_70x4", ALL, lambda dt, d: a(dt, 2, 64, 2, 70, 4, 1, d, accumulate=True))
    add("attention", "simt_d40_70x64_div2", HALF, lambda dt, d: a(dt, 2, 40, 4, 70, 64, 2, d, impl="simt"))
    # wgmma attention: self D 40 / 64 (L % 128), D 80 (L % 256, the v block of the fused row is poison), cross with T = 0 / 4 / 16
    add("wgmma_attention", "self_d40", HALF, lambda dt, d: H.self_tc_case(dt, 40, 2, 256, 3, d))
    add("wgmma_attention", "self_d64", HALF, lambda dt, d: H.self_tc_case(dt, 64, 2, 256, 2, d))
    add("wgmma_attention", "self_d80", HALF, lambda dt, d: H.self_tc_case(dt, 80, 2, 256, 2, d))
    add("wgmma_attention", "cross_d40_T0", HALF, _widened(lambda dt, d: H.cross_tc_case(dt, 3, 40, 4, 200, 77, 0, 2, d), _cross_d40_q_atom))
    add("wgmma_attention", "cross_d40_T16", HALF, _widened(lambda dt, d: H.cross_tc_case(dt, 3, 40, 4, 200, 77, 16, 2, d), _cross_d40_q_atom))
    add("wgmma_attention", "cross_d64_T4", HALF, lambda dt, d: H.cross_tc_case(dt, 2, 64, 2, 130, 64, 4, 1, d))
    add("wgmma_attention", "cross_d80_T16", HALF, lambda dt, d: H.cross_tc_case(dt, 2, 80, 4, 129, 5, 16, 4, d))
    tm = H.temporal_case
    # fyc_temporal_attention: the mma kernel for frame counts on both sides of 16 and 32, D 40 / 80 / 160; the CUDA-core kernel
    for Fr, D in ((1, 40), (2, 80), (15, 160), (16, 40), (17, 80), (24, 40), (31, 160), (32, 80)):
        add("temporal", f"mma_F{Fr}_D{D}", HALF, lambda dt, d, Fr=Fr, D=D: tm(dt, 2, Fr, 5, 2, D, d))
    add("temporal", "simt_F17_D40", [torch.float32], lambda dt, d: tm(dt, 2, 17, 5, 2, 40, d))
    add("temporal", "simt_F9_D36", HALF, lambda dt, d: tm(dt, 1, 9, 6, 2, 36, d))
    add("glue", "transpose_tokens", HALF, lambda dt, d: H.transpose_case(dt, 2, 130, 72, 8, d))
    add("glue", "softmax_rows", ALL, lambda dt, d: H.softmax_case(dt, 37, 300, d))
    return c


CASES = _cases()


@pytest.fixture(scope="module")
def ratios(tmp_path_factory):
    r = {}
    yield r
    path = tmp_path_factory.mktemp("cones") / "cone_ratios.json"
    fam = {}
    for cid, v in r.items():
        f = fam.setdefault(CASES[cid][0], dict(cases=0, max_ratio=0.0))
        f["cases"] += 1
        f["max_ratio"] = max(f["max_ratio"], v)
    path.write_text(json.dumps(dict(c=H.C_BOUND, families=fam, cases=r), indent=1))
    print(f"\nbound ratios (c = {H.C_BOUND}): {json.dumps(fam)} -> {path}")


@pytest.mark.parametrize("cid", list(CASES))
def test_kernel_cone(cuda, cid, ratios):
    from followyourclick_b200 import ops
    ops.set_impl("auto")
    case = CASES[cid][1]("cuda")
    res = H.run_checks(case)
    ratios[cid] = res["bound"]["ratio"]
    bad_cones = [c for c in res["cones"] if not c["ok"]]
    problems = ([] if res["surround"]["ok"] else [("surround", res["surround"])]) + [("cone", c) for c in bad_cones] + \
               ([] if res["bound"]["ok"] else [("bound", res["bound"])])
    assert not problems, problems


def test_unfused_geglu_rejects_a_strided_output(cuda):
    """Regression: the CUDA-core GEGLU epilogue (fyc_geglu) writes packed rows; given an output view with a wider row stride, ops.gemm
    used to place rows 62.. in the stride padding and leave the view's tail unwritten.  It now refuses such a view."""
    from followyourclick_b200 import _lib, ops
    A, W = H.rnd((70, 40), 1, torch.float32, "cuda"), H.rnd((256, 40), 2, torch.float32, "cuda")
    bias = H.rnd((256,), 3, torch.float32, "cuda")
    out, _ = H.embedded((70, 128), torch.float32, float("nan"), ld=128 + H.PAD, device="cuda")
    with pytest.raises(_lib.FycError, match="contiguous"):
        ops.gemm(A, W, bias=bias, geglu=True, out=out)
    assert bool(torch.isnan(out).all())
