"""CPU self-test of the cone / bound harness (tests/cone_helpers.py) that tests/test_kernel_cones_gpu.py runs on the kernels.

The case builders run at small shapes with every ops entry point replaced by tests/ops_emulator.py (the fyc.h contract in fp32 with one
storage rounding).  The emulator must pass all three checks; each deliberately broken variant of it below must be caught by the check
named for it - evidence that the checks can fail before they are trusted to pass on the GPU.
"""
import pytest
import torch
import torch.nn.functional as F

from tests import cone_helpers as H
from tests import ops_emulator as E

BF, F32 = torch.bfloat16, torch.float32


@pytest.fixture(autouse=True)
def _emulated(monkeypatch):
    E.install(monkeypatch)
    yield


def _gemm():
    return H.gemm_case(BF, 130, 48, 40, "cpu", residual=True, alpha=0.5)


def _attention():
    return H.attention_case(BF, 2, 8, 4, 10, 5, 2, "cpu")


def _conv():
    return H.conv_case(BF, 2, 4, 4, 8, 16, "cpu")


def _groupnorm():
    return H.groupnorm_case(BF, 4, 6, 16, 4, 2, "cpu")


def _temporal():
    return H.temporal_case(BF, 1, 3, 2, 2, 8, "cpu")


CASES = {
    "gemm": _gemm,
    "gemm_lnfold_rowbias": lambda: H.gemm_case(BF, 256, 32, 24, "cpu", ln=True, rpg=128),
    "gemm_two_segment": lambda: H.gemm_case(BF, 70, 32, 64, "cpu", K2=24),
    "gemm_geglu": lambda: H.gemm_case(BF, 66, 512, 24, "cpu", geglu=True),
    "gemm_batched_f32out": lambda: H.gemm_case(BF, 20, 16, 8, "cpu", bias=False, alpha=0.25, out_f32=True, batch=2),
    "gemm_f32": lambda: H.gemm_case(F32, 9, 24, 16, "cpu", residual=True, rpg=4),
    "conv": _conv,
    "conv_stride2_pad1_rowbias": lambda: H.conv_case(BF, 4, 4, 4, 8, 16, "cpu", stride=2, pad_mode=1, ipg=2),
    "conv_up2_phases": lambda: H.conv_case(BF, 2, 4, 8, 8, 16, "cpu", up=2, phases=True),
    "conv_f32_residual": lambda: H.conv_case(F32, 2, 4, 5, 8, 4, "cpu", residual=True),
    "groupnorm": _groupnorm,
    "groupnorm_concat": lambda: H.groupnorm_case(F32, 2, 5, 12, 4, 2, "cpu", silu=True, C2=8),
    "layernorm_pe": lambda: H.layernorm_case(BF, 70, 16, "cpu", pe=True),
    "layernorm_stats": lambda: H.layernorm_case(BF, 9, 24, "cpu", stats_only=True),
    "attention": _attention,
    "attention_second_context": lambda: H.attention_case(F32, 2, 8, 2, 6, 5, 1, "cpu", T=3),
    "attention_accumulate": lambda: H.attention_case(BF, 2, 8, 2, 6, 5, 1, "cpu", accumulate=True),
    "cross_tc_d40": lambda: H.cross_tc_case(BF, 3, 40, 2, 9, 6, 4, 2, "cpu"),
    "self_tc_d64": lambda: H.self_tc_case(BF, 64, 1, 16, 2, "cpu", wide_out=False),
    "self_tc_d80": lambda: H.self_tc_case(BF, 80, 1, 16, 2, "cpu", wide_out=False),
    "temporal": _temporal,
    "transpose": lambda: H.transpose_case(BF, 2, 6, 8, 8, "cpu"),
    "softmax": lambda: H.softmax_case(BF, 3, 7, "cpu"),
}


def _failures(res):
    f = set()
    if not res["surround"]["ok"]:
        f.add("surround")
    if any(not c["ok"] for c in res["cones"]):
        f.add("cone")
    if not res["bound"]["ok"]:
        f.add("values")
    return f


@pytest.mark.parametrize("name", list(CASES))
def test_emulator_passes_every_check(name):
    case = CASES[name]()
    assert case.seeds
    res = H.run_checks(case)
    assert not _failures(res), res


# ---- mutants: small wrappers around the emulator, each with one fault ----------------------------------------------------------

def _gemm_reads_past_k(A, W, *a, **kw):
    """reads column K of A through the view's storage (multiplied by a zero weight column)"""
    M, K = A.shape
    wide = A.as_strided((M, K + 1), A.stride())
    return E.gemm(wide, torch.cat([W, torch.zeros_like(W[:, :1])], dim=1), *a, **kw)


def _attention_wrong_last_group(q, k, v, heads, scale, kv_batch_div=1, **kw):
    """the last image reads the context of the group before its own"""
    idx = torch.arange(q.shape[0]) // kv_batch_div
    idx[-1] = max(int(idx[-1]) - 1, 0)
    return E.attention(q, k[idx], v[idx], heads, scale, kv_batch_div=1, **kw)


def _conv_reads_neighbour_row(x, w, bias=None, **kw):
    """image n's top padding row holds image n - 1's bottom row"""
    xp = F.pad(x.float().permute(0, 3, 1, 2), (1, 1, 1, 1))
    xp[1:, :, 0, 1:-1] = x.float().permute(0, 3, 1, 2)[:-1, :, -1, :]
    y = F.conv2d(xp, w.float().permute(0, 3, 1, 2), bias)
    return y.permute(0, 2, 3, 1).to(x.dtype).contiguous()


def _groupnorm_across_stat_batches(x, gamma, beta, groups, eps, stat_batches=None, **kw):
    return E.groupnorm(x, gamma, beta, groups, eps, stat_batches=max((stat_batches or x.shape[0]) // 2, 1), **kw)


def _temporal_unmasked_pad_frame(qkv, heads, scale):
    """softmax over F + 1 keys: the zero-filled padding frame F takes part"""
    pad = torch.zeros_like(qkv[:, :1])
    full = E.temporal_attention(torch.cat([qkv, pad], dim=1), heads, scale)
    return full[:, :-1].contiguous()


def _gemm_one_element_off(A, W, bias=None, residual=None, alpha=1.0, out=None, **kw):
    y = E.gemm(A, W, bias=bias, residual=residual, alpha=alpha, **kw)
    o = dict(A=A.double(), W=W.double())
    if bias is not None:
        o["bias"] = bias.double()
    if residual is not None:
        o["residual"] = residual.double()
    ref, mag = H.gemm_ref(o, alpha), H.gemm_mag(o, alpha)
    b = H.bound(ref, mag, y.dtype)
    y = y.double()
    y[3, 5] = ref[3, 5] + 4 * b[3, 5]
    y = y.to(A.dtype)
    if out is not None:
        out.copy_(y)
        return out
    return y


def _gemm_block_one_row_down(A, W, *a, out=None, **kw):
    y = E.gemm(A, W, *a, **kw)
    out[:64] = y[:64]
    out[65:129] = y[64:128]
    out[129:] = y[129:]
    return out


MUTANTS = [
    ("gemm_reads_one_column_past_k", "gemm", _gemm_reads_past_k, _gemm, {"surround"}),
    ("attention_last_image_wrong_kv_group", "attention", _attention_wrong_last_group, _attention, {"cone"}),
    ("conv_reads_neighbour_edge_row", "conv3x3", _conv_reads_neighbour_row, _conv, {"cone"}),
    ("groupnorm_stats_cross_stat_batches", "groupnorm", _groupnorm_across_stat_batches, _groupnorm, {"cone"}),
    ("temporal_pad_frame_unmasked", "temporal_attention", _temporal_unmasked_pad_frame, _temporal, {"values"}),
    ("output_element_off_by_4_bounds", "gemm", _gemm_one_element_off, _gemm, {"values"}),
    ("row_block_stored_one_row_down", "gemm", _gemm_block_one_row_down, _gemm, {"surround", "cone"}),
]


@pytest.mark.parametrize("name,fn,mutant,build,caught_by", MUTANTS, ids=[m[0] for m in MUTANTS])
def test_mutant_is_caught(monkeypatch, name, fn, mutant, build, caught_by):
    from followyourclick_b200 import ops
    monkeypatch.setattr(ops, fn, mutant)
    res = H.run_checks(build())
    assert caught_by <= _failures(res), (caught_by, res)
