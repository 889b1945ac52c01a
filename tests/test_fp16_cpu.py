"""CPU: the opt-in fp16 tensor-core mode - C ABI constant, the compute-dtype API, the fp16 LN-folded weights, and the host logic of the
UNet / VAE / pipeline in fp16 with every kernel launch emulated (tests/ops_emulator.py; the tensor-core routes are the ones the rules of
followyourclick_b200.ops pick for fp16).  The real fp16 kernels are checked by tests/test_fp16_gpu.py.
"""
import os
import re

import pytest
import torch

from followyourclick_b200 import _lib, ops
from tests import ops_emulator
from tests.fp16_helpers import literal_fp16_to

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def emulated(monkeypatch):
    ops_emulator.install(monkeypatch)
    literal_fp16_to(monkeypatch)
    torch.set_num_threads(8)
    yield


# ---- C ABI ----------------------------------------------------------------------------------------------------------------------
def test_f16_code_agrees_between_header_and_binding():
    hdr = open(os.path.join(ROOT, "include", "fyc.h")).read()
    enum = dict((k, int(v)) for k, v in re.findall(r"(FYC_(?:F32|BF16|F16)) = (\d+)", hdr))
    assert enum == {"FYC_F32": _lib.F32, "FYC_BF16": _lib.BF16, "FYC_F16": _lib.F16} == {"FYC_F32": 0, "FYC_BF16": 1, "FYC_F16": 2}
    assert _lib.dtype_code(torch.float16) == _lib.F16 and _lib.dtype_code(torch.bfloat16) == _lib.BF16
    # every fp16 twin of a dtype-less wgmma attention entry point is declared with the bf16 entry point's arguments
    for base in ("fyc_self_attention_tc", "fyc_self_attention_tc_d80", "fyc_cross_attention_tc"):
        args = lambda name: re.search(r"int32_t " + name + r"\(([^;]*)\);", hdr).group(1).count(",")
        assert args(base + "_f16") == args(base)
        assert _lib.SIGNATURES[base + "_f16"] == _lib.SIGNATURES[base]


# ---- compute-dtype API ----------------------------------------------------------------------------------------------------------
def _mini_models():
    from followyourclick_b200 import AutoencoderKL, UNet2DConditionModel, UNet3DConditionModel
    from tests.cfgs import MINI_UNET2D
    from tests.engine_helpers import mini_unet_ref_kwargs
    vae = AutoencoderKL(in_channels=3, out_channels=3, down_block_types=("DownEncoderBlock2D",) * 2, up_block_types=("UpDecoderBlock2D",) * 2,
                        block_out_channels=(32, 64), layers_per_block=1, latent_channels=4, norm_num_groups=32)
    return UNet3DConditionModel(**mini_unet_ref_kwargs("base")), UNet2DConditionModel(**MINI_UNET2D), vae


def test_set_compute_dtype_selects_fp16_and_rejects_other_dtypes():
    from followyourclick_b200.ip_adapter import IPAttnProcessor
    proc = IPAttnProcessor(hidden_size=64, cross_attention_dim=32)
    for m in list(_mini_models()) + [proc]:
        for dt in (torch.float16, torch.bfloat16, torch.float32):
            assert m.set_compute_dtype(dt) is m and m._compute_dtype == dt
        for bad in (torch.float64, torch.int8, torch.float8_e4m3fn, "float16"):
            with pytest.raises(ValueError):
                m.set_compute_dtype(bad)
        assert m._compute_dtype == torch.float32


def test_set_compute_dtype_invalidates_packed_weights():
    unet, _, _ = _mini_models()
    v = unet._pack_version
    unet._pack_cache["x"] = 1
    unet.set_compute_dtype(torch.float16)
    assert unet._pack_version == v + 1 and unet._pack_cache == {} and unet.dtype == torch.float16


def test_to_float16_and_half_still_select_bf16():
    for m in _mini_models():
        assert m.to(torch.float16).dtype == torch.bfloat16
        m.set_compute_dtype(torch.float32)
        assert m.half().dtype == torch.bfloat16
        assert m.to(dtype=torch.float16).dtype == torch.bfloat16
        m.set_compute_dtype(torch.float16)
        assert m.to(torch.float16).dtype == torch.bfloat16          # .to() keeps its mapping even from fp16 mode


def test_pipeline_and_ip_adapter_forward_the_compute_dtype():
    from followyourclick_b200 import AnimationPipeline, DDIMScheduler
    from followyourclick_b200.ip_adapter import MyIPAdapter
    from followyourclick_b200.unet import ImageProjModel
    unet, _, vae = _mini_models()
    unet.image_proj_model = ImageProjModel(cross_attention_dim=768, clip_embeddings_dim=32, clip_extra_context_tokens=4)
    ipa = MyIPAdapter(unet, device="cpu", image_encoder=None, clip_embeddings_dim=32)
    pipe = AnimationPipeline(vae=vae, text_encoder=None, tokenizer=None, unet=unet, scheduler=DDIMScheduler(), ip_adapter=ipa)
    assert pipe.set_compute_dtype(torch.float16) is pipe
    assert unet.dtype == vae.dtype == ipa.image_proj_model.dtype == unet.image_proj_model.dtype == torch.float16
    pipe.set_compute_dtype(torch.bfloat16)
    assert unet.dtype == vae.dtype == ipa.image_proj_model.dtype == torch.bfloat16
    with pytest.raises(ValueError):
        pipe.set_compute_dtype(torch.float64)
    assert unet.dtype == torch.bfloat16


# ---- LN-folded weights ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_ln_fold_weight_rows_sum_to_zero(dtype):
    g = torch.Generator().manual_seed(3)
    N, K = 96, 320
    w = torch.randn(N, K, generator=g) * 0.05
    w[:, :7] *= 40                                            # a few large columns: the row sum's rounding error is dominated by them
    gamma = 1 + 0.1 * torch.randn(K, generator=g)
    wp = ops.ln_fold_weight(w, gamma, dtype)
    assert wp.dtype == dtype and wp.shape == (N, K)
    exact = w * gamma[None, :]
    exact = exact - exact.mean(dim=1, keepdim=True)
    plain = exact.to(dtype).float()
    frac = {torch.float16: 10, torch.bfloat16: 7}[dtype]
    spacing = torch.exp2(torch.floor(torch.log2(plain.abs().clamp_min(1e-30))) - frac)
    # at most 12 one-ulp steps per row (one per balancing pass) away from the once-rounded centred weight, and the rows sum to ~0
    steps = (wp.float() - plain).abs() / spacing
    assert float(steps.sum(dim=1).max()) <= 12 * 2 + 1e-6
    rowsum = wp.double().sum(dim=1).abs()
    assert float(rowsum.max()) < 1e-5 * float(exact.abs().max()) * K ** 0.5, float(rowsum.max())
    assert float(plain.double().sum(dim=1).abs().max()) > 10 * float(rowsum.max())      # the balancing did something


def test_fp16_balancing_is_finer_than_bf16():
    g = torch.Generator().manual_seed(4)
    w, gamma = torch.randn(64, 640, generator=g) * 0.02, torch.ones(640)
    e16 = (ops.ln_fold_weight(w, gamma, torch.float16).float() - (w - w.mean(dim=1, keepdim=True))).norm()
    eb16 = (ops.ln_fold_weight(w, gamma, torch.bfloat16).float() - (w - w.mean(dim=1, keepdim=True))).norm()
    assert e16 * 4 < eb16


# ---- host logic in fp16 against the reference fixtures, kernels emulated ---------------------------------------------------------
# fp16 tolerances: the bf16 ones (tests/test_host_emulated_cpu.py: rel-L2 3e-2, PSNR 30 dB) tightened by the 8x finer rounding.  One UNet
# variant and the VAE decoder here (the emulated forwards are slow on CPU); every variant runs on the GPU in tests/test_fp16_gpu.py.
def test_unet_host_logic_fp16_vs_reference_golden_on_tensor_core_routes(emulated, monkeypatch):
    from tests.engine_helpers import run_unet_case
    sb = run_unet_case("base", torch.bfloat16, device="cpu")
    seen = {}
    for name in ("conv3x3", "self_attention_tc", "cross_attention_tc", "temporal_attention", "groupnorm"):
        fn = getattr(ops, name)

        def spy(*a, _fn=fn, _name=name, **kw):
            seen.setdefault(_name, set()).add(a[0].dtype)
            return _fn(*a, **kw)
        monkeypatch.setattr(ops, name, spy)
    s16 = run_unet_case("base", torch.float16, device="cpu")
    assert s16["finite"] and s16["rel_l2"] < 1e-2 and s16["rel_l2"] < sb["rel_l2"], (s16, sb)
    assert seen == {k: {torch.float16} for k in ("conv3x3", "self_attention_tc", "cross_attention_tc", "temporal_attention", "groupnorm")}, seen


def test_vae_and_pipeline_host_logic_fp16_vs_reference_golden(emulated):
    from tests.engine_helpers import run_pipeline_case, run_vae_case
    s16 = run_vae_case(torch.float16, device="cpu")
    assert s16["finite"] and s16["rel_l2"] < 1e-2, s16
    r16 = run_pipeline_case(torch.float16, steps=3, against="golden", device="cpu")
    assert r16["finite"] and r16["shape"] == (1, 3, 4, 64, 64) and r16["psnr"] > 40.0, r16
