// C-ABI entry points that choose between the wgmma tensor-core kernels and the CUDA-core kernels.
// Both are device code of this library; there is no CPU fallback anywhere.
#include "common.cuh"

int32_t fyc_gemm_simt(const fyc_gemm_args* g, cudaStream_t st);
int32_t fyc_gemm_tc(const fyc_gemm_args* g, cudaStream_t st);
bool fyc_gemm_tc_eligible(const fyc_gemm_args* g);
int32_t fyc_conv3x3_simt(const fyc_conv3x3_args* c, cudaStream_t st);
int32_t fyc_conv3x3_tc(const fyc_conv3x3_args* c, const void* x_planes, cudaStream_t st);
bool fyc_conv3x3_tc_eligible(const fyc_conv3x3_args* c);
int32_t fyc_conv3x3_up2_tc(const fyc_conv3x3_args* c, cudaStream_t st);
bool fyc_conv3x3_up2_tc_eligible(const fyc_conv3x3_args* c);
int32_t fyc_space_to_planes(const void* x, void* out, int64_t NB, int64_t H, int64_t W, int64_t C, cudaStream_t st);
int32_t fyc_attention_simt(const fyc_attention_args* a, cudaStream_t st);
int32_t fyc_attention_mma(const fyc_attention_args* a, cudaStream_t st);
bool fyc_attention_mma_eligible(const fyc_attention_args* a);
bool fyc_gemv_eligible(const fyc_gemm_args* g);
int32_t fyc_gemv(const fyc_gemm_args* g, cudaStream_t st);
bool fyc_conv_small_n_eligible(const fyc_conv3x3_args* c);
int32_t fyc_conv_small_n(const fyc_conv3x3_args* c, cudaStream_t st);

extern "C" int32_t fyc_gemm(const fyc_gemm_args* g, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  FYC_CHECK(g && g->A && g->W && g->out, "gemm: null pointer");
  FYC_CHECK(g->M > 0 && g->N > 0 && g->K > 0 && g->batch >= 1, "gemm: bad shape M=%lld N=%lld K=%lld batch=%lld", (long long)g->M,
            (long long)g->N, (long long)g->K, (long long)g->batch);
  FYC_CHECK(!(g->epilogue & FYC_EPI_BIAS) || g->bias, "gemm: FYC_EPI_BIAS without bias");
  FYC_CHECK(!(g->epilogue & FYC_EPI_RESIDUAL) || g->residual, "gemm: FYC_EPI_RESIDUAL without residual");
  FYC_CHECK(!(g->epilogue & FYC_EPI_ROWBIAS) || (g->rowbias && g->rows_per_group > 0), "gemm: FYC_EPI_ROWBIAS without rowbias/rows_per_group");
  FYC_CHECK(!(g->epilogue & FYC_EPI_OUT_F32) || fyc_is_16bit(g->dtype) || g->dtype == FYC_F32, "gemm: bad dtype");
  if (g->A2)
    FYC_CHECK(g->impl != FYC_IMPL_SIMT && fyc_gemm_tc_eligible(g), "gemm: the two-segment A (A2) is a tensor-core-path feature (bf16, K1 %% 64 == 0); "
              "other callers materialise the concatenation with fyc_concat_channels");
  if (g->epilogue & FYC_EPI_LNFOLD)
    FYC_CHECK(g->impl != FYC_IMPL_SIMT && fyc_gemm_tc_eligible(g), "gemm: FYC_EPI_LNFOLD is a tensor-core-path epilogue (bf16, N %% 8 == 0, alpha 1, "
              "ln_rowstats / ln_colsum set); the CUDA-core path runs fyc_layernorm + fyc_gemm");
  if (g->impl == FYC_IMPL_TCGEN05) return fyc_gemm_tc(g, st);
  if (g->impl == FYC_IMPL_AUTO && fyc_gemm_tc_eligible(g)) return fyc_gemm_tc(g, st);
  if (g->impl == FYC_IMPL_AUTO && fyc_gemv_eligible(g)) return fyc_gemv(g, st);
  return fyc_gemm_simt(g, st);
}

extern "C" size_t fyc_conv3x3_workspace_bytes(const fyc_conv3x3_args* c) {
  if (fyc_is_16bit(c->dtype) && c->stride == 2 && c->upsample == 1) return (size_t)(c->NB * c->H * c->W * c->Cin * 2);
  return 0;
}

extern "C" int32_t fyc_conv3x3_up2_eligible(const fyc_conv3x3_args* c) {
  return (c && c->impl != FYC_IMPL_SIMT && fyc_tcgen05_available() == 1 && fyc_conv3x3_up2_tc_eligible(c)) ? 1 : 0;
}

// The route of a fyc_conv3x3 call (workspace as given): the one rule for both the launch below and fyc_conv3x3_tc_route.
enum ConvRoute { CONV_SIMT, CONV_TC, CONV_TC_UP2 };
static ConvRoute conv3x3_route(const fyc_conv3x3_args* c) {
  if (c->impl == FYC_IMPL_SIMT) return CONV_SIMT;
  if (c->upsample == 2 && c->w_phases && fyc_conv3x3_up2_tc_eligible(c)) return CONV_TC_UP2;
  if (!fyc_conv3x3_tc_eligible(c)) return CONV_SIMT;
  if (c->stride == 2 && (!c->workspace || c->workspace_bytes < fyc_conv3x3_workspace_bytes(c))) return CONV_SIMT;
  return CONV_TC;
}

extern "C" int32_t fyc_conv3x3_tc_route(const fyc_conv3x3_args* c) {
  return (c && conv3x3_route(c) != CONV_SIMT) ? 1 : 0;
}

extern "C" int32_t fyc_conv3x3(const fyc_conv3x3_args* c, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  FYC_CHECK(c && c->x && c->w && c->out, "conv3x3: null pointer");
  FYC_CHECK(c->stride == 1 || c->stride == 2, "conv3x3: stride %d", c->stride);
  FYC_CHECK(c->upsample == 1 || c->upsample == 2, "conv3x3: upsample %d", c->upsample);
  FYC_CHECK(c->pad_mode == 0 || (c->pad_mode == 1 && c->stride == 2 && c->upsample == 1 && c->H % 2 == 0 && c->W % 2 == 0),
            "conv3x3: pad_mode %d needs stride 2, no upsampling and even H, W", c->pad_mode);
  FYC_CHECK(!(c->epilogue & FYC_EPI_BIAS) || c->bias, "conv3x3: FYC_EPI_BIAS without bias");
  FYC_CHECK(!(c->epilogue & FYC_EPI_RESIDUAL) || c->residual, "conv3x3: FYC_EPI_RESIDUAL without residual");
  FYC_CHECK(!(c->epilogue & FYC_EPI_ROWBIAS) || (c->rowbias && c->images_per_group > 0), "conv3x3: FYC_EPI_ROWBIAS without rowbias");
  const ConvRoute route = conv3x3_route(c);
  if (route == CONV_TC_UP2) return fyc_conv3x3_up2_tc(c, st);
  if (route == CONV_SIMT) {
    FYC_CHECK(c->impl != FYC_IMPL_TCGEN05 || c->stride != 2 || !fyc_conv3x3_tc_eligible(c),
              "conv3x3(tensor cores): stride-2 needs %zu workspace bytes", fyc_conv3x3_workspace_bytes(c));
    FYC_CHECK(c->impl != FYC_IMPL_TCGEN05, "conv3x3: tensor-core path requested but shape not eligible");
    if (c->impl == FYC_IMPL_AUTO && fyc_conv_small_n_eligible(c)) return fyc_conv_small_n(c, st);
    return fyc_conv3x3_simt(c, st);
  }
  if (c->stride == 2) {
    int32_t rc = fyc_space_to_planes(c->x, c->workspace, c->NB, c->H, c->W, c->Cin, st);
    if (rc) return rc;
    return fyc_conv3x3_tc(c, c->workspace, st);
  }
  return fyc_conv3x3_tc(c, nullptr, st);
}

extern "C" int32_t fyc_attention(const fyc_attention_args* a, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  FYC_CHECK(a && a->q && a->k && a->v && a->out, "attention: null pointer");
  FYC_CHECK(a->batch > 0 && a->heads > 0 && a->Lq > 0 && a->Lk > 0 && a->D > 0 && a->kv_batch_div >= 1, "attention: bad shape");
  FYC_CHECK((a->k2 == nullptr) == (a->v2 == nullptr) && (!a->k2 || a->Lk2 > 0), "attention: second context needs k2, v2 and Lk2 > 0");
  if (a->impl == FYC_IMPL_TCGEN05) {
    FYC_CHECK(fyc_attention_mma_eligible(a), "attention: tensor-core path requested but shape not eligible");
    return fyc_attention_mma(a, st);
  }
  if (a->impl == FYC_IMPL_AUTO && fyc_attention_mma_eligible(a)) return fyc_attention_mma(a, st);
  if (a->k2) {     // CUDA-core path (strict-fp32 mode): the two softmaxes as two passes of the same kernel, the second accumulating in fp32
    fyc_attention_args p1 = *a, p2 = *a;
    p1.k2 = p1.v2 = nullptr;
    p2.k = a->k2; p2.v = a->v2; p2.Lk = a->Lk2; p2.ldk = a->ldk2; p2.ldv = a->ldv2; p2.bsk = a->bsk2; p2.bsv = a->bsv2;
    p2.k2 = p2.v2 = nullptr; p2.out_alpha = a->alpha2; p2.accumulate = 1;
    const int32_t rc = fyc_attention_simt(&p1, st);
    return rc ? rc : fyc_attention_simt(&p2, st);
  }
  return fyc_attention_simt(a, st);
}
