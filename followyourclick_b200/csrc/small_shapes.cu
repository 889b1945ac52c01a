// Memory-bound special cases of the GEMM / conv families that neither tile shape serves well:
//   * gemv_small_m_kernel : M <= 8 rows (time / fps / flow embedding MLPs and the 22 time_emb_proj Linears,
//                           unet.py:526-558, resnet.py:307) - one warp per output column streams the weight row once.
//   * conv3x3_small_n_kernel : Cout <= 8 (conv_out 320 -> 4, unet.py:351; VAE conv_out 128 -> 3, vae.py:205) - one thread
//                           per output pixel, 16-byte channel vectors, weights in shared memory; reads the input once
//                           from HBM (the 9-tap reuse is served by L1/L2).
#include "common.cuh"

namespace {

template <typename T, typename TO, int MAXM>
__global__ void __launch_bounds__(256) gemv_small_m_kernel(const T* __restrict__ A, const T* __restrict__ W, TO* __restrict__ out,
                                                           int M, int64_t N, int64_t K, int64_t lda, int64_t ldw, int64_t ldo,
                                                           const float* __restrict__ bias, const TO* __restrict__ residual,
                                                           int64_t ldr, float alpha) {
  const int lane = threadIdx.x & 31;
  const int64_t n = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (n >= N) return;
  float acc[MAXM];
#pragma unroll
  for (int m = 0; m < MAXM; ++m) acc[m] = 0.f;
  const T* wr = W + n * ldw;
  for (int64_t k = lane * 4; k < K; k += 128) {       // K % 4 == 0 checked by the host
    float w[4];
    Vec4<T>::load(wr + k, w);
#pragma unroll
    for (int m = 0; m < MAXM; ++m) {
      if (m < M) {
        float a[4];
        Vec4<T>::load(A + m * lda + k, a);
        acc[m] = fmaf(a[0], w[0], fmaf(a[1], w[1], fmaf(a[2], w[2], fmaf(a[3], w[3], acc[m]))));
      }
    }
  }
#pragma unroll
  for (int m = 0; m < MAXM; ++m) acc[m] = warp_sum(acc[m]);
  if (lane == 0) {
#pragma unroll
    for (int m = 0; m < MAXM; ++m) {
      if (m < M) {
        float v = acc[m] * alpha;
        if (bias) v += bias[n];
        if (residual) v += to_f(residual[m * ldr + n]);
        out[m * ldo + n] = from_f<TO>(v);
      }
    }
  }
}

template <typename T, typename TO, int CO>
__global__ void __launch_bounds__(128) conv3x3_small_n_kernel(const T* __restrict__ x, const T* __restrict__ w, TO* __restrict__ out,
                                                              const float* __restrict__ bias, int64_t NB, int H, int W, int Cin,
                                                              int Cout) {
  extern __shared__ float sw[];     // [9][Cin][CO]
  for (int i = threadIdx.x; i < 9 * Cin * CO; i += blockDim.x) {
    int co = i % CO, rest = i / CO;           // rest = tap * Cin + c
    sw[i] = co < Cout ? to_f(w[(int64_t)co * 9 * Cin + rest]) : 0.f;
  }
  __syncthreads();
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= NB * H * W) return;
  const int ow = (int)(p % W), oh = (int)((p / W) % H);
  const int64_t n = p / ((int64_t)W * H);
  float acc[CO];
#pragma unroll
  for (int co = 0; co < CO; ++co) acc[co] = 0.f;
  for (int tap = 0; tap < 9; ++tap) {
    const int ih = oh + tap / 3 - 1, iw = ow + tap % 3 - 1;
    if (ih < 0 || iw < 0 || ih >= H || iw >= W) continue;
    const T* xr = x + ((n * H + ih) * W + iw) * Cin;
    const float* wt = sw + tap * Cin * CO;
    for (int c = 0; c < Cin; c += 8) {
      float f[8];
      Vec8<T>::load(xr + c, f);
#pragma unroll
      for (int e = 0; e < 8; ++e)
#pragma unroll
        for (int co = 0; co < CO; ++co) acc[co] = fmaf(f[e], wt[(c + e) * CO + co], acc[co]);
    }
  }
  TO* o = out + p * Cout;
#pragma unroll
  for (int co = 0; co < CO; ++co)
    if (co < Cout) o[co] = from_f<TO>(acc[co] + (bias ? bias[co] : 0.f));
}

template <typename T, typename TO>
int32_t launch_small_n(const fyc_conv3x3_args* c, cudaStream_t st) {
  const int64_t M = c->NB * c->H * c->W;
  const size_t smem = (size_t)9 * c->Cin * 4 * sizeof(float);
  auto kern = conv3x3_small_n_kernel<T, TO, 4>;
  if (smem > 48 * 1024) FYC_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kern<<<(unsigned)ceil_div64(M, 128), 128, smem, st>>>((const T*)c->x, (const T*)c->w, (TO*)c->out, (c->epilogue & FYC_EPI_BIAS) ? c->bias : nullptr,
                                                         c->NB, (int)c->H, (int)c->W, (int)c->Cin, (int)c->Cout);
  FYC_LAUNCH_CHECK();
  return FYC_OK;
}

}  // namespace

bool fyc_gemv_eligible(const fyc_gemm_args* g) {
  return g->M <= 8 && g->batch == 1 && g->K % 4 == 0 && g->lda % 4 == 0 && g->ldw % 4 == 0 &&
         !(g->epilogue & (FYC_EPI_GEGLU | FYC_EPI_ROWBIAS)) && (((uintptr_t)g->A | (uintptr_t)g->W) % 16 == 0);
}

int32_t fyc_gemv(const fyc_gemm_args* g, cudaStream_t st) {
  const unsigned grid = (unsigned)ceil_div64(g->N, 8);
  const float* bias = (g->epilogue & FYC_EPI_BIAS) ? g->bias : nullptr;
  const void* res = (g->epilogue & FYC_EPI_RESIDUAL) ? g->residual : nullptr;
  const bool f32out = (g->epilogue & FYC_EPI_OUT_F32) != 0;
  if (g->dtype == FYC_F32) {
    gemv_small_m_kernel<float, float, 8><<<grid, 256, 0, st>>>((const float*)g->A, (const float*)g->W, (float*)g->out, (int)g->M, g->N, g->K,
                                                                 g->lda, g->ldw, g->ldo, bias, (const float*)res, g->ldr, g->alpha);
  } else {
    FYC_DISPATCH16(g->dtype, {
      if (f32out)
        gemv_small_m_kernel<T, float, 8><<<grid, 256, 0, st>>>((const T*)g->A, (const T*)g->W, (float*)g->out, (int)g->M, g->N, g->K,
                                                               g->lda, g->ldw, g->ldo, bias, (const float*)res, g->ldr, g->alpha);
      else
        gemv_small_m_kernel<T, T, 8><<<grid, 256, 0, st>>>((const T*)g->A, (const T*)g->W, (T*)g->out, (int)g->M, g->N, g->K,
                                                           g->lda, g->ldw, g->ldo, bias, (const T*)res, g->ldr, g->alpha);
    })
  }
  FYC_LAUNCH_CHECK();
  return FYC_OK;
}

bool fyc_conv_small_n_eligible(const fyc_conv3x3_args* c) {
  return c->Cout <= 4 && c->Cin % 8 == 0 && c->stride == 1 && c->upsample == 1 && !(c->epilogue & ~(FYC_EPI_BIAS | FYC_EPI_OUT_F32)) &&
         ((uintptr_t)c->x % 16 == 0) && (size_t)9 * c->Cin * 4 * sizeof(float) <= 200 * 1024;
}

int32_t fyc_conv_small_n(const fyc_conv3x3_args* c, cudaStream_t st) {
  const bool f32out = (c->epilogue & FYC_EPI_OUT_F32) != 0;
  if (c->dtype == FYC_F32) return launch_small_n<float, float>(c, st);
  FYC_DISPATCH16(c->dtype, {
    if (f32out) return launch_small_n<T, float>(c, st);
    return launch_small_n<T, T>(c, st);
  })
  return FYC_OK;
}
