// CUDA-core (FFMA) GEMM and implicit-GEMM 3x3 convolution with fp32 accumulation.
//
// Role: (1) the strict-fp32 parity path (dtype = FYC_F32: every product and sum in fp32, the on-GPU
// restatement the tensor-core kernels are themselves checked against), and (2) shapes the tensor-core path does not
// take (Cin = 9 / 4 stems, Cout = 4 / 3 heads, M = 2 time-embedding MLPs).  The 16-bit hot path is gemm_tc.cu.
//
// Tiling: 128 x 64 x 16 CTA tile, 256 threads, 8 x 4 register tile per thread, smem double buffering with
// register prefetch.  The A-operand loader is a functor so the same main loop serves plain row-major A and the
// on-the-fly im2col view of an NHWC image (stride 1/2, nearest-2x upsample folded into the index).
#include "common.cuh"

namespace {

constexpr int BM = 128, BN = 64, BK = 16, NT = 256;
constexpr int BMP = BM + 4, BNP = BN + 4;

struct Epilogue {
  const float* bias;
  const void* residual;
  const float* rowbias;
  int64_t ldo, ldr, rows_per_group;
  float alpha;
  int flags;
  int64_t ldrb;            // row stride of rowbias (elements)
};

// ---- A loaders: fetch 8 consecutive k of logical row m (zero outside the matrix) -------------------------
template <typename T>
struct PlainA {
  const T* A; int64_t lda, M, K;
  bool vec;  // K % 8 == 0 && lda % 8 == 0 and aligned base
  __device__ __forceinline__ void load8(int64_t m, int64_t k0, float* f) const {
    if (m < M && vec && k0 + 8 <= K) { Vec8<T>::load(A + m * lda + k0, f); return; }
#pragma unroll
    for (int e = 0; e < 8; ++e) f[e] = (m < M && k0 + e < K) ? to_f(A[m * lda + k0 + e]) : 0.f;
  }
};

template <typename T>
struct ConvA {   // logical A[m, k]: m = (n, oh, ow), k = (kh, kw, c);  x is NHWC (pre-upsample dims H, W)
  const T* x; int64_t NB, H, W, Cin, Ho, Wo, M, K;
  int stride, up;
  int pad = 1;   // rows / columns of zero padding BEFORE the image (0 for pad_mode 1: bottom / right padding only)
  bool vec;  // Cin % 8 == 0
  __device__ __forceinline__ float at(int64_t n, int64_t oh, int64_t ow, int64_t k) const {
    int tap = (int)(k / Cin); int64_t c = k - (int64_t)tap * Cin;
    int64_t ih = oh * stride + tap / 3 - pad, iw = ow * stride + tap % 3 - pad;
    if (ih < 0 || iw < 0 || ih >= H * up || iw >= W * up) return 0.f;
    return to_f(x[((n * H + ih / up) * W + iw / up) * Cin + c]);
  }
  __device__ __forceinline__ void load8(int64_t m, int64_t k0, float* f) const {
    if (m >= M) {
#pragma unroll
      for (int e = 0; e < 8; ++e) f[e] = 0.f;
      return;
    }
    int64_t ow = m % Wo; int64_t t = m / Wo; int64_t oh = t % Ho; int64_t n = t / Ho;
    if (vec && k0 + 8 <= K) {   // 8 consecutive k stay inside one tap because Cin % 8 == 0
      int tap = (int)(k0 / Cin); int64_t c = k0 - (int64_t)tap * Cin;
      int64_t ih = oh * stride + tap / 3 - pad, iw = ow * stride + tap % 3 - pad;
      if (ih < 0 || iw < 0 || ih >= H * up || iw >= W * up) {
#pragma unroll
        for (int e = 0; e < 8; ++e) f[e] = 0.f;
      } else {
        Vec8<T>::load(x + ((n * H + ih / up) * W + iw / up) * Cin + c, f);
      }
      return;
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) f[e] = (k0 + e < K) ? at(n, oh, ow, k0 + e) : 0.f;
  }
};

template <typename T>
__device__ __forceinline__ void load_w8(const T* W, int64_t ldw, int64_t N, int64_t K, bool vec, int64_t n, int64_t k0, float* f) {
  if (n < N && vec && k0 + 8 <= K) { Vec8<T>::load(W + n * ldw + k0, f); return; }
#pragma unroll
  for (int e = 0; e < 8; ++e) f[e] = (n < N && k0 + e < K) ? to_f(W[n * ldw + k0 + e]) : 0.f;
}

template <typename T, typename TO, typename ALoader>
__global__ void __launch_bounds__(NT) gemm_simt_kernel(ALoader al, const T* __restrict__ Wg, TO* __restrict__ out,
                                                       int64_t M, int64_t N, int64_t K, int64_t ldw, bool wvec,
                                                       int64_t strideA, int64_t strideW, int64_t strideO, Epilogue ep) {
  __shared__ __align__(16) float As[2][BK][BMP];
  __shared__ __align__(16) float Bs[2][BK][BNP];
  const int tid = threadIdx.x;
  const int64_t m0 = (int64_t)blockIdx.x * BM, n0 = (int64_t)blockIdx.y * BN;
  const int64_t bz = blockIdx.z;
  ALoader a = al;
  a.shift(bz * strideA);
  const T* Wb = Wg + bz * strideW;
  TO* ob = out + bz * strideO;

  // global->smem mapping: A tile 128 x 16 = 256 threads x 8;  W tile 64 x 16 = 128 threads x 8
  const int a_row = tid >> 1, a_k = (tid & 1) * 8;
  const int w_row = (tid & 127) >> 1, w_k = (tid & 1) * 8;
  const bool w_active = tid < 128;
  const int ty = tid >> 4, tx = tid & 15;   // compute mapping: rows ty*8.., cols tx*4..

  float acc[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  float ra[8], rw[8];
  const int64_t nk = (K + BK - 1) / BK;
  a.load8(m0 + a_row, a_k, ra);
  if (w_active) load_w8(Wb, ldw, N, K, wvec, n0 + w_row, w_k, rw);
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    As[0][a_k + e][a_row] = ra[e];
    if (w_active) Bs[0][w_k + e][w_row] = rw[e];
  }
  __syncthreads();

  for (int64_t kb = 0; kb < nk; ++kb) {
    const int cur = (int)(kb & 1);
    if (kb + 1 < nk) {
      a.load8(m0 + a_row, (kb + 1) * BK + a_k, ra);
      if (w_active) load_w8(Wb, ldw, N, K, wvec, n0 + w_row, (kb + 1) * BK + w_k, rw);
    }
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float4 a0 = *reinterpret_cast<const float4*>(&As[cur][k][ty * 8]);
      float4 a1 = *reinterpret_cast<const float4*>(&As[cur][k][ty * 8 + 4]);
      float4 b0 = *reinterpret_cast<const float4*>(&Bs[cur][k][tx * 4]);
      float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      float bv[4] = {b0.x, b0.y, b0.z, b0.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    if (kb + 1 < nk) {
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        As[cur ^ 1][a_k + e][a_row] = ra[e];
        if (w_active) Bs[cur ^ 1][w_k + e][w_row] = rw[e];
      }
    }
    __syncthreads();
  }

  // epilogue: alpha * acc + bias[n] + rowbias[m / rpg, n] + residual[m, n]
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int64_t m = m0 + ty * 8 + i;
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int64_t n = n0 + tx * 4 + j;
      if (n >= N) continue;
      float v = acc[i][j] * ep.alpha;
      if (ep.flags & FYC_EPI_BIAS) v += ep.bias[n];
      if (ep.flags & FYC_EPI_ROWBIAS) v += ep.rowbias[(m / ep.rows_per_group) * ep.ldrb + n];
      if (ep.flags & FYC_EPI_RESIDUAL) v += to_f(reinterpret_cast<const TO*>(ep.residual)[bz * strideO + m * ep.ldr + n]);
      ob[m * ep.ldo + n] = from_f<TO>(v);
    }
  }
}

template <typename T> struct PlainAS : PlainA<T> { __device__ __forceinline__ void shift(int64_t off) { this->A += off; } };
template <typename T> struct ConvAS : ConvA<T> { __device__ __forceinline__ void shift(int64_t) {} };

template <typename T, typename TO, typename AL>
int32_t launch(const AL& al, const T* W, TO* out, int64_t M, int64_t N, int64_t K, int64_t ldw, int64_t batch,
               int64_t sA, int64_t sW, int64_t sO, const Epilogue& ep, cudaStream_t st) {
  bool wvec = (K % 8 == 0) && (ldw % 8 == 0) && (((uintptr_t)W) % 32 == 0) && (sW % 8 == 0);
  dim3 grid((unsigned)ceil_div64(M, BM), (unsigned)ceil_div64(N, BN), (unsigned)batch);
  FYC_CHECK(grid.y < 65536 && grid.z < 65536, "gemm_simt: grid too large");
  gemm_simt_kernel<T, TO, AL><<<grid, NT, 0, st>>>(al, W, out, M, N, K, ldw, wvec, sA, sW, sO, ep);
  FYC_LAUNCH_CHECK();
  return FYC_OK;
}

}  // namespace

int32_t fyc_gemm_simt(const fyc_gemm_args* g, cudaStream_t st) {
  Epilogue ep{g->bias, g->residual, g->rowbias, g->ldo, g->ldr, g->rows_per_group > 0 ? g->rows_per_group : 1, g->alpha, g->epilogue, g->N};
  FYC_CHECK(!(g->epilogue & FYC_EPI_GEGLU), "gemm_simt: GEGLU epilogue is a separate kernel on this path (fyc_geglu)");
  const bool f32out = (g->epilogue & FYC_EPI_OUT_F32) != 0;
  if (g->dtype == FYC_F32) {
    PlainAS<float> al; al.A = (const float*)g->A; al.lda = g->lda; al.M = g->M; al.K = g->K;
    al.vec = (g->K % 8 == 0) && (g->lda % 8 == 0) && (((uintptr_t)g->A) % 32 == 0) && (g->strideA % 8 == 0);
    return launch<float, float>(al, (const float*)g->W, (float*)g->out, g->M, g->N, g->K, g->ldw, g->batch, g->strideA, g->strideW, g->strideO, ep, st);
  } else if (fyc_is_16bit(g->dtype)) {
    FYC_DISPATCH16(g->dtype, {
      PlainAS<T> al; al.A = (const T*)g->A; al.lda = g->lda; al.M = g->M; al.K = g->K;
      al.vec = (g->K % 8 == 0) && (g->lda % 8 == 0) && (((uintptr_t)g->A) % 16 == 0) && (g->strideA % 8 == 0);
      if (f32out) return launch<T, float>(al, (const T*)g->W, (float*)g->out, g->M, g->N, g->K, g->ldw, g->batch, g->strideA, g->strideW, g->strideO, ep, st);
      return launch<T, T>(al, (const T*)g->W, (T*)g->out, g->M, g->N, g->K, g->ldw, g->batch, g->strideA, g->strideW, g->strideO, ep, st);
    })
  }
  FYC_CHECK(false, "gemm: unknown dtype %d", g->dtype);
}

int32_t fyc_conv3x3_simt(const fyc_conv3x3_args* c, cudaStream_t st) {
  const int up = c->upsample, s = c->stride;
  const int pad = c->pad_mode == 1 ? 0 : 1;       // pad_mode 1: the single padding row / column is on the bottom / right
  const int64_t Ho = (c->H * up + 2 - 3) / s + 1, Wo = (c->W * up + 2 - 3) / s + 1;   // = H / 2 for stride 2 in both modes (even H)
  const int64_t M = c->NB * Ho * Wo, K = 9 * c->Cin, N = c->Cout;
  Epilogue ep{c->bias, c->residual, c->rowbias, N, N, (c->images_per_group > 0 ? c->images_per_group : 1) * Ho * Wo, 1.0f, c->epilogue,
              c->ld_rowbias > 0 ? c->ld_rowbias : N};
  const bool f32out = (c->epilogue & FYC_EPI_OUT_F32) != 0;
  if (c->dtype == FYC_F32) {
    ConvAS<float> al; al.x = (const float*)c->x; al.NB = c->NB; al.H = c->H; al.W = c->W; al.Cin = c->Cin; al.Ho = Ho; al.Wo = Wo;
    al.M = M; al.K = K; al.stride = s; al.up = up; al.pad = pad; al.vec = (c->Cin % 8 == 0) && (((uintptr_t)c->x) % 32 == 0);
    return launch<float, float>(al, (const float*)c->w, (float*)c->out, M, N, K, K, 1, 0, 0, 0, ep, st);
  } else if (fyc_is_16bit(c->dtype)) {
    FYC_DISPATCH16(c->dtype, {
      ConvAS<T> al; al.x = (const T*)c->x; al.NB = c->NB; al.H = c->H; al.W = c->W; al.Cin = c->Cin; al.Ho = Ho; al.Wo = Wo;
      al.M = M; al.K = K; al.stride = s; al.up = up; al.pad = pad; al.vec = (c->Cin % 8 == 0) && (((uintptr_t)c->x) % 16 == 0);
      if (f32out) return launch<T, float>(al, (const T*)c->w, (float*)c->out, M, N, K, K, 1, 0, 0, 0, ep, st);
      return launch<T, T>(al, (const T*)c->w, (T*)c->out, M, N, K, K, 1, 0, 0, 0, ep, st);
    })
  }
  FYC_CHECK(false, "conv3x3: unknown dtype %d", c->dtype);
}
