// Temporal self-attention on tensor cores (bf16 or fp16 storage): one warp per (clip, pixel, head) item.
// The F x F problem (F <= 32 frames) is tiny - 16 x 16 x D per head - so the CUDA-core version was instruction-bound
// (issue-bound at a small fraction of HBM bandwidth).  Here the warp stages q, k, v (F rows, strided by
// H*W*3C in the fused qkv activation) in shared memory with cp.async and runs S = Q K^T and O = P V as a handful of
// mma.sync m16n8k16 instructions (11 for F = 16, D = 40), with the softmax on the accumulator fragment.
#include "common.cuh"

namespace {

// FP = frames padded to 16 or 32; DP = head dim padded to a multiple of 16; T = the 16-bit storage type (bf16 | f16)
template <int FP, int DP, typename T>
__global__ void __launch_bounds__(256) temporal_attention_mma_kernel(const T* __restrict__ qkv, T* __restrict__ out, int64_t B,
                                                                     int F, int64_t HW, int heads, int D, float scale_log2e) {
  constexpr int LDS = DP + 8;
  constexpr int MT = FP / 16;          // m-tiles (query frames)
  constexpr int NT = FP / 8;           // 8-key n-tiles of S
  constexpr int KS = DP / 16;          // k-steps of QK^T
  constexpr int KK = FP / 16;          // k-steps of PV
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  T* base = reinterpret_cast<T*>(smem_raw) + (size_t)w * 3 * FP * LDS;
  T* sq = base; T* sk = base + FP * LDS; T* sv = base + 2 * FP * LDS;
  const int64_t item = (int64_t)blockIdx.x * (blockDim.x >> 5) + w;
  if (item >= B * HW * heads) return;
  const int h = (int)(item % heads);
  const int64_t bp = item / heads;
  const int64_t p = bp % HW, b = bp / HW;
  const int C = heads * D;
  const int64_t row_stride = HW * 3 * (int64_t)C;
  const T* src = qkv + (b * F * HW + p) * 3 * C + h * D;
  // zero the padding (rows >= F, cols >= D) once, then async-copy the valid region
  const int ch = DP / 8, chv = D / 8;
  for (int i = lane; i < 3 * FP * ch; i += 32) {
    int seg = i / (FP * ch), r = (i / ch) % FP, c = (i % ch) * 8;
    T* dst = base + (seg * FP + r) * LDS + c;
    if (r < F && (i % ch) < chv) cp_async16(dst, src + (int64_t)r * row_stride + seg * C + c);
    else *reinterpret_cast<uint4*>(dst) = make_uint4(0, 0, 0, 0);
  }
  cp_async_commit();
  cp_async_wait<0>();
  __syncwarp();
  const int g = lane >> 2, t = lane & 3, mi = lane >> 3;
#pragma unroll
  for (int mt = 0; mt < MT; ++mt) {
    float s[NT][4];
#pragma unroll
    for (int j = 0; j < NT; ++j) { s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f; }
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
      uint32_t a[4];
      ldmatrix_x4(a, sq + (mt * 16 + (lane & 15)) * LDS + ks * 16 + (lane >> 4) * 8);
#pragma unroll
      for (int jp = 0; jp < NT / 2; ++jp) {
        uint32_t bb[4];
        ldmatrix_x4(bb, sk + (jp * 16 + (lane & 7) + (mi >> 1) * 8) * LDS + ks * 16 + (mi & 1) * 8);
        mma16816<T>(s[2 * jp], a, bb[0], bb[1]);
        mma16816<T>(s[2 * jp + 1], a, bb[2], bb[3]);
      }
    }
    float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
    for (int j = 0; j < NT; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        bool ok = 8 * j + 2 * t + e < F;
        s[j][e] = ok ? s[j][e] * scale_log2e : -INFINITY;
        s[j][2 + e] = ok ? s[j][2 + e] * scale_log2e : -INFINITY;
        mx0 = fmaxf(mx0, s[j][e]); mx1 = fmaxf(mx1, s[j][2 + e]);
      }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    float l0 = 0.f, l1 = 0.f;
    uint32_t pf[KK][4];
#pragma unroll
    for (int j = 0; j < NT; ++j) {
      float p0 = ex2_approx(s[j][0] - mx0), p1 = ex2_approx(s[j][1] - mx0), p2 = ex2_approx(s[j][2] - mx1), p3 = ex2_approx(s[j][3] - mx1);
      l0 += p0 + p1; l1 += p2 + p3;
      pf[j >> 1][(j & 1) * 2] = pack_u32<T>(p0, p1);
      pf[j >> 1][(j & 1) * 2 + 1] = pack_u32<T>(p2, p3);
    }
    l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
    l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
    const float i0 = 1.0f / l0, i1 = 1.0f / l1;
    const int f0 = mt * 16 + g, f1 = f0 + 8;
    T* o0 = out + ((b * F + f0) * HW + p) * C + h * D;
    T* o1 = out + ((b * F + f1) * HW + p) * C + h * D;
#pragma unroll
    for (int np = 0; np < DP / 16; ++np) {
      float o[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
#pragma unroll
      for (int kk = 0; kk < KK; ++kk) {
        uint32_t bb[4];
        ldmatrix_x4_trans(bb, sv + (kk * 16 + (lane & 7) + (mi & 1) * 8) * LDS + np * 16 + (mi >> 1) * 8);
        mma16816<T>(o[0], pf[kk], bb[0], bb[1]);
        mma16816<T>(o[1], pf[kk], bb[2], bb[3]);
      }
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const int col = np * 16 + q * 8 + 2 * t;
        if (col < D) {
          if (f0 < F) *reinterpret_cast<typename Pair16<T>::type*>(o0 + col) = Pair16<T>::pack(o[q][0] * i0, o[q][1] * i0);
          if (f1 < F) *reinterpret_cast<typename Pair16<T>::type*>(o1 + col) = Pair16<T>::pack(o[q][2] * i1, o[q][3] * i1);
        }
      }
    }
  }
}

template <int FP, int DP, typename T>
int32_t launch(const T* qkv, T* out, int64_t B, int F, int64_t HW, int heads, int D, float scale, cudaStream_t st) {
  const size_t per_warp = (size_t)3 * FP * (DP + 8) * sizeof(T);
  int wpb = (int)((100 * 1024) / per_warp);
  if (wpb > 8) wpb = 8;
  if (wpb < 1) wpb = 1;
  const size_t smem = per_warp * wpb;
  auto kern = temporal_attention_mma_kernel<FP, DP, T>;
  FYC_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int64_t items = B * HW * heads;
  kern<<<(unsigned)ceil_div64(items, wpb), wpb * 32, smem, st>>>(qkv, out, B, F, HW, heads, D, scale * 1.4426950408889634f);
  FYC_LAUNCH_CHECK();
  return FYC_OK;
}

}  // namespace

bool fyc_temporal_mma_eligible(int64_t F, int64_t D, int64_t heads, int32_t dtype, const void* qkv, const void* out) {
  return fyc_is_16bit(dtype) && F >= 1 && F <= 32 && D % 8 == 0 && D <= 160 && (((uintptr_t)qkv) % 16 == 0) && (((uintptr_t)out) % 4 == 0);
}

int32_t fyc_temporal_attention_mma(const void* qkv, void* out, int64_t B, int64_t F, int64_t HW, int64_t heads, int64_t D, float scale,
                                   int32_t dtype, cudaStream_t st) {
#define FYC_TM(FP)                                                                                                       \
  if (D <= 48) return launch<FP, 48, T>((const T*)qkv, (T*)out, B, (int)F, HW, (int)heads, (int)D, scale, st);           \
  if (D <= 80) return launch<FP, 80, T>((const T*)qkv, (T*)out, B, (int)F, HW, (int)heads, (int)D, scale, st);           \
  return launch<FP, 160, T>((const T*)qkv, (T*)out, B, (int)F, HW, (int)heads, (int)D, scale, st);
  FYC_DISPATCH16(dtype, if (F <= 16) { FYC_TM(16) } FYC_TM(32))
#undef FYC_TM
  return FYC_OK;
}
