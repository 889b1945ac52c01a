// CUDA-core attention kernels (fp32 math, online softmax, score matrix never materialised):
//   * attention_simt_kernel: generic multi-head attention, any Lq/Lk, D <= 256 - the strict-fp32 parity path for
//     attn1/attn2/IP, and the fallback for head dims the tensor-core kernel does not instantiate;
//   * temporal_attention_kernel: self-attention over the frame axis (F <= 32 keys), one warp per
//     (clip, pixel, head); q/k/v are read strided along F straight out of the fused qkv activation, so the
//     reference's two '(b f) d c <-> (b d) f c' transposing copies disappear.  Pure HBM-bound work.
#include "common.cuh"

namespace {

// ---------------------------------------------------------------------------------------------------------
// generic: block = 4 warps; each warp owns 4 query rows; K/V streamed through smem in chunks of 32 keys.
constexpr int QW = 4;        // queries per warp
constexpr int NW = 4;        // warps per block
constexpr int KC = 32;       // keys per chunk

template <typename T, int DI>   // DI = ceil(D / 32) upper bound
__global__ void __launch_bounds__(NW * 32) attention_simt_kernel(fyc_attention_args a) {
  extern __shared__ __align__(16) float smem[];
  const int D = (int)a.D, DP = D + 4;
  float* ks = smem;                       // [KC][DP]
  float* vs = ks + KC * DP;               // [KC][DP]
  float* qs = vs + KC * DP;               // [NW*QW][D]
  float* ps = qs + NW * QW * D;           // [NW][KC][QW]
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int64_t n = blockIdx.z, h = blockIdx.y;
  const int64_t q0 = (int64_t)blockIdx.x * (NW * QW);
  const T* qg = (const T*)a.q + n * a.bsq + h * D;
  const int64_t nk = n / a.kv_batch_div;
  const T* kg = (const T*)a.k + nk * a.bsk + h * D;
  const T* vg = (const T*)a.v + nk * a.bsv + h * D;

  for (int i = tid; i < NW * QW * D; i += NW * 32) {
    int r = i / D, d = i % D;
    int64_t qi = q0 + r;
    qs[i] = qi < a.Lq ? to_f(qg[qi * a.ldq + d]) * a.scale : 0.f;
  }
  float m[QW], l[QW], o[QW][DI];
#pragma unroll
  for (int qi = 0; qi < QW; ++qi) {
    m[qi] = -INFINITY; l[qi] = 0.f;
#pragma unroll
    for (int i = 0; i < DI; ++i) o[qi][i] = 0.f;
  }
  const float* qw = qs + w * QW * D;
  float* pw = ps + w * KC * QW;

  for (int64_t j0 = 0; j0 < a.Lk; j0 += KC) {
    __syncthreads();
    for (int i = tid; i < KC * D; i += NW * 32) {
      int r = i / D, d = i % D;
      int64_t j = j0 + r;
      ks[r * DP + d] = j < a.Lk ? to_f(kg[j * a.ldk + d]) : 0.f;
      vs[r * DP + d] = j < a.Lk ? to_f(vg[j * a.ldv + d]) : 0.f;
    }
    __syncthreads();
    // S = q . k for key `lane`
    float s[QW];
#pragma unroll
    for (int qi = 0; qi < QW; ++qi) s[qi] = 0.f;
    const float* kr = ks + lane * DP;
    for (int d = 0; d < D; d += 4) {
      float4 kv = *reinterpret_cast<const float4*>(kr + d);
#pragma unroll
      for (int qi = 0; qi < QW; ++qi) {
        float4 qv = *reinterpret_cast<const float4*>(qw + qi * D + d);
        s[qi] = fmaf(qv.x, kv.x, fmaf(qv.y, kv.y, fmaf(qv.z, kv.z, fmaf(qv.w, kv.w, s[qi]))));
      }
    }
    const bool valid = j0 + lane < a.Lk;
    float corr[QW];
#pragma unroll
    for (int qi = 0; qi < QW; ++qi) {
      float sv = valid ? s[qi] : -INFINITY;
      float mn = fmaxf(m[qi], warp_max(sv));
      float p = valid ? expf(sv - mn) : 0.f;
      corr[qi] = (m[qi] == -INFINITY) ? 0.f : expf(m[qi] - mn);
      l[qi] = l[qi] * corr[qi] + warp_sum(p);
      m[qi] = mn;
      pw[lane * QW + qi] = p;
    }
    __syncwarp();
    // O = O * corr + P V ; lane owns columns d = lane + 32 i
#pragma unroll
    for (int qi = 0; qi < QW; ++qi)
#pragma unroll
      for (int i = 0; i < DI; ++i) o[qi][i] *= corr[qi];
    for (int j = 0; j < KC; ++j) {
      float4 pj = *reinterpret_cast<const float4*>(pw + j * QW);
      float pv[QW] = {pj.x, pj.y, pj.z, pj.w};
#pragma unroll
      for (int i = 0; i < DI; ++i) {
        int d = lane + 32 * i;
        float vv = d < D ? vs[j * DP + d] : 0.f;
#pragma unroll
        for (int qi = 0; qi < QW; ++qi) o[qi][i] = fmaf(pv[qi], vv, o[qi][i]);
      }
    }
    __syncwarp();
  }
  T* og = (T*)a.out + n * a.bso + h * D;
#pragma unroll
  for (int qi = 0; qi < QW; ++qi) {
    int64_t q = q0 + w * QW + qi;
    if (q >= a.Lq) continue;
    float inv = a.out_alpha / l[qi];
#pragma unroll
    for (int i = 0; i < DI; ++i) {
      int d = lane + 32 * i;
      if (d < D) {
        float r = o[qi][i] * inv;
        T* dst = og + q * a.ldo + d;
        if (a.accumulate) r += to_f(*dst);
        *dst = from_f<T>(r);
      }
    }
  }
}

template <typename T, int DI>
int32_t launch_attn(const fyc_attention_args* a, cudaStream_t st) {
  const int D = (int)a->D;
  size_t smem = (size_t)(2 * KC * (D + 4) + NW * QW * D + NW * KC * QW) * sizeof(float);
  auto kern = attention_simt_kernel<T, DI>;
  FYC_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  dim3 grid((unsigned)ceil_div64(a->Lq, NW * QW), (unsigned)a->heads, (unsigned)a->batch);
  kern<<<grid, NW * 32, smem, st>>>(*a);
  FYC_LAUNCH_CHECK();
  return FYC_OK;
}

// ---------------------------------------------------------------------------------------------------------
// temporal: one warp per (b, pixel, head).  Lane = (query frame i, d-split s): FP = pow2 >= F, S = 32 / FP.
template <typename T, int FP>
__global__ void __launch_bounds__(256) temporal_attention_kernel(const T* __restrict__ qkv, T* __restrict__ out, int64_t B,
                                                                 int F, int64_t HW, int heads, int D, float scale) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  constexpr int S = 32 / FP;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int C = heads * D;
  // per-warp staging: q, k, v as [F][D] in T
  T* base = reinterpret_cast<T*>(smem_raw) + (size_t)w * 3 * F * D;
  T* qs = base; T* ks = base + F * D; T* vs = base + 2 * F * D;
  const int64_t item = (int64_t)blockIdx.x * (blockDim.x >> 5) + w;   // consecutive warps = consecutive (pixel, head) items
  const int64_t total = B * HW * heads;
  if (item >= total) return;
  const int h = (int)(item % heads);
  const int64_t bp = item / heads;
  const int64_t p = bp % HW, b = bp / HW;
  const int64_t row_stride = HW * 3 * C;                     // frame stride in the qkv tensor
  const T* src = qkv + (b * F * HW + p) * 3 * C + h * D;
  // cooperative load: 3 segments x F rows x D elements, 4-element (8 B bf16 / fp16, 16 B fp32) vectors
  const int dv = D / 4;
  for (int i = lane; i < 3 * F * dv; i += 32) {
    int seg = i / (F * dv);
    int r = (i / dv) % F;
    int c4 = (i % dv) * 4;
    float f[4];
    Vec4<T>::load(src + (int64_t)r * row_stride + seg * C + c4, f);
    Vec4<T>::store(base + (seg * F + r) * D + c4, f);
  }
  __syncwarp();
  const int qi = lane % FP, sp = lane / FP;
  float s[FP];
#pragma unroll
  for (int j = 0; j < FP; ++j) s[j] = 0.f;
  if (qi < F) {
    for (int c = sp; c < dv; c += S) {
      float qv[4];
      Vec4<T>::load(qs + qi * D + c * 4, qv);
#pragma unroll
      for (int j = 0; j < FP; ++j) {
        if (j < F) {
          float kv[4];
          Vec4<T>::load(ks + j * D + c * 4, kv);
          s[j] = fmaf(qv[0], kv[0], fmaf(qv[1], kv[1], fmaf(qv[2], kv[2], fmaf(qv[3], kv[3], s[j]))));
        }
      }
    }
  }
  // combine the S partial dot products (lanes qi + FP * sp)
#pragma unroll
  for (int j = 0; j < FP; ++j) {
#pragma unroll
    for (int o = FP; o < 32; o <<= 1) s[j] += __shfl_xor_sync(0xffffffffu, s[j], o);
  }
  float mx = -INFINITY;
#pragma unroll
  for (int j = 0; j < FP; ++j) if (j < F) { s[j] *= scale; mx = fmaxf(mx, s[j]); }
  float sum = 0.f;
#pragma unroll
  for (int j = 0; j < FP; ++j) { s[j] = (j < F) ? expf(s[j] - mx) : 0.f; sum += s[j]; }
  const float inv = 1.0f / sum;
  if (qi < F) {
    T* dst = out + ((b * F + qi) * HW + p) * C + h * D;
    for (int c = sp; c < dv; c += S) {
      float o4[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int j = 0; j < FP; ++j) {
        if (j < F) {
          float vv[4];
          Vec4<T>::load(vs + j * D + c * 4, vv);
#pragma unroll
          for (int e = 0; e < 4; ++e) o4[e] = fmaf(s[j], vv[e], o4[e]);
        }
      }
#pragma unroll
      for (int e = 0; e < 4; ++e) o4[e] *= inv;
      Vec4<T>::store(dst + c * 4, o4);
    }
  }
}

template <typename T, int FP>
int32_t launch_temporal(const T* qkv, T* out, int64_t B, int F, int64_t HW, int heads, int D, float scale, cudaStream_t st) {
  const size_t per_warp = (size_t)3 * F * D * sizeof(T);
  int wpb = (int)((96 * 1024) / per_warp);          // <= 96 KB per CTA keeps >= 2 CTAs resident per SM
  if (wpb > 8) wpb = 8;
  FYC_CHECK(wpb >= 1, "temporal_attention: F*D too large for shared memory (%zu B per warp)", per_warp);
  const size_t smem = per_warp * wpb;
  auto kern = temporal_attention_kernel<T, FP>;
  FYC_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int64_t items = B * HW * heads;
  kern<<<(unsigned)ceil_div64(items, wpb), wpb * 32, smem, st>>>(qkv, out, B, F, HW, heads, D, scale);
  FYC_LAUNCH_CHECK();
  return FYC_OK;
}

}  // namespace

int32_t fyc_attention_simt(const fyc_attention_args* a, cudaStream_t st) {
  FYC_CHECK(a->D % 4 == 0 && a->D <= 256, "attention(simt): head dim %lld must be a multiple of 4 and <= 256", (long long)a->D);
  FYC_CHECK(a->heads < 65536 && a->batch < 65536, "attention(simt): grid too large");
  const int di = (int)((a->D + 31) / 32);
#define FYC_ATTN_DI(T)                                                   \
  if (di <= 2) return launch_attn<T, 2>(a, st);                          \
  if (di <= 3) return launch_attn<T, 3>(a, st);                          \
  if (di <= 5) return launch_attn<T, 5>(a, st);                          \
  return launch_attn<T, 8>(a, st);
  if (a->dtype == FYC_F32) { FYC_ATTN_DI(float) }
  if (a->dtype == FYC_BF16) { FYC_ATTN_DI(bf16) }
  if (a->dtype == FYC_F16) { FYC_ATTN_DI(f16) }
#undef FYC_ATTN_DI
  FYC_CHECK(false, "attention: unknown dtype %d", a->dtype);
}

bool fyc_temporal_mma_eligible(int64_t F, int64_t D, int64_t heads, int32_t dtype, const void* qkv, const void* out);
int32_t fyc_temporal_attention_mma(const void* qkv, void* out, int64_t B, int64_t F, int64_t HW, int64_t heads, int64_t D, float scale,
                                   int32_t dtype, cudaStream_t st);

extern "C" int32_t fyc_temporal_attention(const void* qkv, void* out, int64_t B, int64_t F, int64_t HW, int64_t heads,
                                          int64_t D, float scale, int32_t dtype, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  FYC_CHECK(F >= 1 && F <= 32, "temporal_attention: F=%lld must be in [1, 32]", (long long)F);
  FYC_CHECK(D % 4 == 0, "temporal_attention: head dim %lld must be a multiple of 4", (long long)D);
  if (fyc_temporal_mma_eligible(F, D, heads, dtype, qkv, out)) return fyc_temporal_attention_mma(qkv, out, B, F, HW, heads, D, scale, dtype, st);
#define FYC_TA(T)                                                                                             \
  if (F <= 4) return launch_temporal<T, 4>((const T*)qkv, (T*)out, B, (int)F, HW, (int)heads, (int)D, scale, st);   \
  if (F <= 8) return launch_temporal<T, 8>((const T*)qkv, (T*)out, B, (int)F, HW, (int)heads, (int)D, scale, st);   \
  if (F <= 16) return launch_temporal<T, 16>((const T*)qkv, (T*)out, B, (int)F, HW, (int)heads, (int)D, scale, st); \
  return launch_temporal<T, 32>((const T*)qkv, (T*)out, B, (int)F, HW, (int)heads, (int)D, scale, st);
  if (dtype == FYC_F32) { FYC_TA(float) }
  if (dtype == FYC_BF16) { FYC_TA(bf16) }
  if (dtype == FYC_F16) { FYC_TA(f16) }
#undef FYC_TA
  FYC_CHECK(false, "temporal_attention: unknown dtype %d", dtype);
}
