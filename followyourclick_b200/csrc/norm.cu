// GroupNorm (cross-frame or per-frame statistics) and LayerNorm.  Both are HBM-bound: one read for the
// statistics, one read + one write for the apply; statistics are accumulated in fp32 per thread, combined in
// fp64 across CTAs so that E[x^2]-E[x]^2 does not cancel.
#include <stdlib.h>

#include <type_traits>

#include "common.cuh"

// FYC_ZIGZAG (default 1): the norm kernels walk their input back to front.  Activations at the 64x64 level are 84 MB, the L2 is 50
// MB: a consumer that starts where its producer stopped finds the most recently written half still cached, one that starts at the
// front finds nothing.  GEMM / conv / attention write front to back, so the norms between them run back to front.
static int fyc_zigzag() {
  const char* e = getenv("FYC_ZIGZAG");
  return (e && e[0] == '0') ? 0 : 1;
}

// Waves of resident statistics CTAs (4 per SM) the GroupNorm statistics pass is cut into (A/B switch FYC_GN_WAVES=1|2|3, default 2).  More
// waves mean shorter streams per CTA (at 3 waves: 13 rows per thread at level 0 - the stream ends before the 8-deep load pipeline pays, and
// every CTA has its shared-memory reduction and partial write).
static int fyc_gn_waves() {
  static int w = -1;
  if (w < 0) {
    const char* e = getenv("FYC_GN_WAVES");
    w = (e && e[0] >= '1' && e[0] <= '3') ? e[0] - '0' : 2;
  }
  return w;
}

namespace {
// one 32-bit word holding two 16-bit T (bf16 | f16) <-> two floats (element 0 in the low half); a 16-byte vector of eight <-> float[8]
template <typename T> __device__ __forceinline__ void u2_to_f2(uint32_t w, float& lo, float& hi) {
  if constexpr (std::is_same<T, bf16>::value) {
    lo = __uint_as_float(w << 16); hi = __uint_as_float(w & 0xffff0000u);
  } else {
    const float2 f = Pair16<T>::unpack(*reinterpret_cast<const typename Pair16<T>::type*>(&w));
    lo = f.x; hi = f.y;
  }
}
template <typename T> __device__ __forceinline__ void u8_to_f(const uint4& raw, float* f) {
  u2_to_f2<T>(raw.x, f[0], f[1]); u2_to_f2<T>(raw.y, f[2], f[3]); u2_to_f2<T>(raw.z, f[4], f[5]); u2_to_f2<T>(raw.w, f[6], f[7]);
}
template <typename T> __device__ __forceinline__ uint4 f_to_u8(const float* f) {
  return make_uint4(pack_u32<T>(f[0], f[1]), pack_u32<T>(f[2], f[3]), pack_u32<T>(f[4], f[5]), pack_u32<T>(f[6], f[7]));
}
// four fp32 parameters with one 16-byte load (scalar parameter loads saturated the LSU queue: lg_throttle)
__device__ __forceinline__ void ldg4(const float* p, float* f) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(p));
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w;
}
}  // namespace

// ---------------------------------------------------------------------------------------------------------
// stats: x viewed as [NB, R, C]; grid (chunks, NB); each CTA reduces rows [r0, r1) for all channels and writes ONE
// partial (sum, sumsq) per group.  No atomics anywhere: the per-thread channel sums are combined through shared
// memory in a fixed order and the per-CTA partials are summed in chunk order by gn_finalize_kernel, so the
// statistics (and therefore the whole engine) are bit-reproducible run to run.
// Two-source form (x2 != nullptr): the normalised tensor is the channel concatenation [x (C1 channels) | x2 (C - C1 channels)] of two
// tensors that are never concatenated in memory - the skip connections of the up blocks (torch.cat at unet_blocks.py:763,885 followed
// by ResnetBlock3D.norm1).  A thread's channel vector lies wholly in one source (C1 % V == 0).
template <typename T, int V>
__global__ void __launch_bounds__(256, 4) gn_stats_kernel(const T* __restrict__ x, float2* __restrict__ partials, int64_t R,
                                                       int C, int G, int64_t rows_per_cta, int rev, const T* __restrict__ x2, int C1) {
  extern __shared__ float s_ch[];   // [RY][C][2]
  const int cpg = C / G;
  const int cvn = C / V;
  const int TX = cvn < 256 ? cvn : 256;
  const int RY = 256 / TX;
  const int tx = threadIdx.x % TX, ry = threadIdx.x / TX;
  // rev: walk the tensor back to front (zig-zag against the producer, which wrote it front to back: its tail is what L2 still holds)
  const int64_t nb = rev ? gridDim.y - 1 - blockIdx.y : blockIdx.y;
  const int64_t bx = rev ? gridDim.x - 1 - blockIdx.x : blockIdx.x;
  const int64_t r0 = bx * rows_per_cta;
  const int64_t r1 = (r0 + rows_per_cta < R) ? r0 + rows_per_cta : R;
  if (ry < RY) {
    for (int cv = tx; cv < cvn; cv += TX) {
      // row pointer and row stride of this channel vector's source; below `base + r * C + cv * V` addresses row r
      const bool second = x2 != nullptr && cv * V >= C1;
      const int ldx = x2 == nullptr ? C : (second ? C - C1 : C1);
      const T* base0 = second ? x2 + nb * R * ldx + (cv * V - C1) : x + nb * R * ldx + cv * V;
      float s[V], q[V];
#pragma unroll
      for (int e = 0; e < V; ++e) { s[e] = 0.f; q[e] = 0.f; }
      int64_t r = r0 + ry;
      if constexpr (sizeof(T) == 2 && V == 8) {
        // 16-bit: 8 independent 16-byte loads in flight per thread, kept packed until they are summed (the 4-deep version was
        // latency-bound: long-scoreboard stalls)
        for (; r + 7 * RY < r1; r += 8 * RY) {
          uint4 raw[8];
#pragma unroll
          for (int u = 0; u < 8; ++u) raw[u] = __ldg(reinterpret_cast<const uint4*>(base0 + (r + (int64_t)u * RY) * ldx));
#pragma unroll
          for (int u = 0; u < 8; ++u) {
            float f[8];
            u8_to_f<T>(raw[u], f);
#pragma unroll
            for (int e = 0; e < 8; ++e) { s[e] = __fadd_rn(s[e], f[e]); q[e] = __fmaf_rn(f[e], f[e], q[e]); }
          }
        }
      }
      for (; r + 3 * RY < r1; r += 4 * RY) {      // 4 independent 16-byte loads in flight per thread
        float f[4][8];
#pragma unroll
        for (int u = 0; u < 4; ++u) load_vec<T, V>(base0 + (r + (int64_t)u * RY) * ldx, f[u]);
#pragma unroll
        for (int u = 0; u < 4; ++u)
#pragma unroll
          for (int e = 0; e < V; ++e) { s[e] += f[u][e]; q[e] = fmaf(f[u][e], f[u][e], q[e]); }
      }
      for (; r < r1; r += RY) {
        float f[8];
        load_vec<T, V>(base0 + r * ldx, f);
#pragma unroll
        for (int e = 0; e < V; ++e) { s[e] += f[e]; q[e] = fmaf(f[e], f[e], q[e]); }
      }
#pragma unroll
      for (int e = 0; e < V; ++e) {
        s_ch[((size_t)ry * C + cv * V + e) * 2] = s[e];
        s_ch[((size_t)ry * C + cv * V + e) * 2 + 1] = q[e];
      }
    }
  }
  __syncthreads();
  for (int g = threadIdx.x; g < G; g += 256) {
    float as = 0.f, aq = 0.f;
    for (int y = 0; y < RY; ++y)
      for (int c = g * cpg; c < (g + 1) * cpg; ++c) { as += s_ch[((size_t)y * C + c) * 2]; aq += s_ch[((size_t)y * C + c) * 2 + 1]; }
    partials[((int64_t)nb * gridDim.x + bx) * G + g] = make_float2(as, aq);      // slot = logical chunk: the finalize order is unchanged
  }
}

// finalize: one CTA per (group, nb).  mean/rstd of the group from the chunk partials (fp64, fixed reduction tree), then per channel
// scale = rstd * gamma, shift = beta - mean * scale   (same form as ATen's CPU kernel).  (One CTA per nb walked all chunks x groups
// with 8 warps: 26 us for the cross-frame case NB = 2 - as long as the statistics pass itself.)
__global__ void __launch_bounds__(128) gn_finalize_kernel(const float2* __restrict__ partials, int chunks,
                                                          const float* __restrict__ gamma, const float* __restrict__ beta,
                                                          float* __restrict__ scale, float* __restrict__ shift, int C, int G,
                                                          double count, float eps) {
  __shared__ double s_red[2][4];
  __shared__ float s_stat[2];
  const int g = blockIdx.x;
  const int64_t nb = blockIdx.y;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  double s = 0.0, q = 0.0;
  for (int k = threadIdx.x; k < chunks; k += 128) { const float2 p = partials[(nb * chunks + k) * G + g]; s += (double)p.x; q += (double)p.y; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { s += __shfl_xor_sync(0xffffffffu, s, o); q += __shfl_xor_sync(0xffffffffu, q, o); }
  if (lane == 0) { s_red[0][wid] = s; s_red[1][wid] = q; }
  __syncthreads();
  if (threadIdx.x == 0) {
    const double st = (s_red[0][0] + s_red[0][1]) + (s_red[0][2] + s_red[0][3]);
    const double qt = (s_red[1][0] + s_red[1][1]) + (s_red[1][2] + s_red[1][3]);
    const double mean = st / count;
    double var = qt / count - mean * mean;
    if (var < 0) var = 0;
    s_stat[0] = (float)mean;
    s_stat[1] = (float)(1.0 / sqrt(var + (double)eps));
  }
  __syncthreads();
  const int cpg = C / G;
  for (int c = g * cpg + threadIdx.x; c < (g + 1) * cpg; c += 128) {
    const float sc = s_stat[1] * gamma[c];
    scale[nb * C + c] = sc;
    shift[nb * C + c] = beta[c] - s_stat[0] * sc;
  }
}

template <typename T, int V, bool SILU>
__global__ void __launch_bounds__(256) gn_apply_kernel(const T* __restrict__ x, const float* __restrict__ scale,
                                                       const float* __restrict__ shift, T* __restrict__ out, int64_t R,
                                                       int C, int64_t total_vec, const T* __restrict__ x2, int C1) {
  const int cvn = C / V;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  constexpr int U = 4;     // vectors in flight per thread
  // (channel vector, row) of vector i0 and of one grid stride, so that the loop advances them by addition: the 64-bit
  // div / mod per vector of the first version cost more issue slots than the loads
  const int64_t i00 = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  int cv = (int)(i00 % cvn);
  int64_t row = i00 / cvn;            // row over all NB images
  const int dcv = (int)(stride % cvn);
  const int64_t drow = stride / cvn;
  for (int64_t i0 = i00; i0 < total_vec; i0 += stride * U) {
    float f[U][8];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t i = i0 + u * stride;
      if (i < total_vec) {
        const T* src = x + i * V;
        if (x2 != nullptr) {                      // two-source form: (row, channel vector) of vector i -> its source tensor
          const int64_t rw = i / cvn; const int c = (int)(i - rw * cvn) * V;
          src = c < C1 ? x + rw * C1 + c : x2 + rw * (C - C1) + (c - C1);
        }
        load_vec<T, V>(src, f[u]);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t i = i0 + u * stride;
      if (i < total_vec) {
        const int64_t nb = (int64_t)((uint32_t)row / (uint32_t)R);      // NB * R < 2^31 (checked by the caller)
        const float* sc = scale + nb * C + cv * V;
        const float* sh = shift + nb * C + cv * V;
        float scv[V], shv[V];
        if constexpr (V >= 4) {
#pragma unroll
          for (int e = 0; e < V; e += 4) { ldg4(sc + e, scv + e); ldg4(sh + e, shv + e); }
        } else {
          scv[0] = __ldg(sc); shv[0] = __ldg(sh);
        }
#pragma unroll
        for (int e = 0; e < V; ++e) {
          float y = fmaf(f[u][e], scv[e], shv[e]);
          f[u][e] = SILU ? (sizeof(T) == 2 ? silu_fast(y) : silu_f(y)) : y;
        }
        store_vec<T, V>(out + i * V, f[u]);
      }
      cv += dcv; row += drow;
      if (cv >= cvn) { cv -= cvn; ++row; }
    }
  }
}

// 16-bit apply, second form: a thread owns ONE 8-channel vector (scale / shift live in 16 registers, loaded once) and walks rows,
// U rows in flight.  The grid-stride form above re-derived (image, channel) and re-loaded four
// parameter vectors for every 16 bytes of data: 160 issued instructions per vector, 51 us for an 84 MB tensor.
// [r2] Row blocks (RY x U consecutive rows) are dealt to the CTAs round-robin - neighbouring CTAs stream neighbouring memory at the same
// time instead of 1184 far-apart private chunks - and the NEXT block's loads are issued before the current block's SiLU math (register
// double buffer), so a CTA always has 2 x U x 16 bytes per thread in flight.  SiLU = y (0.5 + 0.5 tanh(y / 2)): one MUFU.TANH per
// element instead of EX2 + RCP (the apply kernel spent a third of its issue slots and all of its MUFU slots there).
__device__ __forceinline__ float tanh_fast(float x) { float y; asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }

template <typename T, bool SILU>
__global__ void __launch_bounds__(256, 3) gn_apply_rows_kernel(const T* __restrict__ x, const float* __restrict__ scale,
                                                            const float* __restrict__ shift, T* __restrict__ out, int64_t R,
                                                            int C, const T* __restrict__ x2, int C1) {
  constexpr int U = 4;
  const int cvn = C / 8;
  const int TX = cvn < 256 ? cvn : 256;
  const int RY = 256 / TX;
  const int tx = threadIdx.x % TX, ry = threadIdx.x / TX;
  if (ry >= RY) return;
  const int64_t nb = blockIdx.y;
  const int64_t blk_rows = (int64_t)RY * U;                     // rows one CTA iteration covers
  const int64_t nblk = (R + blk_rows - 1) / blk_rows;
  T* ob = out + nb * R * C;
  for (int cv = tx; cv < cvn; cv += TX) {
    const bool second = x2 != nullptr && cv * 8 >= C1;
    const int ldx = x2 == nullptr ? C : (second ? C - C1 : C1);
    const T* xb = second ? x2 + nb * R * ldx + (cv * 8 - C1) : x + nb * R * ldx + cv * 8;     // row r of this channel vector: xb + r * ldx
    float sc[8], sh[8];
    ldg4(scale + nb * C + cv * 8, sc); ldg4(scale + nb * C + cv * 8 + 4, sc + 4);
    ldg4(shift + nb * C + cv * 8, sh); ldg4(shift + nb * C + cv * 8 + 4, sh + 4);
    auto load_blk = [&](int64_t blk, uint4* raw) {
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int64_t rr = blk * blk_rows + (int64_t)u * RY + ry;
        raw[u] = make_uint4(0, 0, 0, 0);
        if (blk < nblk && rr < R) raw[u] = __ldg(reinterpret_cast<const uint4*>(xb + rr * ldx));
      }
    };
    uint4 cur[U], nxt[U];
    int64_t blk = blockIdx.x;
    load_blk(blk, cur);
    for (; blk < nblk; blk += gridDim.x) {
      load_blk(blk + gridDim.x, nxt);                             // next block's rows are in flight during this block's math
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int64_t rr = blk * blk_rows + (int64_t)u * RY + ry;
        if (rr >= R) break;
        const uint32_t w[4] = {cur[u].x, cur[u].y, cur[u].z, cur[u].w};
        uint32_t o[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          float y0, y1;
          u2_to_f2<T>(w[e], y0, y1);
          y0 = __fmaf_rn(y0, sc[2 * e], sh[2 * e]); y1 = __fmaf_rn(y1, sc[2 * e + 1], sh[2 * e + 1]);
          if (SILU) {                       // y * sigmoid(y) = y * (0.5 + 0.5 tanh(y / 2))
            const float h0 = __fmul_rn(y0, 0.5f), h1 = __fmul_rn(y1, 0.5f);
            y0 = __fmul_rn(y0, __fmaf_rn(tanh_fast(h0), 0.5f, 0.5f)); y1 = __fmul_rn(y1, __fmaf_rn(tanh_fast(h1), 0.5f, 0.5f));
          }
          o[e] = pack_u32<T>(y0, y1);
        }
        *reinterpret_cast<uint4*>(ob + rr * C + cv * 8) = make_uint4(o[0], o[1], o[2], o[3]);
      }
#pragma unroll
      for (int u = 0; u < U; ++u) cur[u] = nxt[u];
    }
  }
}

static int64_t gn_max_chunks(int64_t NB) { return ((int64_t)fyc_sm_count() * 12 + NB - 1) / NB + 1; }   // ~3 waves of 4 CTAs per SM
static int64_t gn_partials(int64_t NB, int64_t G) { return (NB * gn_max_chunks(NB) * G + 1) / 2 * 2; }   // even: keeps scale/shift 16-byte aligned

extern "C" size_t fyc_groupnorm_workspace_bytes(int64_t NB, int64_t C, int64_t G) {
  return (size_t)(gn_partials(NB, G) * sizeof(float2) + NB * C * 2 * sizeof(float));
}

template <typename T, int V>
static int32_t groupnorm_impl(const T* x, const float* gamma, const float* beta, T* out, int64_t NB, int64_t R, int C,
                              int G, float eps, int silu, void* ws, cudaStream_t st, const T* x2 = nullptr, int C1 = 0) {
  float2* partials = (float2*)ws;
  float* scale = (float*)(partials + gn_partials(NB, G));
  float* shift = scale + NB * C;
  const int cvn = C / V;
  const int TX = cvn < 256 ? cvn : 256;
  const int RY = 256 / TX;
  int64_t target = ceil_div64((int64_t)fyc_sm_count() * 4 * fyc_gn_waves(), NB);   // CTAs per nb (<= gn_max_chunks(NB) - 1, the workspace bound)
  int64_t rows_per_cta = ceil_div64(R, target);
  if (rows_per_cta < 8 * RY) rows_per_cta = 8 * RY;
  rows_per_cta = ceil_div64(rows_per_cta, RY) * RY;
  const int chunks = (int)ceil_div64(R, rows_per_cta);
  FYC_CHECK(chunks <= gn_max_chunks(NB), "groupnorm: internal chunk count");
  const size_t smem = (size_t)RY * C * 2 * sizeof(float);
  FYC_CHECK(smem <= 200 * 1024, "groupnorm: C=%d too large", C);
  auto kern = gn_stats_kernel<T, V>;
  if (smem > 48 * 1024) FYC_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  dim3 grid((unsigned)chunks, (unsigned)NB);
  kern<<<grid, 256, smem, st>>>(x, partials, R, C, G, rows_per_cta, fyc_zigzag(), x2, C1);
  FYC_LAUNCH_CHECK();
  gn_finalize_kernel<<<dim3((unsigned)G, (unsigned)NB), 128, 0, st>>>(partials, chunks, gamma, beta, scale, shift, C, G,
                                                                       (double)R * (C / G), eps);
  FYC_LAUNCH_CHECK();
  if constexpr (sizeof(T) == 2 && V == 8) {
    // one wave of resident CTAs (3 per SM); each walks the row blocks (RY x 4 rows) round-robin
    int64_t want = ceil_div64((int64_t)fyc_sm_count() * 3, NB);
    const int64_t nblk = ceil_div64(R, (int64_t)RY * 4);
    if (want > nblk) want = nblk;
    dim3 ga((unsigned)want, (unsigned)NB);
    if (silu) gn_apply_rows_kernel<T, true><<<ga, 256, 0, st>>>(x, scale, shift, out, R, C, x2, C1);
    else gn_apply_rows_kernel<T, false><<<ga, 256, 0, st>>>(x, scale, shift, out, R, C, x2, C1);
    FYC_LAUNCH_CHECK();
    return FYC_OK;
  }
  int64_t total_vec = NB * R * cvn;
  int64_t blocks = ceil_div64(total_vec, 256);
  int64_t cap = (int64_t)fyc_sm_count() * 16;
  unsigned gb = (unsigned)(blocks > cap ? cap : blocks);
  if (silu) gn_apply_kernel<T, V, true><<<gb, 256, 0, st>>>(x, scale, shift, out, R, C, total_vec, x2, C1);
  else gn_apply_kernel<T, V, false><<<gb, 256, 0, st>>>(x, scale, shift, out, R, C, total_vec, x2, C1);
  FYC_LAUNCH_CHECK();
  return FYC_OK;
}

// the argument checks fyc_groupnorm and fyc_groupnorm_concat share (C: all normalised channels)
static int32_t gn_check_args(const char* who, int64_t NB, int64_t R, int64_t C, int64_t G, const void* workspace, size_t workspace_bytes) {
  FYC_CHECK(G > 0 && C % G == 0, "%s: C=%lld not divisible by G=%lld", who, (long long)C, (long long)G);
  FYC_CHECK(workspace && workspace_bytes >= fyc_groupnorm_workspace_bytes(NB, C, G), "%s: workspace too small", who);
  FYC_CHECK(NB > 0 && NB < 65536 && R > 0 && C < (1 << 20) && NB * R < (1ll << 31), "%s: bad shape", who);
  return FYC_OK;
}

extern "C" int32_t fyc_groupnorm(const void* x, const float* gamma, const float* beta, void* out, int64_t NB, int64_t R,
                                 int64_t C, int64_t G, float eps, int32_t silu, int32_t dtype, void* workspace,
                                 size_t workspace_bytes, void* stream) {
  if (const int32_t err = gn_check_args("groupnorm", NB, R, C, G, workspace, workspace_bytes)) return err;
  cudaStream_t st = (cudaStream_t)stream;
  if (fyc_is_16bit(dtype)) {
    FYC_DISPATCH16(dtype, {
      if (C % 8 == 0) return groupnorm_impl<T, 8>((const T*)x, gamma, beta, (T*)out, NB, R, (int)C, (int)G, eps, silu, workspace, st);
      return groupnorm_impl<T, 1>((const T*)x, gamma, beta, (T*)out, NB, R, (int)C, (int)G, eps, silu, workspace, st);
    })
  } else if (dtype == FYC_F32) {
    if (C % 4 == 0) return groupnorm_impl<float, 4>((const float*)x, gamma, beta, (float*)out, NB, R, (int)C, (int)G, eps, silu, workspace, st);
    return groupnorm_impl<float, 1>((const float*)x, gamma, beta, (float*)out, NB, R, (int)C, (int)G, eps, silu, workspace, st);
  }
  FYC_CHECK(false, "groupnorm: unknown dtype %d", dtype);
}

extern "C" int32_t fyc_groupnorm_concat(const void* x1, int64_t C1, const void* x2, int64_t C2, const float* gamma, const float* beta,
                                        void* out, int64_t NB, int64_t R, int64_t G, float eps, int32_t silu, int32_t dtype,
                                        void* workspace, size_t workspace_bytes, void* stream) {
  const int64_t C = C1 + C2;
  FYC_CHECK(x1 && x2 && C1 > 0 && C2 > 0, "groupnorm_concat: bad arguments");
  if (const int32_t err = gn_check_args("groupnorm_concat", NB, R, C, G, workspace, workspace_bytes)) return err;
  cudaStream_t st = (cudaStream_t)stream;
  if (fyc_is_16bit(dtype)) {
    FYC_CHECK(C1 % 8 == 0 && C2 % 8 == 0 && ((((uintptr_t)x1 | (uintptr_t)x2 | (uintptr_t)out)) & 15) == 0, "groupnorm_concat(bf16): channel counts must be multiples of 8, pointers 16-byte aligned");
    FYC_DISPATCH16(dtype, return groupnorm_impl<T, 8>((const T*)x1, gamma, beta, (T*)out, NB, R, (int)C, (int)G, eps, silu, workspace, st, (const T*)x2, (int)C1))
  } else if (dtype == FYC_F32) {
    FYC_CHECK(C1 % 4 == 0 && C2 % 4 == 0, "groupnorm_concat(f32): channel counts must be multiples of 4");
    return groupnorm_impl<float, 4>((const float*)x1, gamma, beta, (float*)out, NB, R, (int)C, (int)G, eps, silu, workspace, st, (const float*)x2, (int)C1);
  }
  FYC_CHECK(false, "groupnorm_concat: unknown dtype %d", dtype);
}

// ---------------------------------------------------------------------------------------------------------
// LayerNorm.  fyc_layernorm_stats must produce exactly the rstd fyc_layernorm would have used (the LN-folded GEMM replaces the
// normalised copy by that rstd), so each normalising kernel shares its row statistics with its statistics-only twin.

// warp-per-row form (layernorm_kernel, ln_stats_kernel): loads row xr into registers - lane `lane` holds the channel vectors
// lane + 32 i below cvn = C / V - and returns its two-pass mean / centred variance
template <typename T, int V, int NV>
__device__ __forceinline__ void ln_warp_row_stats(const T* xr, int lane, int cvn, int C, float eps, float (&v)[NV][V], float& mean, float& rstd) {
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int cv = lane + 32 * i;
    if (cv < cvn) {
      load_vec<T, V>(xr + cv * V, v[i]);
#pragma unroll
      for (int e = 0; e < V; ++e) sum += v[i][e];
    }
  }
  mean = warp_sum(sum) / (float)C;
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i)
    if (lane + 32 * i < cvn) {
#pragma unroll
      for (int e = 0; e < V; ++e) { const float d = v[i][e] - mean; sq = fmaf(d, d, sq); }
    }
  rstd = rsqrtf(warp_sum(sq) / (float)C + eps);
}

// LPR form (layernorm_lpr_kernel, ln_stats_lpr_kernel): LPR lanes share a row of C = 40 * LPR channels, five 16-byte vectors per
// lane.  From a lane's raw vectors to the centred values v, the row's mean and rstd: two-pass, even and odd elements accumulated
// separately, combined over the row's lanes by xor-shuffle - every lane of the warp must take part.
template <typename T, int LPR>
__device__ __forceinline__ void ln_lpr_row_stats(const uint4 (&raw)[5], float eps, float (&v)[5][8], float& mean, float& rstd) {
  const float inv_c = 1.0f / (float)(LPR * 40);
  float s0 = 0.f, s1 = 0.f;
#pragma unroll
  for (int i = 0; i < 5; ++i) {
    u8_to_f<T>(raw[i], v[i]);
#pragma unroll
    for (int e = 0; e < 8; e += 2) { s0 = __fadd_rn(s0, v[i][e]); s1 = __fadd_rn(s1, v[i][e + 1]); }
  }
  float sum = s0 + s1;
#pragma unroll
  for (int o = 1; o < LPR; o <<= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  mean = sum * inv_c;
  float q0 = 0.f, q1 = 0.f;
#pragma unroll
  for (int i = 0; i < 5; ++i)
#pragma unroll
    for (int e = 0; e < 8; e += 2) {
      v[i][e] = __fadd_rn(v[i][e], -mean); v[i][e + 1] = __fadd_rn(v[i][e + 1], -mean);
      q0 = __fmaf_rn(v[i][e], v[i][e], q0); q1 = __fmaf_rn(v[i][e + 1], v[i][e + 1], q1);
    }
  float sq = q0 + q1;
#pragma unroll
  for (int o = 1; o < LPR; o <<= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
  rstd = rsqrtf(sq * inv_c + eps);
}

// one warp per row, row held in registers, optional PE add
template <typename T, int V, int NV>
__global__ void __launch_bounds__(256) layernorm_kernel(const T* __restrict__ x, const float* __restrict__ gamma,
                                                        const float* __restrict__ beta, T* __restrict__ out, int64_t M,
                                                        int C, float eps, const float* __restrict__ pe,
                                                        int64_t rows_per_frame, int64_t frames) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= M) return;
  const int cvn = C / V;
  float v[NV][V], mean, rstd;
  ln_warp_row_stats<T, V, NV>(x + row * C, lane, cvn, C, eps, v, mean, rstd);
  const float* per = pe ? pe + ((row / rows_per_frame) % frames) * C : nullptr;
  T* orow = out + row * C;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    int cv = lane + 32 * i;
    if (cv < cvn) {
      float o[V], gm[V], bt[V];
#pragma unroll
      for (int e = 0; e < V; e += 4) { ldg4(gamma + cv * V + e, gm + e); ldg4(beta + cv * V + e, bt + e); }
      if (per) {
#pragma unroll
        for (int e = 0; e < V; e += 4) {
          float p4[4];
          ldg4(per + cv * V + e, p4);
          bt[e] += p4[0]; bt[e + 1] += p4[1]; bt[e + 2] += p4[2]; bt[e + 3] += p4[3];
        }
      }
#pragma unroll
      for (int e = 0; e < V; ++e) o[e] = (v[i][e] - mean) * rstd * gm[e] + bt[e];
      store_vec<T, V>(orow + cv * V, o);
    }
  }
}

// 16-bit LayerNorm, RPW rows per warp: every row's 16-byte vectors are requested before any is used (RPW x NV loads in
// flight per lane instead of NV), gamma / beta are read once per warp instead of once per row.  The one-row kernel ran at
// 2.6 TB/s of the 6.6 TB/s the copy benchmark reaches: too few bytes in flight per SM and ~5 parameter loads per data load.
// (Its statistics multiply by 1 / C where the warp-per-row pair divides by C: it has no statistics-only twin to agree with.)
template <typename T, int NV, int RPW>
__global__ void __launch_bounds__(256) layernorm_rows_kernel(const T* __restrict__ x, const float* __restrict__ gamma,
                                                             const float* __restrict__ beta, T* __restrict__ out, int64_t M,
                                                             int C, float eps, const float* __restrict__ pe,
                                                             int64_t rows_per_frame, int64_t frames) {
  const int lane = threadIdx.x & 31;
  const int64_t row0 = ((int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * RPW;
  if (row0 >= M) return;
  const int cvn = C / 8;
  uint4 raw[RPW][NV];
#pragma unroll
  for (int r = 0; r < RPW; ++r)
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int cv = lane + 32 * i;
      raw[r][i] = make_uint4(0, 0, 0, 0);
      if (cv < cvn && row0 + r < M) raw[r][i] = __ldg(reinterpret_cast<const uint4*>(x + (row0 + r) * C + cv * 8));
    }
  float gm[NV][8], bt[NV][8];
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int cv = lane + 32 * i;
    if (cv < cvn) {
#pragma unroll
      for (int e = 0; e < 8; e += 4) { ldg4(gamma + cv * 8 + e, gm[i] + e); ldg4(beta + cv * 8 + e, bt[i] + e); }
    }
  }
  const float inv_c = 1.0f / (float)C;
#pragma unroll
  for (int r = 0; r < RPW; ++r) {
    const int64_t row = row0 + r;
    if (row >= M) break;                      // warp-uniform
    float v[NV][8];
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      u8_to_f<T>(raw[r][i], v[i]);
      if (lane + 32 * i < cvn) {
#pragma unroll
        for (int e = 0; e < 8; ++e) sum += v[i][e];
      }
    }
    const float mean = warp_sum(sum) * inv_c;
    float sq = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i)
      if (lane + 32 * i < cvn) {
#pragma unroll
        for (int e = 0; e < 8; ++e) { const float d = v[i][e] - mean; sq = fmaf(d, d, sq); }
      }
    const float rstd = rsqrtf(warp_sum(sq) * inv_c + eps);
    const float* per = pe ? pe + ((row / rows_per_frame) % frames) * C : nullptr;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int cv = lane + 32 * i;
      if (cv < cvn) {
        float o[8], pb[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        if (per) { ldg4(per + cv * 8, pb); ldg4(per + cv * 8 + 4, pb + 4); }
#pragma unroll
        for (int e = 0; e < 8; ++e) o[e] = (v[i][e] - mean) * rstd * gm[i][e] + (bt[i][e] + pb[e]);
        Vec8<T>::store(out + row * C + cv * 8, o);
      }
    }
  }
}

// 16-bit LayerNorm for C = 40 * LPR (320 / 640 / 1280): LPR lanes share a row, five 16-byte vectors per lane - every lane is busy
// (the warp-per-row kernels idle 24 of 32 lanes on the second vector of a 320-wide row), 32 / LPR rows per warp pass, PASSES passes
// with all loads of a pass issued up front.  gamma stays in registers for the warp's lifetime; the arithmetic is the same
// two-pass (mean, then centred variance) as the reference kernel in explicitly rounded, never contracted fp32 steps: ~5 issued
// instructions per element instead of ~18.
template <typename T, int LPR, int PASSES, bool HAS_PE>
__global__ void __launch_bounds__(256, 2) layernorm_lpr_kernel(const T* __restrict__ x, const float* __restrict__ gamma,
                                                               const float* __restrict__ beta, T* __restrict__ out, int64_t M,
                                                               float eps, const float* __restrict__ pe, int64_t rows_per_frame,
                                                               int64_t frames, int rev) {
  constexpr int C = LPR * 40, RPP = 32 / LPR;           // channels; rows per warp pass
  constexpr int VS = LPR * 8;                           // element stride between a lane's consecutive vectors
  const int lane = threadIdx.x & 31, sub = lane % LPR, rr = lane / LPR;
  // rev: CTAs take the row blocks back to front - the GEMM that produced x wrote it front to back (its tail is still in L2) and the
  // GEMM that consumes `out` reads front to back (the front is what this kernel then wrote last)
  const int64_t bxl = rev ? (int64_t)gridDim.x - 1 - blockIdx.x : (int64_t)blockIdx.x;
  const int64_t row_base = (bxl * (blockDim.x >> 5) + (threadIdx.x >> 5)) * (RPP * PASSES);
  if (row_base >= M) return;
  float gm[5][8];                                       // beta is re-read from L1 per vector: 40 more registers would halve the occupancy
  const float* gp = gamma + sub * 8;
  const float* bp = beta + sub * 8;
#pragma unroll
  for (int i = 0; i < 5; ++i) { ldg4(gp + i * VS, gm[i]); ldg4(gp + i * VS + 4, gm[i] + 4); }
#pragma unroll 1
  for (int ps = 0; ps < PASSES; ++ps) {
    const int64_t row = row_base + ps * RPP + rr;
    const bool ok = row < M;
    const int64_t rowc = ok ? row : M - 1;            // out-of-range lanes shadow the last row (shuffles stay full-warp), never store
    const T* xr = x + rowc * C + sub * 8;
    uint4 raw[5];
#pragma unroll
    for (int i = 0; i < 5; ++i) raw[i] = __ldg(reinterpret_cast<const uint4*>(xr + i * VS));
    float v[5][8], mean, rstd;
    ln_lpr_row_stats<T, LPR>(raw, eps, v, mean, rstd);
    const float* pp = HAS_PE ? pe + ((rowc / rows_per_frame) % frames) * C + sub * 8 : nullptr;
    T* orow = out + rowc * C + sub * 8;
#pragma unroll
    for (int i = 0; i < 5; ++i) {
      float bb[8], o[8];
      ldg4(bp + i * VS, bb); ldg4(bp + i * VS + 4, bb + 4);
      if (HAS_PE) {
        float pb[8];
        ldg4(pp + i * VS, pb); ldg4(pp + i * VS + 4, pb + 4);
#pragma unroll
        for (int e = 0; e < 8; ++e) bb[e] = __fadd_rn(bb[e], pb[e]);
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) o[e] = __fmaf_rn(__fmul_rn(v[i][e], rstd), gm[i][e], bb[e]);
      const uint4 packed = f_to_u8<T>(o);
      if (ok) *reinterpret_cast<uint4*>(orow + i * VS) = packed;
    }
  }
}

// LayerNorm STATISTICS only (fyc_layernorm_stats): per row rstd (fp32) and the 8-column 16-bit "aug" row [m_hi, m_hi, m_lo, m_lo, 0, 0, 0, 0]
// (mean = m_hi + m_lo) that the LN-folded GEMM appends to its K dimension (fyc.h FYC_EPI_LNFOLD).  Same lane layout and the same
// row statistics as layernorm_lpr_kernel - one read of x, no write of a normalised copy.  PASSES x 5 independent 16-byte loads
// per lane are requested before the first is used.
// AT: the aug element type.  bf16: hi + lo keeps 16 significand bits of the mean (relative error <= 2^-17).  fp16: hi + lo keeps 22
// bits while m_lo is a normal number (|mean| >= 2^-3); below that m_lo is subnormal and the absolute error stays <= 2^-25, which is
// <= 2^-17 |mean| for every |mean| >= 2^-8 - so the fp16 pair is at least as exact as the bf16 one except for means under 0.004, where
// it is off by at most 3e-8.  |mean| never exceeds the fp16 range: it averages fp16 values.
template <typename AT>
__device__ __forceinline__ void ln_write_stats(float* __restrict__ rstd_out, AT* __restrict__ aug, int64_t row, float mean, float rstd) {
  rstd_out[row] = rstd;
  if (aug == nullptr) return;
  const AT hi = from_f<AT>(mean);
  const AT lo = from_f<AT>(mean - to_f(hi));
  const uint32_t hh = (uint32_t)*reinterpret_cast<const uint16_t*>(&hi) * 0x10001u, ll = (uint32_t)*reinterpret_cast<const uint16_t*>(&lo) * 0x10001u;
  *reinterpret_cast<uint4*>(aug + row * 8) = make_uint4(hh, ll, 0u, 0u);
}

template <typename T, int LPR, int PASSES>
__global__ void __launch_bounds__(256, 2) ln_stats_lpr_kernel(const T* __restrict__ x, float* __restrict__ rstd_out, T* __restrict__ aug,
                                                              int64_t M, float eps, int rev) {
  constexpr int C = LPR * 40, RPP = 32 / LPR, VS = LPR * 8;
  const int lane = threadIdx.x & 31, sub = lane % LPR, rr = lane / LPR;
  const int64_t bxl = rev ? (int64_t)gridDim.x - 1 - blockIdx.x : (int64_t)blockIdx.x;
  const int64_t row_base = (bxl * (blockDim.x >> 5) + (threadIdx.x >> 5)) * (RPP * PASSES);
  if (row_base >= M) return;
  uint4 raw[PASSES][5];
#pragma unroll
  for (int ps = 0; ps < PASSES; ++ps) {
    const int64_t row = row_base + ps * RPP + rr;
    const int64_t rowc = row < M ? row : M - 1;       // out-of-range lanes shadow the last row (shuffles stay full-warp), never store
    const T* xr = x + rowc * C + sub * 8;
#pragma unroll
    for (int i = 0; i < 5; ++i) raw[ps][i] = __ldg(reinterpret_cast<const uint4*>(xr + i * VS));
  }
#pragma unroll
  for (int ps = 0; ps < PASSES; ++ps) {
    const int64_t row = row_base + ps * RPP + rr;
    float v[5][8], mean, rstd;
    ln_lpr_row_stats<T, LPR>(raw[ps], eps, v, mean, rstd);
    if (sub == 0 && row < M) ln_write_stats(rstd_out, aug, row, mean, rstd);
  }
}

// generic widths (C % 8 == 0, C <= 2048; 16-bit) and fp32 rows (bf16 aug): one warp per row
template <typename T, int V, int NV, typename AT>
__global__ void __launch_bounds__(256) ln_stats_kernel(const T* __restrict__ x, float* __restrict__ rstd_out, AT* __restrict__ aug, int64_t M, int C, float eps) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= M) return;
  const int cvn = C / V;
  float v[NV][V], mean, rstd;
  ln_warp_row_stats<T, V, NV>(x + row * C, lane, cvn, C, eps, v, mean, rstd);
  if (lane == 0) ln_write_stats(rstd_out, aug, row, mean, rstd);
}

// The row-width classes of fyc_layernorm and fyc_layernorm_stats (C already checked: a multiple of V, <= 2048): calls
// f(LPR, NV) with compile-time constants - LPR != 0: an LPR kernel (16-bit, C = 40 * LPR); LPR == 0: a warp-per-row kernel with
// NV vectors of V = 16 / sizeof(T) elements per lane.
template <int N> using int_c = std::integral_constant<int, N>;
template <typename T, typename F>
static void ln_for_width(int64_t C, F f) {
  if constexpr (sizeof(T) == 2) {
    if (C == 320) f(int_c<8>(), int_c<5>());
    else if (C == 640) f(int_c<16>(), int_c<5>());
    else if (C == 1280) f(int_c<32>(), int_c<5>());
    else if (C <= 8 * 32 * 5) f(int_c<0>(), int_c<5>());
    else f(int_c<0>(), int_c<8>());
  } else {
    if (C <= 4 * 32 * 5) f(int_c<0>(), int_c<5>());
    else if (C <= 4 * 32 * 10) f(int_c<0>(), int_c<10>());
    else f(int_c<0>(), int_c<16>());
  }
}

template <typename T, typename AT>
static void layernorm_stats_launch(const T* x, float* rstd, AT* aug, int64_t M, int64_t C, float eps, cudaStream_t st) {
  ln_for_width<T>(C, [&](auto lpr, auto nv) {
    constexpr int LPR = decltype(lpr)::value, NV = decltype(nv)::value, PASSES = 4;
    if constexpr (LPR != 0)
      ln_stats_lpr_kernel<T, LPR, PASSES><<<(unsigned)ceil_div64(M, 8 * (32 / LPR) * PASSES), 256, 0, st>>>(x, rstd, aug, M, eps, fyc_zigzag());
    else
      ln_stats_kernel<T, 16 / sizeof(T), NV, AT><<<(unsigned)ceil_div64(M, 8), 256, 0, st>>>(x, rstd, aug, M, (int)C, eps);
  });
}

extern "C" int32_t fyc_layernorm_stats(const void* x, float* rstd, void* aug, int64_t M, int64_t C, float eps, int32_t dtype, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  FYC_CHECK(x && rstd && M > 0 && C > 0, "layernorm_stats: bad arguments");
  FYC_CHECK((((uintptr_t)x | (uintptr_t)aug) & 15) == 0 && (((uintptr_t)rstd) & 3) == 0, "layernorm_stats: alignment");
  if (fyc_is_16bit(dtype)) {
    FYC_CHECK(C % 8 == 0 && C <= 2048, "layernorm_stats(bf16): C=%lld must be a multiple of 8 and <= 2048", (long long)C);
    FYC_DISPATCH16(dtype, layernorm_stats_launch((const T*)x, rstd, (T*)aug, M, C, eps, st))
  } else if (dtype == FYC_F32) {
    FYC_CHECK(C % 4 == 0 && C <= 2048, "layernorm_stats(f32): C=%lld must be a multiple of 4 and <= 2048", (long long)C);
    layernorm_stats_launch((const float*)x, rstd, (bf16*)aug, M, C, eps, st);
  } else {
    FYC_CHECK(false, "layernorm_stats: unknown dtype %d", dtype);
  }
  FYC_LAUNCH_CHECK();
  return FYC_OK;
}

template <typename T>
static void layernorm_launch(const T* x, const float* gamma, const float* beta, T* out, int64_t M, int64_t C, float eps, const float* pe,
                             int64_t rows_per_frame, int64_t frames, cudaStream_t st) {
  ln_for_width<T>(C, [&](auto lpr, auto nv) {
    constexpr int LPR = decltype(lpr)::value, NV = decltype(nv)::value, PASSES = 2;
    if constexpr (LPR != 0) {
      const unsigned grid = (unsigned)ceil_div64(M, 8 * (32 / LPR) * PASSES);
      if (pe) layernorm_lpr_kernel<T, LPR, PASSES, true><<<grid, 256, 0, st>>>(x, gamma, beta, out, M, eps, pe, rows_per_frame, frames, fyc_zigzag());
      else layernorm_lpr_kernel<T, LPR, PASSES, false><<<grid, 256, 0, st>>>(x, gamma, beta, out, M, eps, pe, rows_per_frame, frames, fyc_zigzag());
    } else {
      if constexpr (sizeof(T) == 2) {       // narrow 16-bit rows: several rows per warp
        if (C <= 8 * 32 * 2) return layernorm_rows_kernel<T, 2, 4><<<(unsigned)ceil_div64(M, 8 * 4), 256, 0, st>>>(x, gamma, beta, out, M, (int)C, eps, pe, rows_per_frame, frames);
        if (C <= 8 * 32 * 3) return layernorm_rows_kernel<T, 3, 2><<<(unsigned)ceil_div64(M, 8 * 2), 256, 0, st>>>(x, gamma, beta, out, M, (int)C, eps, pe, rows_per_frame, frames);
      }
      layernorm_kernel<T, 16 / sizeof(T), NV><<<(unsigned)ceil_div64(M, 8), 256, 0, st>>>(x, gamma, beta, out, M, (int)C, eps, pe, rows_per_frame, frames);
    }
  });
}

extern "C" int32_t fyc_layernorm(const void* x, const float* gamma, const float* beta, void* out, int64_t M, int64_t C,
                                 float eps, const float* pe, int64_t rows_per_frame, int64_t frames, int32_t dtype,
                                 void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  FYC_CHECK(M > 0 && C > 0, "layernorm: bad shape");
  if (pe) FYC_CHECK(rows_per_frame > 0 && frames > 0, "layernorm: pe needs rows_per_frame/frames");
  if (fyc_is_16bit(dtype)) {
    FYC_CHECK(C % 8 == 0 && C <= 8 * 32 * 8, "layernorm(bf16): C=%lld must be a multiple of 8 and <= 2048", (long long)C);
    FYC_CHECK((((uintptr_t)x | (uintptr_t)out) & 15) == 0 && (((uintptr_t)gamma | (uintptr_t)beta | (uintptr_t)pe) & 15) == 0, "layernorm(bf16): 16-byte alignment");
    FYC_DISPATCH16(dtype, layernorm_launch((const T*)x, gamma, beta, (T*)out, M, C, eps, pe, rows_per_frame, frames, st))
  } else if (dtype == FYC_F32) {
    FYC_CHECK(C % 4 == 0 && C <= 4 * 32 * 16, "layernorm(f32): C=%lld must be a multiple of 4 and <= 2048", (long long)C);
    layernorm_launch((const float*)x, gamma, beta, (float*)out, M, C, eps, pe, rows_per_frame, frames, st);
  } else {
    FYC_CHECK(false, "layernorm: unknown dtype %d", dtype);
  }
  FYC_LAUNCH_CHECK();
  return FYC_OK;
}
