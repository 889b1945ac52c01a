// Fused multi-head attention on tensor cores (bf16 or fp16 operands, fp32 accumulation, online softmax in registers):
// spatial self-attention (N up to 9216 keys), text cross-attention (77 keys) and the IP-adapter pass (4/16 keys).
// The score matrix lives only in registers: S = Q K^T (mma.sync m16n8k16) -> warp-shuffle row max/sum ->
// P (16-bit, re-used in place as the A operand) -> O += P V.  K/V tiles are double-buffered with cp.async.
// Head dims 40/80/160 (SD-1.5: C/8) are padded to 48/80/160 in shared memory only.
//
// It serves the shapes the wgmma kernels of attention_tc.cu do not take (head dim 160, ragged or unpacked contexts).
#include <stdlib.h>

#include "common.cuh"

namespace {

constexpr int BQ = 64, BKV = 64, NTHR = 128;

// copy a [64 x DP] tile (rows row0.., valid while < L, columns < D; everything else zero) into smem
template <int D, int DP, int LDS, bool ONES_COL = false, typename T>
__device__ __forceinline__ void load_tile(T* dst, const T* src, int64_t ld, int64_t row0, int64_t L, int tid) {
  constexpr int CH = DP / 8;
  for (int i = tid; i < 64 * CH; i += NTHR) {
    int r = i / CH, c = (i % CH) * 8;
    bool ok = (row0 + r < L) && (c < D);
    if (ONES_COL && c == D) {
      // V padding chunk: [1, 0, 0, ...] for valid keys (row sum via the PV MMA), zeros for keys past the end
      uint4 v = make_uint4((row0 + r < L) ? Pair16<T>::ONE : 0u, 0u, 0u, 0u);     // T(1.0) in the low half
      *reinterpret_cast<uint4*>(dst + r * LDS + c) = v;
      continue;
    }
    const T* s = ok ? src + (row0 + r) * ld + c : src;
    cp_async16(dst + r * LDS + c, s, ok ? 16 : 0);
  }
}

template <int D, int DP, typename T>
__global__ void __launch_bounds__(NTHR) attention_mma_kernel(fyc_attention_args a) {
  constexpr int LDS = DP + 8;          // padded row stride: ldmatrix row addresses hit distinct bank groups
  constexpr int KS = DP / 16;          // k-steps of QK^T
  constexpr int NO = DP / 8;           // n-tiles of the output
  constexpr bool ONES = DP > D;        // V's first padding column (col D) holds ones -> O[:, D] accumulates the softmax row sum
  extern __shared__ __align__(16) unsigned char smem_raw[];
  T* sQ = reinterpret_cast<T*>(smem_raw);
  T* sK = sQ + 64 * LDS;            // [2][64][LDS]
  T* sV = sK + 2 * 64 * LDS;        // [2][64][LDS]
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int64_t n = blockIdx.z, h = blockIdx.y;
  const int64_t q0 = (int64_t)blockIdx.x * BQ;
  const int64_t nk = n / a.kv_batch_div;
  const T* qg = (const T*)a.q + n * a.bsq + h * D;
  const T* kg = (const T*)a.k + nk * a.bsk + h * D;
  const T* vg = (const T*)a.v + nk * a.bsv + h * D;
  const int nkt = (int)((a.Lk + BKV - 1) / BKV);

  load_tile<D, DP, LDS>(sQ, qg, a.ldq, q0, a.Lq, tid);
  load_tile<D, DP, LDS>(sK, kg, a.ldk, 0, a.Lk, tid);
  load_tile<D, DP, LDS, (DP > D)>(sV, vg, a.ldv, 0, a.Lk, tid);
  cp_async_commit();

  uint32_t qf[KS][4];
  float o[NO][4];
#pragma unroll
  for (int i = 0; i < NO; ++i) { o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f; }
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;   // rows g and g+8 of this warp's 16-row slab
  const float sl2 = a.scale * 1.4426950408889634f;             // fold log2(e): p = 2^((s - m) * sl2)

  for (int kt = 0; kt < nkt; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < nkt) {
      load_tile<D, DP, LDS>(sK + (buf ^ 1) * 64 * LDS, kg, a.ldk, (int64_t)(kt + 1) * BKV, a.Lk, tid);
      load_tile<D, DP, LDS, (DP > D)>(sV + (buf ^ 1) * 64 * LDS, vg, a.ldv, (int64_t)(kt + 1) * BKV, a.Lk, tid);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    if (kt == 0) {
#pragma unroll
      for (int ks = 0; ks < KS; ++ks)
        ldmatrix_x4(qf[ks], sQ + (w * 16 + (lane & 15)) * LDS + ks * 16 + (lane >> 4) * 8);
    }
    const T* kb = sK + buf * 64 * LDS;
    const T* vb = sV + buf * 64 * LDS;
    // ---- S = Q K^T : 16 x 64 per warp
    float s[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) { s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f; }
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
#pragma unroll
      for (int jp = 0; jp < 4; ++jp) {       // pairs of 8-key n-tiles
        uint32_t b[4];
        const int mi = lane >> 3;
        ldmatrix_x4(b, kb + (jp * 16 + (lane & 7) + (mi >> 1) * 8) * LDS + ks * 16 + (mi & 1) * 8);
        mma16816<T>(s[2 * jp], qf[ks], b[0], b[1]);
        mma16816<T>(s[2 * jp + 1], qf[ks], b[2], b[3]);
      }
    }
    // ---- online softmax on the raw scores (rows g, g+8; this thread holds cols 8j + 2t, +1).
    // Instruction diet (the kernel is issue-bound): the logit scale is folded into one FFMA per
    // element (p = 2^(s*sl2 - m*sl2)), masking runs only on the last, ragged KV tile, and for D < DP the row sum comes
    // out of the PV MMA itself through a column of ones planted in V's padding (col D) - no per-element FADD.
    if (kt == nkt - 1 && (a.Lk & (BKV - 1))) {
      const int64_t kbase = (int64_t)kt * BKV;
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (kbase + 8 * j + 2 * t + e >= a.Lk) { s[j][e] = -INFINITY; s[j][2 + e] = -INFINITY; }
    }
    float mx0 = s[0][0], mx1 = s[0][2];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      mx0 = fmaxf(mx0, fmaxf(s[j][0], s[j][1]));
      mx1 = fmaxf(mx1, fmaxf(s[j][2], s[j][3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);           // running maxima of the RAW scores (scale > 0)
    const float c0 = (m0 == -INFINITY) ? 0.f : ex2_approx((m0 - mn0) * sl2), c1 = (m1 == -INFINITY) ? 0.f : ex2_approx((m1 - mn1) * sl2);
    m0 = mn0; m1 = mn1;
    const float nb0 = -mn0 * sl2, nb1 = -mn1 * sl2;
    float rs0 = 0.f, rs1 = 0.f;
    uint32_t pf[4][4];   // P as A fragments: k-step kk covers keys 16kk..16kk+15 = n-tiles 2kk, 2kk+1
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float p0 = ex2_approx(fmaf(s[j][0], sl2, nb0)), p1 = ex2_approx(fmaf(s[j][1], sl2, nb0));
      float p2 = ex2_approx(fmaf(s[j][2], sl2, nb1)), p3 = ex2_approx(fmaf(s[j][3], sl2, nb1));
      if constexpr (!ONES) { rs0 += p0 + p1; rs1 += p2 + p3; }
      pf[j >> 1][(j & 1) * 2 + 0] = pack_u32<T>(p0, p1);
      pf[j >> 1][(j & 1) * 2 + 1] = pack_u32<T>(p2, p3);
    }
    if constexpr (!ONES) {
      rs0 += __shfl_xor_sync(0xffffffffu, rs0, 1); rs0 += __shfl_xor_sync(0xffffffffu, rs0, 2);
      rs1 += __shfl_xor_sync(0xffffffffu, rs1, 1); rs1 += __shfl_xor_sync(0xffffffffu, rs1, 2);
      l0 = l0 * c0 + rs0; l1 = l1 * c1 + rs1;
    }
#pragma unroll
    for (int i = 0; i < NO; ++i) { o[i][0] *= c0; o[i][1] *= c0; o[i][2] *= c1; o[i][3] *= c1; }
    // ---- O += P V
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
      for (int np = 0; np < NO / 2; ++np) {   // pairs of 8-wide output n-tiles
        uint32_t b[4];
        const int mi = lane >> 3;
        ldmatrix_x4_trans(b, vb + (kk * 16 + (lane & 7) + (mi & 1) * 8) * LDS + np * 16 + (mi >> 1) * 8);
        mma16816<T>(o[2 * np], pf[kk], b[0], b[1]);
        mma16816<T>(o[2 * np + 1], pf[kk], b[2], b[3]);
      }
    }
    __syncthreads();
  }
  // ---- epilogue: O / l * out_alpha (+ existing out)
  if constexpr (ONES) {   // column D of O is sum_j P_ij: lives in n-tile D/8, element 0/2 of the lane with 2t == D % 8
    constexpr int NTL = D / 8, SRC = (D % 8) / 2;
    l0 = __shfl_sync(0xffffffffu, o[NTL][0], (lane & ~3) | SRC);
    l1 = __shfl_sync(0xffffffffu, o[NTL][2], (lane & ~3) | SRC);
  }
  const float i0 = a.out_alpha / l0, i1 = a.out_alpha / l1;
  T* og = (T*)a.out + n * a.bso + h * D;
  const int64_t r0 = q0 + w * 16 + g, r1 = r0 + 8;
#pragma unroll
  for (int i = 0; i < NO; ++i) {
    const int col = i * 8 + 2 * t;
    if (col < D) {
      if (r0 < a.Lq) {
        typename Pair16<T>::type* dst = reinterpret_cast<typename Pair16<T>::type*>(og + r0 * a.ldo + col);
        float x = o[i][0] * i0, y = o[i][1] * i0;
        if (a.accumulate) { float2 e = Pair16<T>::unpack(*dst); x += e.x; y += e.y; }
        *dst = Pair16<T>::pack(x, y);
      }
      if (r1 < a.Lq) {
        typename Pair16<T>::type* dst = reinterpret_cast<typename Pair16<T>::type*>(og + r1 * a.ldo + col);
        float x = o[i][2] * i1, y = o[i][3] * i1;
        if (a.accumulate) { float2 e = Pair16<T>::unpack(*dst); x += e.x; y += e.y; }
        *dst = Pair16<T>::pack(x, y);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
// Short-context variant (Lk <= 128: the 77 text tokens of every cross-attention; optional SECOND context of <= 64 keys: the 4 / 16
// image-prompt tokens of the IP-Adapter).  The generic kernel above launches one CTA per 64 query rows, and each of those 16 K CTAs
// at the 64x64 level re-stages the same K / V tiles and pays the full launch -> cp.async -> barrier latency for ~100 MMAs of work
// (a small fraction of the HBM stream).  Here a CTA owns one (image, head), stages K and V (and K_ip, V_ip) ONCE, and
// walks a strided set of query tiles with the next Q tile prefetched (cp.async double buffer) while the current one is in the
// tensor cores.
//
// Fused IP cross-attention (IPCrossAttention.forward animatediff/models/attention.py:92-120 == IPAttnProcessor.__call__
// ip_adapter/attention_processor.py:137-168): with a.k2 != NULL the same query fragments run a second, independent softmax over
// the image keys and the kernel writes  out_alpha * softmax(q K_t^T s) V_t + alpha2 * softmax(q K_i^T s) V_i  ONCE - the reference's
// two attention passes + add, without the second launch, the second read of Q, or a read-modify-write of `out`.
// Only the 16-key groups that hold valid keys are multiplied (77 keys = 5 groups of the 8 staged; 4 / 16 image keys = 1 group).
template <int D, int DP, typename T>
__global__ void __launch_bounds__(NTHR) attention_mma_shortk_kernel(fyc_attention_args a, int nqt) {
  constexpr int LDS = DP + 8;
  constexpr int KS = DP / 16;
  constexpr int NO = DP / 8;
  constexpr bool ONES = DP > D;
  constexpr bool PACKED = DP > 80;                // D = 160: the first context's result waits as packed 16-bit pairs (register budget)
  extern __shared__ __align__(16) unsigned char smem_raw[];
  T* sQ = reinterpret_cast<T*>(smem_raw);   // [2][64][LDS]
  T* sK = sQ + 2 * 64 * LDS;                   // [3][64][LDS]  key tiles 0, 1 of the first context, tile 2 = second context
  T* sV = sK + 3 * 64 * LDS;                   // [3][64][LDS]
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int64_t n = blockIdx.z, h = blockIdx.y;
  const int64_t nk = n / a.kv_batch_div;
  const T* qg = (const T*)a.q + n * a.bsq + h * D;
  const T* kg = (const T*)a.k + nk * a.bsk + h * D;
  const T* vg = (const T*)a.v + nk * a.bsv + h * D;
  T* og = (T*)a.out + n * a.bso + h * D;
  const int nkt = (int)((a.Lk + BKV - 1) / BKV);  // 1 or 2
  const int npass = a.k2 ? 2 : 1;
  const float sl2 = a.scale * 1.4426950408889634f;

  for (int kt = 0; kt < nkt; ++kt) {
    load_tile<D, DP, LDS>(sK + kt * 64 * LDS, kg, a.ldk, (int64_t)kt * BKV, a.Lk, tid);
    load_tile<D, DP, LDS, (DP > D)>(sV + kt * 64 * LDS, vg, a.ldv, (int64_t)kt * BKV, a.Lk, tid);
  }
  if (a.k2) {
    load_tile<D, DP, LDS>(sK + 2 * 64 * LDS, (const T*)a.k2 + nk * a.bsk2 + h * D, a.ldk2, 0, a.Lk2, tid);
    load_tile<D, DP, LDS, (DP > D)>(sV + 2 * 64 * LDS, (const T*)a.v2 + nk * a.bsv2 + h * D, a.ldv2, 0, a.Lk2, tid);
  }
  int qt = blockIdx.x;
  if (qt < nqt) load_tile<D, DP, LDS>(sQ, qg, a.ldq, (int64_t)qt * BQ, a.Lq, tid);
  cp_async_commit();

  for (int it = 0; qt < nqt; qt += gridDim.x, ++it) {
    const int qb = it & 1;
    const int nq = qt + (int)gridDim.x;
    if (nq < nqt) {
      load_tile<D, DP, LDS>(sQ + (qb ^ 1) * 64 * LDS, qg, a.ldq, (int64_t)nq * BQ, a.Lq, tid);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    uint32_t qf[KS][4];
#pragma unroll
    for (int ks = 0; ks < KS; ++ks)
      ldmatrix_x4(qf[ks], sQ + qb * 64 * LDS + (w * 16 + (lane & 15)) * LDS + ks * 16 + (lane >> 4) * 8);
    float o[NO][4];
    float accf[PACKED ? 1 : NO][4];                 // first context's finished result (fp32), or ...
    uint32_t accp[PACKED ? NO : 1][2];              // ... packed 16-bit pairs (rows g, g+8)

#pragma unroll 1
    for (int pass = 0; pass < npass; ++pass) {
      const int tile0 = pass ? 2 : 0, ntl = pass ? 1 : nkt;
      const int64_t Lp = pass ? a.Lk2 : a.Lk;
#pragma unroll
      for (int i = 0; i < NO; ++i) { o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f; }
      float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;

      for (int kt = 0; kt < ntl; ++kt) {
        const T* kb = sK + (tile0 + kt) * 64 * LDS;
        const T* vb = sV + (tile0 + kt) * 64 * LDS;
        const int nvalid = (int)min((int64_t)BKV, Lp - (int64_t)kt * BKV);     // valid keys of this tile (>= 1)
        const int ngrp = (nvalid + 15) >> 4;                                    // 16-key groups that hold any
        float s[8][4];
#pragma unroll
        for (int j = 0; j < 8; ++j) { s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f; }
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
#pragma unroll
          for (int jp = 0; jp < 4; ++jp) {
            if (jp < ngrp) {
              uint32_t b[4];
              const int mi = lane >> 3;
              ldmatrix_x4(b, kb + (jp * 16 + (lane & 7) + (mi >> 1) * 8) * LDS + ks * 16 + (mi & 1) * 8);
              mma16816<T>(s[2 * jp], qf[ks], b[0], b[1]);
              mma16816<T>(s[2 * jp + 1], qf[ks], b[2], b[3]);
            }
          }
        }
        if (nvalid < BKV) {
#pragma unroll
          for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e)
              if (8 * j + 2 * t + e >= nvalid) { s[j][e] = -INFINITY; s[j][2 + e] = -INFINITY; }
        }
        float mx0 = s[0][0], mx1 = s[0][2];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          mx0 = fmaxf(mx0, fmaxf(s[j][0], s[j][1]));
          mx1 = fmaxf(mx1, fmaxf(s[j][2], s[j][3]));
        }
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
        const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
        const float c0 = (m0 == -INFINITY) ? 0.f : ex2_approx((m0 - mn0) * sl2), c1 = (m1 == -INFINITY) ? 0.f : ex2_approx((m1 - mn1) * sl2);
        m0 = mn0; m1 = mn1;
        const float nb0 = -mn0 * sl2, nb1 = -mn1 * sl2;
        float rs0 = 0.f, rs1 = 0.f;
        uint32_t pf[4][4];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if ((j >> 1) < ngrp) {
            float p0 = ex2_approx(fmaf(s[j][0], sl2, nb0)), p1 = ex2_approx(fmaf(s[j][1], sl2, nb0));
            float p2 = ex2_approx(fmaf(s[j][2], sl2, nb1)), p3 = ex2_approx(fmaf(s[j][3], sl2, nb1));
            if constexpr (!ONES) { rs0 += p0 + p1; rs1 += p2 + p3; }
            pf[j >> 1][(j & 1) * 2 + 0] = pack_u32<T>(p0, p1);
            pf[j >> 1][(j & 1) * 2 + 1] = pack_u32<T>(p2, p3);
          }
        }
        if constexpr (!ONES) {
          rs0 += __shfl_xor_sync(0xffffffffu, rs0, 1); rs0 += __shfl_xor_sync(0xffffffffu, rs0, 2);
          rs1 += __shfl_xor_sync(0xffffffffu, rs1, 1); rs1 += __shfl_xor_sync(0xffffffffu, rs1, 2);
          l0 = l0 * c0 + rs0; l1 = l1 * c1 + rs1;
        }
        if (kt > 0) {
#pragma unroll
          for (int i = 0; i < NO; ++i) { o[i][0] *= c0; o[i][1] *= c0; o[i][2] *= c1; o[i][3] *= c1; }
        }
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          if (kk < ngrp) {
#pragma unroll
            for (int np = 0; np < NO / 2; ++np) {
              uint32_t b[4];
              const int mi = lane >> 3;
              ldmatrix_x4_trans(b, vb + (kk * 16 + (lane & 7) + (mi & 1) * 8) * LDS + np * 16 + (mi >> 1) * 8);
              mma16816<T>(o[2 * np], pf[kk], b[0], b[1]);
              mma16816<T>(o[2 * np + 1], pf[kk], b[2], b[3]);
            }
          }
        }
      }
      if constexpr (ONES) {
        constexpr int NTL = D / 8, SRC = (D % 8) / 2;
        l0 = __shfl_sync(0xffffffffu, o[NTL][0], (lane & ~3) | SRC);
        l1 = __shfl_sync(0xffffffffu, o[NTL][2], (lane & ~3) | SRC);
      }
      const float wgt = pass ? a.alpha2 : a.out_alpha;
      const float i0 = wgt / l0, i1 = wgt / l1;
      if (pass == 0 && npass == 2) {                 // park  out_alpha * softmax(q K_t^T) V_t  while the image keys are processed
#pragma unroll
        for (int i = 0; i < NO; ++i) {
          if constexpr (PACKED) { accp[i][0] = pack_u32<T>(o[i][0] * i0, o[i][1] * i0); accp[i][1] = pack_u32<T>(o[i][2] * i1, o[i][3] * i1); }
          else { accf[i][0] = o[i][0] * i0; accf[i][1] = o[i][1] * i0; accf[i][2] = o[i][2] * i1; accf[i][3] = o[i][3] * i1; }
        }
      } else {
#pragma unroll
        for (int i = 0; i < NO; ++i) {
          o[i][0] *= i0; o[i][1] *= i0; o[i][2] *= i1; o[i][3] *= i1;
          if (pass == 1) {
            if constexpr (PACKED) {
              const float2 e0 = Pair16<T>::unpack(*reinterpret_cast<const typename Pair16<T>::type*>(&accp[i][0]));
              const float2 e1 = Pair16<T>::unpack(*reinterpret_cast<const typename Pair16<T>::type*>(&accp[i][1]));
              o[i][0] += e0.x; o[i][1] += e0.y; o[i][2] += e1.x; o[i][3] += e1.y;
            } else { o[i][0] += accf[i][0]; o[i][1] += accf[i][1]; o[i][2] += accf[i][2]; o[i][3] += accf[i][3]; }
          }
        }
      }
    }
    const int64_t r0 = (int64_t)qt * BQ + w * 16 + g, r1 = r0 + 8;
#pragma unroll
    for (int i = 0; i < NO; ++i) {
      const int col = i * 8 + 2 * t;
      if (col < D) {
        if (r0 < a.Lq) {
          typename Pair16<T>::type* dst = reinterpret_cast<typename Pair16<T>::type*>(og + r0 * a.ldo + col);
          float x = o[i][0], y = o[i][1];
          if (a.accumulate) { float2 e = Pair16<T>::unpack(*dst); x += e.x; y += e.y; }
          *dst = Pair16<T>::pack(x, y);
        }
        if (r1 < a.Lq) {
          typename Pair16<T>::type* dst = reinterpret_cast<typename Pair16<T>::type*>(og + r1 * a.ldo + col);
          float x = o[i][2], y = o[i][3];
          if (a.accumulate) { float2 e = Pair16<T>::unpack(*dst); x += e.x; y += e.y; }
          *dst = Pair16<T>::pack(x, y);
        }
      }
    }
    __syncthreads();      // every warp is done with sQ[qb] before the next iteration's prefetch refills it
  }
}

static bool shortk_enabled() {
  const char* e = getenv("FYC_ATTN_SHORTK");
  return !(e && e[0] == '0');
}

template <int D, int DP, typename T>
int32_t launch_mma_shortk(const fyc_attention_args* a, cudaStream_t st) {
  constexpr int LDS = DP + 8;
  const size_t smem = (size_t)8 * 64 * LDS * sizeof(T);     // 2 Q + 3 K + 3 V tiles
  auto kern = attention_mma_shortk_kernel<D, DP, T>;
  FYC_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int nqt = (int)ceil_div64(a->Lq, BQ);
  // CTAs per (image, head): enough to fill the machine (~227 KB of shared memory per SM), at most one per query tile
  const int64_t per_sm = (int64_t)(227 * 1024) / (int64_t)(smem + 1024);
  const int64_t pairs = a->heads * a->batch;
  int64_t gx = ceil_div64((int64_t)fyc_sm_count() * (per_sm > 8 ? 8 : per_sm), pairs);
  if (gx < 1) gx = 1;
  if (gx > nqt) gx = nqt;
  dim3 grid((unsigned)gx, (unsigned)a->heads, (unsigned)a->batch);
  kern<<<grid, NTHR, smem, st>>>(*a, nqt);
  FYC_LAUNCH_CHECK();
  return FYC_OK;
}

template <int D, int DP, typename T>
int32_t launch_mma(const fyc_attention_args* a, cudaStream_t st) {
  if (a->k2) {     // fused two-context form (IP cross-attention): one launch when both contexts fit the resident kernel, else two passes
    if (a->Lk <= 2 * BKV && a->Lk2 <= BKV) return launch_mma_shortk<D, DP, T>(a, st);
    fyc_attention_args p1 = *a, p2 = *a;
    p1.k2 = p1.v2 = nullptr;
    p2.k = a->k2; p2.v = a->v2; p2.Lk = a->Lk2; p2.ldk = a->ldk2; p2.ldv = a->ldv2; p2.bsk = a->bsk2; p2.bsv = a->bsv2;
    p2.k2 = p2.v2 = nullptr; p2.out_alpha = a->alpha2; p2.accumulate = 1;
    const int32_t rc = launch_mma<D, DP, T>(&p1, st);
    return rc ? rc : launch_mma<D, DP, T>(&p2, st);
  }
  if (a->Lk <= 2 * BKV && a->Lq >= 4 * BQ && DP <= 80 && shortk_enabled()) return launch_mma_shortk<D, DP, T>(a, st);
  constexpr int LDS = DP + 8;
  const size_t smem = (size_t)5 * 64 * LDS * sizeof(T);
  auto kern = attention_mma_kernel<D, DP, T>;
  FYC_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  dim3 grid((unsigned)ceil_div64(a->Lq, BQ), (unsigned)a->heads, (unsigned)a->batch);
  kern<<<grid, NTHR, smem, st>>>(*a);
  FYC_LAUNCH_CHECK();
  return FYC_OK;
}

}  // namespace

bool fyc_attention_mma_eligible(const fyc_attention_args* a) {
  if (!fyc_is_16bit(a->dtype)) return false;
  if (a->D != 40 && a->D != 80 && a->D != 160 && a->D != 64) return false;
  if ((a->ldq | a->ldk | a->ldv | a->bsq | a->bsk | a->bsv) % 8) return false;
  if ((a->ldo | a->bso) % 2) return false;
  if (((uintptr_t)a->q | (uintptr_t)a->k | (uintptr_t)a->v) & 15) return false;
  if (a->k2 && (((a->ldk2 | a->ldv2 | a->bsk2 | a->bsv2) % 8) || (((uintptr_t)a->k2 | (uintptr_t)a->v2) & 15))) return false;
  if ((uintptr_t)a->out & 3) return false;
  if (a->heads >= 65536 || a->batch >= 65536) return false;
  return true;
}

int32_t fyc_attention_mma(const fyc_attention_args* a, cudaStream_t st) {
  FYC_DISPATCH16(a->dtype, switch (a->D) {
    case 40: return launch_mma<40, 48, T>(a, st);
    case 64: return launch_mma<64, 64, T>(a, st);
    case 80: return launch_mma<80, 80, T>(a, st);
    case 160: return launch_mma<160, 160, T>(a, st);
  })
  FYC_CHECK(false, "attention(mma): unsupported head dim %lld", (long long)a->D);
}
