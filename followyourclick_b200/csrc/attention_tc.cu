// Spatial self-attention and short-context cross-attention on Hopper tensor cores (wgmma), for the long-sequence, small-head
// cases that dominate the UNet (SD-1.5: level 0 4096 tokens, 8 heads x 40 dims, level 1 1024 tokens, head dim 80; SD-2.x: head dim 64
// at every level).
//
// Self-attention: one CTA = 128 query rows of one (image, head), two warpgroups of 64 rows each.  Per 128-key tile:
//   S = Q K^T     wgmma m64n128k16, Q and K straight from 128B-swizzled TMA tiles, fp32 S in registers
//   softmax       running max per row (4 lanes share a row), p = ex2(s * scale*log2e - m), O rescaled in registers
//   O += P V      wgmma m64nDVk16 with P (bf16) as the register A operand and V^T (keys contiguous) as the K-major B operand
// K and V^T tiles arrive through a 2-stage TMA ring; the score matrix never leaves registers.
// Operand prerequisites (prepared by the host side once per layer call, see unet.py::_transformer):
//   q, k : [NB, L, heads * 64] bf16 (zero columns 40..63 per head come for free from zero rows in the packed projection weight;
//          head dim 64: the fused [q | k | v] projection as is, one 64-column atom per head, 4 k-steps)
//          or, head dim 80, the fused [q | k | v] projection as is (two 64-column atoms per head, 5 k-steps)
//   v^T  : [NB, heads * D, L] bf16 (fyc_transpose_tokens)
//
// Cross-attention: a SHORT, step-invariant context (the 77 text tokens, padded to 80 keys; optionally the IP-Adapter's 4 / 16 image
// tokens, padded to 16) against long query sequences (CrossAttention._attention diffusers/models/attention.py:649-678 for attn2;
// IPCrossAttention.forward animatediff/models/attention.py:92-120 == IPAttnProcessor.__call__ ip_adapter/attention_processor.py:137-168).
// One CTA = one (image, head): K_t, V_t^T (and K_i, V_i^T) are loaded ONCE and stay in shared memory while the CTA walks its query
// tiles (double-buffered Q).  Per tile: S_t = Q K_t^T (N = 80) and S_i = Q K_i^T (N = 16) -> two INDEPENDENT softmaxes, normalised
// in registers (the whole context is one tile: no online rescaling) and pre-scaled by out_alpha / l_t and alpha2 / l_i -> P_t, P_i
// (bf16 registers) -> O = P_t V_t + P_i V_i in ONE accumulator -> bf16 out, written once.  Padding keys are masked to -inf.
#include <stdlib.h>

#include "tma.cuh"
#include "wgmma.cuh"

namespace {

constexpr int BQ = 128, BKV = 128;
constexpr int ATOM_BYTES = BQ * 128;                            // 16 KB: 128 rows x 64 bf16 columns
constexpr int NTHREADS = 256;                                   // two warpgroups

__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}
// register accumulator of n-tiles [2 kk, 2 kk + 1] (rows r, r + 8) -> the A fragment of k-step kk, as pairs of T
template <typename T>
__device__ __forceinline__ void pack_a(const float* p, int kk, uint32_t* a) {
  a[0] = pack_u32<T>(p[8 * kk + 0], p[8 * kk + 1]);
  a[1] = pack_u32<T>(p[8 * kk + 2], p[8 * kk + 3]);
  a[2] = pack_u32<T>(p[8 * kk + 4], p[8 * kk + 5]);
  a[3] = pack_u32<T>(p[8 * kk + 6], p[8 * kk + 7]);
}
// out[row, col .. col + 1] for the n-tiles of a 64 x DV accumulator that hold real columns (< D)
template <int DV, int D, typename T>
__device__ __forceinline__ void store_rows(T* og, int64_t ldo, int64_t r0, int64_t nrows, const float* o, float s0, float s1, int q) {
  typedef typename Pair16<T>::type P;
#pragma unroll
  for (int j = 0; j < DV / 8; ++j) {
    const int col = 8 * j + 2 * q;
    if (col >= D) continue;
    if (r0 < nrows) *reinterpret_cast<P*>(og + r0 * ldo + col) = Pair16<T>::pack(o[4 * j] * s0, o[4 * j + 1] * s0);
    if (r0 + 8 < nrows) *reinterpret_cast<P*>(og + (r0 + 8) * ldo + col) = Pair16<T>::pack(o[4 * j + 2] * s1, o[4 * j + 3] * s1);
  }
}

struct AttnTcParams {
  void* out; int64_t ldo, bso;      // out[n, token, h*D + d]
  int L, heads;
  float scale_log2e;
};

// KA: 64-column atoms per q / k head (1: D = 40 zero-padded to 64 or D = 64, 2: D = 80), KS: k-steps of QK^T that hold data, DV: PV accumulator
// columns (D rounded up to a multiple of 16 rows of V^T; the extra rows belong to the next head and only feed unstored columns); T: the
// 16-bit operand / output type (bf16 | f16)
template <int KA, int KS, int DV, int D, typename T>
__global__ void __launch_bounds__(NTHREADS, 1)
attention_tc_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k, const __grid_constant__ CUtensorMap map_v,
                    const AttnTcParams p) {
  constexpr int VBOX = DV * 128;                   // one V^T box: DV rows x 64 keys
  constexpr int K_BYTES = KA * ATOM_BYTES, V_BYTES = 2 * VBOX;
  constexpr int OFF_K = KA * ATOM_BYTES, OFF_V = OFF_K + 2 * K_BYTES, OFF_BAR = OFF_V + 2 * V_BYTES;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + pad1024(smem_raw);
  uint64_t* qbar = reinterpret_cast<uint64_t*>(smem + OFF_BAR);
  uint64_t* full = qbar + 1;                       // [2]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2, q = lane & 3;
  const int q0 = blockIdx.x * BQ, h = blockIdx.y, n = blockIdx.z;
  const int nkv = p.L / BKV;

  auto load_kv = [&](int j) {
    const int s = j & 1;
    mbar_expect_tx(&full[s], K_BYTES + V_BYTES);
#pragma unroll
    for (int a = 0; a < KA; ++a) tma_load_4d(&map_k, &full[s], smem + OFF_K + s * K_BYTES + a * ATOM_BYTES, 64 * a, j * BKV, h, n);
#pragma unroll
    for (int b = 0; b < 2; ++b) tma_load_3d(&map_v, &full[s], smem + OFF_V + s * V_BYTES + b * VBOX, j * BKV + 64 * b, h * D, n);
  };
  if (threadIdx.x == 0) {
    mbar_init(qbar, 1); mbar_init(&full[0], 1); mbar_init(&full[1], 1);
    mbar_init_fence();
    mbar_expect_tx(qbar, KA * ATOM_BYTES);
#pragma unroll
    for (int a = 0; a < KA; ++a) tma_load_4d(&map_q, qbar, smem + a * ATOM_BYTES, 64 * a, q0, h, n);
    load_kv(0);
    if (nkv > 1) load_kv(1);
  }
  __syncthreads();

  float o[DV / 2];
#pragma unroll
  for (int i = 0; i < DV / 2; ++i) o[i] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;     // rows r, r + 8; l is this thread's partial row sum
  const float sl2 = p.scale_log2e;
  const uint32_t sq = smem_u32(smem) + (uint32_t)wg * (64 * 128);
  mbar_wait(qbar, 0);
  for (int j = 0; j < nkv; ++j) {
    const int s = j & 1;
    mbar_wait(&full[s], (uint32_t)(j >> 1) & 1u);
    float sc[BKV / 2];
    const uint32_t sk = smem_u32(smem + OFF_K + s * K_BYTES), sv = smem_u32(smem + OFF_V + s * V_BYTES);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < KS; ++ks)
      Wgmma<BKV, T>::ss(sc, wgmma_desc_sw128(sq + (ks >> 2) * ATOM_BYTES) + 2 * (ks & 3), wgmma_desc_sw128(sk + (ks >> 2) * ATOM_BYTES) + 2 * (ks & 3),
                     ks > 0 ? 1 : 0);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs<BKV / 2>(sc);
    float mx0 = sc[0], mx1 = sc[2];
#pragma unroll
    for (int t = 0; t < BKV / 8; ++t) {
      mx0 = fmaxf(mx0, fmaxf(sc[4 * t], sc[4 * t + 1]));
      mx1 = fmaxf(mx1, fmaxf(sc[4 * t + 2], sc[4 * t + 3]));
    }
    const float mn0 = fmaxf(m0, quad_max(mx0)), mn1 = fmaxf(m1, quad_max(mx1));   // running maxima of the RAW scores (scale > 0)
    const float c0 = ex2_approx((m0 - mn0) * sl2), c1 = ex2_approx((m1 - mn1) * sl2);
    m0 = mn0; m1 = mn1;
    const float nb0 = -mn0 * sl2, nb1 = -mn1 * sl2;
    float rs0 = 0.f, rs1 = 0.f;
#pragma unroll
    for (int t = 0; t < BKV / 8; ++t) {
      sc[4 * t] = ex2_approx(fmaf(sc[4 * t], sl2, nb0)); sc[4 * t + 1] = ex2_approx(fmaf(sc[4 * t + 1], sl2, nb0));
      sc[4 * t + 2] = ex2_approx(fmaf(sc[4 * t + 2], sl2, nb1)); sc[4 * t + 3] = ex2_approx(fmaf(sc[4 * t + 3], sl2, nb1));
      rs0 += sc[4 * t] + sc[4 * t + 1]; rs1 += sc[4 * t + 2] + sc[4 * t + 3];
    }
    l0 = l0 * c0 + rs0; l1 = l1 * c1 + rs1;
#pragma unroll
    for (int t = 0; t < DV / 8; ++t) { o[4 * t] *= c0; o[4 * t + 1] *= c0; o[4 * t + 2] *= c1; o[4 * t + 3] *= c1; }
    uint32_t pa[BKV / 16][4];
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk) pack_a<T>(sc, kk, pa[kk]);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk) Wgmma<DV, T>::rs(o, pa[kk], wgmma_desc_sw128(sv + (kk >> 2) * VBOX) + 2 * (kk & 3), 1);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs<DV / 2>(o);
    __syncthreads();                                 // both warpgroups are done with stage s
    if (threadIdx.x == 0 && j + 2 < nkv) load_kv(j + 2);
  }
  l0 = quad_sum(l0); l1 = quad_sum(l1);
  T* og = (T*)p.out + (int64_t)n * p.bso + (int64_t)h * D;
  const int64_t r0 = q0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
  store_rows<DV, D, T>(og, p.ldo, r0, p.L, o, 1.0f / l0, 1.0f / l1, q);
}

// ------------------------------------------------------------------------------------------------------------------------------
struct AttnCxParams {
  void* out; int64_t ldo, bso;
  int Lq, heads, Lk, Lk2, kv_div, nqt;
  float scale_log2e, out_alpha, alpha2;
};
constexpr int CX_LK = 80, CX_LK2 = 16;

// softmax over the first Lk keys of a single-tile context (NT n-tiles), normalised and pre-scaled by its weight
template <int NT>
__device__ __forceinline__ void softmax_ctx(float* sc, int Lk, float wgt, float sl2, int q) {
  float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
  for (int t = 0; t < NT; ++t)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const bool ok = 8 * t + 2 * q + e < Lk;
      sc[4 * t + e] = ok ? sc[4 * t + e] : -INFINITY; sc[4 * t + 2 + e] = ok ? sc[4 * t + 2 + e] : -INFINITY;
      mx0 = fmaxf(mx0, sc[4 * t + e]); mx1 = fmaxf(mx1, sc[4 * t + 2 + e]);
    }
  const float nb0 = -quad_max(mx0) * sl2, nb1 = -quad_max(mx1) * sl2;
  float rs0 = 0.f, rs1 = 0.f;
#pragma unroll
  for (int t = 0; t < NT; ++t) {
    sc[4 * t] = ex2_approx(fmaf(sc[4 * t], sl2, nb0)); sc[4 * t + 1] = ex2_approx(fmaf(sc[4 * t + 1], sl2, nb0));
    sc[4 * t + 2] = ex2_approx(fmaf(sc[4 * t + 2], sl2, nb1)); sc[4 * t + 3] = ex2_approx(fmaf(sc[4 * t + 3], sl2, nb1));
    rs0 += sc[4 * t] + sc[4 * t + 1]; rs1 += sc[4 * t + 2] + sc[4 * t + 3];
  }
  const float f0 = wgt / quad_sum(rs0), f1 = wgt / quad_sum(rs1);
#pragma unroll
  for (int t = 0; t < NT; ++t) { sc[4 * t] *= f0; sc[4 * t + 1] *= f0; sc[4 * t + 2] *= f1; sc[4 * t + 3] *= f1; }
}

template <int KA, int KS, int DV, int D, typename T>
__global__ void __launch_bounds__(NTHREADS, 1)
attention_cx_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k, const __grid_constant__ CUtensorMap map_v,
                    const __grid_constant__ CUtensorMap map_k2, const __grid_constant__ CUtensorMap map_v2, const AttnCxParams p) {
  constexpr int VBOX = DV * 128;
  constexpr int KT_ATOM = CX_LK * 128, KI_ATOM = CX_LK2 * 128;    // 10 KB / 2 KB per 64-column atom
  constexpr int Q_BYTES = KA * ATOM_BYTES;
  constexpr int OFF_KT = 2 * Q_BYTES, OFF_VT = OFF_KT + KA * KT_ATOM, OFF_KI = OFF_VT + 2 * VBOX, OFF_VI = OFF_KI + KA * KI_ATOM;
  constexpr int OFF_BAR = OFF_VI + VBOX;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + pad1024(smem_raw);
  uint64_t* cbar = reinterpret_cast<uint64_t*>(smem + OFF_BAR);
  uint64_t* qfull = cbar + 1;                      // [2]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2, q = lane & 3;
  const int h = blockIdx.y, n = blockIdx.z, nc = n / p.kv_div;
  const bool two = p.Lk2 > 0;

  auto load_q = [&](int it) {
    const int qt = blockIdx.x + it * gridDim.x;
    mbar_expect_tx(&qfull[it & 1], Q_BYTES);
#pragma unroll
    for (int a = 0; a < KA; ++a) tma_load_3d(&map_q, &qfull[it & 1], smem + (it & 1) * Q_BYTES + a * ATOM_BYTES, h * D + 64 * a, qt * BQ, n);
  };
  if (threadIdx.x == 0) {
    mbar_init(cbar, 1); mbar_init(&qfull[0], 1); mbar_init(&qfull[1], 1);
    mbar_init_fence();
    const int dkp = KA == 1 ? 64 : D;
    mbar_expect_tx(cbar, KA * KT_ATOM + 2 * VBOX + (two ? KA * KI_ATOM + VBOX : 0));
#pragma unroll
    for (int a = 0; a < KA; ++a) tma_load_3d(&map_k, cbar, smem + OFF_KT + a * KT_ATOM, h * dkp + 64 * a, 0, nc);
    for (int b = 0; b < 2; ++b) tma_load_3d(&map_v, cbar, smem + OFF_VT + b * VBOX, 64 * b, h * D, nc);
    if (two) {
#pragma unroll
      for (int a = 0; a < KA; ++a) tma_load_3d(&map_k2, cbar, smem + OFF_KI + a * KI_ATOM, h * dkp + 64 * a, 0, nc);
      tma_load_3d(&map_v2, cbar, smem + OFF_VI, 0, h * D, nc);
    }
    if ((int)blockIdx.x < p.nqt) load_q(0);
    if ((int)blockIdx.x + (int)gridDim.x < p.nqt) load_q(1);
  }
  __syncthreads();
  mbar_wait(cbar, 0);
  const float sl2 = p.scale_log2e;
  const uint32_t skt = smem_u32(smem + OFF_KT), svt = smem_u32(smem + OFF_VT), ski = smem_u32(smem + OFF_KI), svi = smem_u32(smem + OFF_VI);
  T* og = (T*)p.out + (int64_t)n * p.bso + (int64_t)h * D;
  for (int it = 0, qt = blockIdx.x; qt < p.nqt; ++it, qt += gridDim.x) {
    mbar_wait(&qfull[it & 1], (uint32_t)(it >> 1) & 1u);
    const uint32_t sq = smem_u32(smem + (it & 1) * Q_BYTES) + (uint32_t)wg * (64 * 128);
    float st[CX_LK / 2], si[CX_LK2 / 2];
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < KS; ++ks)
      Wgmma<CX_LK, T>::ss(st, wgmma_desc_sw128(sq + (ks >> 2) * ATOM_BYTES) + 2 * (ks & 3), wgmma_desc_sw128(skt + (ks >> 2) * KT_ATOM) + 2 * (ks & 3),
                       ks > 0 ? 1 : 0);
    if (two) {
#pragma unroll
      for (int ks = 0; ks < KS; ++ks)
        Wgmma<CX_LK2, T>::ss(si, wgmma_desc_sw128(sq + (ks >> 2) * ATOM_BYTES) + 2 * (ks & 3), wgmma_desc_sw128(ski + (ks >> 2) * KI_ATOM) + 2 * (ks & 3),
                          ks > 0 ? 1 : 0);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs<CX_LK / 2>(st);
    wgmma_fence_regs<CX_LK2 / 2>(si);
    softmax_ctx<CX_LK / 8>(st, p.Lk, p.out_alpha, sl2, q);
    if (two) softmax_ctx<CX_LK2 / 8>(si, p.Lk2, p.alpha2, sl2, q);
    uint32_t pt[CX_LK / 16][4], pi[4];
#pragma unroll
    for (int kk = 0; kk < CX_LK / 16; ++kk) pack_a<T>(st, kk, pt[kk]);
    pack_a<T>(si, 0, pi);
    float o[DV / 2];
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < CX_LK / 16; ++kk) Wgmma<DV, T>::rs(o, pt[kk], wgmma_desc_sw128(svt + (kk >> 2) * VBOX) + 2 * (kk & 3), kk > 0 ? 1 : 0);
    if (two) Wgmma<DV, T>::rs(o, pi, wgmma_desc_sw128(svi), 1);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs<DV / 2>(o);
    const int64_t r0 = (int64_t)qt * BQ + wg * 64 + (warp & 3) * 16 + (lane >> 2);
    store_rows<DV, D, T>(og, p.ldo, r0, p.Lq, o, 1.0f, 1.0f, q);
    __syncthreads();                                 // both warpgroups are done with this Q buffer
    if (threadIdx.x == 0 && qt + 2 * (int)gridDim.x < p.nqt) load_q(it + 2);
  }
}

template <int KA, int KS, int DV, int D> constexpr int self_smem() { return KA * ATOM_BYTES + 2 * (KA * ATOM_BYTES + 2 * DV * 128) + 64 + 1024; }
template <int KA, int DV> constexpr int cx_smem() { return 2 * KA * ATOM_BYTES + KA * CX_LK * 128 + 2 * DV * 128 + KA * CX_LK2 * 128 + DV * 128 + 64 + 1024; }

// [NB, L, ld] (columns col0 .. col0+C) -> [NB, C, L]   (V -> V^T so that keys are the contiguous, K-major dimension of PV).  It only moves
// 16-bit values, so it serves bf16 and fp16 alike.
__global__ void __launch_bounds__(256) transpose_tokens_kernel(const bf16* __restrict__ in, bf16* __restrict__ out, int L, int C,
                                                               int64_t ld, int64_t col0) {
  __shared__ bf16 tile[64][66];
  const int n = blockIdx.z, t0 = blockIdx.x * 64, c0 = blockIdx.y * 64;
  const bf16* src = in + (int64_t)n * L * ld + col0;
  for (int i = threadIdx.x; i < 64 * 32; i += 256) {        // 64 tokens x 32 channel pairs
    int t = i >> 5, cp = (i & 31) * 2;
    __nv_bfloat162 v = __floats2bfloat162_rn(0.f, 0.f);
    if (t0 + t < L && c0 + cp < C) v = *reinterpret_cast<const __nv_bfloat162*>(src + (int64_t)(t0 + t) * ld + c0 + cp);
    tile[t][cp] = v.x; tile[t][cp + 1] = v.y;
  }
  __syncthreads();
  bf16* dst = out + (int64_t)n * C * L;
  for (int i = threadIdx.x; i < 64 * 32; i += 256) {        // 64 channels x 32 token pairs
    int c = i >> 5, tp = (i & 31) * 2;
    if (c0 + c < C && t0 + tp < L) {
      __nv_bfloat162 v;
      v.x = tile[tp][c]; v.y = tile[tp + 1][c];
      *reinterpret_cast<__nv_bfloat162*>(dst + (int64_t)(c0 + c) * L + t0 + tp) = v;
    }
  }
}

template <int KA, int KS, int DV, int D, typename T>
int32_t launch_self(const CUtensorMap& mq, const CUtensorMap& mk, const CUtensorMap& mv, const AttnTcParams& p, int64_t NB, cudaStream_t st) {
  constexpr int smem = self_smem<KA, KS, DV, D>();
  auto kern = attention_tc_kernel<KA, KS, DV, D, T>;
  static bool attr = false;
  if (!attr) { FYC_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem)); attr = true; }
  dim3 grid((unsigned)(p.L / BQ), (unsigned)p.heads, (unsigned)NB);
  kern<<<grid, NTHREADS, smem, st>>>(mq, mk, mv, p);
  FYC_LAUNCH_CHECK();
  return FYC_OK;
}

template <int KA, int KS, int DV, int D, typename T>
int32_t launch_cx(const CUtensorMap& mq, const CUtensorMap& mk, const CUtensorMap& mv, const CUtensorMap& mk2, const CUtensorMap& mv2,
                  const AttnCxParams& p, dim3 grid, cudaStream_t st) {
  constexpr int smem = cx_smem<KA, DV>();
  auto kern = attention_cx_kernel<KA, KS, DV, D, T>;
  static bool attr = false;
  if (!attr) { FYC_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem)); attr = true; }
  kern<<<grid, NTHREADS, smem, st>>>(mq, mk, mv, mk2, mv2, p);
  FYC_LAUNCH_CHECK();
  return FYC_OK;
}

}  // namespace

extern "C" int32_t fyc_transpose_tokens(const void* in, void* out, int64_t NB, int64_t L, int64_t C, int64_t ld, int64_t col0,
                                        void* stream) {
  FYC_CHECK(C % 2 == 0 && L % 2 == 0 && ld % 2 == 0 && col0 % 2 == 0 && NB < 65536, "transpose_tokens: even sizes required");
  dim3 grid((unsigned)ceil_div64(L, 64), (unsigned)ceil_div64(C, 64), (unsigned)NB);
  transpose_tokens_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((const bf16*)in, (bf16*)out, (int)L, (int)C, ld, col0);
  FYC_LAUNCH_CHECK();
  return FYC_OK;
}

// qk: [NB, L, ldqk] 16-bit (dt) with q head h at columns [q_col0 + 64h, +64) and k head h at [k_col0 + 64h, +64) (D = 40: cols 40..63 zero;
// D = 64: the unpadded fused projection); vt: [NB, heads*D, L]; out: [NB, L, ldo] (head h at columns [h*D, (h+1)*D)).
static int32_t self_attention_tc(int32_t dt, const void* qk, int64_t ldqk, int64_t q_col0, int64_t k_col0, const void* vt, void* out,
                                         int64_t ldo, int64_t NB, int64_t heads, int64_t L, int64_t D, float scale, void* stream) {
  FYC_CHECK(D == 40 || D == 64, "self_attention_tc: built for head dims 40 and 64 (got %lld)", (long long)D);
  FYC_CHECK(L % 128 == 0 && L >= 128, "self_attention_tc: sequence length %lld must be a multiple of 128", (long long)L);
  FYC_CHECK(ldqk % 8 == 0 && q_col0 % 8 == 0 && k_col0 % 8 == 0 && ldo % 8 == 0, "self_attention_tc: 16-byte alignment");
  FYC_CHECK((((uintptr_t)qk | (uintptr_t)vt | (uintptr_t)out) & 15) == 0, "self_attention_tc: pointers must be 16-byte aligned");
  FYC_CHECK(NB < 65536 && heads < 65536, "self_attention_tc: grid too large");
  CUtensorMap mq, mk, mv;
  {
    uint64_t dims[4] = {64, (uint64_t)L, (uint64_t)heads, (uint64_t)NB};
    uint64_t str[3] = {(uint64_t)ldqk * 2, 128, (uint64_t)L * ldqk * 2};
    uint32_t box[4] = {64, (uint32_t)BQ, 1, 1};
    int32_t rc = encode_map(&mq, (const uint16_t*)qk + q_col0, 4, dims, str, box, tma_dtype(dt));
    if (rc) return rc;
    rc = encode_map(&mk, (const uint16_t*)qk + k_col0, 4, dims, str, box, tma_dtype(dt));
    if (rc) return rc;
  }
  {
    uint64_t dims[3] = {(uint64_t)L, (uint64_t)(heads * D), (uint64_t)NB};
    uint64_t str[2] = {(uint64_t)L * 2, (uint64_t)L * heads * D * 2};
    uint32_t box[3] = {64, D == 40 ? 48u : 64u, 1};
    int32_t rc = encode_map(&mv, vt, 3, dims, str, box, tma_dtype(dt));
    if (rc) return rc;
  }
  AttnTcParams p;
  p.out = out; p.ldo = ldo; p.bso = L * ldo; p.L = (int)L; p.heads = (int)heads;
  p.scale_log2e = scale * 1.4426950408889634f;
  FYC_DISPATCH16(dt, {
    if (D == 64) return launch_self<1, 4, 64, 64, T>(mq, mk, mv, p, NB, (cudaStream_t)stream);
    return launch_self<1, 3, 48, 40, T>(mq, mk, mv, p, NB, (cudaStream_t)stream);      // k-step 3 would multiply the zero columns 48..63
  })
  return FYC_OK;
}

// Head dim 80 (level-1 self-attention): qkv [NB, L, ldqkv] 16-bit (dt) with q head h at columns [q_col0 + 80 h, +80), k at [k_col0 + 80 h, +80) -
// UNPADDED, the fused [q | k | v] projection as the GEMM wrote it (reads up to column k_col0 + 80 heads + 47: the buffer must hold at
// least 48 more columns after k's last head, which the v block provides); vt: [NB, heads * 80, L]; out: [NB, L, ldo].
static int32_t self_attention_tc_d80(int32_t dt, const void* qkv, int64_t ldqkv, int64_t q_col0, int64_t k_col0, const void* vt, void* out,
                                             int64_t ldo, int64_t NB, int64_t heads, int64_t L, float scale, void* stream) {
  constexpr int D = 80;
  FYC_CHECK(L % (2 * BQ) == 0 && L >= 2 * BQ, "self_attention_tc_d80: sequence length %lld must be a multiple of 256", (long long)L);
  FYC_CHECK(ldqkv % 8 == 0 && q_col0 % 8 == 0 && k_col0 % 8 == 0 && ldo % 8 == 0, "self_attention_tc_d80: 16-byte alignment");
  FYC_CHECK((((uintptr_t)qkv | (uintptr_t)vt | (uintptr_t)out) & 15) == 0, "self_attention_tc_d80: pointers must be 16-byte aligned");
  FYC_CHECK(NB < 65536 && heads < 65536, "self_attention_tc_d80: grid too large");
  FYC_CHECK(q_col0 + heads * D + 48 <= ldqkv && k_col0 + heads * D + 48 <= ldqkv, "self_attention_tc_d80: the row must extend 48 columns past the last head");
  CUtensorMap mq, mk, mv;
  {
    // inner extent 128 columns per head although heads are 160 bytes apart: overlapping tensor-map dimensions are legal, and the second
    // atom's foreign columns are never multiplied (5 k-steps)
    uint64_t dims[4] = {128, (uint64_t)L, (uint64_t)heads, (uint64_t)NB};
    uint64_t str[3] = {(uint64_t)ldqkv * 2, (uint64_t)D * 2, (uint64_t)L * ldqkv * 2};
    uint32_t box[4] = {64, (uint32_t)BQ, 1, 1};
    int32_t rc = encode_map(&mq, (const uint16_t*)qkv + q_col0, 4, dims, str, box, tma_dtype(dt));
    if (rc) return rc;
    rc = encode_map(&mk, (const uint16_t*)qkv + k_col0, 4, dims, str, box, tma_dtype(dt));
    if (rc) return rc;
  }
  {
    uint64_t dims[3] = {(uint64_t)L, (uint64_t)(heads * D), (uint64_t)NB};
    uint64_t str[2] = {(uint64_t)L * 2, (uint64_t)L * heads * D * 2};
    uint32_t box[3] = {64, (uint32_t)D, 1};
    int32_t rc = encode_map(&mv, vt, 3, dims, str, box, tma_dtype(dt));
    if (rc) return rc;
  }
  AttnTcParams p;
  p.out = out; p.ldo = ldo; p.bso = L * ldo; p.L = (int)L; p.heads = (int)heads;
  p.scale_log2e = scale * 1.4426950408889634f;
  FYC_DISPATCH16(dt, return launch_self<2, 5, 80, 80, T>(mq, mk, mv, p, NB, (cudaStream_t)stream))
  return FYC_OK;
}

// Cross-attention with a resident short context on tensor cores (head dim 40, 64 or 80).  q: [NB, Lq, ldq] 16-bit (dt), head h at columns [q_col0 + D h, +D),
// UNPADDED, ldq >= heads * D;
// k: [NBc, 80, ldk] with head h at columns [DKP h, +D), DKP = 64 for D = 40 (columns D..63 ZERO) or 64, 80 for D = 80, rows Lk..79 zero;
// vt: [NBc, heads * D, 80]; optional second context k2 [NBc, 16, ldk2], vt2 [NBc, heads * D, 16] (rows / columns Lk2..15 zero).
// out[n, i, h D + :] = out_alpha softmax_j<Lk(scale q k^T) v + alpha2 softmax_j<Lk2(scale q k2^T) v2, NBc = NB / kv_batch_div.
static int32_t cross_attention_tc(int32_t dt, const void* q, int64_t ldq, int64_t q_col0, const void* k, int64_t ldk, const void* vt,
                                          const void* k2, int64_t ldk2, const void* vt2, void* out, int64_t ldo, int64_t NB, int64_t heads,
                                          int64_t Lq, int64_t D, int64_t Lk, int64_t Lk2, int64_t kv_batch_div, float scale, float out_alpha,
                                          float alpha2, void* stream) {
  FYC_CHECK(D == 40 || D == 64 || D == 80, "cross_attention_tc: head dim %lld (40, 64 or 80)", (long long)D);
  FYC_CHECK(Lk >= 1 && Lk <= CX_LK && Lk2 >= 0 && Lk2 <= CX_LK2 && Lq >= 1 && kv_batch_div >= 1 && NB % kv_batch_div == 0, "cross_attention_tc: bad shape");
  FYC_CHECK((k2 != nullptr) == (Lk2 > 0) && (vt2 != nullptr) == (Lk2 > 0), "cross_attention_tc: second context needs k2, vt2 and Lk2 > 0");
  FYC_CHECK(ldq % 8 == 0 && q_col0 % 8 == 0 && ldk % 8 == 0 && ldo % 8 == 0 && (k2 == nullptr || ldk2 % 8 == 0), "cross_attention_tc: 16-byte alignment");
  FYC_CHECK((((uintptr_t)q | (uintptr_t)k | (uintptr_t)vt | (uintptr_t)out | (uintptr_t)k2 | (uintptr_t)vt2) & 15) == 0, "cross_attention_tc: pointers must be 16-byte aligned");
  FYC_CHECK(NB < 65536 && heads < 65536, "cross_attention_tc: grid too large");
  const int64_t NBc = NB / kv_batch_div;
  const int64_t DKP = D == 80 ? 80 : 64;
  const uint32_t DV = D == 40 ? 48 : (uint32_t)D;
  CUtensorMap mq, mk, mv, mk2, mv2;
  {
    // q and k as 3-D maps over the WHOLE head-packed row (box origin = the head's first column): columns past the row end - the tail
    // of the last head's 64-column atom - are out of bounds for TMA and zero-filled instead of read
    uint64_t dims[3] = {(uint64_t)(heads * D), (uint64_t)Lq, (uint64_t)NB};
    uint64_t str[2] = {(uint64_t)ldq * 2, (uint64_t)Lq * ldq * 2};
    uint32_t box[3] = {64, (uint32_t)BQ, 1};
    int32_t rc = encode_map(&mq, (const uint16_t*)q + q_col0, 3, dims, str, box, tma_dtype(dt));
    if (rc) return rc;
  }
  {
    uint64_t dims[3] = {(uint64_t)(heads * DKP), (uint64_t)CX_LK, (uint64_t)NBc};
    uint64_t str[2] = {(uint64_t)ldk * 2, (uint64_t)CX_LK * ldk * 2};
    uint32_t box[3] = {64, (uint32_t)CX_LK, 1};
    int32_t rc = encode_map(&mk, k, 3, dims, str, box, tma_dtype(dt));
    if (rc) return rc;
    uint64_t vd[3] = {(uint64_t)CX_LK, (uint64_t)(heads * D), (uint64_t)NBc};
    uint64_t vs[2] = {CX_LK * 2, (uint64_t)(CX_LK * heads * D * 2)};
    uint32_t vb[3] = {64, DV, 1};
    rc = encode_map(&mv, vt, 3, vd, vs, vb, tma_dtype(dt));
    if (rc) return rc;
  }
  mk2 = mk; mv2 = mv;
  if (k2) {
    uint64_t dims[3] = {(uint64_t)(heads * DKP), (uint64_t)CX_LK2, (uint64_t)NBc};
    uint64_t str[2] = {(uint64_t)ldk2 * 2, (uint64_t)CX_LK2 * ldk2 * 2};
    uint32_t box[3] = {64, (uint32_t)CX_LK2, 1};
    int32_t rc = encode_map(&mk2, k2, 3, dims, str, box, tma_dtype(dt));
    if (rc) return rc;
    uint64_t vd[3] = {(uint64_t)CX_LK2, (uint64_t)(heads * D), (uint64_t)NBc};
    uint64_t vs[2] = {CX_LK2 * 2, (uint64_t)(CX_LK2 * heads * D * 2)};
    uint32_t vb[3] = {64, DV, 1};
    rc = encode_map(&mv2, vt2, 3, vd, vs, vb, tma_dtype(dt));
    if (rc) return rc;
  }
  AttnCxParams p;
  p.out = out; p.ldo = ldo; p.bso = Lq * ldo; p.Lq = (int)Lq; p.heads = (int)heads; p.Lk = (int)Lk; p.Lk2 = (int)Lk2;
  p.kv_div = (int)kv_batch_div; p.scale_log2e = scale * 1.4426950408889634f; p.out_alpha = out_alpha; p.alpha2 = alpha2;
  p.nqt = (int)((Lq + BQ - 1) / BQ);
  // CTAs per (image, head): enough to fill the machine once (one CTA per SM), at most one per pair of query tiles - the context load is
  // paid once per CTA
  int64_t gx = ((int64_t)fyc_sm_count() + heads * NB - 1) / (heads * NB);
  if (gx < 1) gx = 1;
  if (gx > (p.nqt + 1) / 2) gx = (p.nqt + 1) / 2;
  dim3 grid((unsigned)gx, (unsigned)heads, (unsigned)NB);
  cudaStream_t st = (cudaStream_t)stream;
  FYC_DISPATCH16(dt, {
    if (D == 40) return launch_cx<1, 3, 48, 40, T>(mq, mk, mv, mk2, mv2, p, grid, st);
    if (D == 64) return launch_cx<1, 4, 64, 64, T>(mq, mk, mv, mk2, mv2, p, grid, st);
    return launch_cx<2, 5, 80, 80, T>(mq, mk, mv, mk2, mv2, p, grid, st);
  })
  return FYC_OK;
}

extern "C" int32_t fyc_self_attention_tc(const void* qk, int64_t ldqk, int64_t q_col0, int64_t k_col0, const void* vt, void* out,
                                         int64_t ldo, int64_t NB, int64_t heads, int64_t L, int64_t D, float scale, void* stream) {
  return self_attention_tc(FYC_BF16, qk, ldqk, q_col0, k_col0, vt, out, ldo, NB, heads, L, D, scale, stream);
}
extern "C" int32_t fyc_self_attention_tc_f16(const void* qk, int64_t ldqk, int64_t q_col0, int64_t k_col0, const void* vt, void* out,
                                             int64_t ldo, int64_t NB, int64_t heads, int64_t L, int64_t D, float scale, void* stream) {
  return self_attention_tc(FYC_F16, qk, ldqk, q_col0, k_col0, vt, out, ldo, NB, heads, L, D, scale, stream);
}
extern "C" int32_t fyc_self_attention_tc_d80(const void* qkv, int64_t ldqkv, int64_t q_col0, int64_t k_col0, const void* vt, void* out,
                                             int64_t ldo, int64_t NB, int64_t heads, int64_t L, float scale, void* stream) {
  return self_attention_tc_d80(FYC_BF16, qkv, ldqkv, q_col0, k_col0, vt, out, ldo, NB, heads, L, scale, stream);
}
extern "C" int32_t fyc_self_attention_tc_d80_f16(const void* qkv, int64_t ldqkv, int64_t q_col0, int64_t k_col0, const void* vt, void* out,
                                                 int64_t ldo, int64_t NB, int64_t heads, int64_t L, float scale, void* stream) {
  return self_attention_tc_d80(FYC_F16, qkv, ldqkv, q_col0, k_col0, vt, out, ldo, NB, heads, L, scale, stream);
}
extern "C" int32_t fyc_cross_attention_tc(const void* q, int64_t ldq, int64_t q_col0, const void* k, int64_t ldk, const void* vt,
                                          const void* k2, int64_t ldk2, const void* vt2, void* out, int64_t ldo, int64_t NB, int64_t heads,
                                          int64_t Lq, int64_t D, int64_t Lk, int64_t Lk2, int64_t kv_batch_div, float scale, float out_alpha,
                                          float alpha2, void* stream) {
  return cross_attention_tc(FYC_BF16, q, ldq, q_col0, k, ldk, vt, k2, ldk2, vt2, out, ldo, NB, heads, Lq, D, Lk, Lk2, kv_batch_div, scale,
                            out_alpha, alpha2, stream);
}
extern "C" int32_t fyc_cross_attention_tc_f16(const void* q, int64_t ldq, int64_t q_col0, const void* k, int64_t ldk, const void* vt,
                                              const void* k2, int64_t ldk2, const void* vt2, void* out, int64_t ldo, int64_t NB, int64_t heads,
                                              int64_t Lq, int64_t D, int64_t Lk, int64_t Lk2, int64_t kv_batch_div, float scale, float out_alpha,
                                              float alpha2, void* stream) {
  return cross_attention_tc(FYC_F16, q, ldq, q_col0, k, ldk, vt, k2, ldk2, vt2, out, ldo, NB, heads, Lq, D, Lk, Lk2, kv_batch_div, scale,
                            out_alpha, alpha2, stream);
}
