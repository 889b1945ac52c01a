// Hopper (sm_90a) tensor-core GEMM / implicit-GEMM 3x3 convolution.
//
//   out[p, n] = epilogue( alpha * sum_{tap, c} X[pixel(p) + (dy,dx)(tap), c] * W[n, tap, c] )
//
// One persistent CTA per SM, 9 warps:
//   warp 8 (1 lane)  TMA producer : cp.async.bulk.tensor (4-D box for the activation patch, 3-D box for the weight slab) into a
//                                   3- or 4-stage 128B-swizzled shared-memory ring, mbarrier expect_tx
//   warps 0..7       two consumer warpgroups, 64 rows of the 128-row tile each: wgmma.mma_async m64 x BN x 16 (bf16 or fp16 -> fp32
//                    register accumulators) straight from the swizzled stages, then the fused epilogue (bias / time-embedding
//                    row bias / residual / GEGLU / LayerNorm fold / alpha) on the registers into the warpgroup's own shared-memory
//                    staging buffer, which one thread writes out with TMA stores (clipped at the output's true extent).
// The producer runs ahead across tile boundaries, so the next tile's operands stream in while the consumers run the epilogue.
// The residual half-tile is TMA-loaded into the staging buffer at the start of the tile, so it lands during the mainloop; the
// TMA stores of a tile drain while the warpgroup runs the next tile's MMAs.
// The 3x3 convolution never builds an im2col matrix: for each filter tap the producer loads the SAME 4-D box shifted
// by (dy, dx); TMA's out-of-bounds zero fill implements the padding halo.  A plain GEMM is the 1-tap special case.
// Stride-2 convolutions run on a parity-plane split of the input (fyc_space_to_planes), which turns every tap into
// a unit-stride shifted read of one plane (tap_img selects the plane).
#include "tma.cuh"
#include "wgmma.cuh"

namespace {

constexpr int BM = 128;            // rows (output pixels) per tile: two warpgroups x 64
constexpr int BK = 64;             // K per stage = one 128-byte swizzle row of bf16
constexpr int STAGES = 4;          // plain-mode stages when the ring has room for them
constexpr int A_BYTES = BM * BK * 2;           // 16 KB
constexpr int MAX_STAGES = 8;                   // barrier slots; the W-resident mode runs up to 8 A-only stages
constexpr int MAX_RING_BYTES = 192 * 1024;      // operand ring (or W slab + A ring): 4 stages of a BN = 256 tile
constexpr int SMEM_LIMIT = 232448;              // 227 KB: the per-block opt-in maximum of sm_90
constexpr int SMEM_EXTRA = 256 + 1024;          // barriers + slack to align the ring to 1024 B
// Output staging: each warpgroup writes its 64-row half-tile into its own buffer as 32-byte-wide column boxes (16 bf16 or 8 fp32
// columns, 64 rows x 32 B = 2 KB each, CU_TENSOR_MAP_SWIZZLE_32B).  Every BN is a multiple of 16, so a tile is a whole number of
// boxes and no box reaches into the next tile's columns; a warp's 4- or 8-byte fragment stores hit 32 distinct banks per wavefront.
constexpr int OUT_BOX_BYTES = 32;
constexpr int OUT_BOX_SMEM = 64 * OUT_BOX_BYTES;   // 2 KB
constexpr int NUM_THREADS = 288;          // 2 consumer warpgroups + the TMA warp

struct TcParams {
  // problem
  int64_t M;                 // valid output rows (pixels)
  int N, N_out;              // accumulator columns / stored columns (N/2 for GEGLU)
  int taps, cin_blocks;      // K loop = taps x cin_blocks
  int BN, n_tiles;
  // output-pixel tiling: tile = bn images x bh rows x bw cols; Wt = ceil(Wo / bw) tiles per row, etc.
  int bw, bh, bn, Wo, Ho, w_tiles, h_tiles;
  int lg_bw, lg_bh;          // log2 of bw, bh (both powers of two)
  int64_t m_tiles;
  int tap_dy[9], tap_dx[9], tap_img[9];
  // epilogue; the output and residual are addressed by their tensor maps
  const float* bias; const float* rowbias;
  int64_t rows_per_group;
  int64_t ldrb;              // row stride of rowbias (elements; N unless the caller passes a slice of a wider table)
  float alpha;
  int flags;
  // two-segment K (fyc_gemm_args.A2): k blocks [0, cb_split) of a tap come from map_a, the rest from map_a2 (INT_MAX: single source)
  int cb_split;
  // LayerNorm folded into the GEMM (FYC_EPI_LNFOLD): per-row rstd; the mean subtraction is in the (row-centred) weights
  const float* ln_rs;
  // W-resident mode (small K): the CTA keeps its whole BN x K weight slab in shared memory and only streams A
  int resident, a_stages;
  // shared memory: [operand ring: ring_bytes][staging warpgroup 0 | 1: stg_bytes each][barriers]
  int ring_bytes, stg_bytes;
  // output / residual box origin of warpgroup 1's half-tile relative to warpgroup 0's, in (w, h, image): the patch is halved
  // along its outermost dimension that is wider than 1
  int half_dw, half_dh, half_dn;
};

// ---------------------------------------------------------------------------------------------- warpgroup barrier
// named barrier over one consumer warpgroup (id 0 is __syncthreads)
__device__ __forceinline__ void warpgroup_sync(int wg) {
  if (wg == 0) asm volatile("bar.sync 1, 128;" ::: "memory");
  else asm volatile("bar.sync 2, 128;" ::: "memory");
}

// ---------------------------------------------------------------------------------------------- tile coordinates
struct TileCoord { int n, w, h, i; };   // n block; patch column / row / image-group of the 128-pixel m block
__device__ __forceinline__ TileCoord tile_coord(const TcParams& p, int64_t t) {
  TileCoord c;
  const uint32_t tile = (uint32_t)t;
  c.n = (int)(tile % (uint32_t)p.n_tiles);
  const uint32_t m_blk = tile / (uint32_t)p.n_tiles;
  c.w = (int)(m_blk % (uint32_t)p.w_tiles);
  const uint32_t m2 = m_blk / (uint32_t)p.w_tiles;
  c.h = (int)(m2 % (uint32_t)p.h_tiles);
  c.i = (int)(m2 / (uint32_t)p.h_tiles);
  return c;
}

// output pixel of patch row r of tile c (-1: outside the output)
__device__ __forceinline__ int64_t tile_pixel(const TcParams& p, const TileCoord& c, int r) {
  const int ow = c.w * p.bw + (r & (p.bw - 1)), oh = c.h * p.bh + ((r >> p.lg_bw) & (p.bh - 1));
  const int img = c.i * p.bn + (r >> (p.lg_bw + p.lg_bh));
  const int64_t pix = ((int64_t)img * p.Ho + oh) * p.Wo + ow;
  return ((ow < p.Wo) && (oh < p.Ho) && (pix < p.M)) ? pix : -1;
}

// ---------------------------------------------------------------------------------------------- epilogue
// Byte offset of (row, col) of a half-tile in the staging layout: column box col / (32 / esize), then row, in the 32-byte
// swizzle TMA applies (16-byte chunk index XOR row bit 2; the staging buffers are 1024-byte aligned).
__device__ __forceinline__ uint32_t stage_off(int row, int col, int esize) {
  const int cpb = OUT_BOX_BYTES / esize;
  const uint32_t in_box = (uint32_t)(row * OUT_BOX_BYTES + (col % cpb) * esize);
  return (uint32_t)(col / cpb) * OUT_BOX_SMEM + (in_box ^ (((in_box >> 7) & 1u) << 4));
}

// The accumulator of warpgroup wg holds rows wg*64 + 16*warp + lane/4 (+8) of the tile; n-tile j (8 columns) sits in acc[4j .. 4j+3]:
// columns 8j + 2(lane%4) + {0, 1} of the first row, then of the second.  The results go to the warpgroup's staging buffer `stg`,
// which holds the residual half-tile on entry when there is one; each thread reads its residual where it then writes its result.
template <int BN, typename T>
__device__ __forceinline__ void epilogue(const TcParams& p, const TileCoord& c, const float* acc, int wg, int warp4, int lane, uint8_t* stg) {
  const int q = lane & 3;
  const int flags = p.flags;
  const bool geglu = flags & FYC_EPI_GEGLU, out_f32 = flags & FYC_EPI_OUT_F32, lnf = flags & FYC_EPI_LNFOLD;
  const bool has_bias = flags & FYC_EPI_BIAS, has_res = flags & FYC_EPI_RESIDUAL, has_rb = flags & FYC_EPI_ROWBIAS;
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    const int row = warp4 * 16 + (lane >> 2) + 8 * half;       // row of the warpgroup's 64-row half-tile
    const int64_t pix = tile_pixel(p, c, wg * 64 + row);
    if (pix < 0) continue;                                      // beyond M: the TMA store clips the row
    const float rs = lnf ? __ldg(p.ln_rs + pix) : 1.0f;
    const float* rb = has_rb ? p.rowbias + (pix / p.rows_per_group) * p.ldrb : nullptr;
    if (geglu) {
      if constexpr (BN == 256) {
        // columns [0,128) of the tile are `a`, [128,256) the matching gate (weight rows pre-interleaved per 128 outputs)
        const float* bp = p.bias + c.n * 256;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int col = 8 * j + 2 * q;
          if (c.n * 128 + col >= p.N_out) continue;
          const float2 ba = __ldg(reinterpret_cast<const float2*>(bp + col)), bg = __ldg(reinterpret_cast<const float2*>(bp + 128 + col));
          const float a0 = acc[4 * j + 2 * half], a1 = acc[4 * j + 2 * half + 1];
          const float g0 = acc[4 * (j + 16) + 2 * half], g1 = acc[4 * (j + 16) + 2 * half + 1];
          const float x = fmaf(a0, rs, ba.x) * gelu_erf_fast(fmaf(g0, rs, bg.x));
          const float y = fmaf(a1, rs, ba.y) * gelu_erf_fast(fmaf(g1, rs, bg.y));
          *reinterpret_cast<typename Pair16<T>::type*>(stg + stage_off(row, col, 2)) = Pair16<T>::pack(x, y);
        }
      }
      continue;
    }
    const float scale = lnf ? rs : p.alpha;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int col = 8 * j + 2 * q, n = c.n * BN + col;
      if (n >= p.N) continue;
      float x = acc[4 * j + 2 * half] * scale, y = acc[4 * j + 2 * half + 1] * scale;
      if (has_bias) { const float2 b = __ldg(reinterpret_cast<const float2*>(p.bias + n)); x += b.x; y += b.y; }
      if (has_rb) { const float2 b = __ldg(reinterpret_cast<const float2*>(rb + n)); x += b.x; y += b.y; }
      if (out_f32) {
        float2* s = reinterpret_cast<float2*>(stg + stage_off(row, col, 4));
        if (has_res) { const float2 r = *s; x += r.x; y += r.y; }
        *s = make_float2(x, y);
      } else {
        typename Pair16<T>::type* s = reinterpret_cast<typename Pair16<T>::type*>(stg + stage_off(row, col, 2));
        if (has_res) { const float2 r = Pair16<T>::unpack(*s); x += r.x; y += r.y; }
        *s = Pair16<T>::pack(x, y);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------- kernel
// T: the 16-bit operand / output type (bf16 | f16)
template <int BN, typename T>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_w, const __grid_constant__ CUtensorMap map_a2,
               const __grid_constant__ CUtensorMap map_out, const __grid_constant__ CUtensorMap map_res, const TcParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + pad1024(smem_raw);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + p.ring_bytes + 2 * p.stg_bytes);
  uint64_t* full = bars;                       // [MAX_STAGES]
  uint64_t* empty = bars + MAX_STAGES;         // [MAX_STAGES]
  uint64_t* wbar = bars + 2 * MAX_STAGES;      // W-resident mode: the weight slab has landed
  uint64_t* rbar = wbar + 1;                   // [2] the residual half-tile of warpgroup 0 / 1 has landed in its staging buffer
  // operand ring, two layouts:
  //   plain     [A 16 KB | W BN x 128 B] x a_stages
  //   resident  [W slab k_iters x BN x 128 B][A 16 KB x a_stages]
  const int nstages = p.a_stages;
  const uint32_t slab_kb = (uint32_t)BN * (BK * 2);
  const uint32_t a_base = p.resident ? (uint32_t)(p.taps * p.cin_blocks) * slab_kb : 0u;
  const uint32_t a_stride = p.resident ? (uint32_t)A_BYTES : (uint32_t)A_BYTES + slab_kb;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int k_iters = p.taps * p.cin_blocks;
  const int64_t num_tiles = p.m_tiles * p.n_tiles;

  if (threadIdx.x == 0) {
    for (int s = 0; s < MAX_STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 256); }   // empty: one arrival per consumer thread
    mbar_init(wbar, 1);
    mbar_init(&rbar[0], 1); mbar_init(&rbar[1], 1);
    mbar_init_fence();
  }
  __syncthreads();

  if (warp == 8) {
    // ================================================================== TMA producer
    if (lane == 0) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_a)) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_w)) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_a2)) : "memory");
      int stage = 0; uint32_t phase = 0;
      const uint32_t tx_bytes = p.resident ? (uint32_t)A_BYTES : A_BYTES + slab_kb;
      if (p.resident) {   // grid % n_tiles == 0, so this CTA's n block never changes: load its weight slab once
        const int n_blk = (int)(blockIdx.x % p.n_tiles);
        mbar_expect_tx(wbar, (uint32_t)k_iters * slab_kb);
        for (int k = 0; k < k_iters; ++k)
          tma_load_3d(&map_w, wbar, smem + (uint32_t)k * slab_kb, (k % p.cin_blocks) * BK, k / p.cin_blocks, n_blk * BN);
      }
      for (int64_t tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const TileCoord tc = tile_coord(p, tile);
        const int ow0 = tc.w * p.bw, oh0 = tc.h * p.bh, img0 = tc.i * p.bn;
        for (int tap = 0; tap < p.taps; ++tap) {
          for (int cb = 0; cb < p.cin_blocks; ++cb) {
            mbar_wait(&empty[stage], phase ^ 1);
            uint8_t* sa = smem + a_base + (uint32_t)stage * a_stride;
            const bool seg2 = cb >= p.cb_split;                    // second K segment: the other source tensor, its own channel origin
            const CUtensorMap* ma = seg2 ? &map_a2 : &map_a;
            const int ka = (seg2 ? cb - p.cb_split : cb) * BK;
            mbar_expect_tx(&full[stage], tx_bytes);
            tma_load_4d(ma, &full[stage], sa, ka, ow0 + p.tap_dx[tap], oh0 + p.tap_dy[tap], img0 + p.tap_img[tap]);
            if (!p.resident) tma_load_3d(&map_w, &full[stage], sa + A_BYTES, cb * BK, tap, tc.n * BN);
            if (++stage == nstages) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
    return;
  }
  // ==================================================================== consumer warpgroups
  const int wg = warp >> 2, warp4 = warp & 3;
  // Everything below except rphase is re-derived from the kernel parameters where it is used, so that it does not hold registers
  // across the mainloop (BN = 256 needs 128 of the 168 for its accumulator).
  const bool elected = (threadIdx.x & 127) == 0;                // issues the warpgroup's TMA stores / residual loads
  auto stg = [&]() { return smem + p.ring_bytes + wg * p.stg_bytes; };
  const bool has_res = p.flags & FYC_EPI_RESIDUAL;
  auto cpb = [&]() { return (p.flags & FYC_EPI_OUT_F32) ? OUT_BOX_BYTES / 4 : OUT_BOX_BYTES / 2; };
  if (elected) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_out)) : "memory");
    if (has_res) asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&map_res)) : "memory");
  }
  float acc[BN / 2];
  int stage = 0; uint32_t phase = 0, rphase = 0;
  if (p.resident) mbar_wait(wbar, 0);
  // this warpgroup's half of tile t: output columns [col0, col0 + nbox * cpb), box origin (bw0, bh0, bn0); live is false only for
  // the rows past M of a plain GEMM's last tile.  Evaluated before and again after the mainloop, so nothing of it stays in registers
  // across the MMAs.
  auto half_tile = [&](int64_t t, int& col0, int& nbox, int& bw0, int& bh0, int& bn0) {
    const TileCoord tc = tile_coord(p, t);
    const int bn_out = (p.flags & FYC_EPI_GEGLU) ? BN / 2 : BN;
    col0 = tc.n * bn_out;
    nbox = min(bn_out, p.N_out - col0) / cpb();
    bw0 = tc.w * p.bw + wg * p.half_dw; bh0 = tc.h * p.bh + wg * p.half_dh; bn0 = tc.i * p.bn + wg * p.half_dn;
    return tile_pixel(p, tc, wg * 64) >= 0;
  };
  for (int64_t tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    if (has_res && elected) {
      int col0, nbox, bw0, bh0, bn0;
      if (half_tile(tile, col0, nbox, bw0, bh0, bn0)) {
        bulk_wait_read();                                        // the previous tile's stores have read the staging buffer
        mbar_expect_tx(&rbar[wg], (uint32_t)(nbox * OUT_BOX_SMEM));
        for (int b = 0; b < nbox; ++b) tma_load_4d(&map_res, &rbar[wg], stg() + b * OUT_BOX_SMEM, col0 + b * cpb(), bw0, bh0, bn0);
      }
    }
    int prev = -1;
    for (int k = 0; k < k_iters; ++k) {
      mbar_wait(&full[stage], phase);
      const uint32_t sa = smem_u32(smem + a_base + (uint32_t)stage * a_stride) + (uint32_t)wg * (64 * BK * 2);
      const uint64_t a_desc = wgmma_desc_sw128(sa);
      const uint64_t b_desc = wgmma_desc_sw128(p.resident ? smem_u32(smem) + (uint32_t)k * slab_kb : smem_u32(smem + (uint32_t)stage * a_stride) + A_BYTES);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < BK / 16; ++kk)
        Wgmma<BN, T>::ss(acc, a_desc + (uint64_t)(2 * kk), b_desc + (uint64_t)(2 * kk), (k > 0 || kk > 0) ? 1 : 0);
      wgmma_commit();
      wgmma_wait<1>();                                   // the previous stage's MMAs have retired: hand it back to the producer
      if (prev >= 0) mbar_arrive(&empty[prev]);
      prev = stage;
      if (++stage == nstages) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_fence_regs<BN / 2>(acc);
    mbar_arrive(&empty[prev]);
    int col0, nbox, bw0, bh0, bn0;
    if (!half_tile(tile, col0, nbox, bw0, bh0, bn0)) continue;
    if (elected) bulk_wait_read();
    warpgroup_sync(wg);                                          // the staging buffer is free (and holds the residual, if any)
    if (has_res) { mbar_wait(&rbar[wg], rphase); rphase ^= 1; }
    epilogue<BN, T>(p, tile_coord(p, tile), acc, wg, warp4, lane, stg());
    fence_async_smem();
    warpgroup_sync(wg);
    if (elected) {
      for (int b = 0; b < nbox; ++b) tma_store_4d(&map_out, stg() + b * OUT_BOX_SMEM, col0 + b * cpb(), bw0, bh0, bn0);
      bulk_commit();
    }
  }
  // no CTA may exit while its TMA stores still read its shared memory
  if (elected) bulk_wait_all();
}

// parity-plane split for stride-2 convolutions: x [NB, H, W, C] -> planes [4, NB, H/2, W/2, C], plane = 2*(h&1) + (w&1).  A pure copy of
// 16-byte vectors: it serves every 16-bit element type.
__global__ void space_to_planes_kernel(const bf16* __restrict__ x, bf16* __restrict__ out, int64_t NB, int64_t H, int64_t W, int64_t C) {
  const int64_t cv = C / 8, H2 = H / 2, W2 = W / 2;
  const int64_t total = NB * H * W * cv;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t c = (i % cv) * 8; int64_t t = i / cv;
    int64_t w = t % W; t /= W;
    int64_t h = t % H; int64_t n = t / H;
    int64_t plane = 2 * (h & 1) + (w & 1);
    bf16* dst = out + ((((plane * NB + n) * H2) + h / 2) * W2 + w / 2) * C + c;
    *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(x + i * 8);
  }
}

// ---------------------------------------------------------------------------------------------- host side
// Output (or residual) map of a launch: `cols` channels by W x H x NB pixels at `base`, pixel (w, h, n) at element offset
// w * sw + h * sh + n * sn.  The dimensions are the tensor's true extent, so TMA clips the rows past M and the columns past N_out.
// Box: one 32-byte column box of a warpgroup's half patch (choose_tiles sets the split).
int32_t encode_out_map(CUtensorMap* m, const void* base, const TcParams& p, int32_t dt, uint64_t cols, uint64_t W, uint64_t H, uint64_t NB,
                       uint64_t sw, uint64_t sh, uint64_t sn) {
  const bool f32 = (p.flags & FYC_EPI_OUT_F32) != 0;
  const uint64_t es = f32 ? 4 : 2;
  uint64_t dims[4] = {cols, W, H, NB};
  uint64_t str[3] = {sw * es, sh * es, sn * es};
  uint32_t box[4] = {(uint32_t)(OUT_BOX_BYTES / es), (uint32_t)(p.half_dw ? p.half_dw : p.bw), (uint32_t)(p.half_dh ? p.half_dh : p.bh),
                     (uint32_t)(p.half_dn ? p.half_dn : p.bn)};
  return encode_map(m, base, 4, dims, str, box, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : tma_dtype(dt),
                    CU_TENSOR_MAP_SWIZZLE_32B);
}

// accumulator widths with a kernel instantiation (wgmma N)
constexpr int BN_CHOICES[] = {256, 192, 160, 128, 96, 80, 64, 48, 32, 16};
// fp32 output: BN <= 128 keeps a warpgroup's staging buffer (64 x BN x 4 B) within 32 KB
constexpr int MAX_BN_F32 = 128;

int pick_bn(int64_t N, bool geglu, bool f32) {
  if (geglu) return 256;
  for (int bn : BN_CHOICES)
    if (N % bn == 0 && (!f32 || bn <= MAX_BN_F32)) return bn;
  return 16;                            // N % 16 == 0 checked by the caller
}

// Shared-memory budget of one CTA (227 KB opt-in = 232 448 B):
//   staging  2 x 64 x BN_out x (2 or 4 B)  <= 64 KB  (bf16 BN = 256: 2 x 32 KB; GEGLU: 2 x 16 KB; fp32 BN <= 128: 2 x 32 KB)
//   barriers + alignment slack  1 280 B
//   operand ring  the rest rounded down to 1 KB, at most 192 KB: bf16 BN = 256 -> 161 KB (3 plain stages of 48 KB),
//                 BN = 160 -> 185 KB (4 plain stages of 36 KB; W-resident K = 320: 100 KB slab + 5 A stages), GEGLU -> 192 KB
int stg_bytes_for(int bn, int flags) {
  const int bn_out = (flags & FYC_EPI_GEGLU) ? bn / 2 : bn;
  return 64 * bn_out * ((flags & FYC_EPI_OUT_F32) ? 4 : 2);
}
int ring_bytes_for(int bn, int flags) {
  const int avail = (SMEM_LIMIT - SMEM_EXTRA - 2 * stg_bytes_for(bn, flags)) & ~1023;
  return avail < MAX_RING_BYTES ? avail : MAX_RING_BYTES;
}

// Tile width, operand-staging mode and grid for one launch.
//  * default: the largest instantiated BN <= 256 dividing N (fewest re-reads of the A tiles through L2);
//  * few rounds of tiles per SM (small M): BN that minimises rounds x (BN + fixed cost) - a 2.2-round launch at BN = 256 runs as
//    3 full rounds, the same problem at a narrower BN as more, shorter rounds (ragged last N tile is zero-filled by TMA and clipped
//    by the output map);
//  * small K (the slab k_iters x BN x 128 B leaves room for >= 3 A stages) and many tiles per CTA: W-resident - the grid is
//    rounded down to a multiple of n_tiles so a CTA's n block is fixed, its weight slab is loaded once, and the ring streams only A
//    (L2 -> SM traffic per tile drops from (128 + BN) x K to 128 x K elements).
// Also sets the shared-memory split and the warpgroup half of the output patch.
void choose_tiles(TcParams& p, int* grid_out) {
  const int sms = fyc_sm_count();
  const bool geglu = (p.flags & FYC_EPI_GEGLU) != 0, f32 = (p.flags & FYC_EPI_OUT_F32) != 0;
  const int max_bn = f32 ? MAX_BN_F32 : 256;
  const int k_iters = p.taps * p.cin_blocks;
  p.resident = 0;
  p.BN = pick_bn(p.N, geglu, f32);
  p.n_tiles = (int)ceil_div64(p.N, p.BN);
  p.half_dw = p.half_dh = p.half_dn = 0;
  if (p.bn >= 2) p.half_dn = p.bn / 2;
  else if (p.bh >= 2) p.half_dh = p.bh / 2;
  else p.half_dw = p.bw / 2;
  int grid = 0;
  if (!geglu) {
    // W-resident candidate
    int rbn = 0;
    for (int min_stages = 4; min_stages >= 3 && !rbn; --min_stages)      // prefer a slab that leaves a 4-stage A ring; settle for 3
      for (int bn : BN_CHOICES)
        if (bn >= 128 && bn <= max_bn && p.N % bn == 0 &&
            (int64_t)k_iters * bn * 128 <= ring_bytes_for(bn, p.flags) - min_stages * A_BYTES) { rbn = bn; break; }
    if (rbn) {
      const int nt = p.N / rbn;
      const int rgrid = (sms / nt) * nt;
      if (nt <= sms && rgrid * 16 >= sms * 15 && p.m_tiles * nt >= (int64_t)rgrid * 4) {
        p.resident = 1; p.BN = rbn; p.n_tiles = nt;
        grid = rgrid;
      }
    }
    const int64_t rounds0 = ceil_div64(p.m_tiles * p.n_tiles, sms);
    if (!p.resident && rounds0 < 8) {
      // per k block a tile costs max(MMA, operand feed) clocks: 128 x bn x 64 MACs at 1024 MAC/clk per SM (H100 dense bf16), and
      // (128 + bn) x 128 B of operands at ~24 B/clk per SM of L2 bandwidth, plus a fixed per-tile overhead (epilogue, pipeline fill)
      auto cost_of = [&](int bn, int64_t nt) {
        const int64_t mma = 8 * bn, feed = (int64_t)(5.3 * (128 + bn));
        return ceil_div64(p.m_tiles * nt, sms) * ((mma > feed ? mma : feed) + 400);
      };
      int64_t best = cost_of(p.BN, p.n_tiles);
      for (int bn : BN_CHOICES) {
        if (bn > p.N || bn < 64 || bn > max_bn) continue;
        const int64_t nt = ceil_div64(p.N, bn);
        const int64_t cost = cost_of(bn, nt);
        if (cost < best) { best = cost; p.BN = bn; p.n_tiles = (int)nt; }
      }
    }
  }
  p.stg_bytes = stg_bytes_for(p.BN, p.flags);
  p.ring_bytes = ring_bytes_for(p.BN, p.flags);
  const int slab = k_iters * p.BN * 128;
  const int st = p.resident ? (p.ring_bytes - slab) / A_BYTES : p.ring_bytes / (A_BYTES + p.BN * 128);
  p.a_stages = st > (p.resident ? MAX_STAGES : STAGES) ? (p.resident ? MAX_STAGES : STAGES) : st;
  if (!p.resident) {
    const int64_t tiles = p.m_tiles * p.n_tiles;
    grid = (int)(tiles < sms ? tiles : sms);
  }
  *grid_out = grid;
}

template <int BN, typename T>
int32_t launch_bn(const CUtensorMap& ma, const CUtensorMap& mw, const CUtensorMap& ma2, const CUtensorMap& mo, const CUtensorMap& mr,
                  const TcParams& p, int grid, cudaStream_t st) {
  static bool attr_set = false;
  if (!attr_set) {
    FYC_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<BN, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_LIMIT));
    attr_set = true;
  }
  const int smem = p.ring_bytes + 2 * p.stg_bytes + SMEM_EXTRA;
  FYC_CHECK(smem <= SMEM_LIMIT && p.a_stages >= 2 && p.a_stages <= MAX_STAGES, "tensor-core GEMM: shared-memory plan does not fit (BN %d)", BN);
  gemm_tc_kernel<BN, T><<<grid, NUM_THREADS, smem, st>>>(ma, mw, ma2, mo, mr, p);
  FYC_LAUNCH_CHECK();
  return FYC_OK;
}

// mr: the residual map (FYC_EPI_RESIDUAL only; otherwise unused)
int32_t launch_tc(int32_t dt, const CUtensorMap& ma, const CUtensorMap& mw, const CUtensorMap& mo, const CUtensorMap* mr, TcParams p, int grid,
                  cudaStream_t st, const CUtensorMap* ma2p = nullptr) {
  const CUtensorMap& ma2 = ma2p ? *ma2p : ma;
  const CUtensorMap& mres = mr ? *mr : mo;
  if (!ma2p) p.cb_split = 0x7fffffff;
  FYC_CHECK(!(p.flags & FYC_EPI_RESIDUAL) || mr, "tensor-core GEMM: residual epilogue without a residual map");
  FYC_CHECK((p.bw & (p.bw - 1)) == 0 && (p.bh & (p.bh - 1)) == 0 && p.bw > 0 && p.bh > 0, "tensor-core GEMM: patch dims must be powers of two");
  p.lg_bw = 0; while ((1 << p.lg_bw) < p.bw) ++p.lg_bw;
  p.lg_bh = 0; while ((1 << p.lg_bh) < p.bh) ++p.lg_bh;
  const int64_t tiles = p.m_tiles * p.n_tiles;
  FYC_CHECK(tiles < (1ll << 31) && p.M < (1ll << 31) && p.rows_per_group < (1ll << 31), "tensor-core GEMM: problem exceeds the 32-bit tile index range");
  if (grid > tiles) grid = (int)tiles;
  FYC_DISPATCH16(dt, switch (p.BN) {
    case 256: return launch_bn<256, T>(ma, mw, ma2, mo, mres, p, grid, st);
    case 192: return launch_bn<192, T>(ma, mw, ma2, mo, mres, p, grid, st);
    case 160: return launch_bn<160, T>(ma, mw, ma2, mo, mres, p, grid, st);
    case 128: return launch_bn<128, T>(ma, mw, ma2, mo, mres, p, grid, st);
    case 96: return launch_bn<96, T>(ma, mw, ma2, mo, mres, p, grid, st);
    case 80: return launch_bn<80, T>(ma, mw, ma2, mo, mres, p, grid, st);
    case 64: return launch_bn<64, T>(ma, mw, ma2, mo, mres, p, grid, st);
    case 48: return launch_bn<48, T>(ma, mw, ma2, mo, mres, p, grid, st);
    case 32: return launch_bn<32, T>(ma, mw, ma2, mo, mres, p, grid, st);
    case 16: return launch_bn<16, T>(ma, mw, ma2, mo, mres, p, grid, st);
  })
  FYC_CHECK(false, "tensor-core GEMM: no kernel for BN = %d", p.BN);
}

}  // namespace

// Is this GEMM eligible for the tensor-core path?
bool fyc_gemm_tc_eligible(const fyc_gemm_args* g) {
  if (!fyc_is_16bit(g->dtype)) return false;
  if (g->K % 8 || g->lda % 8 || g->ldw % 8 || g->N % 16 || g->M < 64) return false;
  if (((uintptr_t)g->A | (uintptr_t)g->W) & 15) return false;
  if (g->batch > 1 && ((g->strideA | g->strideW | g->strideO) % 8)) return false;
  const int64_t n_out = (g->epilogue & FYC_EPI_GEGLU) ? g->N / 2 : g->N;
  if (g->ldo % 8 || ((uintptr_t)g->out & 15)) return false;
  if ((g->epilogue & FYC_EPI_RESIDUAL) && (g->ldr % 8 || ((uintptr_t)g->residual & 15))) return false;
  if ((g->epilogue & FYC_EPI_GEGLU) && (g->N % 256 || !(g->epilogue & FYC_EPI_BIAS) || (g->epilogue & ~(FYC_EPI_GEGLU | FYC_EPI_BIAS | FYC_EPI_LNFOLD)))) return false;
  if (g->A2) {
    if (g->batch != 1 || g->K1 <= 0 || g->K1 >= g->K || g->K1 % BK || g->lda2 % 8 || (((uintptr_t)g->A2) & 15)) return false;
  }
  if (g->epilogue & FYC_EPI_LNFOLD) {
    if (!g->ln_rowstats || (((uintptr_t)g->ln_rowstats) & 3)) return false;
    if (g->alpha != 1.0f || (g->epilogue & (FYC_EPI_OUT_F32 | FYC_EPI_RESIDUAL)) || g->N % 8) return false;
    if ((g->epilogue & FYC_EPI_ROWBIAS) && g->rows_per_group % 128) return false;     // a warp's 32 rows never straddle two row-bias groups
  }
  if ((g->epilogue & FYC_EPI_BIAS) && ((uintptr_t)g->bias & 15)) return false;
  if ((g->epilogue & FYC_EPI_ROWBIAS) && ((uintptr_t)g->rowbias & 15)) return false;
  (void)n_out;
  return tma_available();
}

int32_t fyc_gemm_tc(const fyc_gemm_args* g, cudaStream_t st) {
  FYC_CHECK(fyc_gemm_tc_eligible(g), "gemm(tensor cores): shape/alignment not eligible (M=%lld N=%lld K=%lld)", (long long)g->M,
            (long long)g->N, (long long)g->K);
  const bool geglu = (g->epilogue & FYC_EPI_GEGLU) != 0;
  const bool f32 = (g->epilogue & FYC_EPI_OUT_F32) != 0;
  for (int64_t b = 0; b < g->batch; ++b) {
    const uint16_t* A = (const uint16_t*)g->A + b * g->strideA;     // 16-bit elements
    const uint16_t* W = (const uint16_t*)g->W + b * g->strideW;
    CUtensorMap ma, mw, ma2;
    const int64_t Ka = g->A2 ? g->K1 : g->K;          // columns of the first (or only) source
    {
      uint64_t dims[4] = {(uint64_t)Ka, (uint64_t)g->M, 1, 1};
      uint64_t str[3] = {(uint64_t)g->lda * 2, (uint64_t)g->lda * 2 * (uint64_t)g->M, (uint64_t)g->lda * 2 * (uint64_t)g->M};
      uint32_t box[4] = {BK, BM, 1, 1};
      int32_t rc = encode_map(&ma, A, 4, dims, str, box, tma_dtype(g->dtype));
      if (rc) return rc;
    }
    if (g->A2) {
      uint64_t dims[4] = {(uint64_t)(g->K - g->K1), (uint64_t)g->M, 1, 1};
      uint64_t str[3] = {(uint64_t)g->lda2 * 2, (uint64_t)g->lda2 * 2 * (uint64_t)g->M, (uint64_t)g->lda2 * 2 * (uint64_t)g->M};
      uint32_t box[4] = {BK, BM, 1, 1};
      int32_t rc = encode_map(&ma2, g->A2, 4, dims, str, box, tma_dtype(g->dtype));
      if (rc) return rc;
    }
    TcParams p{};
    p.M = g->M; p.N = (int)g->N; p.N_out = geglu ? (int)g->N / 2 : (int)g->N;
    p.taps = 1; p.cin_blocks = (int)ceil_div64(g->K, BK);
    p.bw = BM; p.bh = 1; p.bn = 1; p.Wo = (int)g->M; p.Ho = 1;
    p.w_tiles = (int)ceil_div64(g->M, BM); p.h_tiles = 1; p.m_tiles = p.w_tiles;
    p.flags = g->epilogue;
    int grid = 0;
    choose_tiles(p, &grid);
    p.tap_dy[0] = p.tap_dx[0] = p.tap_img[0] = 0;
    {
      uint64_t dims[3] = {(uint64_t)g->K, 1, (uint64_t)g->N};
      uint64_t str[2] = {(uint64_t)g->ldw * 2, (uint64_t)g->ldw * 2};
      uint32_t box[3] = {BK, 1, (uint32_t)p.BN};
      int32_t rc = encode_map(&mw, W, 3, dims, str, box, tma_dtype(g->dtype));
      if (rc) return rc;
    }
    FYC_CHECK(g->M < (1ll << 31), "gemm(tensor cores): M too large");
    p.bias = g->bias; p.rowbias = g->rowbias; p.rows_per_group = g->rows_per_group > 0 ? g->rows_per_group : 1; p.ldrb = g->N;
    p.alpha = g->alpha;
    p.ln_rs = g->ln_rowstats;
    p.cb_split = g->A2 ? (int)(g->K1 / BK) : 0x7fffffff;
    // output / residual: N_out x M rows of ldo / ldr elements (ldo may exceed N_out: the caller passes a column slice)
    const int64_t es = f32 ? 4 : 2;
    const uint64_t M = (uint64_t)g->M, No = (uint64_t)p.N_out;
    CUtensorMap mo, mr;
    int32_t rc = encode_out_map(&mo, (const char*)g->out + b * g->strideO * es, p, g->dtype, No, M, 1, 1, g->ldo, g->ldo * M, g->ldo * M);
    if (rc) return rc;
    if (g->epilogue & FYC_EPI_RESIDUAL) {
      rc = encode_out_map(&mr, (const char*)g->residual + b * g->strideO * es, p, g->dtype, No, M, 1, 1, g->ldr, g->ldr * M, g->ldr * M);
      if (rc) return rc;
    }
    rc = launch_tc(g->dtype, ma, mw, mo, (g->epilogue & FYC_EPI_RESIDUAL) ? &mr : nullptr, p, grid, st, g->A2 ? &ma2 : nullptr);
    if (rc) return rc;
  }
  return FYC_OK;
}

// Tile shape for a conv output of Ho x Wo over NB images: bw*bh*bn == 128, all dividing evenly.
static bool pick_patch(int64_t NB, int64_t Ho, int64_t Wo, int* bw, int* bh, int* bn) {
  int w = 1; while (w < 128 && Wo % (w * 2) == 0) w *= 2;
  int h = 1; while (w * h < 128 && Ho % (h * 2) == 0) h *= 2;
  int n = 128 / (w * h);
  if (w * h * n != 128 || NB % n != 0) return false;
  *bw = w; *bh = h; *bn = n;
  return true;
}

bool fyc_conv3x3_tc_eligible(const fyc_conv3x3_args* c) {
  if (!fyc_is_16bit(c->dtype) || c->upsample != 1) return false;
  if (c->stride != 1 && c->stride != 2) return false;
  if (c->Cin % 8 || c->Cout % 16) return false;
  if (c->stride == 2 && (c->H % 2 || c->W % 2)) return false;
  if (((uintptr_t)c->x | (uintptr_t)c->w | (uintptr_t)c->out) & 15) return false;
  if ((c->epilogue & FYC_EPI_RESIDUAL) && ((uintptr_t)c->residual & 15)) return false;
  if ((c->epilogue & FYC_EPI_ROWBIAS) && (((uintptr_t)c->rowbias & 15) || (c->ld_rowbias > 0 && c->ld_rowbias % 4))) return false;
  if (c->epilogue & FYC_EPI_GEGLU) return false;
  int bw, bh, bn;
  if (!pick_patch(c->NB, c->H / c->stride, c->W / c->stride, &bw, &bh, &bn)) return false;
  return tma_available();
}

// x for stride 2 must already be the parity-plane split (see fyc_space_to_planes); H, W are the ORIGINAL dims.
int32_t fyc_conv3x3_tc(const fyc_conv3x3_args* c, const void* x_planes, cudaStream_t st) {
  FYC_CHECK(fyc_conv3x3_tc_eligible(c), "conv3x3(tensor cores): shape/alignment not eligible");
  const int s = c->stride;
  const int64_t Ho = c->H / s, Wo = c->W / s;
  TcParams p{};
  pick_patch(c->NB, Ho, Wo, &p.bw, &p.bh, &p.bn);
  p.M = c->NB * Ho * Wo; p.N = (int)c->Cout; p.N_out = p.N;
  p.taps = 9; p.cin_blocks = (int)ceil_div64(c->Cin, BK);
  p.Wo = (int)Wo; p.Ho = (int)Ho; p.w_tiles = (int)(Wo / p.bw); p.h_tiles = (int)(Ho / p.bh);
  p.m_tiles = (int64_t)p.w_tiles * p.h_tiles * (c->NB / p.bn);
  p.flags = c->epilogue;
  int grid = 0;
  choose_tiles(p, &grid);
  CUtensorMap ma, mw;
  const void* xa = c->x;
  uint64_t imgs = (uint64_t)c->NB;
  for (int t = 0; t < 9; ++t) {
    int kh = t / 3, kw = t % 3;
    if (s == 1) { p.tap_dy[t] = kh - 1; p.tap_dx[t] = kw - 1; p.tap_img[t] = 0; }
    else if (c->pad_mode == 1) {   // ih = 2*oh + kh: kh=0 -> even plane, row oh; kh=1 -> odd plane, row oh; kh=2 -> even plane, row oh+1
      int ph = (kh == 1) ? 1 : 0, pw = (kw == 1) ? 1 : 0;       // (row H/2 of a plane is out of bounds: TMA zero fill = the bottom / right pad)
      p.tap_dy[t] = (kh == 2) ? 1 : 0; p.tap_dx[t] = (kw == 2) ? 1 : 0;
      p.tap_img[t] = (2 * ph + pw) * (int)c->NB;
    } else {   // ih = 2*oh + kh - 1: kh=0 -> odd plane, row oh-1; kh=1 -> even plane, row oh; kh=2 -> odd plane, row oh
      int ph = (kh == 1) ? 0 : 1, pw = (kw == 1) ? 0 : 1;
      p.tap_dy[t] = (kh == 0) ? -1 : 0; p.tap_dx[t] = (kw == 0) ? -1 : 0;
      p.tap_img[t] = (2 * ph + pw) * (int)c->NB;
    }
  }
  if (s == 2) { xa = x_planes; imgs = 4ull * c->NB; FYC_CHECK(x_planes != nullptr, "conv3x3(tensor cores): stride 2 needs the plane-split input"); }
  {
    uint64_t dims[4] = {(uint64_t)c->Cin, (uint64_t)Wo, (uint64_t)Ho, imgs};
    uint64_t str[3] = {(uint64_t)c->Cin * 2, (uint64_t)c->Cin * 2 * Wo, (uint64_t)c->Cin * 2 * Wo * Ho};
    uint32_t box[4] = {BK, (uint32_t)p.bw, (uint32_t)p.bh, (uint32_t)p.bn};
    int32_t rc = encode_map(&ma, xa, 4, dims, str, box, tma_dtype(c->dtype));
    if (rc) return rc;
  }
  {
    uint64_t dims[3] = {(uint64_t)c->Cin, 9, (uint64_t)c->Cout};
    uint64_t str[2] = {(uint64_t)c->Cin * 2, (uint64_t)c->Cin * 2 * 9};
    uint32_t box[3] = {BK, 1, (uint32_t)p.BN};
    int32_t rc = encode_map(&mw, c->w, 3, dims, str, box, tma_dtype(c->dtype));
    if (rc) return rc;
  }
  p.bias = c->bias; p.rowbias = c->rowbias;
  p.ldrb = c->ld_rowbias > 0 ? c->ld_rowbias : c->Cout;
  p.rows_per_group = (c->images_per_group > 0 ? c->images_per_group : 1) * Ho * Wo;
  p.alpha = 1.0f;
  const uint64_t C = (uint64_t)c->Cout;
  CUtensorMap mo, mr;
  int32_t rc = encode_out_map(&mo, c->out, p, c->dtype, C, Wo, Ho, c->NB, C, C * Wo, C * Wo * Ho);
  if (rc) return rc;
  if (c->epilogue & FYC_EPI_RESIDUAL) {
    rc = encode_out_map(&mr, c->residual, p, c->dtype, C, Wo, Ho, c->NB, C, C * Wo, C * Wo * Ho);
    if (rc) return rc;
  }
  return launch_tc(c->dtype, ma, mw, mo, (c->epilogue & FYC_EPI_RESIDUAL) ? &mr : nullptr, p, grid, st);
}

// nearest-x2 upsample + padded 3x3 conv as four 2x2-tap implicit GEMMs on the low-resolution image (fyc.h: w_phases).
// Phase (py, px) produces output pixels (2*oh + py, 2*ow + px).  No kernel change is needed: the A boxes are the usual shifted
// patches of x (TMA zero fill = the conv's zero padding, because an upsampled halo pixel is out of bounds exactly when its source
// pixel is), and the interleaved destination is a strided output map: base out + (py * 2W + px) * Cout, dimensions
// {Cout, W, H, NB} with strides 2 Cout, 4W Cout, 4HW Cout elements, so low-resolution pixel (ow, oh, img) lands at
// ((img * 2H + 2 oh + py) * 2W + 2 ow + px) * Cout, the NHWC offset of the upsampled pixel.
bool fyc_conv3x3_up2_tc_eligible(const fyc_conv3x3_args* c) {
  if (!fyc_is_16bit(c->dtype) || c->upsample != 2 || c->stride != 1 || c->pad_mode != 0 || !c->w_phases) return false;
  if (c->Cin % 8 || c->Cout % 16) return false;
  if (((uintptr_t)c->x | (uintptr_t)c->w_phases | (uintptr_t)c->out) & 15) return false;
  if (c->epilogue & ~FYC_EPI_BIAS) return false;          // the upsamplers carry a bias only (resnet.py:168, diffusers resnet.py:139)
  int bw, bh, bn;
  if (!pick_patch(c->NB, c->H, c->W, &bw, &bh, &bn)) return false;
  return tma_available();
}

int32_t fyc_conv3x3_up2_tc(const fyc_conv3x3_args* c, cudaStream_t st) {
  FYC_CHECK(fyc_conv3x3_up2_tc_eligible(c), "conv3x3 up2(tensor cores): shape/alignment not eligible");
  const int64_t H = c->H, W = c->W;
  TcParams p{};
  pick_patch(c->NB, H, W, &p.bw, &p.bh, &p.bn);
  p.M = c->NB * H * W; p.N = (int)c->Cout; p.N_out = p.N;
  p.taps = 4; p.cin_blocks = (int)ceil_div64(c->Cin, BK);
  p.Wo = (int)W; p.Ho = (int)H; p.w_tiles = (int)(W / p.bw); p.h_tiles = (int)(H / p.bh);
  p.m_tiles = (int64_t)p.w_tiles * p.h_tiles * (c->NB / p.bn);
  p.flags = c->epilogue;
  int grid = 0;
  choose_tiles(p, &grid);
  p.alpha = 1.0f;
  p.bias = c->bias; p.rowbias = nullptr; p.rows_per_group = 1; p.ldrb = p.N;
  CUtensorMap ma;
  {
    uint64_t dims[4] = {(uint64_t)c->Cin, (uint64_t)W, (uint64_t)H, (uint64_t)c->NB};
    uint64_t str[3] = {(uint64_t)c->Cin * 2, (uint64_t)c->Cin * 2 * W, (uint64_t)c->Cin * 2 * W * H};
    uint32_t box[4] = {BK, (uint32_t)p.bw, (uint32_t)p.bh, (uint32_t)p.bn};
    int32_t rc = encode_map(&ma, c->x, 4, dims, str, box, tma_dtype(c->dtype));
    if (rc) return rc;
  }
  for (int ph = 0; ph < 4; ++ph) {
    const int py = ph >> 1, px = ph & 1;
    for (int t = 0; t < 4; ++t) {               // tap (a, b): input row oh + a - 1 + py, column ow + b - 1 + px
      p.tap_dy[t] = (t >> 1) - 1 + py; p.tap_dx[t] = (t & 1) - 1 + px; p.tap_img[t] = 0;
    }
    CUtensorMap mw;
    const uint16_t* wp = (const uint16_t*)c->w_phases + (int64_t)ph * c->Cout * 4 * c->Cin;
    uint64_t dims[3] = {(uint64_t)c->Cin, 4, (uint64_t)c->Cout};
    uint64_t str[2] = {(uint64_t)c->Cin * 2, (uint64_t)c->Cin * 2 * 4};
    uint32_t box[3] = {BK, 1, (uint32_t)p.BN};
    int32_t rc = encode_map(&mw, wp, 3, dims, str, box, tma_dtype(c->dtype));
    if (rc) return rc;
    const uint64_t C = (uint64_t)c->Cout;
    CUtensorMap mo;
    rc = encode_out_map(&mo, (const uint16_t*)c->out + ((int64_t)py * 2 * W + px) * c->Cout, p, c->dtype, C, W, H, c->NB, 2 * C, 4 * W * C, 4 * H * W * C);
    if (rc) return rc;
    rc = launch_tc(c->dtype, ma, mw, mo, nullptr, p, grid, st);
    if (rc) return rc;
  }
  return FYC_OK;
}

int32_t fyc_space_to_planes(const void* x, void* out, int64_t NB, int64_t H, int64_t W, int64_t C, cudaStream_t st) {
  FYC_CHECK(H % 2 == 0 && W % 2 == 0 && C % 8 == 0, "space_to_planes: H, W must be even and C a multiple of 8");
  int64_t total = NB * H * W * C / 8;
  int64_t blocks = ceil_div64(total, 256), cap = (int64_t)fyc_sm_count() * 16;
  space_to_planes_kernel<<<(unsigned)(blocks > cap ? cap : blocks), 256, 0, st>>>((const bf16*)x, (bf16*)out, NB, H, W, C);
  FYC_LAUNCH_CHECK();
  return FYC_OK;
}
