// Shared helpers for libfyc_sm90a (H100 / sm_90a only).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "fyc.h"

typedef __nv_bfloat16 bf16;
typedef __half f16;

void fyc_set_error(const char* fmt, ...);

#define FYC_CHECK(cond, ...)                 \
  do {                                       \
    if (!(cond)) {                           \
      fyc_set_error(__VA_ARGS__);            \
      return FYC_ERR_INVALID;                \
    }                                        \
  } while (0)

#define FYC_CUDA(call)                                                                         \
  do {                                                                                         \
    cudaError_t e_ = (call);                                                                   \
    if (e_ != cudaSuccess) {                                                                   \
      fyc_set_error("%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_));      \
      return FYC_ERR_CUDA;                                                                     \
    }                                                                                          \
  } while (0)

#define FYC_LAUNCH_CHECK() FYC_CUDA(cudaGetLastError())

// switch over the storage dtype; body sees `T`
#define FYC_DISPATCH(dt, ...)                                  \
  switch (dt) {                                                \
    case FYC_F32: { using T = float; __VA_ARGS__; } break;     \
    case FYC_BF16: { using T = bf16; __VA_ARGS__; } break;     \
    case FYC_F16: { using T = f16; __VA_ARGS__; } break;       \
    default: FYC_CHECK(false, "unknown dtype %d", (int)(dt));  \
  }
// the same over the 16-bit storage dtypes only (the tensor-core paths)
#define FYC_DISPATCH16(dt, ...)                                       \
  switch (dt) {                                                       \
    case FYC_BF16: { using T = bf16; __VA_ARGS__; } break;            \
    case FYC_F16: { using T = f16; __VA_ARGS__; } break;              \
    default: FYC_CHECK(false, "unsupported 16-bit dtype %d", (int)(dt)); \
  }
static inline bool fyc_is_16bit(int32_t dt) { return dt == FYC_BF16 || dt == FYC_F16; }

__device__ __forceinline__ float to_f(float v) { return v; }
__device__ __forceinline__ float to_f(bf16 v) { return __bfloat162float(v); }
template <typename T> __device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }
template <> __device__ __forceinline__ bf16 from_f<bf16>(float v) { return __float2bfloat16_rn(v); }
__device__ __forceinline__ float to_f(f16 v) { return __half2float(v); }
template <> __device__ __forceinline__ f16 from_f<f16>(float v) { return __float2half_rn(v); }

// Two 16-bit values in one 32-bit word (element 0 in the low half): Pair16<T>::type is __nv_bfloat162 | __half2, pack() rounds two
// floats once, unpack() widens exactly; ONE is the bit pattern of 1.0.
template <typename T> struct Pair16;
template <> struct Pair16<bf16> {
  typedef __nv_bfloat162 type;
  static constexpr uint32_t ONE = 0x3F80u;
  static __device__ __forceinline__ type pack(float lo, float hi) { return __floats2bfloat162_rn(lo, hi); }
  static __device__ __forceinline__ float2 unpack(type v) { return __bfloat1622float2(v); }
};
template <> struct Pair16<f16> {
  typedef __half2 type;
  static constexpr uint32_t ONE = 0x3C00u;
  static __device__ __forceinline__ type pack(float lo, float hi) { return __floats2half2_rn(lo, hi); }
  static __device__ __forceinline__ float2 unpack(type v) { return __half22float2(v); }
};
template <typename T> __device__ __forceinline__ uint32_t pack_u32(float lo, float hi) {
  typename Pair16<T>::type v = Pair16<T>::pack(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

// 8-element vector of T (16 B for bf16 / fp16, 32 B for fp32) <-> float[8]
template <typename T> struct Vec8 {     // 16-bit T
  typedef typename Pair16<T>::type P;
  static __device__ __forceinline__ void load(const T* p, float* f) {
    uint4 u = *reinterpret_cast<const uint4*>(p);
    const P* h = reinterpret_cast<const P*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) { float2 t = Pair16<T>::unpack(h[i]); f[2 * i] = t.x; f[2 * i + 1] = t.y; }
  }
  static __device__ __forceinline__ void store(T* p, const float* f) {
    uint4 u;
    P* h = reinterpret_cast<P*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = Pair16<T>::pack(f[2 * i], f[2 * i + 1]);
    *reinterpret_cast<uint4*>(p) = u;
  }
};
template <> struct Vec8<float> {
  static __device__ __forceinline__ void load(const float* p, float* f) {
    float4 a = *reinterpret_cast<const float4*>(p), b = *reinterpret_cast<const float4*>(p + 4);
    f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
  }
  static __device__ __forceinline__ void store(float* p, const float* f) {
    *reinterpret_cast<float4*>(p) = make_float4(f[0], f[1], f[2], f[3]);
    *reinterpret_cast<float4*>(p + 4) = make_float4(f[4], f[5], f[6], f[7]);
  }
};

// 4-element vector
template <typename T> struct Vec4 {     // 16-bit T
  typedef typename Pair16<T>::type P;
  static __device__ __forceinline__ void load(const T* p, float* f) {
    uint2 u = *reinterpret_cast<const uint2*>(p);
    const P* h = reinterpret_cast<const P*>(&u);
    float2 a = Pair16<T>::unpack(h[0]), b = Pair16<T>::unpack(h[1]);
    f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y;
  }
  static __device__ __forceinline__ void store(T* p, const float* f) {
    uint2 u;
    P* h = reinterpret_cast<P*>(&u);
    h[0] = Pair16<T>::pack(f[0], f[1]);
    h[1] = Pair16<T>::pack(f[2], f[3]);
    *reinterpret_cast<uint2*>(p) = u;
  }
};
template <> struct Vec4<float> {
  static __device__ __forceinline__ void load(const float* p, float* f) {
    float4 a = *reinterpret_cast<const float4*>(p);
    f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w;
  }
  static __device__ __forceinline__ void store(float* p, const float* f) {
    *reinterpret_cast<float4*>(p) = make_float4(f[0], f[1], f[2], f[3]);
  }
};

// V (8, 4 or 1) consecutive elements of T <-> float[V]
template <typename T, int V> __device__ __forceinline__ void load_vec(const T* p, float* f) {
  if constexpr (V == 8) Vec8<T>::load(p, f);
  else if constexpr (V == 4) Vec4<T>::load(p, f);
  else f[0] = to_f(*p);
}
template <typename T, int V> __device__ __forceinline__ void store_vec(T* p, const float* f) {
  if constexpr (V == 8) Vec8<T>::store(p, f);
  else if constexpr (V == 4) Vec4<T>::store(p, f);
  else *p = from_f<T>(f[0]);
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// 16-byte cp.async global -> shared; the first form reads src_bytes (0 or 16) and zero-fills the rest
__device__ __forceinline__ void cp_async16(void* dst, const void* src, int src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async16(void* dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void ldmatrix_x4(uint32_t* r, const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_u32(p)));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t* r, const void* p) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(smem_u32(p)));
}

// mma.sync m16n8k16, fp32 accumulator c += a b with 16-bit operands T (bf16 | f16)
template <typename T> __device__ __forceinline__ void mma16816(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
  if constexpr (std::is_same<T, f16>::value)
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  else
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ float silu_f(float x) { return x / (1.0f + expf(-x)); }
// 16-bit-storage paths: 2-ulp intrinsics are far below the 2^-9 (bf16) / 2^-12 (fp16) output rounding
__device__ __forceinline__ float silu_fast(float x) { return __fdividef(x, 1.0f + __expf(-x)); }
// exact-erf GELU (F.gelu default; diffusers/models/attention.py:815)
__device__ __forceinline__ float gelu_erf_f(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }

// single MUFU.EX2 (exp2f() adds denormal-range handling: ~4 instructions per element in an issue-bound kernel)
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// exact-erf GELU with erf(z) = 1 - 2^q(z), q = degree-5 least-squares fit of log2(erfc(z)) on [0, 4] (|erf error| <= 7.2e-7,
// |gelu error| <= 1.3e-6 over all x; fit script in DESIGN.md): ONE MUFU.EX2 + 7 FMAs instead of erff()'s ~30 instructions.
// (A first version with Abramowitz-Stegun 7.1.26 needed rcp + ex2 = two MUFU ops per element and made the GEGLU epilogue
// MUFU-bound: 431 vs 636 TFLOP/s on the level-0 FF1 GEMM.)
// |gelu_erf_fast(x) - gelu(x)| <= 1.3e-6 + 2^-23 |x| (polynomial and ex2.approx measured on a dense grid over [-12, 12], plus fp32
// rounding); fminf drops a NaN x, the final multiply by x still returns NaN.
__device__ __forceinline__ float gelu_erf_fast(float x) {
  const float z = fminf(fabsf(x) * 0.70710678118654752440f, 4.0f);
  float q = fmaf(-0.002980560529977083f, z, 0.02972414717078209f);
  q = fmaf(q, z, -0.14882677793502808f);
  q = fmaf(q, z, -0.9184384942054749f);
  q = fmaf(q, z, -1.6278971433639526f);
  q = fmaf(q, z, -2.8457714051910443e-07f);
  const float erfv = copysignf(1.0f - ex2_approx(q), x);
  return 0.5f * x * (1.0f + erfv);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

static inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }
int fyc_sm_count();
