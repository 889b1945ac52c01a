// HBM-bound glue kernels: embeddings, layout changes, CFG + DDIM step, frame finalisation.
// All are coalesced, 16-byte vectorised where the shape allows, grid sized in multiples of the SM count.
#include "common.cuh"

static inline int grid_for(int64_t work_items, int threads) {
  int64_t blocks = ceil_div64(work_items, threads);
  int64_t cap = (int64_t)fyc_sm_count() * 16;
  return (int)(blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
}

// ---------------------------------------------------------------------------------------------------------
// get_timestep_embedding (diffusers/models/embeddings.py:39-56): emb = t * freq; [sin | cos] (or flipped).
__global__ void timestep_embed_kernel(const int64_t* __restrict__ t, const float* __restrict__ freqs,
                                      float* __restrict__ out, int64_t n, int half, int flip) {
  int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (idx >= n * half) return;
  int64_t i = idx / half;
  int k = (int)(idx % half);
  float ang = (float)t[i] * freqs[k];
  float s = sinf(ang), c = cosf(ang);
  float* row = out + i * 2 * half;
  if (flip) { row[k] = c; row[half + k] = s; } else { row[k] = s; row[half + k] = c; }
}

extern "C" int32_t fyc_timestep_embed(const int64_t* t, const float* freqs, float* out, int64_t n, int64_t dim,
                                      int32_t flip, void* stream) {
  FYC_CHECK(dim % 2 == 0 && n > 0, "timestep_embed: dim must be even (got %lld)", (long long)dim);
  int half = (int)(dim / 2);
  timestep_embed_kernel<<<(unsigned)ceil_div64(n * half, 128), 128, 0, (cudaStream_t)stream>>>(t, freqs, out, n, half, flip);
  FYC_LAUNCH_CHECK();
  return FYC_OK;
}

// ---------------------------------------------------------------------------------------------------------
template <typename T>
__global__ void silu_kernel(const T* __restrict__ x, T* __restrict__ out, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = from_f<T>(silu_f(to_f(x[i])));
}
extern "C" int32_t fyc_silu(const void* x, void* out, int64_t n, int32_t dtype, void* stream) {
  FYC_DISPATCH(dtype, silu_kernel<T><<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>((const T*)x, (T*)out, n));
  FYC_LAUNCH_CHECK();
  return FYC_OK;
}

// exact-erf GELU (nn.GELU() of the Perceiver Resampler's feed-forward, ip_adapter/resampler.py:14-21)
template <typename T>
__global__ void gelu_kernel(const T* __restrict__ x, T* __restrict__ out, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = from_f<T>(gelu_erf_f(to_f(x[i])));
}
extern "C" int32_t fyc_gelu(const void* x, void* out, int64_t n, int32_t dtype, void* stream) {
  FYC_DISPATCH(dtype, gelu_kernel<T><<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>((const T*)x, (T*)out, n));
  FYC_LAUNCH_CHECK();
  return FYC_OK;
}

// GEGLU for the SIMT path.  in [M, 2*Hd]: column block t of 256 holds a[128t:128t+128] | gate[128t:128t+128].
template <typename T>
__global__ void geglu_kernel(const T* __restrict__ in, T* __restrict__ out, int64_t M, int64_t Hd) {
  int64_t total = M * Hd / 4;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t m = i / (Hd / 4);
    int64_t j = (i % (Hd / 4)) * 4;
    const T* row = in + m * 2 * Hd + (j / 128) * 256 + (j % 128);
    float a[4], g[4], o[4];
    Vec4<T>::load(row, a);
    Vec4<T>::load(row + 128, g);
#pragma unroll
    for (int e = 0; e < 4; ++e) o[e] = a[e] * gelu_erf_f(g[e]);
    Vec4<T>::store(out + m * Hd + j, o);
  }
}
extern "C" int32_t fyc_geglu(const void* in, void* out, int64_t M, int64_t Hd, int32_t dtype, void* stream) {
  FYC_CHECK(Hd % 128 == 0, "geglu: hidden dim %lld must be a multiple of 128", (long long)Hd);
  FYC_DISPATCH(dtype, geglu_kernel<T><<<grid_for(M * Hd / 4, 256), 256, 0, (cudaStream_t)stream>>>((const T*)in, (T*)out, M, Hd));
  FYC_LAUNCH_CHECK();
  return FYC_OK;
}

// ---------------------------------------------------------------------------------------------------------
// nearest 2x upsample, NHWC (animatediff/models/resnet.py:155; diffusers/models/resnet.py:128)
template <typename T, int V>
__global__ void upsample2x_kernel(const T* __restrict__ x, T* __restrict__ out, int64_t NB, int64_t H, int64_t W, int64_t C) {
  int64_t cv = C / V;
  int64_t total = NB * 2 * H * 2 * W * cv;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t c = (i % cv) * V;
    int64_t p = i / cv;
    int64_t ow = p % (2 * W); p /= (2 * W);
    int64_t oh = p % (2 * H);
    int64_t n = p / (2 * H);
    const T* src = x + ((n * H + oh / 2) * W + ow / 2) * C + c;
    T* dst = out + i * V;
    if (V == 8) *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(src);
    else *dst = *src;
  }
}
extern "C" int32_t fyc_upsample_nearest2x(const void* x, void* out, int64_t NB, int64_t H, int64_t W, int64_t C,
                                          int32_t dtype, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (fyc_is_16bit(dtype) && C % 8 == 0) {     // a 16-byte copy: the bf16 instantiation moves any 16-bit type
    upsample2x_kernel<bf16, 8><<<grid_for(NB * 4 * H * W * C / 8, 256), 256, 0, st>>>((const bf16*)x, (bf16*)out, NB, H, W, C);
  } else {
    FYC_DISPATCH(dtype, upsample2x_kernel<T, 1><<<grid_for(NB * 4 * H * W * C, 256), 256, 0, st>>>((const T*)x, (T*)out, NB, H, W, C));
  }
  FYC_LAUNCH_CHECK();
  return FYC_OK;
}

// channel concat (unet_blocks.py:763,885)
template <typename T, int V>
__global__ void concat_kernel(const T* __restrict__ a, const T* __restrict__ b, T* __restrict__ out, int64_t M, int64_t C1, int64_t C2) {
  int64_t cv = (C1 + C2) / V;
  int64_t total = M * cv;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t m = i / cv, c = (i % cv) * V;
    const T* src = c < C1 ? a + m * C1 + c : b + m * C2 + (c - C1);
    T* dst = out + i * V;
    if (V * sizeof(T) == 16) *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(src);
    else *dst = *src;
  }
}
extern "C" int32_t fyc_concat_channels(const void* a, const void* b, void* out, int64_t M, int64_t C1, int64_t C2,
                                       int32_t dtype, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (fyc_is_16bit(dtype) && C1 % 8 == 0 && C2 % 8 == 0) {     // a 16-byte copy: the bf16 instantiation moves any 16-bit type
    concat_kernel<bf16, 8><<<grid_for(M * (C1 + C2) / 8, 256), 256, 0, st>>>((const bf16*)a, (const bf16*)b, (bf16*)out, M, C1, C2);
  } else if (dtype == FYC_F32 && C1 % 4 == 0 && C2 % 4 == 0) {
    concat_kernel<float, 4><<<grid_for(M * (C1 + C2) / 4, 256), 256, 0, st>>>((const float*)a, (const float*)b, (float*)out, M, C1, C2);
  } else {
    FYC_DISPATCH(dtype, concat_kernel<T, 1><<<grid_for(M * (C1 + C2), 256), 256, 0, st>>>((const T*)a, (const T*)b, (T*)out, M, C1, C2));
  }
  FYC_LAUNCH_CHECK();
  return FYC_OK;
}

// ---------------------------------------------------------------------------------------------------------
// fp32 (b, c, f, hw) <-> T [b, f, hw, c].  Used at the UNet boundary (C = 4 / 9) and by tests.
template <typename T>
__global__ void ncfhw_to_nfhwc_kernel(const float* __restrict__ in, T* __restrict__ out, int64_t B, int64_t C, int64_t F, int64_t HW, float scale) {
  int64_t total = B * F * HW * C;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t c = i % C; int64_t r = i / C;
    int64_t p = r % HW; r /= HW;
    int64_t f = r % F; int64_t b = r / F;
    out[i] = from_f<T>(__fmul_rn(in[((b * C + c) * F + f) * HW + p], scale));
  }
}
template <typename T>
__global__ void nfhwc_to_ncfhw_kernel(const T* __restrict__ in, float* __restrict__ out, int64_t B, int64_t C, int64_t F, int64_t HW, int64_t ldc) {
  int64_t total = B * F * HW * C;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t p = i % HW; int64_t r = i / HW;
    int64_t f = r % F; r /= F;
    int64_t c = r % C; int64_t b = r / C;
    out[i] = to_f(in[((b * F + f) * HW + p) * ldc + c]);
  }
}
extern "C" int32_t fyc_ncfhw_to_nfhwc(const float* in, void* out, int64_t B, int64_t C, int64_t F, int64_t HW, float scale, int32_t dtype, void* stream) {
  FYC_DISPATCH(dtype, ncfhw_to_nfhwc_kernel<T><<<grid_for(B * C * F * HW, 256), 256, 0, (cudaStream_t)stream>>>(in, (T*)out, B, C, F, HW, scale));
  FYC_LAUNCH_CHECK();
  return FYC_OK;
}
extern "C" int32_t fyc_nfhwc_to_ncfhw(const void* in, float* out, int64_t B, int64_t C, int64_t F, int64_t HW, int64_t ldc, int32_t dtype, void* stream) {
  if (ldc <= 0) ldc = C;
  FYC_CHECK(ldc >= C, "nfhwc_to_ncfhw: channel stride %lld < C %lld", (long long)ldc, (long long)C);
  FYC_DISPATCH(dtype, nfhwc_to_ncfhw_kernel<T><<<grid_for(B * C * F * HW, 256), 256, 0, (cudaStream_t)stream>>>((const T*)in, out, B, C, F, HW, ldc));
  FYC_LAUNCH_CHECK();
  return FYC_OK;
}

// ---------------------------------------------------------------------------------------------------------
// UNet input assembly (pipeline_animation.py:625-635,693-711): per pixel [latents(4) | mask(1) | first-frame block(4)],
// duplicated `dup` times along the batch for CFG (:709).
template <typename T>
__global__ void build_unet_input_kernel(const float* __restrict__ lat, const float* __restrict__ mask,
                                        const float* __restrict__ first, T* __restrict__ out, int64_t b, int64_t F,
                                        int64_t HW, int dup, int concat, int c_pad) {
  int Cin = concat ? 9 : 4;
  int64_t total = b * F * HW;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t p = i % HW; int64_t r = i / HW;
    int64_t f = r % F; int64_t bi = r / F;
    float v[9];
#pragma unroll
    for (int c = 0; c < 4; ++c) v[c] = lat[((bi * 4 + c) * F + f) * HW + p];
    if (concat) {
      float m = mask ? fminf(fmaxf(mask[bi * HW + p], 0.f), 1.f) : (f == 0 ? 1.f : 0.f);
      v[4] = m;
#pragma unroll
      for (int c = 0; c < 4; ++c) v[5 + c] = (f == 0) ? first[(bi * 4 + c) * HW + p] : 0.f;
    }
    for (int d = 0; d < dup; ++d) {
      T* o = out + (((d * b + bi) * F + f) * HW + p) * c_pad;
      for (int c = 0; c < Cin; ++c) o[c] = from_f<T>(v[c]);
      for (int c = Cin; c < c_pad; ++c) o[c] = from_f<T>(0.f);
    }
  }
}
extern "C" int32_t fyc_build_unet_input(const float* latents, const float* mask, const float* first, void* out, int64_t b,
                                        int64_t F, int64_t HW, int32_t dup, int32_t c_pad, int32_t dtype, void* stream) {
  FYC_CHECK(dup == 1 || dup == 2, "build_unet_input: dup must be 1 or 2");
  int concat = first != nullptr;
  FYC_CHECK(c_pad >= (concat ? 9 : 4) && c_pad <= 64, "build_unet_input: c_pad=%d", c_pad);
  FYC_DISPATCH(dtype, build_unet_input_kernel<T><<<grid_for(b * F * HW, 256), 256, 0, (cudaStream_t)stream>>>(latents, mask, first, (T*)out, b, F, HW, dup, concat, c_pad));
  FYC_LAUNCH_CHECK();
  return FYC_OK;
}

// The first-frame-conditioned models' step prologue (fyc.h fyc_build_unet_input_first).  One thread per pixel (clip, frame, position):
// under FYC_FIRST_FRAME the frame-0 threads overwrite their own four latents with the first-image latents before reading them, so no
// thread reads what another one writes.
template <typename T>
__global__ void build_unet_input_first_kernel(float* __restrict__ lat, const float* __restrict__ first, T* __restrict__ out, int64_t b,
                                              int64_t F, int64_t HW, int dup, int mode, int c_pad) {
  const int Cin = (mode & FYC_FIRST_CONCAT) ? 8 : 4;
  int64_t total = b * F * HW;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t p = i % HW; int64_t r = i / HW;
    int64_t f = r % F; int64_t bi = r / F;
    float v[8];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      float* src = lat + ((bi * 4 + c) * F + f) * HW + p;
      if ((mode & FYC_FIRST_FRAME) && f == 0) *src = first[(bi * 4 + c) * HW + p];
      v[c] = *src;
      v[4 + c] = first[(bi * 4 + c) * HW + p];
    }
    for (int d = 0; d < dup; ++d) {
      T* o = out + (((d * b + bi) * F + f) * HW + p) * c_pad;
      for (int c = 0; c < Cin; ++c) o[c] = from_f<T>(v[c]);
      for (int c = Cin; c < c_pad; ++c) o[c] = from_f<T>(0.f);
    }
  }
}
extern "C" int32_t fyc_build_unet_input_first(float* latents, const float* first, void* out, int64_t b, int64_t F, int64_t HW, int32_t dup,
                                              int32_t mode, int32_t c_pad, int32_t dtype, void* stream) {
  FYC_CHECK(latents && first && out && b > 0 && F > 0 && HW > 0, "build_unet_input_first: bad arguments");
  FYC_CHECK(dup == 1 || dup == 2, "build_unet_input_first: dup must be 1 or 2");
  FYC_CHECK(mode >= 1 && mode <= (FYC_FIRST_CONCAT | FYC_FIRST_FRAME), "build_unet_input_first: unknown mode %d", mode);
  FYC_CHECK(c_pad >= ((mode & FYC_FIRST_CONCAT) ? 8 : 4) && c_pad <= 64, "build_unet_input_first: c_pad=%d", c_pad);
  FYC_DISPATCH(dtype, build_unet_input_first_kernel<T><<<grid_for(b * F * HW, 256), 256, 0, (cudaStream_t)stream>>>(latents, first, (T*)out, b, F, HW, dup, mode, c_pad));
  FYC_LAUNCH_CHECK();
  return FYC_OK;
}

// Per-image time-embedding rows of the first-frame condition (resnet.py:304-313): frame 0 of every clip reads row B (the t = 0 row the
// UNet appends, unet.py:523-524), frame f > 0 of clip b reads row b.
__global__ void first_frame_temb_rows_kernel(const float* __restrict__ temb, float* __restrict__ out, int64_t B, int64_t F, int64_t N) {
  const int64_t total = B * F * N;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t n = i % N, img = i / N;
    const int64_t f = img % F, bi = img / F;
    out[i] = temb[(f == 0 ? B : bi) * N + n];
  }
}
extern "C" int32_t fyc_first_frame_temb_rows(const float* temb, float* out, int64_t B, int64_t F, int64_t N, void* stream) {
  FYC_CHECK(temb && out && B > 0 && F > 0 && N > 0, "first_frame_temb_rows: bad arguments");
  first_frame_temb_rows_kernel<<<grid_for(B * F * N, 256), 256, 0, (cudaStream_t)stream>>>(temb, out, B, F, N);
  FYC_LAUNCH_CHECK();
  return FYC_OK;
}

// ---------------------------------------------------------------------------------------------------------
// CFG combine + DDIM step.  Operation order and roundings follow the reference line by line so that the fp32
// result is bit-identical to PyTorch eager (each torch op rounds once; no FMA contraction):
//   pipeline_animation.py:764        n   = u + g * (c - u)
//   scheduling_ddim.py:318-325       x0  = (x - sb*n)/sa | n | sa*x - sb*n ;  eps = n | - | sa*n + sb*x
//   scheduling_ddim.py:330           clip x0
//   scheduling_ddim.py:346-349       prev = sap*x0 + dir*eps
//   scheduling_ddim.py:366-368       prev += noise_coef * noise        (eta > 0)
//   pipeline_animation.py:757-761    n   = s + vs * (u - s) + g * (c - u)      (video_scale > 0: s = per-frame prediction)
__global__ void cfg_ddim_kernel(const float* __restrict__ pred, const float* __restrict__ single, float video_scale,
                                const float* __restrict__ sample,
                                const float* __restrict__ noise, float* __restrict__ prev, int64_t n, fyc_ddim_coefs c) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float m;
    if (single) {
      float u = pred[i], t = pred[n + i], s = single[i];
      m = __fadd_rn(__fadd_rn(s, __fmul_rn(video_scale, __fsub_rn(u, s))), __fmul_rn(c.guidance, __fsub_rn(t, u)));
    } else if (c.cfg_pair) {
      float u = pred[i], t = pred[n + i];
      m = __fadd_rn(u, __fmul_rn(c.guidance, __fsub_rn(t, u)));
    } else {
      m = pred[i];
    }
    float x = sample[i];
    float x0, eps;
    if (c.prediction_type == FYC_PRED_EPSILON) {
      x0 = __fdiv_rn(__fsub_rn(x, __fmul_rn(c.sqrt_beta_t, m)), c.sqrt_alpha_t);
      eps = m;
    } else if (c.prediction_type == FYC_PRED_SAMPLE) {
      x0 = m;
      eps = m;   // reference quirk: model_output is passed through unchanged as the direction term
    } else {
      x0 = __fsub_rn(__fmul_rn(c.sqrt_alpha_t, x), __fmul_rn(c.sqrt_beta_t, m));
      eps = __fadd_rn(__fmul_rn(c.sqrt_alpha_t, m), __fmul_rn(c.sqrt_beta_t, x));
    }
    if (c.clip_sample) x0 = fminf(fmaxf(x0, -1.f), 1.f);
    float r = __fadd_rn(__fmul_rn(c.sqrt_alpha_prev, x0), __fmul_rn(c.dir_coef, eps));
    if (noise) r = __fadd_rn(r, __fmul_rn(c.noise_coef, noise[i]));
    prev[i] = r;
  }
}
extern "C" int32_t fyc_cfg_ddim_step(const float* pred, const float* sample, const float* noise, float* prev, int64_t n,
                                     const fyc_ddim_coefs* c, void* stream) {
  FYC_CHECK(c != nullptr && n > 0, "cfg_ddim_step: bad arguments");
  FYC_CHECK(c->prediction_type >= 0 && c->prediction_type <= 2, "cfg_ddim_step: unknown prediction_type %d", c->prediction_type);
  cfg_ddim_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(pred, nullptr, 0.f, sample, noise, prev, n, *c);
  FYC_LAUNCH_CHECK();
  return FYC_OK;
}
extern "C" int32_t fyc_cfg_video_ddim_step(const float* pred, const float* single, float video_scale, const float* sample,
                                           const float* noise, float* prev, int64_t n, const fyc_ddim_coefs* c, void* stream) {
  FYC_CHECK(c != nullptr && n > 0 && pred && single, "cfg_video_ddim_step: bad arguments");
  FYC_CHECK(c->prediction_type >= 0 && c->prediction_type <= 2, "cfg_video_ddim_step: unknown prediction_type %d", c->prediction_type);
  FYC_CHECK(c->cfg_pair != 0, "cfg_video_ddim_step: the per-frame guidance branch exists only under classifier-free guidance");
  cfg_ddim_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(pred, single, video_scale, sample, noise, prev, n, *c);
  FYC_LAUNCH_CHECK();
  return FYC_OK;
}

// ---------------------------------------------------------------------------------------------------------
// decode_latents epilogue (pipeline_animation.py:409-410): [b*F, HW, 3] -> (b, 3, F, HW) fp32, (x/2+0.5).clamp(0,1)
template <typename T>
__global__ void frames_finalize_kernel(const T* __restrict__ x, float* __restrict__ video, int64_t b, int64_t F, int64_t HW, int64_t ldc) {
  int64_t total = b * 3 * F * HW;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t p = i % HW; int64_t r = i / HW;
    int64_t f = r % F; r /= F;
    int64_t c = r % 3; int64_t bi = r / 3;
    float v = to_f(x[((bi * F + f) * HW + p) * ldc + c]);
    v = __fadd_rn(__fdiv_rn(v, 2.0f), 0.5f);
    if constexpr (std::is_same<T, f16>::value)
      // fp16 storage ends at 65504: a value that overflowed anywhere upstream (inf, or the NaN it turns into) reaches the video as NaN
      // instead of being clipped to a black or white pixel (fminf / fmaxf return the non-NaN operand)
      video[i] = isfinite(v) ? fminf(fmaxf(v, 0.f), 1.f) : __int_as_float(0x7fffffff);
    else
      video[i] = fminf(fmaxf(v, 0.f), 1.f);
  }
}
extern "C" int32_t fyc_frames_finalize(const void* x, float* video, int64_t b, int64_t F, int64_t HW, int64_t ldc, int32_t dtype, void* stream) {
  if (ldc <= 0) ldc = 3;
  FYC_CHECK(ldc >= 3, "frames_finalize: channel stride %lld < 3", (long long)ldc);
  FYC_DISPATCH(dtype, frames_finalize_kernel<T><<<grid_for(b * 3 * F * HW, 256), 256, 0, (cudaStream_t)stream>>>((const T*)x, video, b, F, HW, ldc));
  FYC_LAUNCH_CHECK();
  return FYC_OK;
}

// ---------------------------------------------------------------------------------------------------------
// save_videos_grid's per-frame tiling + 8-bit conversion (animatediff/utils/util.py:18-27) on the device: for every frame t the b
// clips are tiled like torchvision.utils.make_grid(nrow, padding, pad_value 0) - a single clip is passed through unpadded - then
// (x [+1)/2 if rescale]) * 255 truncated to uint8.  video (b, 3, F, H, W) fp32 -> out [F, Hg, Wg, 3] uint8: a quarter of the bytes of
// the fp32 video cross PCIe, already in the layout the GIF writer wants.
__global__ void video_grid_u8_kernel(const float* __restrict__ video, uint8_t* __restrict__ out, int64_t b, int64_t F, int64_t H, int64_t W,
                                     int64_t xmaps, int64_t pad, int64_t Hg, int64_t Wg, int rescale) {
  const int64_t total = F * Hg * Wg * 3;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t c = i % 3; int64_t r = i / 3;
    const int64_t x = r % Wg; r /= Wg;
    const int64_t y = r % Hg; const int64_t t = r / Hg;
    float v = 0.f;                                      // pad_value
    const int64_t ch = H + pad, cw = W + pad;           // cell pitch
    const int64_t yy = y - pad, xx = x - pad;
    if (yy >= 0 && xx >= 0) {
      const int64_t gy = yy / ch, gx = xx / cw, iy = yy % ch, ix = xx % cw;
      const int64_t k = gy * xmaps + gx;
      if (gx < xmaps && k < b && iy < H && ix < W) v = video[(((k * 3 + c) * F + t) * H + iy) * W + ix];
    }
    if (rescale) v = __fdiv_rn(__fadd_rn(v, 1.0f), 2.0f);
    v = __fmul_rn(v, 255.0f);
    out[i] = (uint8_t)(int)fminf(fmaxf(v, 0.f), 255.f);     // numpy astype(uint8) of an in-range float truncates toward zero
  }
}
extern "C" int32_t fyc_video_grid_u8(const float* video, uint8_t* out, int64_t b, int64_t F, int64_t H, int64_t W, int64_t nrow,
                                     int64_t padding, int32_t rescale, void* stream) {
  FYC_CHECK(video && out && b > 0 && F > 0 && H > 0 && W > 0 && nrow > 0 && padding >= 0, "video_grid_u8: bad arguments");
  const int64_t pad = (b == 1) ? 0 : padding;            // make_grid returns a single image as is
  const int64_t xmaps = b < nrow ? b : nrow, ymaps = (b + xmaps - 1) / xmaps;
  const int64_t Hg = (H + pad) * ymaps + pad, Wg = (W + pad) * xmaps + pad;
  video_grid_u8_kernel<<<grid_for(F * Hg * Wg * 3, 256), 256, 0, (cudaStream_t)stream>>>(video, out, b, F, H, W, xmaps, pad, Hg, Wg, rescale);
  FYC_LAUNCH_CHECK();
  return FYC_OK;
}

// ---------------------------------------------------------------------------------------------------------
// fp32 row softmax (VAE AttentionBlock, diffusers/models/attention.py:366).  One block per row.
template <typename T>
__global__ void softmax_rows_kernel(const float* __restrict__ s, T* __restrict__ p, int64_t L) {
  const float* row = s + (int64_t)blockIdx.x * L;
  T* out = p + (int64_t)blockIdx.x * L;
  __shared__ float red[32];
  float m = -INFINITY;
  for (int64_t j = threadIdx.x; j < L; j += blockDim.x) m = fmaxf(m, row[j]);
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  m = (threadIdx.x & 31) < (blockDim.x >> 5) ? red[threadIdx.x & 31] : -INFINITY;   // every warp reduces the 8 partials
  m = warp_max(m);
  __syncthreads();
  float sum = 0.f;
  for (int64_t j = threadIdx.x; j < L; j += blockDim.x) sum += expf(row[j] - m);
  sum = warp_sum(sum);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
  __syncthreads();
  sum = (threadIdx.x & 31) < (blockDim.x >> 5) ? red[threadIdx.x & 31] : 0.f;
  sum = warp_sum(sum);
  float inv = 1.0f / sum;
  for (int64_t j = threadIdx.x; j < L; j += blockDim.x) out[j] = from_f<T>(expf(row[j] - m) * inv);
}
extern "C" int32_t fyc_softmax_rows(const float* scores, void* probs, int64_t rows, int64_t L, int32_t dtype, void* stream) {
  FYC_CHECK(rows > 0 && rows < (1ll << 31) && L > 0, "softmax_rows: bad shape");
  FYC_DISPATCH(dtype, softmax_rows_kernel<T><<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>(scores, (T*)probs, L));
  FYC_LAUNCH_CHECK();
  return FYC_OK;
}
