// Host side of the TMA paths: the driver's tensor-map encoder, looked up once through the runtime (no link against libcuda).
#include "tma.cuh"

namespace {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(ptr);
    else
      (void)cudaGetLastError();
  }
  return fn;
}

}  // namespace

bool tma_available() { return get_encode_fn() != nullptr; }

CUtensorMapDataType tma_dtype(int32_t dt) { return dt == FYC_F16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16; }

int32_t encode_map(CUtensorMap* m, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                   const uint32_t* box, CUtensorMapDataType dtype, CUtensorMapSwizzle swizzle) {
  EncodeTiledFn fn = get_encode_fn();
  FYC_CHECK(fn != nullptr, "tensor-core path: cuTensorMapEncodeTiled driver entry point unavailable");
  cuuint64_t gdim[5]; cuuint64_t gstr[4]; cuuint32_t bx[5]; cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) { gdim[i] = dims[i]; bx[i] = box[i]; es[i] = 1; }
  for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
  CUresult r = fn(m, dtype, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bx, es,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  FYC_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed with CUresult %d (rank %d dims %llu %llu %llu %llu)", (int)r, rank,
            (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)(rank > 2 ? dims[2] : 0),
            (unsigned long long)(rank > 3 ? dims[3] : 0));
  return FYC_OK;
}

extern "C" int32_t fyc_tcgen05_available(void) { return tma_available() ? 1 : 0; }
