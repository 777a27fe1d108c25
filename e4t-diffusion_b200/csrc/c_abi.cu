// e4t_b200 — C-ABI plumbing: status/error reporting, launch counter, TMA tensor-map encode.
// The reference (mkshing/e4t-diffusion) has no FFI of its own; this boundary is what its Python
// module API (e4t/weightoffsets.py, e4t/models/*.py, e4t/encoder.py) binds through ctypes.
#include "common.cuh"
#include <stdarg.h>

thread_local char g_e4t_err[512] = {0};
unsigned long long g_e4t_launches = 0;

int e4t_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_e4t_err, sizeof(g_e4t_err), fmt, ap);
  va_end(ap);
  return 1;
}

extern "C" const char* e4t_last_error(void) { return g_e4t_err; }
extern "C" int e4t_version(void) { return 100; }  // 0.1.0
extern "C" unsigned long long e4t_launch_count(void) { return g_e4t_launches; }
extern "C" void e4t_reset_launch_count(void) { g_e4t_launches = 0; }

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static PFN_encodeTiled g_encode = nullptr;

int e4t_tmap_encode(CUtensorMap* map, const void* gptr, int rank, const uint64_t* dims,
                    const uint64_t* strides_bytes, const uint32_t* box, int elem_bytes, int swizzle_bytes,
                    const uint32_t* elem_strides) {
  if (!g_encode) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !fn)
      return e4t_set_error("cuTensorMapEncodeTiled entry point unavailable (%s)", cudaGetErrorString(e));
    g_encode = (PFN_encodeTiled)fn;
  }
  // cuTensorMapEncodeTiled is a DRIVER entry point: it needs the primary context bound to the calling thread, which the
  // runtime only does on a thread's first runtime call.  torch's autograd worker threads can reach this function before
  // making any (first backward of a process: CUDA_ERROR_INVALID_CONTEXT, seen in round 2) — bind it once per thread.
  static thread_local bool ctx_bound = false;
  if (!ctx_bound) {
    cudaFree(0);
    ctx_bound = true;
  }
  cuuint64_t gdim[5], gstr[4];
  cuuint32_t bdim[5], estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bdim[i] = box[i];
    estr[i] = elem_strides ? elem_strides[i] : 1;
    if (i > 0) gstr[i - 1] = strides_bytes[i - 1];
  }
  CUtensorMapDataType dt = elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  CUresult r = g_encode(map, dt, (cuuint32_t)rank, const_cast<void*>(gptr), gdim, gstr, bdim, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE,
                        swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                        : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                        : swizzle_bytes == 32 ? CU_TENSOR_MAP_SWIZZLE_32B : CU_TENSOR_MAP_SWIZZLE_NONE,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    return e4t_set_error(
        "cuTensorMapEncodeTiled failed (%d): rank=%d dims=[%llu,%llu,%llu,%llu] strides=[%llu,%llu,%llu] "
        "box=[%u,%u,%u,%u] ptr=%p",
        (int)r, rank, (unsigned long long)gdim[0], (unsigned long long)(rank > 1 ? gdim[1] : 0),
        (unsigned long long)(rank > 2 ? gdim[2] : 0), (unsigned long long)(rank > 3 ? gdim[3] : 0),
        (unsigned long long)(rank > 1 ? gstr[0] : 0), (unsigned long long)(rank > 2 ? gstr[1] : 0),
        (unsigned long long)(rank > 3 ? gstr[2] : 0), bdim[0], rank > 1 ? bdim[1] : 0, rank > 2 ? bdim[2] : 0,
        rank > 3 ? bdim[3] : 0, gptr);
  }
  return 0;
}

typedef CUresult (*PFN_encodeIm2col)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                     const cuuint64_t*, const int*, const int*, cuuint32_t, cuuint32_t,
                                     const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                     CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static PFN_encodeIm2col g_encode_im2col = nullptr;

int e4t_tmap_encode_im2col(CUtensorMap* map, const void* gptr, const uint64_t* dims, const uint64_t* strides_bytes,
                           const int* lower, const int* upper, uint32_t channels, uint32_t pixels,
                           const uint32_t* elem_strides) {
  if (!g_encode_im2col) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &fn, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || !fn)
      return e4t_set_error("cuTensorMapEncodeIm2col entry point unavailable (%s)", cudaGetErrorString(e));
    g_encode_im2col = (PFN_encodeIm2col)fn;
  }
  static thread_local bool ctx_bound = false;  // as in e4t_tmap_encode
  if (!ctx_bound) {
    cudaFree(0);
    ctx_bound = true;
  }
  cuuint64_t gdim[4], gstr[3];
  cuuint32_t estr[4];
  for (int i = 0; i < 4; ++i) {
    gdim[i] = dims[i];
    estr[i] = elem_strides[i];
    if (i > 0) gstr[i - 1] = strides_bytes[i - 1];
  }
  CUresult r = g_encode_im2col(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(gptr), gdim, gstr, lower,
                               upper, channels, pixels, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                               CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return e4t_set_error(
        "cuTensorMapEncodeIm2col failed (%d): dims=[%llu,%llu,%llu,%llu] corners=[%d,%d]..[%d,%d] pixels=%u "
        "stride=%u ptr=%p",
        (int)r, (unsigned long long)gdim[0], (unsigned long long)gdim[1], (unsigned long long)gdim[2],
        (unsigned long long)gdim[3], lower[0], lower[1], upper[0], upper[1], pixels, estr[1], gptr);
  return 0;
}
