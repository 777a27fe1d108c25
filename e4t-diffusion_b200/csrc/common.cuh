// e4t_b200 — shared device/host helpers for the sm_90a kernels.
// Hand-written PTX wrappers for mbarrier, TMA (cp.async.bulk.tensor), wgmma and mma.sync / ldmatrix.
// No CUTLASS/CuTe dependency: everything the kernels need is spelled out here.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

typedef __nv_bfloat16 bf16;

// ---------------------------------------------------------------------------------------------
// Host-side error plumbing (C-ABI returns int status; message kept per thread)
// ---------------------------------------------------------------------------------------------
extern thread_local char g_e4t_err[512];
int e4t_set_error(const char* fmt, ...);

#define E4T_CHECK(cond, ...)                                   \
  do {                                                         \
    if (!(cond)) return e4t_set_error(__VA_ARGS__);            \
  } while (0)

#define E4T_CUDA(call)                                                                  \
  do {                                                                                  \
    cudaError_t _e = (call);                                                            \
    if (_e != cudaSuccess)                                                              \
      return e4t_set_error("%s:%d CUDA error %s: %s", __FILE__, __LINE__, #call,        \
                           cudaGetErrorString(_e));                                     \
  } while (0)

#define E4T_LAUNCH_CHECK() E4T_CUDA(cudaGetLastError())

// Count of kernels launched by this library (bench.py reports it as gpu_launches).
extern unsigned long long g_e4t_launches;
#define E4T_COUNT_LAUNCH() (++g_e4t_launches)

// Tensor-map encode through the driver entry point (no link-time libcuda dependency).
int e4t_tmap_encode(CUtensorMap* map, const void* gptr, int rank, const uint64_t* dims,
                    const uint64_t* strides_bytes /* rank-1 entries, dims 1.. */,
                    const uint32_t* box, int elem_bytes /*2 = bf16*/, int swizzle_bytes = 128,
                    const uint32_t* elem_strides = nullptr /* traversal stride per dim (box is in global coordinates) */);
// im2col-mode tensor map over an NHWC bf16 tensor, 128-byte swizzle: dims / strides as for e4t_tmap_encode (rank 4,
// {C, W, H, N}); each load reads `pixels` pixels x `channels` channels.  lower / upper {W, H}: the bounding box a load
// walks spans [lower, dim - 1 + upper] in W and H, stepped by elem_strides[1], [2].
int e4t_tmap_encode_im2col(CUtensorMap* map, const void* gptr, const uint64_t* dims, const uint64_t* strides_bytes,
                           const int* lower, const int* upper, uint32_t channels, uint32_t pixels,
                           const uint32_t* elem_strides);

static inline int cdiv(long a, long b) { return (int)((a + b - 1) / b); }

#ifdef __CUDACC__
// ---------------------------------------------------------------------------------------------
// Device helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

// ---- GroupNorm statistics ----------------------------------------------------------------------
// fp32 [B][G][kGNStat] per (image, group) = (p, sum (x - p), sum (x - p)^2) over the group's n elements, where the
// pivot p is the group's first element in that image.  Summing around p instead of 0 keeps E[x^2] - mean^2 from
// cancelling when a group's mean is large against its spread (trained VAE / UNet activations).  Written by
// e4t_groupnorm_fwd; every GroupNorm kernel turns it into (mean, rstd) here and nowhere else.
static constexpr int kGNStat = 3;
__device__ __forceinline__ float2 gn_mean_rstd(const float* __restrict__ st, float inv_n, float eps) {
  const float d = st[1] * inv_n;
  return make_float2(st[0] + d, rsqrtf(fmaxf(st[2] * inv_n - d * d, 0.f) + eps));
}

// ---- mbarrier ------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// non-blocking poll (try_wait may suspend the thread up to a system-defined time limit when the phase is incomplete)
__device__ __forceinline__ bool mbar_test_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ---- proxy fences --------------------------------------------------------------------------
// generic-proxy smem writes -> visible to the async proxy (TMA stores, wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ---- TMA loads (tile mode, mbarrier completion) ----------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
      "[%2];" ::"r"(smem_u32(smem)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// im2col mode (tensor map from e4t_tmap_encode_im2col, NHWC): (c, w, h, n) is the input position of the first pixel's
// top-left tap; the load walks the map's pixelsPerColumn pixels in NHW order through its bounding box, across row and
// image boundaries, and reads each one at (w + off_w, h + off_h), zero-filling reads outside the tensor.
__device__ __forceinline__ void tma_load_im2col_4d(void* smem, const CUtensorMap* m, uint64_t* bar, int c, int w,
                                                   int h, int n, int off_w, int off_h) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, "
      "%6}], [%2], {%7, %8};" ::"r"(smem_u32(smem)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c), "r"(w), "r"(h), "r"(n),
      "h"((uint16_t)off_w), "h"((uint16_t)off_h)
      : "memory");
}

// contiguous global -> shared copy (16-byte aligned, bytes % 16 == 0), mbarrier completion
__device__ __forceinline__ void bulk_load_1d(void* smem, const void* g, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem)),
               "l"(g), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// ---- TMA stores (smem -> global, bulk async group completion) ------------------------------------
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* m, const void* smem, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(smem)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
// smem tile -> global with an element-wise ADD performed by the TMA engine / L2 (type and box come from the tensor map)
__device__ __forceinline__ void tma_reduce_add_3d(const CUtensorMap* m, const void* smem, int c0, int c1, int c2) {
  asm volatile("cp.reduce.async.bulk.tensor.3d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(smem)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ---- wgmma (sm_90a warpgroup MMA) ---------------------------------------------------------------
// Shared-memory matrix descriptor, SWIZZLE_128B.
//   K-major operand : rows of 128 B (64 bf16 of K), 8-row groups 1024 B apart (SBO); LBO unused (1).
//   MN-major operand: rows of 128 B (64 bf16 of M/N), row index = k; 8-k groups 1024 B apart (SBO);
//                     successive 64-wide MN chunks LBO bytes apart.
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFFu) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= 1ull << 62;  // SWIZZLE_128B
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator reads/writes across an asynchronous wgmma
template <int R>
__device__ __forceinline__ void reg_fence(float* d) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// the same for bf16-packed A-operand registers of a register-A wgmma, which the instruction reads until it retires
template <int R>
__device__ __forceinline__ void reg_fence_u32(uint32_t* a) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+r"(a[i])::"memory");
}
// named barrier over `nthreads` threads of the CTA (id 0 is __syncthreads)
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
// warpgroup register re-allocation (producer warpgroup gives registers to the MMA warpgroups)
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R));
}
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R));
}

// ---- warp-level MMA (mma.sync m16n8k16, bf16 -> fp32) and ldmatrix ---------------------------------
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t* r) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t* r) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}
// d[4] += a[4] (16x16, row-major fragment) * b[2] (16x8, column fragment)
__device__ __forceinline__ void mma16816(float* d, const uint32_t* a, const uint32_t* b) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
// 16-byte global -> shared copy (cp.async, L2 only); src_bytes < 16 zero-fills the rest
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// byte offset of 16-byte chunk `c16` (0..7) of row `r` inside a [rows][64 bf16] SWIZZLE_128B tile
__device__ __forceinline__ uint32_t sw128_off(uint32_t r, uint32_t c16) {
  return r * 128u + ((c16 ^ (r & 7u)) << 4);
}

// ---- small math helpers ----------------------------------------------------------------------
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
__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
  __nv_bfloat162 t = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&t);
}
__device__ __forceinline__ float2 unpack_bf16(uint32_t u) {
  __nv_bfloat162 t = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(t);
}
// 2^x on the MUFU pipe, no denormal fix-up code (inputs here are <= 0 or bounded)
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float silu_f(float x) { return x / (1.f + __expf(-x)); }
#endif  // __CUDACC__
