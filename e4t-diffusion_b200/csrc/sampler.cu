// e4t_b200 — one denoising update of the sampling schedulers (e4t/schedulers.py), driven by a coefficient table.
//
// Every scheduler of the reference's inference.py (DDIM, PLMS, LMS, Euler, Euler ancestral, DPM-Solver++) moves the
// latents by a linear combination of the sample, the guided model output, a few earlier outputs, a saved sample and
// noise, with coefficients that depend only on the step index.  The host writes them as an fp64 table (format defined
// in e4t/schedulers.py, column indices mirrored below); a one-thread-block tick publishes row *step_dev as fp32 and the
// next step's timestep, then advances the counter, and the update applies the row elementwise.  Nothing here branches
// on host state, so the whole denoising step replays from a CUDA graph.
#include <algorithm>

#include "common.cuh"

namespace {

// table columns (e4t/schedulers.py)
constexpr int kX = 0, kE = 1, kH0 = 2, kS = 6, kZ = 7, kSlot = 8, kHA = 9, kHB = 10, kSave = 11, kSNext = 12,
              kTNext = 13, kRow = 14, kMaxHist = 4;
constexpr int kThreads = 256;

// *step holds the steps already taken: row min(*step, n_rows - 1) is published, its next-step timestep written to
// *t_out (the UNet's fp32 timestep buffer) when given, and the counter advances.
__global__ void sampler_tick_kernel(const double* __restrict__ table, int n_rows, int* step, float* row, float* t_out) {
  const int s = *step;
  const int i = min(max(s, 0), n_rows - 1);
  __syncthreads();
  if (threadIdx.x < kRow) row[threadIdx.x] = (float)table[(long long)i * kRow + threadIdx.x];
  if (threadIdx.x == 0) {
    if (t_out) *t_out = (float)table[(long long)i * kRow + kTNext];
    *step = s + 1;
  }
}

struct SamplerArgs {
  const float* out;       // [G][n] model output, uncond rows first under guidance
  const float* guidance;  // device scalar (G == 2)
  const float* x;         // [n]
  float* x_next;          // [n], may alias x
  float* hist;            // [n_hist][hist_ld]
  float* saved;           // [n]
  const float* noise;     // [n] or null
  const float* row;       // published fp32 row
  float* model_in;        // [G][n] or null
  long long n, hist_ld;
  int G, n_hist;
};

template <int W>
struct Vec;
template <>
struct Vec<4> {
  static __device__ __forceinline__ void ld(const float* p, long long i, float* v) {
    const float4 t = reinterpret_cast<const float4*>(p)[i];
    v[0] = t.x, v[1] = t.y, v[2] = t.z, v[3] = t.w;
  }
  static __device__ __forceinline__ void st(float* p, long long i, const float* v) {
    reinterpret_cast<float4*>(p)[i] = make_float4(v[0], v[1], v[2], v[3]);
  }
};
template <>
struct Vec<1> {
  static __device__ __forceinline__ void ld(const float* p, long long i, float* v) { v[0] = p[i]; }
  static __device__ __forceinline__ void st(float* p, long long i, const float* v) { p[i] = v[0]; }
};

// W consecutive elements starting at element W*i (vector index i), or one element at index i for W = 1.
template <int W>
__device__ __forceinline__ void sampler_elems(const SamplerArgs& a, const float* r, float g, int slot, long long i) {
  using V = Vec<W>;
  float e[W], x[W], xn[W], t[W];
  V::ld(a.out, i, e);
  if (a.G == 2) {
    V::ld(a.out + a.n, i, t);
#pragma unroll
    for (int j = 0; j < W; ++j) e[j] = e[j] + g * (t[j] - e[j]);
  }
  V::ld(a.x, i, x);
#pragma unroll
  for (int j = 0; j < W; ++j) xn[j] = r[kX] * x[j] + r[kE] * e[j];
#pragma unroll
  for (int k = 0; k < kMaxHist; ++k) {
    if (k < a.n_hist && r[kH0 + k] != 0.f) {
      V::ld(a.hist + k * a.hist_ld, i, t);
#pragma unroll
      for (int j = 0; j < W; ++j) xn[j] += r[kH0 + k] * t[j];
    }
  }
  if (r[kS] != 0.f) {
    V::ld(a.saved, i, t);
#pragma unroll
    for (int j = 0; j < W; ++j) xn[j] += r[kS] * t[j];
  }
  if (r[kZ] != 0.f && a.noise) {
    V::ld(a.noise, i, t);
#pragma unroll
    for (int j = 0; j < W; ++j) xn[j] += r[kZ] * t[j];
  }
  // every read above happens before the writes below (x_next may alias x; no slot is read and written in one step)
  if (slot >= 0) {
#pragma unroll
    for (int j = 0; j < W; ++j) t[j] = r[kHA] * x[j] + r[kHB] * e[j];
    V::st(a.hist + slot * a.hist_ld, i, t);
  }
  if (r[kSave] != 0.f) V::st(a.saved, i, x);
  V::st(a.x_next, i, xn);
  if (a.model_in) {
#pragma unroll
    for (int j = 0; j < W; ++j) t[j] = r[kSNext] * xn[j];
    V::st(a.model_in, i, t);
    if (a.G == 2) V::st(a.model_in + a.n, i, t);
  }
}

__global__ void __launch_bounds__(kThreads) sampler_update_kernel(SamplerArgs a, long long n_vec) {
  __shared__ float r[kRow];
  if (threadIdx.x < kRow) r[threadIdx.x] = a.row[threadIdx.x];
  __syncthreads();
  const float g = a.G == 2 ? *a.guidance : 0.f;
  const int slot0 = (int)r[kSlot];
  const int slot = slot0 < a.n_hist ? slot0 : -1;
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  for (long long i = tid; i < n_vec; i += stride) sampler_elems<4>(a, r, g, slot, i);
  for (long long i = n_vec * 4 + tid; i < a.n; i += stride) sampler_elems<1>(a, r, g, slot, i);
}

inline bool aligned16(const void* p) { return ((uintptr_t)p % 16) == 0; }

}  // namespace

extern "C" int e4t_sampler_step(const float* out, int G, const float* guidance, const float* x, float* x_next,
                                float* hist, int n_hist, long long hist_ld, float* saved, const float* noise,
                                const double* table, int n_rows, int* step_dev, float* row, float* t_out,
                                float* model_in, long long n, void* stream_) {
  E4T_CHECK(G == 1 || G == 2, "e4t_sampler_step: G must be 1 (no guidance) or 2 (uncond + cond rows), got %d", G);
  E4T_CHECK(n > 0, "e4t_sampler_step: empty latents");
  E4T_CHECK(out && x && x_next && saved && table && step_dev && row, "e4t_sampler_step: null buffer");
  E4T_CHECK(G == 1 || guidance, "e4t_sampler_step: guidance scalar needed with G == 2");
  E4T_CHECK(n_hist >= 0 && n_hist <= kMaxHist, "e4t_sampler_step: %d history slots (at most %d)", n_hist, kMaxHist);
  E4T_CHECK(n_hist == 0 || (hist && hist_ld >= n), "e4t_sampler_step: history slots need a row stride >= n");
  E4T_CHECK(n_rows >= 1, "e4t_sampler_step: empty table");
  cudaStream_t st = (cudaStream_t)stream_;
  SamplerArgs a{out, guidance, x, x_next, hist, saved, noise, row, model_in, n, hist_ld, G, n_hist};
  const bool vec = aligned16(out) && aligned16(out + (G - 1) * n) && aligned16(x) && aligned16(x_next) &&
                   aligned16(saved) && (!noise || aligned16(noise)) &&
                   (n_hist == 0 || (aligned16(hist) && hist_ld % 4 == 0)) &&
                   (!model_in || (aligned16(model_in) && aligned16(model_in + (G - 1) * n)));
  const long long n_vec = vec ? n / 4 : 0;
  const long long work = vec ? n_vec + (n - 4 * n_vec) : n;
  // one thread per float4 (or per element without them), capped at one full wave of resident blocks (2048 threads
  // = 8 blocks of 256 per SM); the loops are grid-stride, so larger latents take more iterations per thread
  int sms = 0, dev = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (sms <= 0) sms = 132;
  const int blocks = (int)std::min<long long>((work + kThreads - 1) / kThreads, 8LL * sms);
  sampler_tick_kernel<<<1, 32, 0, st>>>(table, n_rows, step_dev, row, t_out);
  E4T_COUNT_LAUNCH();
  sampler_update_kernel<<<blocks, kThreads, 0, st>>>(a, n_vec);
  E4T_COUNT_LAUNCH();
  E4T_LAUNCH_CHECK();
  return 0;
}
