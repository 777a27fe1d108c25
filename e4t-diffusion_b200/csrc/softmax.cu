// e4t_b200 — row softmax, fp32 scores in, bf16 probabilities out (sm_90a).
//   The VAE mid-block AttentionBlock (one head, dh = 512, 4096 tokens at a 64 x 64 latent; e4t/models/attention.py:152-166
//   in the reference: `torch.softmax(attention_scores.float(), dim=-1).type(attention_scores.dtype)`).  The scores come
//   from the wgmma GEMM engine in fp32 and the probabilities feed the P·V GEMM in bf16.
// One CTA per row; each thread holds up to 16 values of the row in registers (four 16-byte loads), so the row is read
// from global memory once: max and sum are block reductions over registers.  Rows longer than 16384 (a latent above
// 128 x 128 tokens, e.g. 1088 x 1024 px) take a two-pass kernel that re-reads the row instead.
#include "common.cuh"

static constexpr int kSmxVec = 4;                          // float4 loads per thread
static constexpr int kSmxMaxThreads = 1024;
static constexpr int kSmxMaxCols = kSmxMaxThreads * kSmxVec * 4;  // 16384

__device__ __forceinline__ float block_reduce(float v, bool is_max, float* red) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  v = is_max ? warp_max(v) : warp_sum(v);
  __syncthreads();  // red[] may still be read by the previous reduction
  if (lane == 0) red[w] = v;
  __syncthreads();
  float r = lane < nw ? red[lane] : (is_max ? -INFINITY : 0.f);
  r = is_max ? warp_max(r) : warp_sum(r);
  return r;
}

__global__ void __launch_bounds__(kSmxMaxThreads)
softmax_rows_kernel(const float* __restrict__ x, bf16* __restrict__ y, int n, long long ldx, long long ldy) {
  __shared__ float red[32];
  const long long row = blockIdx.x;
  const float* xr = x + row * ldx;
  bf16* yr = y + row * ldy;
  float v[kSmxVec][4];
  float mx = -INFINITY;
#pragma unroll
  for (int k = 0; k < kSmxVec; ++k) {
    const int c = 4 * (threadIdx.x + k * blockDim.x);
    if (c < n) {
      const float4 f = *reinterpret_cast<const float4*>(xr + c);
      v[k][0] = f.x; v[k][1] = f.y; v[k][2] = f.z; v[k][3] = f.w;
    } else {
      v[k][0] = v[k][1] = v[k][2] = v[k][3] = -INFINITY;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) mx = fmaxf(mx, v[k][j]);
  }
  mx = block_reduce(mx, true, red);
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < kSmxVec; ++k)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      v[k][j] = __expf(v[k][j] - mx);  // exp(-inf) = 0 for the padding lanes
      s += v[k][j];
    }
  s = block_reduce(s, false, red);
  const float inv = 1.f / s;
#pragma unroll
  for (int k = 0; k < kSmxVec; ++k) {
    const int c = 4 * (threadIdx.x + k * blockDim.x);
    if (c < n)
      *reinterpret_cast<uint2*>(yr + c) = make_uint2(pack_bf16(v[k][0] * inv, v[k][1] * inv),
                                                     pack_bf16(v[k][2] * inv, v[k][3] * inv));
  }
}

// Rows longer than kSmxMaxCols: one CTA of 1024 threads per row walks the row in chunks of 4096 columns, one float4
// per thread per chunk.  Pass 1 keeps a per-thread online max and sum (the sum rescaled by exp(m_old - m_new) whenever
// the max rises); the block combines them.  Pass 2 re-reads the row (at most a few hundred KB, served from L2) and
// writes bf16.  Same exp (__expf of x - max) and same final scaling as the register kernel.
__global__ void __launch_bounds__(kSmxMaxThreads)
softmax_rows_long_kernel(const float* __restrict__ x, bf16* __restrict__ y, int n, long long ldx, long long ldy) {
  __shared__ float red[32];
  const long long row = blockIdx.x;
  const float* xr = x + row * ldx;
  bf16* yr = y + row * ldy;
  const long long step = 4LL * blockDim.x;
  float m = -INFINITY, s = 0.f;
  for (long long c = 4LL * threadIdx.x; c < n; c += step) {
    const float4 f = *reinterpret_cast<const float4*>(xr + c);
    const float nm = fmaxf(m, fmaxf(fmaxf(f.x, f.y), fmaxf(f.z, f.w)));
    s = s * __expf(m - nm) + (__expf(f.x - nm) + __expf(f.y - nm)) + (__expf(f.z - nm) + __expf(f.w - nm));
    m = nm;
  }
  const float mx = block_reduce(m, true, red);
  s = block_reduce(s * __expf(m - mx), false, red);  // a thread with no column has s = 0, m = -inf
  const float inv = 1.f / s;
  for (long long c = 4LL * threadIdx.x; c < n; c += step) {
    const float4 f = *reinterpret_cast<const float4*>(xr + c);
    *reinterpret_cast<uint2*>(yr + c) = make_uint2(pack_bf16(__expf(f.x - mx) * inv, __expf(f.y - mx) * inv),
                                                   pack_bf16(__expf(f.z - mx) * inv, __expf(f.w - mx) * inv));
  }
}

// y[r][0:n] = bf16(softmax(x[r][0:n])) for r < rows.  x fp32 with row stride ldx, y bf16 with row stride ldy (elements).
// n % 4 == 0; ldx, ldy multiples of 4; x 16-byte and y 8-byte aligned.  n <= 16384 runs from registers, longer rows on
// the two-pass kernel.
extern "C" int e4t_softmax_rows(const float* x, void* y, long long rows, int n, long long ldx, long long ldy,
                                void* stream_) {
  E4T_CHECK(rows >= 0 && n > 0 && n % 4 == 0,
            "e4t_softmax_rows: row length %d must be a positive multiple of 4", n);
  E4T_CHECK(ldx >= n && ldy >= n && ldx % 4 == 0 && ldy % 4 == 0, "e4t_softmax_rows: bad row strides");
  E4T_CHECK(((uintptr_t)x % 16) == 0 && ((uintptr_t)y % 8) == 0, "e4t_softmax_rows: misaligned operands");
  E4T_CHECK(rows <= 0x7fffffffLL, "e4t_softmax_rows: too many rows");
  if (rows == 0) return 0;
  if (n > kSmxMaxCols) {
    softmax_rows_long_kernel<<<(unsigned)rows, kSmxMaxThreads, 0, (cudaStream_t)stream_>>>(x, (bf16*)y, n, ldx, ldy);
    E4T_COUNT_LAUNCH();
    E4T_LAUNCH_CHECK();
    return 0;
  }
  int threads = cdiv(n, 4 * kSmxVec);
  threads = (threads + 31) / 32 * 32;
  softmax_rows_kernel<<<(unsigned)rows, threads, 0, (cudaStream_t)stream_>>>(x, (bf16*)y, n, ldx, ldy);
  E4T_COUNT_LAUNCH();
  E4T_LAUNCH_CHECK();
  return 0;
}
