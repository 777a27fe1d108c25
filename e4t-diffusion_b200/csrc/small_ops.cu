// e4t_b200 — small HBM-bound / short-sequence operators (sm_90a) that complete the E4T step on hand-written kernels:
//   * GELU / quick-GELU forward and backward           (open_clip ViT MLP `nn.GELU`, encoder.py:91-96; HF CLIP text
//                                                        `quick_gelu`, modeling_clip.py:10-82 via CLIPEncoderLayer)
//   * LeakyReLU forward / backward                      (E4TEncoder head, encoder.py:101-105,163-166)
//   * column sum  dbias[n] = sum_m dY[m][n]             (bias gradients of every trainable Linear / conv)
//   * embedding gradient dE[ids[p]] += dX[p]           (CLIP token table under --train_text_encoder), deterministic
//   * short-sequence attention with optional causal mask (N, M <= 128, dh <= 64): the CLIP text tower's 77-token
//     causal self-attention (modeling_clip.py:45-51).  One CTA per (batch, head); Q/K/V/dO live in shared memory as
//     bf16, the score matrix as fp32.  At 77 x 77 x 64 the whole tower's attention is 0.3 GFLOP per step: latency,
//     not throughput, is what matters, and a 128-row tensor-core tile would be 40 % padding.
#include "common.cuh"

// ---------------------------------------------------------------------------------------------
// activations (bf16 in / out, fp32 math); mode 0 = exact erf GELU, 1 = quick GELU x*sigmoid(1.702x), 2 = LeakyReLU(0.01)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float act_f(float x, int mode) {
  if (mode == 0) return 0.5f * x * (1.f + erff(x * 0.70710678118654752f));
  if (mode == 1) return x / (1.f + __expf(-1.702f * x));
  return x > 0.f ? x : 0.01f * x;
}
__device__ __forceinline__ float act_df(float x, int mode) {
  if (mode == 0) {
    const float cdf = 0.5f * (1.f + erff(x * 0.70710678118654752f));
    return cdf + x * 0.3989422804014327f * __expf(-0.5f * x * x);
  }
  if (mode == 1) {
    // beyond |x| = 1e30 the sigmoid is exactly 0 or 1 in fp32; the clamp keeps 1.702x finite, so the product below is
    // 0 * finite instead of 0 * inf = NaN for |x| > 2e38
    x = fminf(fmaxf(x, -1e30f), 1e30f);
    const float s = 1.f / (1.f + __expf(-1.702f * x));
    return s * (1.f + 1.702f * x * (1.f - s));
  }
  return x > 0.f ? 1.f : 0.01f;
}

template <bool BWD>
__global__ void __launch_bounds__(256) act_kernel(const bf16* __restrict__ x, const bf16* __restrict__ dy,
                                                  bf16* __restrict__ out, long long nvec, int mode) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    const uint4 u = reinterpret_cast<const uint4*>(x)[i];
    const uint32_t us[4] = {u.x, u.y, u.z, u.w};
    uint32_t ds[4] = {0, 0, 0, 0};
    if (BWD) {
      const uint4 d = reinterpret_cast<const uint4*>(dy)[i];
      ds[0] = d.x; ds[1] = d.y; ds[2] = d.z; ds[3] = d.w;
    }
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 v = unpack_bf16(us[j]);
      if (BWD) {
        const float2 g = unpack_bf16(ds[j]);
        o[j] = pack_bf16(g.x * act_df(v.x, mode), g.y * act_df(v.y, mode));
      } else {
        o[j] = pack_bf16(act_f(v.x, mode), act_f(v.y, mode));
      }
    }
    reinterpret_cast<uint4*>(out)[i] = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

extern "C" int e4t_act_fwd(const void* x, void* y, long long n, int mode, void* stream_) {
  E4T_CHECK(n % 8 == 0 && mode >= 0 && mode <= 2, "e4t_act_fwd: n %% 8 != 0 or bad mode");
  const long long nvec = n / 8;
  long long blocks = (nvec + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  if (blocks < 1) return 0;
  act_kernel<false><<<(int)blocks, 256, 0, (cudaStream_t)stream_>>>((const bf16*)x, nullptr, (bf16*)y, nvec, mode);
  E4T_COUNT_LAUNCH();
  E4T_LAUNCH_CHECK();
  return 0;
}
extern "C" int e4t_act_bwd(const void* x, const void* dy, void* dx, long long n, int mode, void* stream_) {
  E4T_CHECK(n % 8 == 0 && mode >= 0 && mode <= 2, "e4t_act_bwd: n %% 8 != 0 or bad mode");
  const long long nvec = n / 8;
  long long blocks = (nvec + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  if (blocks < 1) return 0;
  act_kernel<true><<<(int)blocks, 256, 0, (cudaStream_t)stream_>>>((const bf16*)x, (const bf16*)dy, (bf16*)dx, nvec, mode);
  E4T_COUNT_LAUNCH();
  E4T_LAUNCH_CHECK();
  return 0;
}

// ---------------------------------------------------------------------------------------------
// column sum: out[n] += sum_m X[m][n]   (X bf16 [M][ld], out fp32 [N], accumulating -> usable directly on .grad)
// block = 32 x 8 threads: each thread owns 8 consecutive columns (one 16-byte load), the 8 thread-rows stride over m
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) colsum_kernel(const bf16* __restrict__ X, float* __restrict__ out, long long M,
                                                     int N, long long ld, int rows_per_block, int blocks_per_group,
                                                     long long rows_per_group) {
  __shared__ float red[8][256 + 8];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int n0 = (blockIdx.x * 32 + tx) * 8;
  const long long grp = blockIdx.y / blocks_per_group;
  const long long m0 = grp * rows_per_group + (long long)(blockIdx.y % blocks_per_group) * rows_per_block;
  long long m1 = m0 + rows_per_block;
  const long long gend = (grp + 1) * rows_per_group < M ? (grp + 1) * rows_per_group : M;
  if (m1 > gend) m1 = gend;
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (n0 < N) {
    for (long long m = m0 + ty; m < m1; m += 8) {
      const uint4 u = *reinterpret_cast<const uint4*>(X + m * ld + n0);
      const float2 a = unpack_bf16(u.x), b = unpack_bf16(u.y), c = unpack_bf16(u.z), d = unpack_bf16(u.w);
      acc[0] += a.x; acc[1] += a.y; acc[2] += b.x; acc[3] += b.y;
      acc[4] += c.x; acc[5] += c.y; acc[6] += d.x; acc[7] += d.y;
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) red[ty][tx * 8 + j] = acc[j];
  __syncthreads();
  const int c = threadIdx.x;   // 256 columns of this block
  float s = 0.f;
#pragma unroll
  for (int r = 0; r < 8; ++r) s += red[r][c];
  const int n = blockIdx.x * 256 + c;
  if (n < N) atomicAdd(out + grp * N + n, s);
}
// out[g][n] += sum over the rows m of group g (m / rows_per_group == g) of X[m][n]; rows_per_group <= 0: one group.
// Bias gradients (one group) and the per-image time-embedding row gradient of ResnetBlock2D (group = image).
extern "C" int e4t_colsum_acc(const void* X, float* out, long long M, int N, long long ld, long long rows_per_group,
                              void* stream_) {
  E4T_CHECK(N % 8 == 0 && ld % 8 == 0, "e4t_colsum_acc: N and ld must be multiples of 8");
  if (M <= 0) return 0;
  if (rows_per_group <= 0 || rows_per_group > M) rows_per_group = M;
  E4T_CHECK(M % rows_per_group == 0, "e4t_colsum_acc: M must be a multiple of rows_per_group");
  const long long groups = M / rows_per_group;
  const int gx = cdiv(N, 256);
  long long bpg = (132 * 4 + gx * groups - 1) / (gx * groups);
  if (bpg < 1) bpg = 1;
  int rpb = (int)((rows_per_group + bpg - 1) / bpg);
  if (rpb < 64) rpb = 64;
  bpg = (rows_per_group + rpb - 1) / rpb;
  colsum_kernel<<<dim3(gx, (unsigned)(groups * bpg)), 256, 0, (cudaStream_t)stream_>>>((const bf16*)X, out, M, N, ld, rpb,
                                                                                     (int)bpg, rows_per_group);
  E4T_COUNT_LAUNCH();
  E4T_LAUNCH_CHECK();
  return 0;
}

// ---------------------------------------------------------------------------------------------
// embedding gradient: dE[ids[p]][:] += dX[p][:] for p < P (token-embedding backward of the CLIP text tower)
// Deterministic, without atomics.  Block (p, column slice): warp 0 scans ids[] in ballots of 32 and lists, in position
// order, every position that carries ids[p].  Only the block whose p is the first of them (the run's head) goes on: it
// sums the listed rows in list order in fp32 and adds the sum once into the table row, which no other block writes.
// Non-head blocks stop at their id's first occurrence, which in a batch of prompts is almost always in the first row.
// The skewed case (the pad/EOS id fills most of every 77-token prompt: ~1,000 of 1,232 rows at B = 16) is one head per
// column slice summing its run with 8 row loads in flight per thread.  The grid depends on P and D only, so the launch
// can be captured in a CUDA graph.  A row's sum is plain fp32 in position order, so its rounding error grows with its
// run: ~1e-6 of the row's own magnitude for the ~1,000-position pad row, which is ~30x the table's typical row.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float4 load_row4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ float4 load_row4(const bf16* p) {
  const uint2 u = *reinterpret_cast<const uint2*>(p);
  const float2 a = unpack_bf16(u.x), b = unpack_bf16(u.y);
  return make_float4(a.x, a.y, b.x, b.y);
}

constexpr int EMB_THREADS = 64;    // x 4 columns per thread: 256 columns per block, 3 slices at D = 768
constexpr int EMB_MAX_P = 12288;   // the position list lives in dynamic shared memory (<= 48 KiB)

template <typename T>
__global__ void __launch_bounds__(EMB_THREADS) embedding_grad_kernel(const long long* __restrict__ ids,
                                                                     const T* __restrict__ dX, float* __restrict__ dE,
                                                                     int P, int D, long long V) {
  extern __shared__ int run[];
  __shared__ int run_len;
  const int p = blockIdx.x;
  const long long id = ids[p];
  if (threadIdx.x < 32) {
    const int lane = threadIdx.x;
    int n = 0;
    bool head = true;
    for (int base = 0; base < P; base += 32) {
      const int q = base + lane;
      const bool m = q < P && ids[q] == id;
      const unsigned b = __ballot_sync(0xffffffffu, m);
      if (n == 0 && b != 0u && base + __ffs(b) - 1 != p) {   // an earlier position owns this id (warp-uniform)
        head = false;
        break;
      }
      if (m) run[n + __popc(b & ((1u << lane) - 1u))] = q;
      n += __popc(b);
    }
    if (lane == 0) run_len = head ? n : 0;
  }
  __syncthreads();
  const int n = run_len;
  const int c = (blockIdx.y * EMB_THREADS + threadIdx.x) * 4;
  if (n == 0 || id < 0 || id >= V || c >= D) return;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  int i = 0;
  for (; i + 8 <= n; i += 8) {
    float4 v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = load_row4(dX + (long long)run[i + j] * D + c);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      acc.x += v[j].x; acc.y += v[j].y; acc.z += v[j].z; acc.w += v[j].w;
    }
  }
  for (; i < n; ++i) {
    const float4 v = load_row4(dX + (long long)run[i] * D + c);
    acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
  }
  float4* e = reinterpret_cast<float4*>(dE + id * D + c);
  float4 o = *e;
  o.x += acc.x; o.y += acc.y; o.z += acc.z; o.w += acc.w;
  *e = o;
}

extern "C" int e4t_embedding_grad(const long long* ids, const void* dX, int dx_f32, float* dE, long long P, int D,
                                  long long V, void* stream_) {
  E4T_CHECK(P <= EMB_MAX_P, "e4t_embedding_grad: at most %d positions (got %lld)", EMB_MAX_P, P);
  E4T_CHECK(D % 4 == 0 && ((uintptr_t)dX % (dx_f32 ? 16 : 8)) == 0 && ((uintptr_t)dE % 16) == 0,
            "e4t_embedding_grad: D must be a multiple of 4 and dX / dE aligned to 4 elements");
  if (P <= 0 || D <= 0) return 0;
  const dim3 grid((unsigned)P, (unsigned)cdiv(D / 4, EMB_THREADS));
  const size_t smem = (size_t)P * sizeof(int);
  if (dx_f32)
    embedding_grad_kernel<float><<<grid, EMB_THREADS, smem, (cudaStream_t)stream_>>>(ids, (const float*)dX, dE, (int)P,
                                                                                     D, V);
  else
    embedding_grad_kernel<bf16><<<grid, EMB_THREADS, smem, (cudaStream_t)stream_>>>(ids, (const bf16*)dX, dE, (int)P,
                                                                                    D, V);
  E4T_COUNT_LAUNCH();
  E4T_LAUNCH_CHECK();
  return 0;
}

// ---------------------------------------------------------------------------------------------
// affine-parameter gradients of LayerNorm / GroupNorm(+SiLU):  dgamma[c] += sum_r dz[r][c] * xhat[r][c],
// dbeta[c] += sum_r dz[r][c], with xhat = (x - mean) * rstd and dz = dy (LayerNorm, GroupNorm) or dy * silu'(z),
// z = xhat * gamma + beta (GroupNorm+SiLU).  Statistics:
//   PERCOL = false (LayerNorm): stats fp32 [rows][2] = (mean, rstd) per row
//   PERCOL = true  (GroupNorm): st0 = e4t_groupnorm_fwd's stats [rows / rows_per_group][G][kGNStat] (common.cuh)
// ---------------------------------------------------------------------------------------------
template <bool PERCOL>
__global__ void __launch_bounds__(256) norm_param_grad_kernel(const bf16* __restrict__ X, const bf16* __restrict__ dY,
                                                              const float* __restrict__ st0,
                                                              const float* __restrict__ gamma, const float* __restrict__ beta,
                                                              float* __restrict__ dgamma, float* __restrict__ dbeta,
                                                              long long rows, int C, int rows_per_block,
                                                              long long rows_per_group, int G, float eps, int silu) {
  __shared__ float red[2][8][256 + 8];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int n0 = (blockIdx.x * 32 + tx) * 8;
  const long long m0 = (long long)blockIdx.y * rows_per_block;
  long long m1 = m0 + rows_per_block;
  if (m1 > rows) m1 = rows;
  float ag[8] = {0, 0, 0, 0, 0, 0, 0, 0}, ab[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (n0 < C) {
    float gm[8], bt[8], mean[8], rstd[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      gm[j] = gamma[n0 + j];
      bt[j] = beta ? beta[n0 + j] : 0.f;
    }
    const int cpg = PERCOL ? C / G : 1;
    const float inv_n = PERCOL ? 1.f / ((float)rows_per_group * (float)cpg) : 0.f;
    long long img = -1;
    for (long long m = m0 + ty; m < m1; m += 8) {
      const uint4 ux = *reinterpret_cast<const uint4*>(X + m * C + n0);
      const uint4 ud = *reinterpret_cast<const uint4*>(dY + m * C + n0);
      const uint32_t xs[4] = {ux.x, ux.y, ux.z, ux.w}, ds[4] = {ud.x, ud.y, ud.z, ud.w};
      if (PERCOL) {
        if (m / rows_per_group != img) {   // the image changed: this thread's (mean, rstd) of its 8 channels
          img = m / rows_per_group;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float2 mr = gn_mean_rstd(st0 + (img * G + (n0 + j) / cpg) * kGNStat, inv_n, eps);
            mean[j] = mr.x;
            rstd[j] = mr.y;
          }
        }
      } else {
        const float mu = st0[m * 2], rs = st0[m * 2 + 1];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          mean[j] = mu;
          rstd[j] = rs;
        }
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float2 xv = unpack_bf16(xs[q]), dv = unpack_bf16(ds[q]);
        const float xin[2] = {xv.x, xv.y}, din[2] = {dv.x, dv.y};
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int j = 2 * q + u;
          const float xh = (xin[u] - mean[j]) * rstd[j];
          float dz = din[u];
          if (silu) {
            const float z = xh * gm[j] + bt[j];
            const float sg = 1.f / (1.f + __expf(-z));
            dz *= sg * (1.f + z * (1.f - sg));
          }
          ag[j] += dz * xh;
          ab[j] += dz;
        }
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    red[0][ty][tx * 8 + j] = ag[j];
    red[1][ty][tx * 8 + j] = ab[j];
  }
  __syncthreads();
  const int c = threadIdx.x;
  float sg = 0.f, sb = 0.f;
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    sg += red[0][r][c];
    sb += red[1][r][c];
  }
  const int n = blockIdx.x * 256 + c;
  if (n < C) {
    atomicAdd(dgamma + n, sg);
    atomicAdd(dbeta + n, sb);
  }
}
static void norm_grid(long long rows, int C, int& gx, long long& gy, int& rpb) {
  gx = cdiv(C, 256);
  gy = (132 * 4 + gx - 1) / gx;
  rpb = (int)((rows + gy - 1) / gy);
  if (rpb < 64) rpb = 64;
  gy = (rows + rpb - 1) / rpb;
}
// LayerNorm: x, dy bf16 [rows][C]; stats fp32 [rows][2] (mean, rstd) as written by e4t_layernorm_fwd.
extern "C" int e4t_layernorm_param_grad(const void* x, const void* dy, const float* stats, const float* gamma,
                                        float* dgamma, float* dbeta, long long rows, int C, void* stream_) {
  E4T_CHECK(C % 8 == 0, "e4t_layernorm_param_grad: C %% 8 != 0");
  if (rows <= 0) return 0;
  int gx, rpb; long long gy;
  norm_grid(rows, C, gx, gy, rpb);
  norm_param_grad_kernel<false><<<dim3(gx, (unsigned)gy), 256, 0, (cudaStream_t)stream_>>>(
      (const bf16*)x, (const bf16*)dy, stats, gamma, nullptr, dgamma, dbeta, rows, C, rpb, 1, 1, 0.f, 0);
  E4T_COUNT_LAUNCH();
  E4T_LAUNCH_CHECK();
  return 0;
}
// GroupNorm(+SiLU): x, dy bf16 [B*HW][C]; stats fp32 [B][G][kGNStat] as written by e4t_groupnorm_fwd.
extern "C" int e4t_groupnorm_param_grad(const void* x, const void* dy, const float* stats, const float* gamma,
                                        const float* beta, float* dgamma, float* dbeta, int B, int HW, int C, int G,
                                        float eps, int act_silu, void* stream_) {
  E4T_CHECK(C % 8 == 0 && C % G == 0, "e4t_groupnorm_param_grad: unsupported C=%d G=%d", C, G);
  const long long rows = (long long)B * HW;
  if (rows <= 0) return 0;
  int gx, rpb; long long gy;
  norm_grid(rows, C, gx, gy, rpb);
  norm_param_grad_kernel<true><<<dim3(gx, (unsigned)gy), 256, 0, (cudaStream_t)stream_>>>(
      (const bf16*)x, (const bf16*)dy, stats, gamma, beta, dgamma, dbeta, rows, C, rpb, HW, G, eps, act_silu);
  E4T_COUNT_LAUNCH();
  E4T_LAUNCH_CHECK();
  return 0;
}

// ---------------------------------------------------------------------------------------------
// weight gradients of the UNet's two narrow convolutions (conv_in 4 -> C, conv_out C -> 4; 3x3, pad 1):
//   acc[w][n][tap] += sum_{b,y,x} wide[b][y][x][w] * narrow[b][n][y + sgn*(ky-1)][x + sgn*(kx-1)]
// wide: bf16 NHWC [B][H][W][Cw]; narrow: fp32 NCHW [B][Cn][H][W] (Cn <= 4); acc fp32 [Cw][Cn][9].
//   conv_in  (unet_2d_condition.py:481): wide = dY, narrow = latent input, sgn = +1 -> acc = dW[co][ci][ky][kx]
//   conv_out (unet_2d_condition.py:557): wide = X,  narrow = dY,           sgn = -1 -> acc[ci][co][tap] = dW[co][ci][ky][kx]
// one thread per wide channel, 36 register accumulators; a block walks `rows_per_block` image rows.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(320) narrow_conv_wgrad_kernel(const bf16* __restrict__ wide,
                                                                const float* __restrict__ narrow, float* __restrict__ acc,
                                                                int H, int W, int Cw, int Cn, int sgn, int rows_per_block) {
  extern __shared__ float patch[];   // [Cn][rows_per_block + 2][W + 2]
  const int b = blockIdx.z, y0 = blockIdx.y * rows_per_block;
  const int w = blockIdx.x * blockDim.x + threadIdx.x;
  const int PW = W + 2, PH = rows_per_block + 2;
  for (int i = threadIdx.x; i < Cn * PH * PW; i += blockDim.x) {
    const int n = i / (PH * PW), r = (i / PW) % PH, c = i % PW;
    const int y = y0 + r - 1, x = c - 1;
    patch[i] = (y >= 0 && y < H && x >= 0 && x < W) ? narrow[(((long long)b * Cn + n) * H + y) * W + x] : 0.f;
  }
  __syncthreads();
  if (w >= Cw) return;
  float a[4][9];
#pragma unroll
  for (int n = 0; n < 4; ++n)
#pragma unroll
    for (int t = 0; t < 9; ++t) a[n][t] = 0.f;
  for (int r = 0; r < rows_per_block && y0 + r < H; ++r) {
    for (int x = 0; x < W; ++x) {
      const float v = __bfloat162float(wide[(((long long)b * H + y0 + r) * W + x) * Cw + w]);
#pragma unroll
      for (int n = 0; n < 4; ++n) {
        if (n < Cn) {
#pragma unroll
          for (int t = 0; t < 9; ++t) {
            const int dy = sgn * (t / 3 - 1), dx = sgn * (t % 3 - 1);
            a[n][t] += v * patch[(n * PH + r + 1 + dy) * PW + x + 1 + dx];
          }
        }
      }
    }
  }
#pragma unroll
  for (int n = 0; n < 4; ++n)
    if (n < Cn)
#pragma unroll
      for (int t = 0; t < 9; ++t) atomicAdd(acc + ((long long)w * Cn + n) * 9 + t, a[n][t]);
}
extern "C" int e4t_narrow_conv_wgrad(const void* wide, const float* narrow, float* acc, int B, int H, int W, int Cw,
                                     int Cn, int sgn, void* stream_) {
  E4T_CHECK(Cn >= 1 && Cn <= 4, "e4t_narrow_conv_wgrad: narrow channel count must be 1..4 (got %d)", Cn);
  E4T_CHECK(sgn == 1 || sgn == -1, "e4t_narrow_conv_wgrad: sgn must be +-1");
  const int rpb = H >= 8 ? 8 : H;
  const size_t smem = (size_t)Cn * (rpb + 2) * (W + 2) * sizeof(float);
  const int threads = Cw >= 320 ? 320 : ((Cw + 31) / 32 * 32);
  narrow_conv_wgrad_kernel<<<dim3(cdiv(Cw, threads), cdiv(H, rpb), B), threads, smem, (cudaStream_t)stream_>>>(
      (const bf16*)wide, narrow, acc, H, W, Cw, Cn, sgn, rpb);
  E4T_COUNT_LAUNCH();
  E4T_LAUNCH_CHECK();
  return 0;
}

// ---------------------------------------------------------------------------------------------
// short-sequence attention (N, M <= 128, dh <= 64, dh % 8 == 0), optional causal mask (key j > query i masked)
// ---------------------------------------------------------------------------------------------
static constexpr int kSA_MAX = 128;      // max sequence
static constexpr int kSA_LD = 64 + 8;    // bf16 row pitch of the Q/K/V/dO tiles (72: 16-byte aligned rows, spreads banks)
static constexpr int kSA_PLD = kSA_MAX + 1;

struct SmallAttnArgs {
  const bf16 *Q, *K, *V, *O, *dO;
  bf16 *Out, *dQ, *dK, *dV;
  float* LSE;
  int B, H, N, M, dh, causal;
  long long ldq, q_bs, ldk, k_bs, ldv, v_bs, ldo, o_bs, lddo, do_bs, lddq, dq_bs, lddk, dk_bs, lddv, dv_bs;
  float scale;
};

__device__ __forceinline__ void sa_load_tile(bf16* s, const bf16* g, int rows, int dh, long long ld) {
  const int vpr = dh / 8;
  for (int i = threadIdx.x; i < rows * vpr; i += blockDim.x) {
    const int r = i / vpr, c = (i % vpr) * 8;
    *reinterpret_cast<uint4*>(s + r * kSA_LD + c) = *reinterpret_cast<const uint4*>(g + (long long)r * ld + c);
  }
}
__device__ __forceinline__ float sa_dot(const bf16* a, const bf16* b, int dh) {
  float acc = 0.f;
  for (int d = 0; d < dh; d += 8) {
    const uint4 x = *reinterpret_cast<const uint4*>(a + d), y = *reinterpret_cast<const uint4*>(b + d);
    const uint32_t xs[4] = {x.x, x.y, x.z, x.w}, ys[4] = {y.x, y.y, y.z, y.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 p = unpack_bf16(xs[j]), q = unpack_bf16(ys[j]);
      acc += p.x * q.x + p.y * q.y;
    }
  }
  return acc;
}

static constexpr int kSA_CH = 32;   // query (fwd, dQ) or key (dK/dV) rows per CTA: blockIdx.z = chunk

// P[i][j] for i in [i0,i1), j in [j0,j1) into sP (row pitch kSA_PLD, indexed [i - i0][j]): softmax over ALL keys when
// lse == nullptr (forward: the CTA owns whole rows, j0 = 0, j1 = M; the row LSE is written to lse_out), otherwise
// exp(s - lse[i]) (backward recomputation).  Masked (causal) entries are exactly 0.
__device__ __forceinline__ void sa_probs(float* sP, const bf16* sQ, const bf16* sK, const SmallAttnArgs& a, int i0, int i1,
                                         int j0, int j1, float* lse_out, const float* lse) {
  const int ni = i1 - i0, nj = j1 - j0;
  for (int idx = threadIdx.x; idx < ni * nj; idx += blockDim.x) {
    const int i = i0 + idx / nj, j = j0 + idx % nj;
    float s = -INFINITY;
    if (!a.causal || j <= i) s = sa_dot(sQ + i * kSA_LD, sK + j * kSA_LD, a.dh) * a.scale;
    sP[(i - i0) * kSA_PLD + j] = s;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int i = i0 + warp; i < i1; i += nw) {
    float* row = sP + (i - i0) * kSA_PLD;
    float l;
    if (lse) {
      l = lse[i];
    } else {
      float mx = -INFINITY;
      for (int j = j0 + lane; j < j1; j += 32) mx = fmaxf(mx, row[j]);
      mx = warp_max(mx);
      float sum = 0.f;
      for (int j = j0 + lane; j < j1; j += 32) sum += __expf(row[j] - mx);
      sum = warp_sum(sum);
      l = mx + logf(sum);
      if (lse_out && lane == 0) lse_out[i] = l;
    }
    for (int j = j0 + lane; j < j1; j += 32) row[j] = __expf(row[j] - l);   // masked entries: exp(-inf) = 0
  }
  __syncthreads();
}

// forward: CTA = (head, batch, chunk of kSA_CH queries)
__global__ void __launch_bounds__(256) attn_small_fwd_kernel(const SmallAttnArgs a) {
  extern __shared__ __align__(16) uint8_t sm[];
  bf16* sQ = reinterpret_cast<bf16*>(sm);
  bf16* sK = sQ + kSA_MAX * kSA_LD;
  bf16* sV = sK + kSA_MAX * kSA_LD;
  float* sP = reinterpret_cast<float*>(sV + kSA_MAX * kSA_LD);   // [kSA_CH][kSA_PLD]
  const int h = blockIdx.x, b = blockIdx.y;
  const int i0 = blockIdx.z * kSA_CH, i1 = min(a.N, i0 + kSA_CH);
  if (i0 >= a.N) return;
  const int mk = a.causal ? min(a.M, i1) : a.M;                  // keys this chunk can see
  sa_load_tile(sQ + i0 * kSA_LD, a.Q + b * a.q_bs + (long long)i0 * a.ldq + h * a.dh, i1 - i0, a.dh, a.ldq);
  sa_load_tile(sK, a.K + b * a.k_bs + h * a.dh, mk, a.dh, a.ldk);
  sa_load_tile(sV, a.V + b * a.v_bs + h * a.dh, mk, a.dh, a.ldv);
  __syncthreads();
  sa_probs(sP, sQ, sK, a, i0, i1, 0, mk, a.LSE + ((long long)b * a.H + h) * a.N, nullptr);
  const int dp = a.dh / 2;
  for (int idx = threadIdx.x; idx < (i1 - i0) * dp; idx += blockDim.x) {
    const int i = i0 + idx / dp, d = (idx % dp) * 2;
    const float* pr = sP + (i - i0) * kSA_PLD;
    float o0 = 0.f, o1 = 0.f;
    const int jmax = a.causal ? min(mk, i + 1) : mk;
    for (int j = 0; j < jmax; ++j) {
      const float2 v = unpack_bf16(*reinterpret_cast<const uint32_t*>(sV + j * kSA_LD + d));
      o0 += pr[j] * v.x;
      o1 += pr[j] * v.y;
    }
    *reinterpret_cast<uint32_t*>(a.Out + b * a.o_bs + (long long)i * a.ldo + h * a.dh + d) = pack_bf16(o0, o1);
  }
}

// backward: WHICH = 0 -> dQ, CTA = (head, batch, chunk of kSA_CH queries); WHICH = 1 -> dK and dV, CTA = chunk of keys.
// Each CTA recomputes its slab of P from the saved LSE (0.4 MFLOP) instead of exchanging partial sums.
template <int WHICH>
__global__ void __launch_bounds__(256) attn_small_bwd_kernel(const SmallAttnArgs a) {
  extern __shared__ __align__(16) uint8_t sm[];
  bf16* sQ = reinterpret_cast<bf16*>(sm);
  bf16* sK = sQ + kSA_MAX * kSA_LD;
  bf16* sV = sK + kSA_MAX * kSA_LD;
  bf16* sdO = sV + kSA_MAX * kSA_LD;
  float* sP = reinterpret_cast<float*>(sdO + kSA_MAX * kSA_LD);   // WHICH 0: [kSA_CH][PLD] (rows = my queries);
  float* sdS = sP + kSA_MAX * kSA_PLD;                            // WHICH 1: [N][PLD] (all queries, my key columns)
  float* sD = sdS + kSA_MAX * kSA_PLD;     // [N] rowsum(dO * O)
  float* sL = sD + kSA_MAX;                // [N] LSE
  const int h = blockIdx.x, b = blockIdx.y;
  const int N = a.N, M = a.M, dh = a.dh;
  int i0, i1, j0, j1;
  if (WHICH == 0) {
    i0 = blockIdx.z * kSA_CH; i1 = min(N, i0 + kSA_CH);
    if (i0 >= N) return;
    j0 = 0; j1 = a.causal ? min(M, i1) : M;
  } else {
    j0 = blockIdx.z * kSA_CH; j1 = min(M, j0 + kSA_CH);
    if (j0 >= M) return;
    i0 = a.causal ? j0 : 0; i1 = N;
    if (i0 >= N) {   // keys no query can see: zero gradients
      for (int idx = threadIdx.x; idx < (j1 - j0) * (dh / 2); idx += blockDim.x) {
        const int j = j0 + idx / (dh / 2), d = (idx % (dh / 2)) * 2;
        *reinterpret_cast<uint32_t*>(a.dK + b * a.dk_bs + (long long)j * a.lddk + h * dh + d) = 0u;
        *reinterpret_cast<uint32_t*>(a.dV + b * a.dv_bs + (long long)j * a.lddv + h * dh + d) = 0u;
      }
      return;
    }
  }
  sa_load_tile(sQ + i0 * kSA_LD, a.Q + b * a.q_bs + (long long)i0 * a.ldq + h * dh, i1 - i0, dh, a.ldq);
  sa_load_tile(sdO + i0 * kSA_LD, a.dO + b * a.do_bs + (long long)i0 * a.lddo + h * dh, i1 - i0, dh, a.lddo);
  sa_load_tile(sK + j0 * kSA_LD, a.K + b * a.k_bs + (long long)j0 * a.ldk + h * dh, j1 - j0, dh, a.ldk);
  sa_load_tile(sV + j0 * kSA_LD, a.V + b * a.v_bs + (long long)j0 * a.ldv + h * dh, j1 - j0, dh, a.ldv);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int i = i0 + warp; i < i1; i += nw) {   // D_i = sum_d dO[i][d] O[i][d]
    const bf16* o = a.O + b * a.o_bs + (long long)i * a.ldo + h * dh;
    const bf16* d = a.dO + b * a.do_bs + (long long)i * a.lddo + h * dh;
    float acc = 0.f;
    for (int c = lane * 2; c < dh; c += 64) {
      const float2 x = unpack_bf16(*reinterpret_cast<const uint32_t*>(o + c));
      const float2 y = unpack_bf16(*reinterpret_cast<const uint32_t*>(d + c));
      acc += x.x * y.x + x.y * y.y;
    }
    acc = warp_sum(acc);
    if (lane == 0) {
      sD[i] = acc;
      sL[i] = a.LSE[((long long)b * a.H + h) * N + i];
    }
  }
  __syncthreads();
  sa_probs(sP, sQ, sK, a, i0, i1, j0, j1, nullptr, sL);
  // dS[i][j] = P (dP - D) * scale, dP[i][j] = dO[i] . V[j]
  const int nj = j1 - j0;
  for (int idx = threadIdx.x; idx < (i1 - i0) * nj; idx += blockDim.x) {
    const int i = i0 + idx / nj, j = j0 + idx % nj;
    const float p = sP[(i - i0) * kSA_PLD + j];
    float ds = 0.f;
    if (p != 0.f) ds = p * (sa_dot(sdO + i * kSA_LD, sV + j * kSA_LD, dh) - sD[i]) * a.scale;
    sdS[(i - i0) * kSA_PLD + j] = ds;
  }
  __syncthreads();
  const int dp = dh / 2;
  if (WHICH == 0) {   // dQ[i][d] = sum_j dS[i][j] K[j][d]
    for (int idx = threadIdx.x; idx < (i1 - i0) * dp; idx += blockDim.x) {
      const int i = i0 + idx / dp, d = (idx % dp) * 2;
      const float* r = sdS + (i - i0) * kSA_PLD;
      float o0 = 0.f, o1 = 0.f;
      const int jmax = a.causal ? min(j1, i + 1) : j1;
      for (int j = 0; j < jmax; ++j) {
        const float2 v = unpack_bf16(*reinterpret_cast<const uint32_t*>(sK + j * kSA_LD + d));
        o0 += r[j] * v.x;
        o1 += r[j] * v.y;
      }
      *reinterpret_cast<uint32_t*>(a.dQ + b * a.dq_bs + (long long)i * a.lddq + h * dh + d) = pack_bf16(o0, o1);
    }
  } else {            // dK[j][d] = sum_i dS[i][j] Q[i][d];  dV[j][d] = sum_i P[i][j] dO[i][d]
    for (int idx = threadIdx.x; idx < nj * dp; idx += blockDim.x) {
      const int j = j0 + idx / dp, d = (idx % dp) * 2;
      float k0 = 0.f, k1 = 0.f, v0 = 0.f, v1 = 0.f;
      const int ia = a.causal ? max(i0, j) : i0;
      for (int i = ia; i < i1; ++i) {
        const float ds = sdS[(i - i0) * kSA_PLD + j], p = sP[(i - i0) * kSA_PLD + j];
        const float2 q = unpack_bf16(*reinterpret_cast<const uint32_t*>(sQ + i * kSA_LD + d));
        const float2 g = unpack_bf16(*reinterpret_cast<const uint32_t*>(sdO + i * kSA_LD + d));
        k0 += ds * q.x; k1 += ds * q.y;
        v0 += p * g.x;  v1 += p * g.y;
      }
      *reinterpret_cast<uint32_t*>(a.dK + b * a.dk_bs + (long long)j * a.lddk + h * dh + d) = pack_bf16(k0, k1);
      *reinterpret_cast<uint32_t*>(a.dV + b * a.dv_bs + (long long)j * a.lddv + h * dh + d) = pack_bf16(v0, v1);
    }
  }
}

static int sa_checks(int N, int M, int dh, long long ldq, long long ldk, long long ldv) {
  E4T_CHECK(N >= 1 && M >= 1 && N <= kSA_MAX && M <= kSA_MAX, "e4t_attn_small: N, M must be in [1, 128] (got %d, %d)", N, M);
  E4T_CHECK(dh % 8 == 0 && dh >= 8 && dh <= 64, "e4t_attn_small: head dim %d unsupported (dh %% 8 == 0, <= 64)", dh);
  E4T_CHECK(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0, "e4t_attn_small: row strides must be multiples of 8 elements");
  return 0;
}

extern "C" int e4t_attn_small_fwd(const void* Q, const void* K, const void* V, void* O, float* LSE, int B, int H, int N,
                                  int M, int dh, long long ldq, long long q_bs, long long ldk, long long k_bs,
                                  long long ldv, long long v_bs, long long ldo, long long o_bs, float scale, int causal,
                                  void* stream_) {
  if (int e = sa_checks(N, M, dh, ldq, ldk, ldv)) return e;
  SmallAttnArgs a;
  memset(&a, 0, sizeof(a));
  a.Q = (const bf16*)Q; a.K = (const bf16*)K; a.V = (const bf16*)V; a.Out = (bf16*)O; a.LSE = LSE;
  a.B = B; a.H = H; a.N = N; a.M = M; a.dh = dh; a.causal = causal;
  a.ldq = ldq; a.q_bs = q_bs; a.ldk = ldk; a.k_bs = k_bs; a.ldv = ldv; a.v_bs = v_bs; a.ldo = ldo; a.o_bs = o_bs;
  a.scale = scale;
  const size_t smem = (size_t)3 * kSA_MAX * kSA_LD * 2 + (size_t)kSA_CH * kSA_PLD * 4;
  static bool attr = false;
  if (!attr) {
    E4T_CUDA(cudaFuncSetAttribute(attn_small_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr = true;
  }
  attn_small_fwd_kernel<<<dim3(H, B, cdiv(N, kSA_CH)), 256, smem, (cudaStream_t)stream_>>>(a);
  E4T_COUNT_LAUNCH();
  E4T_LAUNCH_CHECK();
  return 0;
}

extern "C" int e4t_attn_small_bwd(const void* Q, const void* K, const void* V, const void* O, const void* dO,
                                  const float* LSE, void* dQ, void* dK, void* dV, int B, int H, int N, int M, int dh,
                                  long long ldq, long long q_bs, long long ldk, long long k_bs, long long ldv,
                                  long long v_bs, long long ldo, long long o_bs, long long lddo, long long do_bs,
                                  long long lddq, long long dq_bs, long long lddk, long long dk_bs, long long lddv,
                                  long long dv_bs, float scale, int causal, void* stream_) {
  if (int e = sa_checks(N, M, dh, ldq, ldk, ldv)) return e;
  E4T_CHECK(lddo % 8 == 0, "e4t_attn_small_bwd: dO row stride must be a multiple of 8 elements");
  SmallAttnArgs a;
  memset(&a, 0, sizeof(a));
  a.Q = (const bf16*)Q; a.K = (const bf16*)K; a.V = (const bf16*)V; a.O = (const bf16*)O; a.dO = (const bf16*)dO;
  a.LSE = const_cast<float*>(LSE);
  a.dQ = (bf16*)dQ; a.dK = (bf16*)dK; a.dV = (bf16*)dV;
  a.B = B; a.H = H; a.N = N; a.M = M; a.dh = dh; a.causal = causal;
  a.ldq = ldq; a.q_bs = q_bs; a.ldk = ldk; a.k_bs = k_bs; a.ldv = ldv; a.v_bs = v_bs; a.ldo = ldo; a.o_bs = o_bs;
  a.lddo = lddo; a.do_bs = do_bs; a.lddq = lddq; a.dq_bs = dq_bs; a.lddk = lddk; a.dk_bs = dk_bs;
  a.lddv = lddv; a.dv_bs = dv_bs;
  a.scale = scale;
  const size_t smem = (size_t)4 * kSA_MAX * kSA_LD * 2 + (size_t)2 * kSA_MAX * kSA_PLD * 4 + 2 * kSA_MAX * 4;
  static bool attr = false;
  if (!attr) {
    E4T_CUDA(cudaFuncSetAttribute(attn_small_bwd_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    E4T_CUDA(cudaFuncSetAttribute(attn_small_bwd_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr = true;
  }
  attn_small_bwd_kernel<0><<<dim3(H, B, cdiv(N, kSA_CH)), 256, smem, (cudaStream_t)stream_>>>(a);
  E4T_COUNT_LAUNCH();
  attn_small_bwd_kernel<1><<<dim3(H, B, cdiv(M, kSA_CH)), 256, smem, (cudaStream_t)stream_>>>(a);
  E4T_COUNT_LAUNCH();
  E4T_LAUNCH_CHECK();
  return 0;
}
