// e4t — token merging (ToMe, bipartite soft matching on a 2-D grid) for the UNet's transformer blocks.
//
// A call of a merging block runs, per image of the batch:
//   partition  which tokens are dst (one per sy x sx cell, at the cell's drawn pattern offset; the pattern is shared by
//              the batch) and which are src; both lists in raster order.  One CTA for the whole batch.
//   normalise  fp32 inverse row norms, the unit-norm src and dst rows in bf16 (compact [B][Ns][C] and [B][Nd][C]).
//   match      cos(src i, dst j) on wgmma from TMA-loaded K panels; per src row the maximum and its (lowest raster
//              index) argmax stay in registers across the dst tiles, so no Ns x Nd score matrix reaches memory.
//   select     one CTA per image: the r src tokens with the largest node_max (ties: lower raster index) are merged;
//              a bitwise radix select finds the r-th key, block prefix sums place the kept tokens and a stable
//              split-based radix sort groups the merged tokens by their dst.  Output: pos[N] (merged row of each
//              token's representative), the CSR member lists of the N - r merged rows (members in ascending raster
//              order) and 1 / (1 + count) per merged row.  No atomics: the result is a function of the inputs only.
//   gather     reduce: N' rows, each the weighted fp32 sum of its CSR members in list order (merge forward with weight
//              1 / len, unmerge backward with weight 1); expand: N rows, out[i] = w[pos i] * y[pos i] (+ residual[i])
//              (unmerge forward with the residual fused, merge backward).  16-byte vector I/O, bf16 in and out.
// Every size follows from the shapes and r: the kernels never synchronise with the host and are graph-capturable.
#include "common.cuh"
#include "wgmma.cuh"

static constexpr int kMatchThreads = 384;    // warpgroup 0: TMA producer; 1, 2: 64 src rows each
static constexpr int kMatchStages = 4;
static constexpr uint32_t kPanel = 128 * 128;   // 128 rows x 64 bf16, SWIZZLE_128B
static constexpr uint32_t kMatchStage = 2 * kPanel;
static constexpr size_t kMatchSmem = 1024 + kMatchStages * kMatchStage + 16 * kMatchStages;
static constexpr int kSelectThreads = 1024;
static constexpr int kSelectMaxTokens = 16384;  // 14-bit raster indices and dst ranks in the packed sort keys
static constexpr int kScanThreads = 1024;

// ---------------------------------------------------------------------------------------------
// block-wide exclusive prefix sum of one int per thread (blockDim.x a multiple of 32, <= 1024); sh: 33 ints
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ int block_excl_scan(int v, int* sh, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) sh[warp] = x;
  __syncthreads();
  if (warp == 0) {
    int s = lane < nw ? sh[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += y;
    }
    sh[lane] = s;
  }
  __syncthreads();
  const int base = warp > 0 ? sh[warp - 1] : 0;
  *total = sh[nw - 1];
  __syncthreads();
  return base + x - v;
}

__device__ __forceinline__ int block_sum(int v, int* sh) {
  int t;
  block_excl_scan(v, sh, &t);
  return t;
}

// contiguous chunk [lo, hi) of n items owned by this thread (so that a block scan over chunk counts is a raster scan)
__device__ __forceinline__ void chunk_of(int n, int& lo, int& hi) {
  const int per = (n + blockDim.x - 1) / blockDim.x;
  lo = min(n, (int)threadIdx.x * per);
  hi = min(n, lo + per);
}

// ---------------------------------------------------------------------------------------------
// partition: slot[t] = src rank (>= 0) or -(dst rank + 1); src_idx / dst_idx the raster indices of each list
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ bool is_dst(int t, int w, int hc, int wc, int sy, int sx, const int* pattern) {
  const int y = t / w, x = t % w, cy = y / sy, cx = x / sx;
  if (cy >= hc || cx >= wc) return false;
  return (y - cy * sy) * sx + (x - cx * sx) == pattern[cy * wc + cx];
}

__global__ void __launch_bounds__(kScanThreads) tome_partition_kernel(const int* __restrict__ pattern, int h, int w,
                                                                     int sy, int sx, int* __restrict__ slot,
                                                                     int* __restrict__ src_idx,
                                                                     int* __restrict__ dst_idx) {
  __shared__ int sh[33];
  const int N = h * w, hc = h / sy, wc = w / sx;
  int lo, hi;
  chunk_of(N, lo, hi);
  int nd = 0;
  for (int t = lo; t < hi; ++t) nd += is_dst(t, w, hc, wc, sy, sx, pattern);
  int total;
  int d = block_excl_scan(nd, sh, &total);
  for (int t = lo; t < hi; ++t) {
    if (is_dst(t, w, hc, wc, sy, sx, pattern)) {
      slot[t] = -(d + 1);
      dst_idx[d++] = t;
    } else {
      slot[t] = t - d;
      src_idx[t - d] = t;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// normalise: one warp per token row; fp32 sum of squares in a fixed order, rows scaled by 1 / max(|x|, 1e-12)
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) tome_normalize_kernel(const bf16* __restrict__ x, const int* __restrict__ slot,
                                                            bf16* __restrict__ src_n, bf16* __restrict__ dst_n, int B,
                                                            int N, int Ns, int Nd, int C) {
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= (long long)B * N) return;
  const int lane = threadIdx.x & 31, b = (int)(row / N), t = (int)(row % N), nv = C / 8;
  const uint4* xr = reinterpret_cast<const uint4*>(x + row * C);
  float ss = 0.f;
  for (int v = lane; v < nv; v += 32) {
    const uint4 u = xr[v];
    const uint32_t* p = reinterpret_cast<const uint32_t*>(&u);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 f = unpack_bf16(p[k]);
      ss = fmaf(f.x, f.x, ss);
      ss = fmaf(f.y, f.y, ss);
    }
  }
  const float inv = rsqrtf(fmaxf(warp_sum(ss), 1e-24f));
  const int s = slot[t];
  bf16* out = s >= 0 ? src_n + ((long long)b * Ns + s) * C : dst_n + ((long long)b * Nd + (-s - 1)) * C;
  uint4* orow = reinterpret_cast<uint4*>(out);
  for (int v = lane; v < nv; v += 32) {
    const uint4 u = xr[v];
    const uint32_t* p = reinterpret_cast<const uint32_t*>(&u);
    uint4 o;
    uint32_t* q = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 f = unpack_bf16(p[k]);
      q[k] = pack_bf16(f.x * inv, f.y * inv);
    }
    orow[v] = o;
  }
}

// ---------------------------------------------------------------------------------------------
// match: CTA = (128 src rows, image); S = src · dstᵀ per 128-column dst tile, K streamed in 64-column panels
// ---------------------------------------------------------------------------------------------
// (v, i) beats (bv, bi): larger similarity, ties to the lower dst rank (dst ranks follow raster order)
__device__ __forceinline__ bool beats(float v, int i, float bv, int bi) { return v > bv || (v == bv && i < bi); }

__global__ void __launch_bounds__(kMatchThreads, 1)
tome_match_kernel(const __grid_constant__ CUtensorMap mapS, const __grid_constant__ CUtensorMap mapD, int Ns, int Nd,
                  int C, const int* __restrict__ dst_idx, float* __restrict__ node_max, int* __restrict__ node_idx) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kMatchStages * kMatchStage);
  uint64_t* empty_bar = full_bar + kMatchStages;
  const int wg = threadIdx.x >> 7, b = blockIdx.y, m0 = blockIdx.x * 128;
  const int KP = C / 64, ntile = (Nd + 127) / 128, total = ntile * KP;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&mapS);
    tma_prefetch_desc(&mapD);
    for (int i = 0; i < kMatchStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 256);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (threadIdx.x != 0) return;
    for (int it = 0; it < total; ++it) {
      const int s = it % kMatchStages, t = it / KP, kp = it % KP;
      mbar_wait(&empty_bar[s], ((uint32_t)(it / kMatchStages) & 1u) ^ 1u);
      uint8_t* st = smem + s * kMatchStage;
      mbar_expect_tx(&full_bar[s], kMatchStage);
      tma_load_3d(st, &mapS, &full_bar[s], 64 * kp, m0, b);
      tma_load_3d(st + kPanel, &mapD, &full_bar[s], 64 * kp, 128 * t, b);
    }
    return;
  }

  setmaxnreg_inc<232>();
  const int cw = wg - 1, lane = threadIdx.x & 31, warp = (threadIdx.x >> 5) & 3;
  const uint32_t s0 = smem_u32(smem);
  float acc[64];
  float best[2] = {-INFINITY, -INFINITY};
  int bidx[2] = {0, 0};
  int it = 0;
  for (int t = 0; t < ntile; ++t) {
    for (int kp = 0; kp < KP; ++kp, ++it) {
      const int s = it % kMatchStages;
      mbar_wait(&full_bar[s], (uint32_t)(it / kMatchStages) & 1u);
      const uint64_t da = wgmma_desc(s0 + s * kMatchStage + 64 * 128 * cw, 16, 1024);
      const uint64_t db = wgmma_desc(s0 + s * kMatchStage + kPanel, 16, 1024);
      reg_fence<64>(acc);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) Wgmma<128, 0, 0>::mma(acc, da + 2 * k, db + 2 * k, (kp > 0 || k > 0) ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence<64>(acc);
      mbar_arrive(&empty_bar[s]);
    }
    // columns of this thread rise with j and e: a strict > keeps the lowest index among equal values
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = 128 * t + 8 * j + 2 * (lane & 3) + e;
        if (col < Nd) {
#pragma unroll
          for (int hr = 0; hr < 2; ++hr) {
            const float v = acc[4 * j + 2 * hr + e];
            if (v > best[hr]) {
              best[hr] = v;
              bidx[hr] = col;
            }
          }
        }
      }
  }
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
#pragma unroll
    for (int o = 1; o <= 2; o <<= 1) {
      const float v = __shfl_xor_sync(0xffffffffu, best[hr], o);
      const int i = __shfl_xor_sync(0xffffffffu, bidx[hr], o);
      if (beats(v, i, best[hr], bidx[hr])) {
        best[hr] = v;
        bidx[hr] = i;
      }
    }
    const int row = m0 + 64 * cw + 16 * warp + (lane >> 2) + 8 * hr;
    if ((lane & 3) == 0 && row < Ns) {
      node_max[(long long)b * Ns + row] = best[hr];
      node_idx[(long long)b * Ns + row] = dst_idx[bidx[hr]];
    }
  }
}

// ---------------------------------------------------------------------------------------------
// select: one CTA per image
// ---------------------------------------------------------------------------------------------
// order-preserving map of fp32 to uint32 (larger float -> larger key)
__device__ __forceinline__ uint32_t f32_key(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__global__ void __launch_bounds__(kSelectThreads, 1)
tome_select_kernel(const float* __restrict__ node_max, const int* __restrict__ node_idx, const int* __restrict__ slot,
                   const int* __restrict__ src_idx, int N, int Ns, int Nd, int r, int* __restrict__ seg,
                   int* __restrict__ pos_g, int* __restrict__ row_off, int* __restrict__ members,
                   float* __restrict__ wrow) {
  extern __shared__ __align__(16) uint8_t smem_sel[];
  uint32_t* bufA = reinterpret_cast<uint32_t*>(smem_sel);   // keys, then sort ping-pong
  uint32_t* bufB = bufA + Ns;
  int* pos = reinterpret_cast<int*>(bufB + Ns);
  uint8_t* kept = reinterpret_cast<uint8_t*>(pos + N);
  __shared__ int sh[33];
  const int b = blockIdx.x, Nm = N - r;
  const float* nm = node_max + (long long)b * Ns;
  const int* ni = node_idx + (long long)b * Ns;
  int* seg_lo = seg + (long long)b * 2 * Nd;
  int* seg_hi = seg_lo + Nd;
  for (int i = threadIdx.x; i < Ns; i += blockDim.x) bufA[i] = f32_key(nm[i]);
  for (int t = threadIdx.x; t < N; t += blockDim.x) kept[t] = 1;
  for (int d = threadIdx.x; d < Nd; d += blockDim.x) seg_lo[d] = seg_hi[d] = 0;
  __syncthreads();

  // 1. threshold key T = the r-th largest key, one bit per pass from the top
  uint32_t T = 0;
  if (r > 0) {
    for (int bit = 31; bit >= 0; --bit) {
      const uint32_t cand = T | (1u << bit);
      int c = 0;
      for (int i = threadIdx.x; i < Ns; i += blockDim.x) c += bufA[i] >= cand;
      if (block_sum(c, sh) >= r) T = cand;
    }
  }
  // 2. merged: key > T, and of the keys == T the lowest src ranks (src ranks follow raster order) up to r in all
  int lo, hi, tot;
  chunk_of(Ns, lo, hi);
  int gt = 0, eq = 0;
  if (r > 0)
    for (int i = lo; i < hi; ++i) {
      gt += bufA[i] > T;
      eq += bufA[i] == T;
    }
  const int e_take = r - block_sum(gt, sh);
  const int eq_before = block_excl_scan(eq, sh, &tot);
  int nsel = 0;
  for (int i = lo, q = eq_before; i < hi && r > 0; ++i) nsel += bufA[i] > T || (bufA[i] == T && q++ < e_take);
  // 3. the merged tokens, compacted in raster order as (dst rank << 14) | raster index, and the kept flags
  int k = block_excl_scan(nsel, sh, &tot);
  for (int i = lo, q = eq_before; i < hi && r > 0; ++i) {
    if (bufA[i] > T || (bufA[i] == T && q++ < e_take)) {
      const int t = src_idx[i];
      bufB[k++] = ((uint32_t)(-slot[ni[i]] - 1) << 14) | (uint32_t)t;
      kept[t] = 0;
    }
  }
  __syncthreads();

  // 4. merged-row position of every kept token (raster order)
  chunk_of(N, lo, hi);
  int nk = 0;
  for (int t = lo; t < hi; ++t) nk += kept[t];
  int p = block_excl_scan(nk, sh, &tot);
  for (int t = lo; t < hi; ++t)
    if (kept[t]) pos[t] = p++;
  __syncthreads();

  // 5. stable split sort of the r packed keys by dst rank (bits 14 ..), ping-pong bufB <-> bufA
  int nbits = 0;
  while ((1 << nbits) < Nd) ++nbits;
  uint32_t* src = bufB;
  uint32_t* dst = bufA;
  chunk_of(r, lo, hi);
  for (int bit = 0; bit < nbits; ++bit) {
    int z = 0;
    for (int q = lo; q < hi; ++q) z += ((src[q] >> (14 + bit)) & 1u) == 0;
    int zall;
    int zb = block_excl_scan(z, sh, &zall);
    int ob = zall + (lo - zb);
    for (int q = lo; q < hi; ++q) {
      const uint32_t v = src[q];
      if (((v >> (14 + bit)) & 1u) == 0) dst[zb++] = v;
      else dst[ob++] = v;
    }
    __syncthreads();
    uint32_t* tmp = src;
    src = dst;
    dst = tmp;
  }
  // 6. the segment of every dst in the sorted list; merged tokens take their dst's row
  for (int q = threadIdx.x; q < r; q += blockDim.x) {
    const uint32_t v = src[q];
    const int d = (int)(v >> 14);
    if (q == 0 || (int)(src[q - 1] >> 14) != d) seg_lo[d] = q;
    if (q == r - 1 || (int)(src[q + 1] >> 14) != d) seg_hi[d] = q + 1;
  }
  __syncthreads();
  for (int q = threadIdx.x; q < r; q += blockDim.x) {
    const int t = (int)(src[q] & 0x3FFFu);
    pos[t] = pos[ni[slot[t]]];
  }
  __syncthreads();
  int* pg = pos_g + (long long)b * N;
  for (int t = threadIdx.x; t < N; t += blockDim.x) pg[t] = pos[t];

  // 7. CSR rows in merged order: a kept src is alone, a dst row is the dst and its segment, raster-sorted
  chunk_of(N, lo, hi);
  int len = 0;
  for (int t = lo; t < hi; ++t) {
    if (!kept[t]) continue;
    const int s = slot[t];
    len += 1 + (s < 0 ? seg_hi[-s - 1] - seg_lo[-s - 1] : 0);
  }
  int off = block_excl_scan(len, sh, &tot);
  int* ro = row_off + (long long)b * (Nm + 1);
  int* mem = members + (long long)b * N;
  float* wr = wrow + (long long)b * Nm;
  for (int t = lo; t < hi; ++t) {
    if (!kept[t]) continue;
    const int s = slot[t], pr = pos[t];
    ro[pr] = off;
    if (s >= 0) {
      mem[off++] = t;
      wr[pr] = 1.f;
      continue;
    }
    const int a = seg_lo[-s - 1], z = seg_hi[-s - 1];
    wr[pr] = 1.f / (float)(1 + z - a);
    bool placed = false;
    for (int q = a; q < z; ++q) {
      const int m = (int)(src[q] & 0x3FFFu);
      if (!placed && t < m) {
        mem[off++] = t;
        placed = true;
      }
      mem[off++] = m;
    }
    if (!placed) mem[off++] = t;
  }
  if (threadIdx.x == 0) ro[Nm] = N;
}

// ---------------------------------------------------------------------------------------------
// gathers (16-byte vectors of 8 channels, fp32 sums in member order)
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) tome_gather_reduce_kernel(const bf16* __restrict__ in,
                                                                const int* __restrict__ row_off,
                                                                const int* __restrict__ members,
                                                                const float* __restrict__ w, bf16* __restrict__ out,
                                                                int B, int n_in, int n_rows, int C) {
  const int nv = C / 8;
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (long long)B * n_rows * nv) return;
  const int v = (int)(g % nv);
  const long long row = g / nv;
  const int b = (int)(row / n_rows), p = (int)(row % n_rows);
  const int* ro = row_off + (long long)b * (n_rows + 1);
  const int* mem = members + (long long)b * n_in;
  const bf16* base = in + (long long)b * n_in * C + 8 * v;
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int k = ro[p], e = ro[p + 1]; k < e; ++k) {
    const uint4 u = *reinterpret_cast<const uint4*>(base + (long long)mem[k] * C);
    const uint32_t* q = reinterpret_cast<const uint32_t*>(&u);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = unpack_bf16(q[i]);
      acc[2 * i] += f.x;
      acc[2 * i + 1] += f.y;
    }
  }
  const float s = w != nullptr ? w[row] : 1.f;
  uint4 o;
  uint32_t* q = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
  for (int i = 0; i < 4; ++i) q[i] = pack_bf16(acc[2 * i] * s, acc[2 * i + 1] * s);
  *reinterpret_cast<uint4*>(out + row * C + 8 * v) = o;
}

__global__ void __launch_bounds__(256) tome_gather_expand_kernel(const bf16* __restrict__ in,
                                                                const int* __restrict__ pos,
                                                                const float* __restrict__ w,
                                                                const bf16* __restrict__ residual,
                                                                bf16* __restrict__ out, int B, int n_in, int n_out,
                                                                int C) {
  const int nv = C / 8;
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= (long long)B * n_out * nv) return;
  const int v = (int)(g % nv);
  const long long row = g / nv;
  const int b = (int)(row / n_out);
  const long long src = (long long)b * n_in + pos[row];
  const uint4 u = *reinterpret_cast<const uint4*>(in + src * C + 8 * v);
  const uint32_t* q = reinterpret_cast<const uint32_t*>(&u);
  const float s = w != nullptr ? w[src] : 1.f;
  uint4 rv = make_uint4(0, 0, 0, 0);
  if (residual != nullptr) rv = *reinterpret_cast<const uint4*>(residual + row * C + 8 * v);
  const uint32_t* rq = reinterpret_cast<const uint32_t*>(&rv);
  uint4 o;
  uint32_t* oq = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 f = unpack_bf16(q[i]);
    const float2 rr = residual != nullptr ? unpack_bf16(rq[i]) : make_float2(0.f, 0.f);
    oq[i] = pack_bf16(fmaf(f.x, s, rr.x), fmaf(f.y, s, rr.y));
  }
  *reinterpret_cast<uint4*>(out + row * C + 8 * v) = o;
}

// =============================================================================================
// Host
// =============================================================================================
static size_t select_smem(int N, int Ns) { return (size_t)8 * Ns + (size_t)5 * N + 16; }

extern "C" int e4t_tome_match(const void* x, const int* pattern, int B, int h, int w, int C, int sy, int sx, int* slot,
                              int* src_idx, int* dst_idx, void* src_n, void* dst_n, float* node_max, int* node_idx,
                              void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const int N = h * w, Nd = (h / sy) * (w / sx), Ns = N - Nd;
  E4T_CHECK(B > 0 && h > 0 && w > 0 && sy > 0 && sx > 0, "tome_match: bad sizes B=%d h=%d w=%d sy=%d sx=%d", B, h, w,
            sy, sx);
  E4T_CHECK(C % 64 == 0 && C > 0, "tome_match: C = %d must be a multiple of 64", C);
  E4T_CHECK(((uintptr_t)x & 15) == 0 && ((uintptr_t)src_n & 15) == 0 && ((uintptr_t)dst_n & 15) == 0,
            "tome_match: tensors must be 16-byte aligned");
  tome_partition_kernel<<<1, kScanThreads, 0, st>>>(pattern, h, w, sy, sx, slot, src_idx, dst_idx);
  E4T_COUNT_LAUNCH();
  E4T_LAUNCH_CHECK();
  tome_normalize_kernel<<<cdiv((long)B * N, 8), 256, 0, st>>>((const bf16*)x, slot, (bf16*)src_n, (bf16*)dst_n, B, N,
                                                               Ns, Nd, C);
  E4T_COUNT_LAUNCH();
  E4T_LAUNCH_CHECK();
  if (Ns == 0 || Nd == 0) return 0;
  CUtensorMap mS, mD;
  {
    const uint64_t dims[3] = {(uint64_t)C, (uint64_t)Ns, (uint64_t)B};
    const uint64_t str[2] = {(uint64_t)C * 2, (uint64_t)Ns * C * 2};
    const uint32_t box[3] = {64, 128, 1};
    if (int e = e4t_tmap_encode(&mS, src_n, 3, dims, str, box, 2)) return e;
  }
  {
    const uint64_t dims[3] = {(uint64_t)C, (uint64_t)Nd, (uint64_t)B};
    const uint64_t str[2] = {(uint64_t)C * 2, (uint64_t)Nd * C * 2};
    const uint32_t box[3] = {64, 128, 1};
    if (int e = e4t_tmap_encode(&mD, dst_n, 3, dims, str, box, 2)) return e;
  }
  E4T_CUDA(cudaFuncSetAttribute(tome_match_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMatchSmem));
  tome_match_kernel<<<dim3(cdiv(Ns, 128), B), kMatchThreads, kMatchSmem, st>>>(mS, mD, Ns, Nd, C, dst_idx, node_max,
                                                                               node_idx);
  E4T_COUNT_LAUNCH();
  E4T_LAUNCH_CHECK();
  return 0;
}

extern "C" int e4t_tome_select(const float* node_max, const int* node_idx, const int* slot, const int* src_idx, int B,
                               int N, int Ns, int Nd, int r, int* seg, int* pos, int* row_off, int* members, float* w,
                               void* stream) {
  E4T_CHECK(N <= kSelectMaxTokens, "tome_select: %d tokens per image; token merging supports at most %d (a 128 x 128 "
            "latent)", N, kSelectMaxTokens);
  E4T_CHECK(B > 0 && Ns >= 0 && Nd >= 0 && Ns + Nd == N && r >= 0 && r <= Ns && (r == 0 || Nd > 0),
            "tome_select: bad sizes N=%d Ns=%d Nd=%d r=%d", N, Ns, Nd, r);
  const size_t smem = select_smem(N, Ns);
  E4T_CUDA(cudaFuncSetAttribute(tome_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  tome_select_kernel<<<B, kSelectThreads, smem, (cudaStream_t)stream>>>(node_max, node_idx, slot, src_idx, N, Ns, Nd, r,
                                                                       seg, pos, row_off, members, w);
  E4T_COUNT_LAUNCH();
  E4T_LAUNCH_CHECK();
  return 0;
}

extern "C" int e4t_tome_gather_reduce(const void* in, const int* row_off, const int* members, const float* w, void* out,
                                      int B, int n_in, int n_rows, int C, void* stream) {
  E4T_CHECK(C % 8 == 0 && ((uintptr_t)in & 15) == 0 && ((uintptr_t)out & 15) == 0,
            "tome_gather_reduce: C %% 8 == 0 and 16-byte aligned tensors needed (C = %d)", C);
  const long long n = (long long)B * n_rows * (C / 8);
  if (n == 0) return 0;
  tome_gather_reduce_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      (const bf16*)in, row_off, members, w, (bf16*)out, B, n_in, n_rows, C);
  E4T_COUNT_LAUNCH();
  E4T_LAUNCH_CHECK();
  return 0;
}

extern "C" int e4t_tome_gather_expand(const void* in, const int* pos, const float* w, const void* residual, void* out,
                                      int B, int n_in, int n_out, int C, void* stream) {
  E4T_CHECK(C % 8 == 0 && ((uintptr_t)in & 15) == 0 && ((uintptr_t)out & 15) == 0 && ((uintptr_t)residual & 15) == 0,
            "tome_gather_expand: C %% 8 == 0 and 16-byte aligned tensors needed (C = %d)", C);
  const long long n = (long long)B * n_out * (C / 8);
  if (n == 0) return 0;
  tome_gather_expand_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      (const bf16*)in, pos, w, (const bf16*)residual, (bf16*)out, B, n_in, n_out, C);
  E4T_COUNT_LAUNCH();
  E4T_LAUNCH_CHECK();
  return 0;
}
