// e4t_b200 — fused attention core softmax(Q Kᵀ / sqrt(dh)) V for the SD-v1.4 UNet on the sm_90a tensor cores
// (mma.sync m16n8k16 bf16 -> fp32, ldmatrix, cp.async double buffering).
// Reference call site: F.scaled_dot_product_attention in AttnProcessor2_0 (e4t/models/cross_attention.py:521-531),
// equivalently get_attention_scores + bmm (cross_attention.py:222-251,313-315).  No mask, no dropout, non-causal
// (the fused backward also takes the causal mask of the CLIP text tower).
//
// Layout: Q [B][N][H*dh], K/V [B][M][H*dh] (token-major, heads are dh-wide column slices; row/batch strides are
// arguments so Q/K/V may alias one fused projection output).  dh % 8 == 0, dh <= 192.  Tiles are staged in shared
// memory with the head dim zero-padded to DP (a multiple of 16, the template parameter) and a row pitch of DP + 8
// elements, which keeps every ldmatrix phase free of bank conflicts.
//
// Forward, per CTA = (64-query tile, head, batch), 4 warps x 16 query rows: Q fragments stay in registers, K_j / V_j
// blocks of 64 keys are double buffered; S = Q·K_jᵀ, online softmax in the exp2 domain, the S accumulators are
// re-packed in registers as the A operand of O += P·V_j.
// Backward recomputes P from the saved log-sum-exp.  dK/dV kernel: CTA = 64 keys, 4 warps x 16 keys, loops over query
// blocks: Sᵀ = K·Qᵀ, dPᵀ = V·dOᵀ, dSᵀ = Pᵀ∘(dPᵀ − D), dV += Pᵀ·dO, dK += dSᵀ·Q; in the single-pass (fused) form the
// same kernel stages dSᵀ in shared memory and reduces dQ += dS·K into an fp32 buffer with atomics.  The two-kernel form
// computes dQ in a kernel of its own (CTA = 64 queries, loop over key blocks).
//
// Which shapes run here: everything except the non-causal forward and single-pass backward with dh = 40, 64 or 80 and
// N, M multiples of 128 and >= 512 (the 4096-token level-0 and 1024-token level-1 self-attention of SD 1.x, the SD 2.x
// self-attention from 512 tokens up; for dh = 64 and 80 only grids of at least half as many 128-query CTAs as SMs),
// which the entry points below hand to the warpgroup kernels of attention_wgmma.cu unless a switch (see "Runtime
// switches") keeps them here.  With dh = 64 that leaves the 77-key cross-attention and the shorter SD 2.x levels to this file.
#include "attention.cuh"
#include <math.h>
#include <stdlib.h>

static constexpr int kAttnThreads = 128;
static constexpr int kBlk = 64;   // query rows of a forward / dQ CTA, key rows of a dK/dV CTA, key block of the loops

// rows [0, nrows) of a head slice -> smem [nrows][DP + 8]; rows >= rows_valid and columns >= dh are zero-filled
template <int DP, int NT = kAttnThreads>
__device__ __forceinline__ void load_rows(bf16* s, const bf16* g, long long ld, int rows_valid, int nrows, int dh) {
  constexpr int CPR = DP / 8, LD = DP + 8;
  const uint32_t sb = smem_u32(s);
  for (int i = threadIdx.x; i < nrows * CPR; i += NT) {
    const int r = i / CPR, c = i - r * CPR;
    const bool ok = r < rows_valid && c * 8 < dh;
    cp_async16(sb + (uint32_t)(r * LD + c * 8) * 2u, ok ? (const void*)(g + (long long)r * ld + c * 8) : (const void*)g,
               ok ? 16u : 0u);
  }
}

// ldmatrix addresses (lane-dependent) inside a [rows][LD] bf16 tile
// A operand 16x16 at (row0, col0), stored row-major [m][k]
__device__ __forceinline__ uint32_t a_addr(const bf16* t, int LD, int row0, int col0) {
  const int l = threadIdx.x & 31;
  return smem_u32(t + (row0 + (l & 15)) * LD + col0 + (l >> 4) * 8);
}
// A operand 16x16 (m x k) stored transposed [k][m] at (k0, m0): ldmatrix.trans
__device__ __forceinline__ uint32_t at_addr(const bf16* t, int LD, int k0, int m0) {
  const int l = threadIdx.x & 31;
  return smem_u32(t + (k0 + (l & 7) + (l >> 4) * 8) * LD + m0 + ((l >> 3) & 1) * 8);
}
// B operands of two n-tiles (16 n x 16 k) stored [n][k] at (n0, k0): ldmatrix (non-trans)
__device__ __forceinline__ uint32_t b_addr(const bf16* t, int LD, int n0, int k0) {
  const int l = threadIdx.x & 31;
  return smem_u32(t + (n0 + (l & 7) + (l >> 4) * 8) * LD + k0 + ((l >> 3) & 1) * 8);
}
// B operands of two n-tiles stored [k][n] at (k0, n0): ldmatrix.trans
__device__ __forceinline__ uint32_t bt_addr(const bf16* t, int LD, int k0, int n0) {
  const int l = threadIdx.x & 31;
  return smem_u32(t + (k0 + (l & 7) + ((l >> 3) & 1) * 8) * LD + n0 + (l >> 4) * 8);
}
// accumulators of two adjacent n-tiles (16 columns) -> bf16 A fragment over those 16 k
__device__ __forceinline__ void pack_a(const float* c0, const float* c1, uint32_t* a) {
  a[0] = pack_bf16(c0[0], c0[1]);
  a[1] = pack_bf16(c0[2], c0[3]);
  a[2] = pack_bf16(c1[0], c1[1]);
  a[3] = pack_bf16(c1[2], c1[3]);
}

// =============================================================================================
// Forward
// =============================================================================================
// 2^x on the FMA pipe (exponent split + degree-6 polynomial of 2^f, f in [0, 1), relative error < 2e-6): lets a share of
// the exponentials bypass the MUFU unit, which the dh = 40 shapes keep busy
__device__ __forceinline__ float exp2_poly(float x) {
  x = fmaxf(x, -126.f);
  const float xi = floorf(x);
  const float f = x - xi;
  float p = 1.5403530e-4f;
  p = fmaf(p, f, 1.3333558e-3f);
  p = fmaf(p, f, 9.6181291e-3f);
  p = fmaf(p, f, 5.5504109e-2f);
  p = fmaf(p, f, 2.4022651e-1f);
  p = fmaf(p, f, 6.9314718e-1f);
  p = fmaf(p, f, 1.0f);
  return __int_as_float(__float_as_int(p) + ((int)xi << 23));
}

// Runtime variants (AttnArgs): stages = 1 / 2 K-V buffers; lazy = 1 rescales O and the row sum only when the row maximum
// grows by more than 2^8 (P then stays below 2^8, exact in fp32 and bf16 range); poly = how many of every 8 exponentials
// go through exp2_poly; p_smem = 1 stages P through shared memory (ldmatrix) instead of re-packing it in registers.
// VAR = false is the default kernel with these fixed at compile time (two buffers, eager rescale, MUFU, registers).
template <int DP, int WARPS, bool VAR>
__global__ void __launch_bounds__(32 * WARPS) attn_fwd_kernel(const AttnArgs a) {
  constexpr int LD = DP + 8, KT = DP / 16, DT = DP / 8, QROWS = 16 * WARPS, PLD = kBlk + 8;
  const int stages = VAR ? a.stages : 2, poly = VAR ? a.poly : 0;
  const bool lazy = VAR && a.lazy, p_smem = VAR && a.p_smem;
  extern __shared__ __align__(16) uint8_t smem_raw[];
  bf16* sQ = reinterpret_cast<bf16*>(smem_raw);
  bf16* sK = sQ + QROWS * LD;                  // [stages][kBlk][LD]
  bf16* sV = sK + stages * kBlk * LD;          // [stages][kBlk][LD]
  bf16* sP = sV + stages * kBlk * LD;          // p_smem: [WARPS][16][PLD]
  const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * QROWS;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bf16* Kg = a.K + b * a.k_bs + h * a.dh;
  const bf16* Vg = a.V + b * a.v_bs + h * a.dh;
  const int nblk = (a.M + kBlk - 1) / kBlk;
  load_rows<DP, 32 * WARPS>(sQ, a.Q + b * a.q_bs + (long long)q0 * a.ldq + h * a.dh, a.ldq, a.N - q0, QROWS, a.dh);
  load_rows<DP, 32 * WARPS>(sK, Kg, a.ldk, a.M, kBlk, a.dh);
  load_rows<DP, 32 * WARPS>(sV, Vg, a.ldv, a.M, kBlk, a.dh);
  cp_async_commit();

  const float sl2 = a.scale * kLog2e;
  float o[DT][4];
#pragma unroll
  for (int i = 0; i < DT; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;
  float m_r[2] = {-INFINITY, -INFINITY}, l_r[2] = {0.f, 0.f};
  uint32_t qf[KT][4];
  for (int j = 0; j < nblk; ++j) {
    int buf = 0;
    if (stages == 2) {
      buf = j & 1;
      if (j + 1 < nblk) {
        const int kn = (j + 1) * kBlk;
        load_rows<DP, 32 * WARPS>(sK + (buf ^ 1) * kBlk * LD, Kg + (long long)kn * a.ldk, a.ldk, a.M - kn, kBlk, a.dh);
        load_rows<DP, 32 * WARPS>(sV + (buf ^ 1) * kBlk * LD, Vg + (long long)kn * a.ldv, a.ldv, a.M - kn, kBlk, a.dh);
      }
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      if (j > 0) {
        load_rows<DP, 32 * WARPS>(sK, Kg + (long long)j * kBlk * a.ldk, a.ldk, a.M - j * kBlk, kBlk, a.dh);
        load_rows<DP, 32 * WARPS>(sV, Vg + (long long)j * kBlk * a.ldv, a.ldv, a.M - j * kBlk, kBlk, a.dh);
        cp_async_commit();
      }
      cp_async_wait<0>();
    }
    __syncthreads();
    if (j == 0) {
#pragma unroll
      for (int kk = 0; kk < KT; ++kk) ldsm_x4(a_addr(sQ, LD, warp * 16, kk * 16), qf[kk]);
    }
    const bf16* k_s = sK + buf * kBlk * LD;
    const bf16* v_s = sV + buf * kBlk * LD;
    float s[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
#pragma unroll
    for (int kk = 0; kk < KT; ++kk) {
#pragma unroll
      for (int np = 0; np < 4; ++np) {
        uint32_t bfr[4];
        ldsm_x4(b_addr(k_s, LD, np * 16, kk * 16), bfr);
        mma16816(s[2 * np], qf[kk], bfr);
        mma16816(s[2 * np + 1], qf[kk], bfr + 2);
      }
    }
    const int k0 = j * kBlk;
    if (k0 + kBlk > a.M) {
#pragma unroll
      for (int nt = 0; nt < 8; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e)
          if (k0 + nt * 8 + 2 * (lane & 3) + (e & 1) >= a.M) s[nt][e] = -INFINITY;
    }
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      float mx = -INFINITY;
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) mx = fmaxf(mx, fmaxf(s[nt][2 * hr], s[nt][2 * hr + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      // every key block holds at least one valid key: mx is finite, and so is mnew after the first block
      const float mx2 = mx * sl2;
      const float mnew = (!lazy || mx2 > m_r[hr] + 8.f) ? fmaxf(m_r[hr], mx2) : m_r[hr];
      const float alpha = exp2f(m_r[hr] - mnew);
      m_r[hr] = mnew;
#pragma unroll
      for (int dt = 0; dt < DT; ++dt) {
        o[dt][2 * hr] *= alpha;
        o[dt][2 * hr + 1] *= alpha;
      }
      float rs = 0.f;
#pragma unroll
      for (int nt = 0; nt < 8; ++nt)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float x = fmaf(s[nt][2 * hr + e], sl2, -mnew);
          const float p = nt < poly ? exp2_poly(x) : exp2f(x);
          s[nt][2 * hr + e] = p;
          rs += p;
        }
      l_r[hr] = l_r[hr] * alpha + rs;
    }
    bf16* sPw = sP + warp * 16 * PLD;
    if (p_smem) {
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const int r = lane >> 2, c = nt * 8 + 2 * (lane & 3);
        *reinterpret_cast<uint32_t*>(sPw + r * PLD + c) = pack_bf16(s[nt][0], s[nt][1]);
        *reinterpret_cast<uint32_t*>(sPw + (r + 8) * PLD + c) = pack_bf16(s[nt][2], s[nt][3]);
      }
      __syncwarp();
    }
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      uint32_t pa[4];
      if (p_smem) ldsm_x4(a_addr(sPw, PLD, 0, kk * 16), pa);
      else pack_a(s[2 * kk], s[2 * kk + 1], pa);
#pragma unroll
      for (int dp = 0; dp < DT / 2; ++dp) {
        uint32_t bfr[4];
        ldsm_x4_t(bt_addr(v_s, LD, kk * 16, dp * 16), bfr);
        mma16816(o[2 * dp], pa, bfr);
        mma16816(o[2 * dp + 1], pa, bfr + 2);
      }
    }
    __syncthreads();   // this buffer is refilled by a later iteration
  }
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    float l = l_r[hr];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const int row = q0 + warp * 16 + (lane >> 2) + 8 * hr;
    if (row >= a.N) continue;
    const float inv = 1.f / l;
    bf16* orow = a.O + b * a.o_bs + (long long)row * a.ldo + h * a.dh;
#pragma unroll
    for (int dt = 0; dt < DT; ++dt) {
      const int d = dt * 8 + 2 * (lane & 3);
      if (d < a.dh) *reinterpret_cast<uint32_t*>(orow + d) = pack_bf16(o[dt][2 * hr] * inv, o[dt][2 * hr + 1] * inv);
    }
    if ((lane & 3) == 0) a.LSE[((long long)b * a.H + h) * a.N + row] = (m_r[hr] + log2f(l)) * (1.f / kLog2e);
  }
}

// =============================================================================================
// D = rowsum(dO ∘ O)  per (b, h, n); one thread per (b, n, h): consecutive threads read consecutive dh-wide slices of
// a token row, so the loads of a warp cover one contiguous span
// =============================================================================================
// one warp per (b, n, h) (E4T_ATTN_DELTA2=0)
__global__ void attn_delta_kernel(const bf16* __restrict__ O, const bf16* __restrict__ dO, float* __restrict__ Dv,
                                  int B, int H, int N, int dh, long long ldo, long long o_bs, long long lddo,
                                  long long do_bs) {
  const long long wid = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (wid >= (long long)B * N * H) return;
  const int h = (int)(wid % H);
  const int n = (int)((wid / H) % N);
  const int b = (int)(wid / ((long long)H * N));
  const bf16* o = O + b * o_bs + (long long)n * ldo + h * dh;
  const bf16* d = dO + b * do_bs + (long long)n * lddo + h * dh;
  float acc = 0.f;
  for (int v = lane; v < dh / 8; v += 32) {
    const uint4 a = *reinterpret_cast<const uint4*>(o + v * 8);
    const uint4 c = *reinterpret_cast<const uint4*>(d + v * 8);
    const uint32_t as[4] = {a.x, a.y, a.z, a.w}, cs[4] = {c.x, c.y, c.z, c.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 x = unpack_bf16(as[i]), y = unpack_bf16(cs[i]);
      acc += x.x * y.x + x.y * y.y;
    }
  }
  acc = warp_sum(acc);
  if (lane == 0) Dv[((long long)b * H + h) * N + n] = acc;
}

__global__ void attn_delta2_kernel(const bf16* __restrict__ O, const bf16* __restrict__ dO, float* __restrict__ Dv,
                                   int B, int H, int N, int dh, long long ldo, long long o_bs, long long lddo,
                                   long long do_bs) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)B * N * H) return;
  const int h = (int)(t % H);
  const int n = (int)((t / H) % N);
  const int b = (int)(t / ((long long)H * N));
  const bf16* o = O + b * o_bs + (long long)n * ldo + h * dh;
  const bf16* d = dO + b * do_bs + (long long)n * lddo + h * dh;
  float acc = 0.f;
  for (int v = 0; v < dh / 8; ++v) {
    const uint4 a = *reinterpret_cast<const uint4*>(o + v * 8);
    const uint4 c = *reinterpret_cast<const uint4*>(d + v * 8);
    const uint32_t as[4] = {a.x, a.y, a.z, a.w}, cs[4] = {c.x, c.y, c.z, c.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 x = unpack_bf16(as[i]), y = unpack_bf16(cs[i]);
      acc += x.x * y.x + x.y * y.y;
    }
  }
  Dv[((long long)b * H + h) * N + n] = acc;
}


// =============================================================================================
// dK / dV (and, DQ = true, the fp32 dQ reduction): CTA = (64-key tile, head, batch)
// =============================================================================================
// BQ: query block of the dK/dV loop (64, or 32 for wide heads: register budget; E4T_ATTN_BWD_BQ=32 selects 32 for all)
template <int DP, int BQ_>
struct BwdCfg {
  static constexpr int LD = DP + 8;
  static constexpr int BQ = BQ_;
  static constexpr int SLD = BQ + 8;              // row pitch of the staged dSᵀ
  static constexpr size_t smem_bytes(bool dq) {
    return (size_t)(2 * kBlk * LD + 4 * BQ * LD) * 2 + (size_t)4 * BQ * 4 + (dq ? (size_t)kBlk * SLD * 2 : 0);
  }
};

template <int DP, int BQ_, bool DQ, bool CAUSAL, int STAGES>
__global__ void __launch_bounds__(kAttnThreads) attn_bwd_kv_kernel(const AttnArgs a) {
  using C = BwdCfg<DP, BQ_>;
  constexpr int LD = C::LD, BQ = C::BQ, SLD = C::SLD, KT = DP / 16, DT = DP / 8, NT = BQ / 8;
  extern __shared__ __align__(16) uint8_t smem_raw[];
  bf16* sK = reinterpret_cast<bf16*>(smem_raw);
  bf16* sV = sK + kBlk * LD;
  bf16* sQ = sV + kBlk * LD;          // [2][BQ][LD]
  bf16* sdO = sQ + 2 * BQ * LD;       // [2][BQ][LD]
  float* sL = reinterpret_cast<float*>(sdO + 2 * BQ * LD);   // [2][BQ] LSE * log2(e)
  float* sD = sL + 2 * BQ;                                   // [2][BQ]
  bf16* sdS = reinterpret_cast<bf16*>(sD + 2 * BQ);          // [kBlk][SLD]
  const int b = blockIdx.z, h = blockIdx.y, k0 = blockIdx.x * kBlk;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long bh = (long long)b * a.H + h;
  const bf16* Qg = a.Q + b * a.q_bs + h * a.dh;
  const bf16* dOg = a.dO + b * a.do_bs + h * a.dh;
  load_rows<DP>(sK, a.K + b * a.k_bs + (long long)k0 * a.ldk + h * a.dh, a.ldk, a.M - k0, kBlk, a.dh);
  load_rows<DP>(sV, a.V + b * a.v_bs + (long long)k0 * a.ldv + h * a.dh, a.ldv, a.M - k0, kBlk, a.dh);
  auto load_q = [&](int i, int buf) {
    const int q0 = i * BQ;
    load_rows<DP>(sQ + buf * BQ * LD, Qg + (long long)q0 * a.ldq, a.ldq, a.N - q0, BQ, a.dh);
    load_rows<DP>(sdO + buf * BQ * LD, dOg + (long long)q0 * a.lddo, a.lddo, a.N - q0, BQ, a.dh);
    for (int t = threadIdx.x; t < BQ; t += kAttnThreads) {
      const bool ok = q0 + t < a.N;
      sL[buf * BQ + t] = ok ? a.LSE[bh * a.N + q0 + t] * kLog2e : 0.f;
      sD[buf * BQ + t] = ok ? a.Dv[bh * a.N + q0 + t] : 0.f;
    }
  };
  const int i0 = CAUSAL ? k0 / BQ : 0;
  const int nq = (a.N + BQ - 1) / BQ;
  load_q(i0, 0);
  cp_async_commit();

  const float sl2 = a.scale * kLog2e;
  float dk[DT][4], dv[DT][4];
#pragma unroll
  for (int i = 0; i < DT; ++i) {
    dk[i][0] = dk[i][1] = dk[i][2] = dk[i][3] = 0.f;
    dv[i][0] = dv[i][1] = dv[i][2] = dv[i][3] = 0.f;
  }
  const int key_r = k0 + warp * 16 + (lane >> 2);
  for (int i = i0; i < nq; ++i) {
    int buf = 0;
    if (STAGES == 2) {   // Q / dO of the next block prefetched while this one is used
      buf = (i - i0) & 1;
      if (i + 1 < nq) load_q(i + 1, buf ^ 1);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      if (i > i0) {
        load_q(i, 0);
        cp_async_commit();
      }
      cp_async_wait<0>();
    }
    __syncthreads();
    const bf16* q_s = sQ + buf * BQ * LD;
    const bf16* do_s = sdO + buf * BQ * LD;
    const float* l_s = sL + buf * BQ;
    const float* d_s = sD + buf * BQ;
    const int q0 = i * BQ;
    float st[NT][4], dpt[NT][4];
#pragma unroll
    for (int n = 0; n < NT; ++n) {
      st[n][0] = st[n][1] = st[n][2] = st[n][3] = 0.f;
      dpt[n][0] = dpt[n][1] = dpt[n][2] = dpt[n][3] = 0.f;
    }
#pragma unroll
    for (int kk = 0; kk < KT; ++kk) {
      uint32_t ka[4], va[4];
      ldsm_x4(a_addr(sK, LD, warp * 16, kk * 16), ka);
      ldsm_x4(a_addr(sV, LD, warp * 16, kk * 16), va);
#pragma unroll
      for (int np = 0; np < NT / 2; ++np) {
        uint32_t bq[4], bo[4];
        ldsm_x4(b_addr(q_s, LD, np * 16, kk * 16), bq);
        ldsm_x4(b_addr(do_s, LD, np * 16, kk * 16), bo);
        mma16816(st[2 * np], ka, bq);
        mma16816(st[2 * np + 1], ka, bq + 2);
        mma16816(dpt[2 * np], va, bo);
        mma16816(dpt[2 * np + 1], va, bo + 2);
      }
    }
    // Pᵀ and dSᵀ (keys are rows, queries columns)
#pragma unroll
    for (int n = 0; n < NT; ++n)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int c = n * 8 + 2 * (lane & 3) + (e & 1);
        const int key = key_r + 8 * (e >> 1);
        float p = exp2f(fmaf(st[n][e], sl2, -l_s[c]));
        if (q0 + c >= a.N || key >= a.M || (CAUSAL && key > q0 + c)) p = 0.f;
        st[n][e] = p;
        dpt[n][e] = p * (dpt[n][e] - d_s[c]);
      }
#pragma unroll
    for (int kq = 0; kq < BQ / 16; ++kq) {
      uint32_t pa[4], sa[4];
      pack_a(st[2 * kq], st[2 * kq + 1], pa);
      pack_a(dpt[2 * kq], dpt[2 * kq + 1], sa);
#pragma unroll
      for (int dp = 0; dp < DT / 2; ++dp) {
        uint32_t bo[4], bq[4];
        ldsm_x4_t(bt_addr(do_s, LD, kq * 16, dp * 16), bo);
        ldsm_x4_t(bt_addr(q_s, LD, kq * 16, dp * 16), bq);
        mma16816(dv[2 * dp], pa, bo);
        mma16816(dv[2 * dp + 1], pa, bo + 2);
        mma16816(dk[2 * dp], sa, bq);
        mma16816(dk[2 * dp + 1], sa, bq + 2);
      }
    }
    if (DQ) {
      // dSᵀ -> smem, then dQ[q][d] += sum_key dS[q][key] K[key][d]: warp = (query group, d half)
#pragma unroll
      for (int n = 0; n < NT; ++n) {
        const int r = warp * 16 + (lane >> 2), c = n * 8 + 2 * (lane & 3);
        *reinterpret_cast<uint32_t*>(sdS + r * SLD + c) = pack_bf16(dpt[n][0], dpt[n][1]);
        *reinterpret_cast<uint32_t*>(sdS + (r + 8) * SLD + c) = pack_bf16(dpt[n][2], dpt[n][3]);
      }
      __syncthreads();
      // the DP/16 16-column pairs of d are split over DSPLIT warps (PPW pairs each, the last warp may get fewer)
      constexpr int QW = BQ / 16, DSPLIT = 4 / QW, NPAIR = DT / 2, PPW = (NPAIR + DSPLIT - 1) / DSPLIT, DTW = 2 * PPW;
      const int qg = warp % QW, dg = warp / QW;
      float dq[DTW][4];
#pragma unroll
      for (int t = 0; t < DTW; ++t) dq[t][0] = dq[t][1] = dq[t][2] = dq[t][3] = 0.f;
#pragma unroll
      for (int kk = 0; kk < kBlk / 16; ++kk) {
        uint32_t af[4];
        ldsm_x4_t(at_addr(sdS, SLD, kk * 16, qg * 16), af);
#pragma unroll
        for (int dp = 0; dp < PPW; ++dp) {
          if (DSPLIT > 1 && dg * PPW + dp >= NPAIR) break;   // warp-uniform
          uint32_t bk[4];
          ldsm_x4_t(bt_addr(sK, LD, kk * 16, (dg * PPW + dp) * 16), bk);
          mma16816(dq[2 * dp], af, bk);
          mma16816(dq[2 * dp + 1], af, bk + 2);
        }
      }
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const int q = q0 + qg * 16 + (lane >> 2) + 8 * hr;
        if (q >= a.N) continue;
        float* dst = a.dQacc + ((long long)b * a.N + q) * ((long long)a.H * a.dh) + h * a.dh;
#pragma unroll
        for (int t = 0; t < DTW; ++t) {
          const int d = (dg * DTW + t) * 8 + 2 * (lane & 3);
          if (dg * DTW + t < DT && d < a.dh) {
            atomicAdd(dst + d, dq[t][2 * hr] * a.scale);
            atomicAdd(dst + d + 1, dq[t][2 * hr + 1] * a.scale);
          }
        }
      }
    }
    __syncthreads();   // the buffers of this block are refilled by the next iteration's prefetch
  }
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int key = key_r + 8 * hr;
    if (key >= a.M) continue;
    bf16* dkr = a.dK + b * a.dk_bs + (long long)key * a.lddk + h * a.dh;
    bf16* dvr = a.dV + b * a.dv_bs + (long long)key * a.lddv + h * a.dh;
#pragma unroll
    for (int dt = 0; dt < DT; ++dt) {
      const int d = dt * 8 + 2 * (lane & 3);
      if (d < a.dh) {
        *reinterpret_cast<uint32_t*>(dkr + d) = pack_bf16(dk[dt][2 * hr] * a.scale, dk[dt][2 * hr + 1] * a.scale);
        *reinterpret_cast<uint32_t*>(dvr + d) = pack_bf16(dv[dt][2 * hr], dv[dt][2 * hr + 1]);
      }
    }
  }
}

// =============================================================================================
// dQ of the two-kernel backward: CTA = (64-query tile, head, batch), loop over key blocks
// =============================================================================================
template <int DP>
__global__ void __launch_bounds__(kAttnThreads) attn_bwd_q_kernel(const AttnArgs a) {
  constexpr int LD = DP + 8, KT = DP / 16, DT = DP / 8;
  extern __shared__ __align__(16) uint8_t smem_raw[];
  bf16* sQ = reinterpret_cast<bf16*>(smem_raw);
  bf16* sdO = sQ + kBlk * LD;
  bf16* sK = sdO + kBlk * LD;       // [2][kBlk][LD]
  bf16* sV = sK + 2 * kBlk * LD;    // [2][kBlk][LD]
  const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * kBlk;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long bh = (long long)b * a.H + h;
  const bf16* Kg = a.K + b * a.k_bs + h * a.dh;
  const bf16* Vg = a.V + b * a.v_bs + h * a.dh;
  load_rows<DP>(sQ, a.Q + b * a.q_bs + (long long)q0 * a.ldq + h * a.dh, a.ldq, a.N - q0, kBlk, a.dh);
  load_rows<DP>(sdO, a.dO + b * a.do_bs + (long long)q0 * a.lddo + h * a.dh, a.lddo, a.N - q0, kBlk, a.dh);
  load_rows<DP>(sK, Kg, a.ldk, a.M, kBlk, a.dh);
  load_rows<DP>(sV, Vg, a.ldv, a.M, kBlk, a.dh);
  cp_async_commit();
  const float sl2 = a.scale * kLog2e;
  float lse2[2], dr[2];
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int q = q0 + warp * 16 + (lane >> 2) + 8 * hr;
    lse2[hr] = q < a.N ? a.LSE[bh * a.N + q] * kLog2e : 0.f;
    dr[hr] = q < a.N ? a.Dv[bh * a.N + q] : 0.f;
  }
  float dq[DT][4];
#pragma unroll
  for (int i = 0; i < DT; ++i) dq[i][0] = dq[i][1] = dq[i][2] = dq[i][3] = 0.f;
  const int nblk = (a.M + kBlk - 1) / kBlk;
  for (int j = 0; j < nblk; ++j) {
    const int buf = j & 1;
    if (j + 1 < nblk) {
      const int kn = (j + 1) * kBlk;
      load_rows<DP>(sK + (buf ^ 1) * kBlk * LD, Kg + (long long)kn * a.ldk, a.ldk, a.M - kn, kBlk, a.dh);
      load_rows<DP>(sV + (buf ^ 1) * kBlk * LD, Vg + (long long)kn * a.ldv, a.ldv, a.M - kn, kBlk, a.dh);
    }
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    const bf16* k_s = sK + buf * kBlk * LD;
    const bf16* v_s = sV + buf * kBlk * LD;
    float s[8][4], dp[8][4];
#pragma unroll
    for (int n = 0; n < 8; ++n) {
      s[n][0] = s[n][1] = s[n][2] = s[n][3] = 0.f;
      dp[n][0] = dp[n][1] = dp[n][2] = dp[n][3] = 0.f;
    }
#pragma unroll
    for (int kk = 0; kk < KT; ++kk) {
      uint32_t qa[4], oa[4];
      ldsm_x4(a_addr(sQ, LD, warp * 16, kk * 16), qa);
      ldsm_x4(a_addr(sdO, LD, warp * 16, kk * 16), oa);
#pragma unroll
      for (int np = 0; np < 4; ++np) {
        uint32_t bk[4], bv[4];
        ldsm_x4(b_addr(k_s, LD, np * 16, kk * 16), bk);
        ldsm_x4(b_addr(v_s, LD, np * 16, kk * 16), bv);
        mma16816(s[2 * np], qa, bk);
        mma16816(s[2 * np + 1], qa, bk + 2);
        mma16816(dp[2 * np], oa, bv);
        mma16816(dp[2 * np + 1], oa, bv + 2);
      }
    }
    const int k0 = j * kBlk;
#pragma unroll
    for (int n = 0; n < 8; ++n)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float p = (k0 + n * 8 + 2 * (lane & 3) + (e & 1) < a.M) ? exp2f(fmaf(s[n][e], sl2, -lse2[e >> 1])) : 0.f;
        s[n][e] = p * (dp[n][e] - dr[e >> 1]);
      }
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      uint32_t sa[4];
      pack_a(s[2 * kk], s[2 * kk + 1], sa);
#pragma unroll
      for (int d2 = 0; d2 < DT / 2; ++d2) {
        uint32_t bk[4];
        ldsm_x4_t(bt_addr(k_s, LD, kk * 16, d2 * 16), bk);
        mma16816(dq[2 * d2], sa, bk);
        mma16816(dq[2 * d2 + 1], sa, bk + 2);
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int q = q0 + warp * 16 + (lane >> 2) + 8 * hr;
    if (q >= a.N) continue;
    bf16* dst = a.dQ + b * a.dq_bs + (long long)q * a.lddq + h * a.dh;
#pragma unroll
    for (int dt = 0; dt < DT; ++dt) {
      const int d = dt * 8 + 2 * (lane & 3);
      if (d < a.dh) *reinterpret_cast<uint32_t*>(dst + d) = pack_bf16(dq[dt][2 * hr] * a.scale, dq[dt][2 * hr + 1] * a.scale);
    }
  }
}

__global__ void cvt_dq_kernel(const float* __restrict__ src, bf16* __restrict__ dst, long long rows_per_b, int C,
                              long long ldd, long long d_bs, long long total_vec) {
  const int vpr = C / 8;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total_vec;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / vpr;
    const int c = (int)(i % vpr) * 8;
    const float4 x = *reinterpret_cast<const float4*>(src + r * C + c);
    const float4 y = *reinterpret_cast<const float4*>(src + r * C + c + 4);
    const long long bb = r / rows_per_b, rr = r % rows_per_b;
    *reinterpret_cast<uint4*>(dst + bb * d_bs + rr * ldd + c) =
        make_uint4(pack_bf16(x.x, x.y), pack_bf16(x.z, x.w), pack_bf16(y.x, y.y), pack_bf16(y.z, y.w));
  }
}

// =============================================================================================
// Host
// =============================================================================================
// padded head dims with a kernel instantiation; dh is rounded up to the next one
#define E4T_ATTN_DPS(X) X(16) X(32) X(48) X(64) X(80) X(96) X(128) X(160) X(192)
static int attn_dp(int dh) {
  static const int dps[] = {16, 32, 48, 64, 80, 96, 128, 160, 192};
  for (int d : dps)
    if (dh <= d) return d;
  return 0;
}

// Runtime switches (read on every call, so that one process can compare the variants; all variants compute the same
// function and are held to each other and to fp32 references by the tests):
//   E4T_ATTN_FWD2      forward variant: unset = two K/V buffers, eager rescale, MUFU exp2, 4 warps (64 queries per CTA);
//                      "0" one buffer and 8 warps; otherwise a letter 'd' (two buffers) / 's' (one buffer) followed by
//                      flags: lazy rescale is on unless 'n' is given, 'p<k>' evaluates k of every 8 exponentials on the
//                      FMA pipe, 'f' uses 8 warps (128 queries per CTA)
//   E4T_ATTN_FWD_PT    0: P goes through shared memory (ldmatrix) instead of being re-packed in registers
//   E4T_ATTN_CG        "<forward warps 4|8>,4,4,<max forward CTAs per SM, 0 = no limit>" (the backward kernels have one
//                      warp count); the limit is imposed by padding the dynamic shared memory
//   E4T_ATTN_DELTA2    0: rowsum(dO∘O) with one warp per row instead of one thread per row
//   E4T_ATTN_BWD_BQ    32: 32-query blocks in the dK/dV kernel for every head dim (default 64 for dh <= 96)
//   E4T_ATTN_BWD_STAGES 1: Q / dO of the dK/dV loop single-buffered (default 2: next block prefetched)
//   E4T_ATTN_BWD_FUSED 0: the non-causal single-pass entry point runs the two-kernel backward instead
//   E4T_ATTN_WGMMA     0: the shapes of the warpgroup kernels (attention_wgmma.cu) run the mma.sync kernels of this file
//                      instead.  Setting any of the kernel-variant switches above except E4T_ATTN_DELTA2 does the same:
//                      they name variants of the mma.sync kernels.
static int env_int(const char* name, int dflt) {
  const char* e = getenv(name);
  return (e && *e) ? atoi(e) : dflt;
}

static bool attn_use_wgmma(int B, int H, int N, int M, int dh) {
  if (!attn_wgmma_shape_ok(B, H, N, M, dh) || !env_int("E4T_ATTN_WGMMA", 1)) return false;
  for (const char* v : {"E4T_ATTN_FWD2", "E4T_ATTN_FWD_PT", "E4T_ATTN_CG", "E4T_ATTN_BWD_FUSED", "E4T_ATTN_BWD_BQ",
                        "E4T_ATTN_BWD_STAGES"})
    if (getenv(v)) return false;
  return true;
}

static int attn_common_checks(int dh, long long ldq, long long ldk, long long ldv) {
  E4T_CHECK(dh % 8 == 0 && dh >= 8 && dh <= 192, "attention: head dim %d unsupported (need dh %% 8 == 0, <= 192)", dh);
  E4T_CHECK(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0, "attention: row strides must be multiples of 8 elements");
  return 0;
}

template <typename Kern>
static int attn_launch(Kern kernel, dim3 grid, size_t smem, const AttnArgs& a, cudaStream_t st,
                       int threads = kAttnThreads) {
  E4T_CHECK(smem <= 227 * 1024, "attention: shared memory budget exceeded (%zu)", smem);
  E4T_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kernel<<<grid, threads, smem, st>>>(a);
  E4T_COUNT_LAUNCH();
  E4T_LAUNCH_CHECK();
  return 0;
}

static void launch_attn_delta(const void* O, const void* dO, float* Dv, int B, int H, int N, int dh, long long ldo,
                              long long o_bs, long long lddo, long long do_bs, cudaStream_t st) {
  if (env_int("E4T_ATTN_DELTA2", 1))
    attn_delta2_kernel<<<cdiv((long long)B * N * H, 256), 256, 0, st>>>((const bf16*)O, (const bf16*)dO, Dv, B, H, N, dh,
                                                                        ldo, o_bs, lddo, do_bs);
  else
    attn_delta_kernel<<<cdiv((long long)B * N * H, 8), 256, 0, st>>>((const bf16*)O, (const bf16*)dO, Dv, B, H, N, dh,
                                                                     ldo, o_bs, lddo, do_bs);
  E4T_COUNT_LAUNCH();
}

static AttnArgs attn_args(const void* Q, const void* K, const void* V, int B, int H, int N, int M, int dh, long long ldq,
                          long long q_bs, long long ldk, long long k_bs, long long ldv, long long v_bs, float scale) {
  AttnArgs a;
  memset(&a, 0, sizeof(a));
  a.B = B; a.H = H; a.N = N; a.M = M; a.dh = dh; a.scale = scale;
  a.Q = (const bf16*)Q; a.ldq = ldq; a.q_bs = q_bs;
  a.K = (const bf16*)K; a.ldk = ldk; a.k_bs = k_bs;
  a.V = (const bf16*)V; a.ldv = ldv; a.v_bs = v_bs;
  return a;
}

extern "C" int e4t_attn_fwd(const void* Q, const void* K, const void* V, void* O, float* LSE, int B, int H, int N,
                            int M, int dh, long long ldq, long long q_bs, long long ldk, long long k_bs,
                            long long ldv, long long v_bs, long long ldo, long long o_bs, float scale,
                            void* stream_) {
  cudaStream_t st = (cudaStream_t)stream_;
  if (int e = attn_common_checks(dh, ldq, ldk, ldv)) return e;
  AttnArgs a = attn_args(Q, K, V, B, H, N, M, dh, ldq, q_bs, ldk, k_bs, ldv, v_bs, scale);
  a.O = (bf16*)O; a.ldo = ldo; a.o_bs = o_bs; a.LSE = LSE;
  if (attn_use_wgmma(B, H, N, M, dh)) return attn_wgmma_fwd(a, st);
  a.stages = 2;
  int warps = 4, cap = 0;
  if (const char* e = getenv("E4T_ATTN_FWD2")) {
    if (e[0] == '0') {
      a.stages = 1;
      warps = 8;
    } else if (e[0] == 'd' || e[0] == 's') {
      a.stages = e[0] == 's' ? 1 : 2;
      a.lazy = 1;
      for (const char* c = e + 1; *c; ++c) {
        if (*c == 'n') a.lazy = 0;
        else if (*c == 'f') warps = 8;
        else if (*c == 'p' && c[1] >= '0' && c[1] <= '8') a.poly = *++c - '0';
      }
    }
  }
  a.p_smem = env_int("E4T_ATTN_FWD_PT", 1) == 0;
  if (const char* e = getenv("E4T_ATTN_CG")) {
    int f = 4, q = 4, k = 4, o = 0;
    sscanf(e, "%d,%d,%d,%d", &f, &q, &k, &o);
    warps = f == 8 ? 8 : 4;
    cap = o > 0 ? o : 0;
  }
  const int dp = attn_dp(dh);
  const dim3 grid(cdiv(N, 16 * warps), H, B);
  size_t smem = ((size_t)16 * warps * (dp + 8) + (size_t)2 * a.stages * kBlk * (dp + 8)) * 2 +
                (a.p_smem ? (size_t)warps * 16 * (kBlk + 8) * 2 : 0);
  if (cap > 0) {   // at most `cap` CTAs fit in an SM's 228 KiB of shared memory
    const size_t floor_bytes = (size_t)228 * 1024 / (cap + 1) + 1024;
    if (smem < floor_bytes) smem = floor_bytes;
  }
  const bool var = a.stages != 2 || a.lazy || a.poly || a.p_smem;
#define E4T_FWD(D)                                                                                      \
  if (dp == D) return warps == 8 ? attn_launch(attn_fwd_kernel<D, 8, true>, grid, smem, a, st, 256)    \
                      : var ? attn_launch(attn_fwd_kernel<D, 4, true>, grid, smem, a, st, 128)          \
                            : attn_launch(attn_fwd_kernel<D, 4, false>, grid, smem, a, st, 128);
  E4T_ATTN_DPS(E4T_FWD)
#undef E4T_FWD
  return e4t_set_error("e4t_attn_fwd: head dim %d unsupported", dh);
}

static int attn_bwd_impl(const void* Q, const void* K, const void* V, const void* O, const void* dO, const float* LSE,
                         float* Dv, float* dQacc, void* dQ, void* dK, void* dV, int B, int H, int N, int M, int dh,
                         long long ldq, long long q_bs, long long ldk, long long k_bs, long long ldv, long long v_bs,
                         long long ldo, long long o_bs, long long lddo, long long do_bs, long long lddq, long long dq_bs,
                         long long lddk, long long dk_bs, long long lddv, long long dv_bs, float scale, bool fused,
                         bool causal, cudaStream_t st) {
  if (int e = attn_common_checks(dh, ldq, ldk, ldv)) return e;
  E4T_CHECK(lddo % 8 == 0 && lddq % 8 == 0 && lddk % 8 == 0 && lddv % 8 == 0, "e4t_attn_bwd: strides %% 8");
  E4T_CHECK(!causal || N == M, "e4t_attn_bwd_fused_causal: needs N == M");
  AttnArgs a = attn_args(Q, K, V, B, H, N, M, dh, ldq, q_bs, ldk, k_bs, ldv, v_bs, scale);
  a.dO = (const bf16*)dO; a.lddo = lddo; a.do_bs = do_bs;
  a.LSE = const_cast<float*>(LSE); a.Dv = Dv; a.dQacc = dQacc;
  a.dQ = (bf16*)dQ; a.lddq = lddq; a.dq_bs = dq_bs;
  a.dK = (bf16*)dK; a.lddk = lddk; a.dk_bs = dk_bs;
  a.dV = (bf16*)dV; a.lddv = lddv; a.dv_bs = dv_bs;
  launch_attn_delta(O, dO, Dv, B, H, N, dh, ldo, o_bs, lddo, do_bs, st);
  E4T_LAUNCH_CHECK();
  if (fused) E4T_CUDA(cudaMemsetAsync(dQacc, 0, (size_t)B * N * H * dh * sizeof(float), st));
  a.stages = env_int("E4T_ATTN_BWD_STAGES", 2) == 1 ? 1 : 2;
  const bool bq32 = env_int("E4T_ATTN_BWD_BQ", 64) == 32;
  const dim3 gkv(cdiv(M, kBlk), H, B), gq(cdiv(N, kBlk), H, B);
  const int dp = attn_dp(dh);
  int r = -1;
  const bool wg = fused && !causal && attn_use_wgmma(B, H, N, M, dh);
  if (wg) r = attn_wgmma_bwd(a, st);
#define E4T_BWD_KV(D, BQ, S)                                                                                     \
  {                                                                                                              \
    const size_t skv = BwdCfg<D, BQ>::smem_bytes(fused);                                                         \
    if (causal) r = attn_launch(attn_bwd_kv_kernel<D, BQ, true, true, S>, gkv, skv, a, st);                      \
    else if (fused) r = attn_launch(attn_bwd_kv_kernel<D, BQ, true, false, S>, gkv, skv, a, st);                 \
    else if (!(r = attn_launch(attn_bwd_kv_kernel<D, BQ, false, false, S>, gkv, skv, a, st)))                    \
      r = attn_launch(attn_bwd_q_kernel<D>, gq, (size_t)6 * kBlk * (D + 8) * 2, a, st);                          \
  }
#define E4T_BWD_BQ(D, BQ)                                                                                        \
  {                                                                                                              \
    if (a.stages == 2) E4T_BWD_KV(D, BQ, 2)                                                                      \
    else E4T_BWD_KV(D, BQ, 1)                                                                                    \
  }
#define E4T_BWD(D)                                                                                               \
  if (!wg && dp == D) {                                                                                               \
    if (D <= 96 && !bq32) E4T_BWD_BQ(D, (D <= 96 ? 64 : 32))                                                      \
    else E4T_BWD_BQ(D, 32)                                                                                       \
  }
  E4T_ATTN_DPS(E4T_BWD)
#undef E4T_BWD
#undef E4T_BWD_BQ
#undef E4T_BWD_KV
  if (r < 0) return e4t_set_error("e4t_attn_bwd: head dim %d unsupported", dh);
  if (r) return r;
  if (fused) {
    const long long total_vec = (long long)B * N * (H * dh / 8);
    long long blocks = (total_vec + 255) / 256;
    if (blocks > 132 * 16) blocks = 132 * 16;
    cvt_dq_kernel<<<(int)blocks, 256, 0, st>>>(dQacc, (bf16*)dQ, N, H * dh, lddq, dq_bs, total_vec);
    E4T_COUNT_LAUNCH();
    E4T_LAUNCH_CHECK();
  }
  return 0;
}

// Two-kernel backward (dK/dV kernel, dQ kernel).  Dv: fp32 scratch [B][H][N].
extern "C" int e4t_attn_bwd(const void* Q, const void* K, const void* V, const void* O, const void* dO,
                            const float* LSE, float* Dv, void* dQ, void* dK, void* dV, int B, int H, int N, int M,
                            int dh, long long ldq, long long q_bs, long long ldk, long long k_bs, long long ldv,
                            long long v_bs, long long ldo, long long o_bs, long long lddo, long long do_bs,
                            long long lddq, long long dq_bs, long long lddk, long long dk_bs, long long lddv,
                            long long dv_bs, float scale, void* stream_) {
  return attn_bwd_impl(Q, K, V, O, dO, LSE, Dv, nullptr, dQ, dK, dV, B, H, N, M, dh, ldq, q_bs, ldk, k_bs, ldv, v_bs, ldo,
                       o_bs, lddo, do_bs, lddq, dq_bs, lddk, dk_bs, lddv, dv_bs, scale, false, false,
                       (cudaStream_t)stream_);
}

// Single-pass backward (one pass over the (key tile, query block) pairs).  dQacc: fp32 scratch [B][N][H*dh] (zeroed
// here).
extern "C" int e4t_attn_bwd_fused(const void* Q, const void* K, const void* V, const void* O, const void* dO,
                                  const float* LSE, float* Dv, float* dQacc, void* dQ, void* dK, void* dV, int B, int H,
                                  int N, int M, int dh, long long ldq, long long q_bs, long long ldk, long long k_bs,
                                  long long ldv, long long v_bs, long long ldo, long long o_bs, long long lddo,
                                  long long do_bs, long long lddq, long long dq_bs, long long lddk, long long dk_bs,
                                  long long lddv, long long dv_bs, float scale, void* stream_) {
  return attn_bwd_impl(Q, K, V, O, dO, LSE, Dv, dQacc, dQ, dK, dV, B, H, N, M, dh, ldq, q_bs, ldk, k_bs, ldv, v_bs, ldo,
                       o_bs, lddo, do_bs, lddq, dq_bs, lddk, dk_bs, lddv, dv_bs, scale,
                       env_int("E4T_ATTN_BWD_FUSED", 1) != 0, false, (cudaStream_t)stream_);
}
// The same with a causal mask (key j contributes to query i only if j <= i; N == M): the backward of the CLIP text
// tower's self-attention (e4t/models/modeling_clip.py:45-51) on the tensor cores.  O and LSE come from the forward that
// applied the same mask (e4t_attn_small_fwd).
extern "C" int e4t_attn_bwd_fused_causal(const void* Q, const void* K, const void* V, const void* O, const void* dO,
                                         const float* LSE, float* Dv, float* dQacc, void* dQ, void* dK, void* dV, int B,
                                         int H, int N, int M, int dh, long long ldq, long long q_bs, long long ldk,
                                         long long k_bs, long long ldv, long long v_bs, long long ldo, long long o_bs,
                                         long long lddo, long long do_bs, long long lddq, long long dq_bs, long long lddk,
                                         long long dk_bs, long long lddv, long long dv_bs, float scale, void* stream_) {
  return attn_bwd_impl(Q, K, V, O, dO, LSE, Dv, dQacc, dQ, dK, dV, B, H, N, M, dh, ldq, q_bs, ldk, k_bs, ldv, v_bs, ldo,
                       o_bs, lddo, do_bs, lddq, dq_bs, lddk, dk_bs, lddv, dv_bs, scale, true, true,
                       (cudaStream_t)stream_);
}
