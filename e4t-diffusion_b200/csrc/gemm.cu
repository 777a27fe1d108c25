// e4t_b200 — wgmma GEMM engine (sm_90a).
//
// One persistent, warp-specialised kernel serves every dense contraction on the E4T hot path:
//   * linear layers   Y[M,N] = A[M,K] · B[N,K]^T            (both operands K-major, e.g. F.linear;
//                                                            reference call sites cross_attention.py:506-518,534,
//                                                            attention.py:429 (GEGLU proj), transformer_2d.py proj_in/out)
//   * weight-gradient  dW[C,R] = dY[m,C]^T · X[m,R]          (both operands MN-major, split-K, fp32 atomic accumulate)
//   * input-gradient   dX[M,K] = dY[M,N] · W[N,K]            (A K-major, B MN-major)
//   * 3x3 convolution  (implicit GEMM over NHWC, 9 taps x Cin/64 K-chunks, halo by TMA out-of-bounds zero fill;
//                       diffusers ResnetBlock2D conv1/conv2, Upsample2D.conv, Downsample2D.conv)
//
// Structure (per CTA, 384 threads = 3 warpgroups): warpgroup 0 is the TMA producer (one thread issues), warpgroups 1
// and 2 each own 64 rows of the 128 x BN output tile and issue wgmma.m64nBNk16 from the shared-memory ring of `stages`
// {A 128x64, B BNx64} bf16 tiles (SWIZZLE_128B).  The accumulator lives in registers; the epilogue (alpha, bias,
// row-group addend, residual) writes each warpgroup's 64 x BN result into its own shared-memory staging buffer, from
// which TMA stores it (bf16 / fp32) or adds it (fp32 atomic mode) while the warpgroup already runs the next tile's
// MMAs.  Outputs TMA cannot address (base, row pitch or batch stride not a multiple of 16 bytes) take a register
// epilogue that stores from the accumulator fragments directly.  A bf16 output's residual, where TMA can address it,
// is loaded by TMA into the staging buffer while the tile's MMAs run, so the epilogue adds it from shared memory.
#include "common.cuh"
#include "wgmma.cuh"
#include <stdlib.h>

struct GemmArgs {
  int M, N, K, batch;
  int BN, m_tiles, n_tiles, splits, kchunks, kper, stages;
  int a_mn, b_mn, a_batched, b_batched;
  // implicit 3x3 convolution (conv = 1: forward / dgrad, 2: weight gradient)
  int conv, H, W, BH, BB, cin_chunks, cout;
  int cstride;   // spatial stride of the forward convolution (1, or 2 = Downsample2D; H, W are the OUTPUT size)
  int cpad;      // top / left zero padding of the forward convolution (1; or 0 = diffusers Downsample2D(padding=0))
  // epilogue
  void* out;
  int out_mode;  // 0 = bf16 store, 1 = fp32 store, 2 = fp32 atomic add
  long long ldo, out_bstride;
  const float* bias;      // [N] or null
  const float* rowgroup;  // [M / rows_per_group][N] fp32 (e.g. time-embedding add per image) or null
  int rows_per_group;
  const bf16* residual;  // [M][ldr] bf16 or null
  long long ldr, res_bstride;
  float alpha;
  int pair_store;  // register epilogue: output rows and base allow two-element (4 / 8-byte) stores
  int epi_tma;     // output staged in shared memory and written by TMA (mapO); 0 = register epilogue
};

static constexpr int kBM = 128;
static constexpr int kBK = 64;
static constexpr int kATileBytes = kBM * kBK * 2;  // 16 KiB
static constexpr int kThreads = 384;               // producer warpgroup + 2 MMA / epilogue warpgroups
// Output staging: each MMA warpgroup owns a 64 x BN bf16-sized buffer (fp32 outputs go through it in two column
// halves), cut into 64-row x 64-byte sub-tiles in the SWIZZLE_64B layout, one TMA box each (32 bf16 / 16 fp32 columns).
static constexpr int kSubBytes = 64 * 64;
template <int BN>
constexpr int kStgBytes = 64 * BN * 2;  // per warpgroup

__device__ __forceinline__ void gemm_decode(const GemmArgs& g, long t, int& n_t, int& m_t, int& sp, int& bz) {
  n_t = (int)(t % g.n_tiles);
  long r = t / g.n_tiles;
  m_t = (int)(r % g.m_tiles);
  r /= g.m_tiles;
  sp = (int)(r % g.splits);
  bz = (int)(r / g.splits);
}

template <int BN, int AMN, int BMN>
__device__ __forceinline__ void gemm_epilogue(const GemmArgs& g, const float* acc, int m_t, int n0, int bz, int wg_row) {
  const int lane = threadIdx.x & 31;
  const int w = (threadIdx.x >> 5) & 3;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = m_t * kBM + wg_row + w * 16 + (lane >> 2) + 8 * h;
    if (m >= g.M) continue;
    const float* rg = g.rowgroup ? g.rowgroup + (long long)(m / g.rows_per_group) * g.N : nullptr;
    const bf16* res = g.residual ? g.residual + (long long)bz * g.res_bstride + (long long)m * g.ldr : nullptr;
    const long long orow = (long long)bz * g.out_bstride + (long long)m * g.ldo;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int n = n0 + 8 * j + 2 * (lane & 3);
      if (n >= g.N) break;
      float f0 = acc[4 * j + 2 * h] * g.alpha, f1 = acc[4 * j + 2 * h + 1] * g.alpha;
      const bool two = n + 1 < g.N;
      if (g.bias) { f0 += g.bias[n]; if (two) f1 += g.bias[n + 1]; }
      if (rg) { f0 += rg[n]; if (two) f1 += rg[n + 1]; }
      if (res) { f0 += __bfloat162float(res[n]); if (two) f1 += __bfloat162float(res[n + 1]); }
      if (g.out_mode == 0) {
        bf16* o = reinterpret_cast<bf16*>(g.out) + orow + n;
        if (two && g.pair_store) {
          *reinterpret_cast<uint32_t*>(o) = pack_bf16(f0, f1);
        } else {
          o[0] = __float2bfloat16(f0);
          if (two) o[1] = __float2bfloat16(f1);
        }
      } else if (g.out_mode == 1) {
        float* o = reinterpret_cast<float*>(g.out) + orow + n;
        if (two && g.pair_store) {
          *reinterpret_cast<float2*>(o) = make_float2(f0, f1);
        } else {
          o[0] = f0;
          if (two) o[1] = f1;
        }
      } else {
        float* o = reinterpret_cast<float*>(g.out) + orow + n;
        atomicAdd(o, f0);
        if (two) atomicAdd(o + 1, f1);
      }
    }
  }
}

// Staged epilogue: the warpgroup applies alpha, bias, row-group addend and residual exactly as gemm_epilogue does,
// writes its 64 x BN rows into its staging buffer, and one thread hands the buffer to TMA (a tile store, or a tile add
// for the fp32-atomic mode).  The stores drain while the warpgroup runs the next tile's MMAs; the buffer is rewritten
// only after TMA has read it.  Rows past M and columns past N are clipped by TMA.
// Staging layout: sub-tile s holds columns [s * kSubCols, (s + 1) * kSubCols) as 64 rows of 64 bytes; the 16-byte chunk
// c of row r sits at chunk c ^ ((r >> 1) & 3) (SWIZZLE_64B), so the 8 rows a warp writes per instruction hit 8
// different bank groups.
// RES_TMA (bf16 output only): the residual tile already sits in the staging buffer, loaded by gemm_residual_load into
// the bytes each thread's outputs go to; the thread waits on res_bar, adds the bf16 pair it finds there in place of
// the global read and overwrites it with the output.  The sum and its order are the same, so the output is too.
// Alpha, bias and row-group addend are applied to the accumulators in place first, in loops without per-column
// branches: a row's bias / row-group loads then issue together, where a branch per column pair made each wait for the
// previous pair's load.  Columns past N add a clamped, in-bounds value (TMA clips them); __fmul_rn / __fadd_rn keep
// every product and sum separately rounded, as in gemm_epilogue, so the outputs do not change.
template <int BN, typename OutT, bool RES_TMA = false>
__device__ __forceinline__ void gemm_epilogue_tma(const GemmArgs& g, const CUtensorMap* mapO, float* acc,
                                                  uint8_t* stg, int m_t, int n0, int bz, int wg_row, uint32_t bar_id,
                                                  uint64_t* res_bar = nullptr, uint32_t res_ph = 0) {
  static_assert(!RES_TMA || sizeof(OutT) == 2, "the TMA-loaded residual fills a bf16 staging buffer");
  constexpr int kEsz = (int)sizeof(OutT);
  constexpr int kSubCols = 64 / kEsz;  // 64-byte sub-tile rows: 32 bf16 or 16 fp32 columns
  constexpr int kSubsPerPass = kStgBytes<BN> / kSubBytes;
  constexpr int kPasses = BN / kSubCols / kSubsPerPass;  // 1 for bf16, 2 for fp32
  const int tid = threadIdx.x & 127;
  const int lane = tid & 31;
  const int w = tid >> 5;
  const int row0 = m_t * kBM + wg_row;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = row0 + w * 16 + (lane >> 2) + 8 * h;
    if (m >= g.M) continue;
    if (g.alpha != 1.f) {  // x * 1 is x
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        acc[4 * j + 2 * h] = __fmul_rn(acc[4 * j + 2 * h], g.alpha);
        acc[4 * j + 2 * h + 1] = __fmul_rn(acc[4 * j + 2 * h + 1], g.alpha);
      }
    }
    if (g.bias) {
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int n = n0 + 8 * j + 2 * (lane & 3);
        acc[4 * j + 2 * h] = __fadd_rn(acc[4 * j + 2 * h], g.bias[min(n, g.N - 1)]);
        acc[4 * j + 2 * h + 1] = __fadd_rn(acc[4 * j + 2 * h + 1], g.bias[min(n + 1, g.N - 1)]);
      }
    }
    if (g.rowgroup) {
      const float* rg = g.rowgroup + (long long)(m / g.rows_per_group) * g.N;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int n = n0 + 8 * j + 2 * (lane & 3);
        acc[4 * j + 2 * h] = __fadd_rn(acc[4 * j + 2 * h], rg[min(n, g.N - 1)]);
        acc[4 * j + 2 * h + 1] = __fadd_rn(acc[4 * j + 2 * h + 1], rg[min(n + 1, g.N - 1)]);
      }
    }
  }
#pragma unroll
  for (int p = 0; p < kPasses; ++p) {
    if constexpr (RES_TMA) {
      // the load was issued after the previous tile's store had been read out of the buffer
      if (row0 < g.M) mbar_wait(res_bar, res_ph);
    } else {
      if (tid == 0) tma_store_wait_read<0>();
      named_bar_sync(bar_id, 128);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = w * 16 + (lane >> 2) + 8 * h;
      const int m = row0 + r;
      if (m >= g.M) continue;
      const bf16* res =
          !RES_TMA && g.residual ? g.residual + (long long)bz * g.res_bstride + (long long)m * g.ldr : nullptr;
      uint8_t* srow = stg + r * 64;
      const int sw = (r >> 1) & 3;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int sub = 8 * j / kSubCols;
        if (sub / kSubsPerPass != p) continue;
        const int n = n0 + 8 * j + 2 * (lane & 3);
        float f0 = acc[4 * j + 2 * h], f1 = acc[4 * j + 2 * h + 1];
        const int byte = (8 * j % kSubCols + 2 * (lane & 3)) * kEsz;
        uint8_t* dst = srow + (sub % kSubsPerPass) * kSubBytes + ((((byte >> 4) ^ sw)) << 4) + (byte & 15);
        if (n < g.N) {
          const bool two = n + 1 < g.N;
          if constexpr (RES_TMA) {
            const float2 rr = unpack_bf16(*reinterpret_cast<const uint32_t*>(dst));
            f0 += rr.x;
            if (two) f1 += rr.y;
          }
          if (res) { f0 += __bfloat162float(res[n]); if (two) f1 += __bfloat162float(res[n + 1]); }
        }
        if (kEsz == 2) *reinterpret_cast<uint32_t*>(dst) = pack_bf16(f0, f1);
        else *reinterpret_cast<float2*>(dst) = make_float2(f0, f1);
      }
    }
    fence_proxy_async_smem();
    named_bar_sync(bar_id, 128);
    if (tid == 0 && row0 < g.M) {
#pragma unroll 1
      for (int s = 0; s < kSubsPerPass; ++s) {
        const int n = n0 + (p * kSubsPerPass + s) * kSubCols;
        if (n >= g.N) break;
        if (g.out_mode == 2) tma_reduce_add_3d(mapO, stg + s * kSubBytes, n, row0, bz);
        else tma_store_3d(mapO, stg + s * kSubBytes, n, row0, bz);
      }
      tma_store_commit();
    }
  }
}

// The residual tile of one MMA warpgroup's 64 output rows, loaded by TMA (mapR: the residual with mapO's geometry, box
// and SWIZZLE_64B) into the warpgroup's staging buffer, each element at the byte its output will be written to.  Boxes
// wholly past N are not issued and not counted; rows past M and columns past N read as zero.
template <int BN>
__device__ __forceinline__ void gemm_residual_load(const GemmArgs& g, const CUtensorMap* mapR, uint8_t* stg,
                                                   uint64_t* bar, int n0, int row0, int bz) {
  constexpr int kSubCols = 32;
  const int subs = min(BN / kSubCols, (g.N - n0 + kSubCols - 1) / kSubCols);
  mbar_expect_tx(bar, (uint32_t)(subs * kSubBytes));
  for (int s = 0; s < subs; ++s) tma_load_3d(stg + s * kSubBytes, mapR, bar, n0 + s * kSubCols, row0, bz);
}

// IM2COL: the implicit convolution's pixel operand (conv = 1: A, conv = 2: B) is an im2col-mode tensor map instead
// of a tiled 4-D box.  RES_TMA: the residual of a bf16 staged-epilogue call is TMA-loaded from mapR (host side:
// out_mode 0, epi_tma, residual addressable by TMA; K-major operands only).  Template arguments rather than GemmArgs
// fields, so the kernels every other call runs compile to exactly the code they had without them; mapR is the last
// parameter, so it moves none of the others.
template <int BN, int AMN, int BMN, bool IM2COL, bool RES_TMA>
__global__ void __launch_bounds__(kThreads, 1)
e4t_gemm_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB,
                const __grid_constant__ CUtensorMap mapO, const GemmArgs g, const __grid_constant__ CUtensorMap mapR) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // align dynamic smem to 1024 B (SWIZZLE_128B atoms)
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  constexpr int kBTileBytes = BN * kBK * 2;
  constexpr int kStageBytes = kATileBytes + kBTileBytes;
  // [stages x {A, B}] [staging of MMA warpgroup 0] [staging of MMA warpgroup 1] [full / empty barriers]
  // [RES_TMA: residual-loaded barrier of each MMA warpgroup]
  uint8_t* staging = smem + (size_t)g.stages * kStageBytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(staging + 2 * kStgBytes<BN>);
  uint64_t* empty_bar = full_bar + g.stages;
  uint64_t* res_bar = empty_bar + g.stages;

  const int wg = threadIdx.x >> 7;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&mapA);
    tma_prefetch_desc(&mapB);
    if (g.epi_tma) tma_prefetch_desc(&mapO);
    for (int i = 0; i < g.stages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 256);
    }
    if constexpr (RES_TMA) {
      tma_prefetch_desc(&mapR);
      mbar_init(&res_bar[0], 1);
      mbar_init(&res_bar[1], 1);
    }
    fence_mbar_init();
  }
  __syncthreads();

  const long total_tiles = (long)g.batch * g.splits * g.m_tiles * g.n_tiles;

  if (wg == 0) {
    // ===================== TMA producer ========================================================================
    setmaxnreg_dec<40>();
    if (threadIdx.x != 0) return;
    int s = 0;
    uint32_t ph = 0;
    for (long t = blockIdx.x; t < total_tiles; t += gridDim.x) {
      int n_t, m_t, sp, bz;
      gemm_decode(g, t, n_t, m_t, sp, bz);
      const int m0 = m_t * kBM, n0 = n_t * BN;
      const int kc0 = sp * g.kper;
      const int kc1 = min(g.kchunks, kc0 + g.kper);
      // (image, row, column) of the tile's first output pixel; with the tiled box the column is non-zero only for
      // rows wider than a tile (W > 128: a tile is 128 pixels of one row), with im2col a tile starts anywhere
      int cb0 = 0, ch0 = 0, cw0 = 0;
      if (g.conv == 1) {
        const int img = g.H * g.W;
        cb0 = m0 / img;
        ch0 = (m0 % img) / g.W;
        cw0 = m0 % g.W;
      }
      for (int kc = kc0; kc < kc1; ++kc) {
        mbar_wait(&empty_bar[s], ph ^ 1u);
        uint8_t* sA = smem + (size_t)s * kStageBytes;
        uint8_t* sB = sA + kATileBytes;
        mbar_expect_tx(&full_bar[s], (uint32_t)kStageBytes);
        if (g.conv == 2) {
          // 3x3 weight gradient: dW[tap][co][ci] = sum_p dY[p][co] * X[p + tap][ci].  A = dY (MN-major, 64 pixels of
          // K per chunk), B = the tap-shifted input pixels (MN-major; same 4-D box + out-of-bounds zero fill as the
          // forward's A operand, 64 pixels x 64 channels per N chunk); batch index = tap
          // (im2col: 64 consecutive pixels from any first pixel, across rows and images; past the last pixel both
          // dY and X read as zero)
          const int tap = bz, dy = tap / 3, dx = tap % 3;
          const int p0 = kc * kBK, img = g.H * g.W;
          const int b0 = p0 / img, h0 = (p0 % img) / g.W;
          tma_load_3d(sA, &mapA, &full_bar[s], m0, p0, 0);
          tma_load_3d(sA + 8192, &mapA, &full_bar[s], m0 + 64, p0, 0);
          for (int i = 0; i < BN / 64; ++i) {
            if constexpr (IM2COL)
              tma_load_im2col_4d(sB + i * 8192, &mapB, &full_bar[s], n0 + 64 * i, p0 % g.W - 1, h0 - 1, b0, dx, dy);
            else
              tma_load_4d(sB + i * 8192, &mapB, &full_bar[s], n0 + 64 * i, dx - 1, h0 + dy - 1, b0);
          }
        } else if (g.conv) {
          const int tap = kc / g.cin_chunks, cc = kc % g.cin_chunks;
          const int dy = tap / 3, dx = tap % 3;
          if constexpr (IM2COL)
            tma_load_im2col_4d(sA, &mapA, &full_bar[s], cc * kBK, g.cstride * cw0 - g.cpad, g.cstride * ch0 - g.cpad,
                               cb0, dx, dy);
          else
            tma_load_4d(sA, &mapA, &full_bar[s], cc * kBK, g.cstride * cw0 + dx - g.cpad,
                        g.cstride * ch0 + dy - g.cpad, cb0);
          tma_load_2d(sB, &mapB, &full_bar[s], cc * kBK, tap * g.cout + n0);
        } else {
          const int ab = g.a_batched ? bz : 0, bb = g.b_batched ? bz : 0;
          if (!AMN) {
            tma_load_3d(sA, &mapA, &full_bar[s], kc * kBK, m0, ab);
          } else {
            tma_load_3d(sA, &mapA, &full_bar[s], m0, kc * kBK, ab);
            tma_load_3d(sA + 8192, &mapA, &full_bar[s], m0 + 64, kc * kBK, ab);
          }
          if (!BMN) {
            tma_load_3d(sB, &mapB, &full_bar[s], kc * kBK, n0, bb);
          } else {
            for (int i = 0; i < BN / 64; ++i)
              tma_load_3d(sB + i * 8192, &mapB, &full_bar[s], n0 + 64 * i, kc * kBK, bb);
          }
        }
        if (++s == g.stages) {
          s = 0;
          ph ^= 1u;
        }
      }
    }
  } else {
    // ===================== MMA + epilogue: warpgroup (wg - 1) owns output rows [64 (wg - 1), 64 wg) ============
    setmaxnreg_inc<232>();
    const int wg_row = (wg - 1) * 64;
    // descriptors of stage 0 / k-step 0 for this warpgroup's 64 rows of A; a later stage or k-step only moves the
    // 14-bit start-address field (all of shared memory is below 256 KiB, so the addition never carries out)
    const uint32_t s0 = smem_u32(smem);
    const uint64_t dA0 = AMN ? wgmma_desc(s0 + 8192u * (wg - 1), 8192, 1024)
                             : wgmma_desc(s0 + 8192u * (wg - 1), 16, 1024);
    const uint64_t dB0 = BMN ? wgmma_desc(s0 + kATileBytes, 8192, 1024) : wgmma_desc(s0 + kATileBytes, 16, 1024);
    constexpr uint32_t a_step = AMN ? (2048u >> 4) : (32u >> 4);
    constexpr uint32_t b_step = BMN ? (2048u >> 4) : (32u >> 4);
    constexpr uint32_t stage_units = (uint32_t)kStageBytes >> 4;
    float acc[BN / 2];
    int s = 0;
    uint32_t ph = 0;
    uint32_t res_ph = 0;
    for (long t = blockIdx.x; t < total_tiles; t += gridDim.x) {
      int n_t, m_t, sp, bz;
      gemm_decode(g, t, n_t, m_t, sp, bz);
      const int kc0 = sp * g.kper;
      const int kc1 = min(g.kchunks, kc0 + g.kper);
      const int row0 = m_t * kBM + wg_row;
      int prev = -1;
      for (int kc = kc0; kc < kc1; ++kc) {
        mbar_wait(&full_bar[s], ph);
        const uint64_t da = dA0 + (uint64_t)((uint32_t)s * stage_units);
        const uint64_t db = dB0 + (uint64_t)((uint32_t)s * stage_units);
        reg_fence<BN / 2>(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBK / 16; ++k)
          Wgmma<BN, AMN, BMN>::mma(acc, da + (uint64_t)(k * a_step), db + (uint64_t)(k * b_step),
                                   (kc > kc0 || k > 0) ? 1u : 0u);
        wgmma_commit();
        reg_fence<BN / 2>(acc);
        if constexpr (RES_TMA) {
          // with the tile's first MMAs under way, the thread that committed the previous tile's store waits until
          // TMA has read the staging buffer out, then has TMA fill it with this tile's residual
          if (kc == kc0 && (threadIdx.x & 127) == 0 && row0 < g.M) {
            tma_store_wait_read<0>();
            gemm_residual_load<BN>(g, &mapR, staging + (wg - 1) * kStgBytes<BN>, &res_bar[wg - 1], n_t * BN, row0, bz);
          }
          __syncwarp();
        }
        // the MMAs of the previous k-chunk have retired: its stage can be refilled
        wgmma_wait<1>();
        reg_fence<BN / 2>(acc);
        if (prev >= 0) mbar_arrive(&empty_bar[prev]);
        prev = s;
        if (++s == g.stages) {
          s = 0;
          ph ^= 1u;
        }
      }
      wgmma_wait<0>();
      reg_fence<BN / 2>(acc);
      if (prev >= 0) mbar_arrive(&empty_bar[prev]);
      if constexpr (RES_TMA) {
        gemm_epilogue_tma<BN, bf16, true>(g, &mapO, acc, staging + (wg - 1) * kStgBytes<BN>, m_t, n_t * BN, bz, wg_row,
                                          wg, &res_bar[wg - 1], res_ph);
        if (row0 < g.M) res_ph ^= 1u;
      } else if (!g.epi_tma) {
        gemm_epilogue<BN, AMN, BMN>(g, acc, m_t, n_t * BN, bz, wg_row);
      } else {
        uint8_t* stg = staging + (wg - 1) * kStgBytes<BN>;
        if (g.out_mode == 0) gemm_epilogue_tma<BN, bf16>(g, &mapO, acc, stg, m_t, n_t * BN, bz, wg_row, wg);
        else gemm_epilogue_tma<BN, float>(g, &mapO, acc, stg, m_t, n_t * BN, bz, wg_row, wg);
      }
    }
    // shared memory must outlive the last TMA reads of the staging buffer
    if (g.epi_tma && (threadIdx.x & 127) == 0) tma_store_wait_all();
  }
}

// ---------------------------------------------------------------------------------------------
// Host side
// ---------------------------------------------------------------------------------------------
static int g_num_sms = 0;
static int num_sms() {
  if (g_num_sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
    if (g_num_sms <= 0) g_num_sms = 132;
  }
  return g_num_sms;
}

// Tile-width choice by a cost model in nominal cycles per CTA, with rates taken from the H100 SXM data sheet (989 dense
// BF16 TFLOP/s over 132 SMs: a 128 x BN x 64 k-chunk is ~3.9 * BN cycles of tensor-core work) plus a fixed per-chunk
// hand-off cost; the epilogue term was fitted to the register epilogue, which wrote each output element once (fp32
// atomics cost several times a store):
//   mainloop per 64-deep k-chunk  = 160 + 3.9 * BN
//   epilogue per tile             = 600 + 12 * BN * (1 + [residual]) * (4 if fp32 atomics)
//   kernel                        = ceil(tiles / SMs) * (mainloop + epilogue)
// The staged epilogue's TMA stores drain under the next tile's MMAs, so the epilogue term now overstates what a tile
// pays; it is kept until it is refitted to measured staged-epilogue timings, since a rough repricing moves the split-K
// factor of the large weight gradients.  The widest tile that does not add a round of the persistent grid wins; wide
// tiles also halve operand traffic.
static int pick_bn(int N, long m_tiles_x_batch, bool b_mn, int force_bn, int kchunks_per_tile = 16,
                   bool residual = false, bool atomic = false, double* cost_out = nullptr) {
  if (force_bn > 0) return force_bn;
  const int step = b_mn ? 64 : 32;
  int best = 0;
  double best_cost = 1e30;
  const double sms = (double)num_sms();
  for (int bn = 256; bn >= 64; bn -= step) {
    const int tiles_n = cdiv(N, bn);
    const double tiles = (double)tiles_n * (double)m_tiles_x_batch;
    const double mainloop = kchunks_per_tile * (160.0 + 3.9 * bn);
    const double epilogue = 600.0 + 12.0 * bn * (residual ? 2.0 : 1.0) * (atomic ? 4.0 : 1.0);
    const double rounds = (double)((long)((tiles + sms - 1) / sms));
    const double cost = rounds * (mainloop + epilogue);
    if (cost < best_cost - 1e-6) {
      best_cost = cost;
      best = bn;
    }
  }
  if (cost_out) *cost_out = best_cost;
  return best;
}

// Split-K factor of an fp32-accumulating GEMM (weight gradients: small M x N, very long K) by the same cost model: the
// factor that minimises rounds x (mainloop + atomic epilogue).
static int auto_splits(int N, long m_tiles_x_batch, bool b_mn, int kchunks) {
  int best = 1;
  double best_cost = 1e30;
  const int smax = kchunks < 64 ? kchunks : 64;
  for (int sp = 1; sp <= smax; ++sp) {
    const int kper = cdiv(kchunks, sp);
    if (cdiv(kchunks, kper) != sp) continue;          // same kper as a smaller factor
    double c = 0;
    pick_bn(N, m_tiles_x_batch * sp, b_mn, 0, kper, false, true, &c);
    if (c < best_cost - 1e-6) {
      best_cost = c;
      best = sp;
    }
  }
  return best;
}

template <int BN, int AMN, int BMN, bool IM2COL, bool RES_TMA>
static int launch_gemm_t(const CUtensorMap& mA, const CUtensorMap& mB, const CUtensorMap& mO, const CUtensorMap& mR,
                         GemmArgs& g, int grid, cudaStream_t stream) {
  constexpr int stage_bytes = kATileBytes + BN * kBK * 2;
  constexpr int res_bars = RES_TMA ? 2 : 0;
  // the ring gets what the two staging buffers, the barriers and the 1 KiB alignment slack leave of 227 KiB
  int stages = (227 * 1024 - 1024 - 2 * kStgBytes<BN> - (16 + res_bars) * (int)sizeof(uint64_t)) / stage_bytes;
  if (stages > 8) stages = 8;
  if (stages > g.kper) stages = g.kper < 2 ? 2 : g.kper;
  g.stages = stages;
  const size_t smem =
      (size_t)stages * stage_bytes + 2 * kStgBytes<BN> + (2 * stages + res_bars) * sizeof(uint64_t) + 1024;
  static bool attr_set = false;
  if (!attr_set) {
    E4T_CUDA(cudaFuncSetAttribute(e4t_gemm_kernel<BN, AMN, BMN, IM2COL, RES_TMA>,
                                  cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    attr_set = true;
  }
  e4t_gemm_kernel<BN, AMN, BMN, IM2COL, RES_TMA><<<grid, kThreads, smem, stream>>>(mA, mB, mO, g, mR);
  E4T_COUNT_LAUNCH();
  E4T_LAUNCH_CHECK();
  return 0;
}

template <int AMN, int BMN, bool IM2COL, bool RES_TMA = false>
static int launch_gemm_bn(const CUtensorMap& mA, const CUtensorMap& mB, const CUtensorMap& mO, const CUtensorMap& mR,
                          GemmArgs& g, int grid, cudaStream_t stream) {
  switch (g.BN) {
    case 64: return launch_gemm_t<64, AMN, BMN, IM2COL, RES_TMA>(mA, mB, mO, mR, g, grid, stream);
    case 128: return launch_gemm_t<128, AMN, BMN, IM2COL, RES_TMA>(mA, mB, mO, mR, g, grid, stream);
    case 192: return launch_gemm_t<192, AMN, BMN, IM2COL, RES_TMA>(mA, mB, mO, mR, g, grid, stream);
    case 256: return launch_gemm_t<256, AMN, BMN, IM2COL, RES_TMA>(mA, mB, mO, mR, g, grid, stream);
  }
  if constexpr (!BMN) {
    switch (g.BN) {
      case 96: return launch_gemm_t<96, AMN, 0, IM2COL, RES_TMA>(mA, mB, mO, mR, g, grid, stream);
      case 160: return launch_gemm_t<160, AMN, 0, IM2COL, RES_TMA>(mA, mB, mO, mR, g, grid, stream);
      case 224: return launch_gemm_t<224, AMN, 0, IM2COL, RES_TMA>(mA, mB, mO, mR, g, grid, stream);
    }
  }
  return e4t_set_error("e4t_gemm_bf16: unsupported tile width BN=%d (b_mn=%d)", g.BN, BMN);
}

// im2col: an implicit convolution whose pixel operand mA (forward) / mB (weight gradient) is an im2col-mode map.
static int launch_gemm(const CUtensorMap& mA, const CUtensorMap& mB, GemmArgs& g, cudaStream_t stream,
                       bool im2col = false) {
  const int esz = g.out_mode == 0 ? 2 : 4;
  g.pair_store = (g.ldo % 2) == 0 && (g.batch == 1 || (g.out_bstride % 2) == 0) && ((uintptr_t)g.out % (2 * esz)) == 0;
  // TMA addresses the output when its base is 16-byte aligned and its row width, row pitch and batch stride are
  // multiples of 16 bytes; anything else, or E4T_GEMM_EPI_PLAIN=0, takes the register epilogue.  (The row width: on
  // the H100 a TMA store whose row ends off a 16-byte boundary writes on to that boundary, so with a row pitch beyond
  // N it overwrote up to 7 bf16 / 3 fp32 elements past N, the neighbouring columns of a column-slice output.)
  const char* p = getenv("E4T_GEMM_EPI_PLAIN");
  const bool want_tma = !(p && *p) || atoi(p) != 0;
  g.epi_tma = want_tma && ((uintptr_t)g.out % 16) == 0 && (g.N * esz) % 16 == 0 && (g.ldo * esz) % 16 == 0 &&
              g.ldo >= g.N &&
              (g.batch == 1 || (g.out_bstride > 0 && (g.out_bstride * esz) % 16 == 0));
  CUtensorMap mO;
  memset(&mO, 0, sizeof(mO));
  if (g.epi_tma) {
    const uint64_t bs = g.batch == 1 ? (uint64_t)g.ldo * g.M : (uint64_t)g.out_bstride;
    uint64_t dims[3] = {(uint64_t)g.N, (uint64_t)g.M, (uint64_t)g.batch};
    uint64_t str[2] = {(uint64_t)g.ldo * esz, bs * esz};
    uint32_t box[3] = {(uint32_t)(64 / esz), 64, 1};
    if (int e = e4t_tmap_encode(&mO, g.out, 3, dims, str, box, esz, 64)) return e;
  }
  // A bf16 staged epilogue's residual is TMA-loaded into the staging buffer under the MMAs when TMA can address it as
  // it addresses the output (the same conditions on base, row pitch and batch stride); fp32 outputs, the register
  // epilogue and other residuals read it from global memory in the epilogue.  Residual calls all have K-major
  // operands, so only those kernels are built with the load.
  const bool res_tma = g.epi_tma && g.out_mode == 0 && g.residual && !g.a_mn && !g.b_mn &&
                       ((uintptr_t)g.residual % 16) == 0 && (g.ldr * 2) % 16 == 0 && g.ldr >= g.N &&
                       (g.batch == 1 || (g.res_bstride > 0 && (g.res_bstride * 2) % 16 == 0));
  CUtensorMap mR;
  memset(&mR, 0, sizeof(mR));
  if (res_tma) {
    const uint64_t bs = g.batch == 1 ? (uint64_t)g.ldr * g.M : (uint64_t)g.res_bstride;
    uint64_t dims[3] = {(uint64_t)g.N, (uint64_t)g.M, (uint64_t)g.batch};
    uint64_t str[2] = {(uint64_t)g.ldr * 2, bs * 2};
    uint32_t box[3] = {32, 64, 1};
    if (int e = e4t_tmap_encode(&mR, g.residual, 3, dims, str, box, 2, 64)) return e;
  }
  const long total = (long)g.batch * g.splits * g.m_tiles * g.n_tiles;
  int grid = (int)(total < num_sms() ? total : num_sms());
  if (grid < 1) return 0;
  // the implicit convolutions load A K-major (wgrad: both operands MN-major, set in a_mn / b_mn)
  if (im2col)
    return g.a_mn ? launch_gemm_bn<1, 1, true>(mA, mB, mO, mR, g, grid, stream)
           : res_tma ? launch_gemm_bn<0, 0, true, true>(mA, mB, mO, mR, g, grid, stream)
                     : launch_gemm_bn<0, 0, true>(mA, mB, mO, mR, g, grid, stream);
  if (g.a_mn)
    return g.b_mn ? launch_gemm_bn<1, 1, false>(mA, mB, mO, mR, g, grid, stream)
                  : launch_gemm_bn<1, 0, false>(mA, mB, mO, mR, g, grid, stream);
  return g.b_mn  ? launch_gemm_bn<0, 1, false>(mA, mB, mO, mR, g, grid, stream)
         : res_tma ? launch_gemm_bn<0, 0, false, true>(mA, mB, mO, mR, g, grid, stream)
                   : launch_gemm_bn<0, 0, false>(mA, mB, mO, mR, g, grid, stream);
}

extern "C" int e4t_gemm_bf16(const void* A, const void* B, void* out, int M, int N, int K, int batch, int a_mn,
                             int b_mn, long long lda, long long ldb, long long a_bstride, long long b_bstride,
                             int out_mode, long long ldo, long long out_bstride, const float* bias,
                             const float* rowgroup, int rows_per_group, const void* residual, long long ldr,
                             long long res_bstride, float alpha, int splits, int force_bn, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  E4T_CHECK(M > 0 && N > 0 && K > 0 && batch > 0, "e4t_gemm_bf16: bad dims M=%d N=%d K=%d batch=%d", M, N, K, batch);
  E4T_CHECK((lda % 8) == 0 && (ldb % 8) == 0, "e4t_gemm_bf16: leading strides must be multiples of 8 elements");
  E4T_CHECK(((uintptr_t)A % 16) == 0 && ((uintptr_t)B % 16) == 0, "e4t_gemm_bf16: operands must be 16-byte aligned");
  E4T_CHECK(out_mode >= 0 && out_mode <= 2, "e4t_gemm_bf16: bad out_mode");
  GemmArgs g;
  memset(&g, 0, sizeof(g));
  g.M = M; g.N = N; g.K = K; g.batch = batch;
  g.a_mn = a_mn; g.b_mn = b_mn;
  g.a_batched = (a_bstride != 0); g.b_batched = (b_bstride != 0);
  g.m_tiles = cdiv(M, kBM);
  g.kchunks = cdiv(K, kBK);
  // every split's epilogue applies bias, row-group addend and residual: split-K takes none of them
  const bool addends = bias || rowgroup || residual;
  if (splits == 0 && out_mode == 2 && force_bn <= 0 && !addends)
    splits = auto_splits(N, (long)g.m_tiles * batch, b_mn != 0, g.kchunks);
  if (splits < 1) splits = 1;
  if (splits > g.kchunks) splits = g.kchunks;
  g.kper = cdiv(g.kchunks, splits);
  g.splits = cdiv(g.kchunks, g.kper);  // no empty split
  g.BN = pick_bn(N, (long)g.m_tiles * batch * g.splits, b_mn != 0, force_bn, g.kper, residual != nullptr, out_mode == 2);
  E4T_CHECK(g.BN >= 64 && g.BN <= 256 && (g.BN % (b_mn ? 64 : 32)) == 0, "e4t_gemm_bf16: bad BN %d", g.BN);
  g.n_tiles = cdiv(N, g.BN);
  E4T_CHECK(g.splits == 1 || out_mode == 2, "e4t_gemm_bf16: split-K requires atomic fp32 output");
  E4T_CHECK(g.splits == 1 || !addends, "e4t_gemm_bf16: split-K would add bias / rowgroup / residual once per split");
  g.out = out; g.out_mode = out_mode; g.ldo = ldo; g.out_bstride = out_bstride;
  g.bias = bias; g.rowgroup = rowgroup; g.rows_per_group = rows_per_group > 0 ? rows_per_group : 1;
  g.residual = (const bf16*)residual; g.ldr = ldr; g.res_bstride = res_bstride;
  g.alpha = alpha;

  CUtensorMap mA, mB;
  {
    const uint64_t nb = g.a_batched ? (uint64_t)batch : 1;
    const uint64_t bs = g.a_batched ? (uint64_t)a_bstride : (uint64_t)lda * (a_mn ? K : M);
    if (!a_mn) {
      uint64_t dims[3] = {(uint64_t)K, (uint64_t)M, nb};
      uint64_t str[2] = {(uint64_t)lda * 2, bs * 2};
      uint32_t box[3] = {kBK, kBM, 1};
      if (int e = e4t_tmap_encode(&mA, A, 3, dims, str, box, 2)) return e;
    } else {
      uint64_t dims[3] = {(uint64_t)M, (uint64_t)K, nb};
      uint64_t str[2] = {(uint64_t)lda * 2, bs * 2};
      uint32_t box[3] = {64, kBK, 1};
      if (int e = e4t_tmap_encode(&mA, A, 3, dims, str, box, 2)) return e;
    }
  }
  {
    const uint64_t nb = g.b_batched ? (uint64_t)batch : 1;
    const uint64_t bs = g.b_batched ? (uint64_t)b_bstride : (uint64_t)ldb * (b_mn ? K : N);
    if (!b_mn) {
      uint64_t dims[3] = {(uint64_t)K, (uint64_t)N, nb};
      uint64_t str[2] = {(uint64_t)ldb * 2, bs * 2};
      uint32_t box[3] = {kBK, (uint32_t)g.BN, 1};
      if (int e = e4t_tmap_encode(&mB, B, 3, dims, str, box, 2)) return e;
    } else {
      uint64_t dims[3] = {(uint64_t)N, (uint64_t)K, nb};
      uint64_t str[2] = {(uint64_t)ldb * 2, bs * 2};
      uint32_t box[3] = {64, kBK, 1};
      if (int e = e4t_tmap_encode(&mB, B, 3, dims, str, box, 2)) return e;
    }
  }
  return launch_gemm(mA, mB, g, stream);
}

// x: NHWC bf16 [B][Hin][Win][Cin];  w: bf16 [9][Cout][Cin] (tap = ky*3+kx);  out: [B*H*W][Cout] (NHWC),
// H = ceil(Hin/stride).
// bias fp32 [Cout]; rowgroup fp32 [B][Cout] (time-embedding projection) ; residual bf16 NHWC.
// Padding: pad_lo zero rows / columns on the top and left (1 = the symmetric pad-1 convolution); the taps of output
// pixel (y, x) read input (stride*y + ky - pad_lo, stride*x + kx - pad_lo), and whatever falls outside the input, on
// either side, is TMA out-of-bounds zero fill.  pad_lo = 0 with stride 2 is diffusers' Downsample2D(padding=0), which
// pads one zero row / column on the bottom and right only.
// stride 2 (diffusers Downsample2D): the A-operand tensor map walks the input with element strides (1,2,2,1), so the
// tile of 128 OUTPUT pixels is gathered directly from every other input pixel — no stride-1 result is computed and
// thrown away (round 1 did exactly that: 4x the FLOPs on the three downsampling convolutions).
// Tiles, tiled box (im2col = 0): an output width W that divides 128 gives tiles of 128 / W whole rows (or whole images
// when H*W < 128); a width W > 128 that is a multiple of 128 gives tiles of 128 consecutive pixels of one row, whose
// first column the producer adds to the A-operand x coordinate.  conv_tiled_fits() is that domain.
// im2col = 1: the A operand is an im2col-mode tensor map, so a tile is any 128 consecutive output pixels in NHW order,
// across row and image boundaries, and every output size works.  Its bounding box starts at -pad_lo and ends on the
// last tap-(0, 0) position, stride*(out - 1) - pad_lo, so each image yields exactly H x W output pixels; the tap's
// (dx, dy) are the load's im2col offsets.  The shared-memory tile is byte-identical to the tiled box's (128 rows of 64
// channels, SWIZZLE_128B), so the MMA warpgroups and the epilogue do not know which load filled it.
// Odd input sides (stride 2, pad 1 only) give ceil(Hin/2) outputs and always take the im2col load: its upper corner
// 2*(H - 1) - 1 - (Hin - 1) is -1 for an odd side (-2 for an even one), and the last output's taps read the bottom /
// right pad as out-of-bounds zeros.
static bool conv_tiled_fits(int H, int W) {
  if (W > 128) return W % 128 == 0;
  if (128 % W) return false;
  return H * W >= 128 ? H % (128 / W) == 0 : 128 % (H * W) == 0;
}

static int conv3x3_impl(const void* x, const void* w, void* out, int B, int Hin, int Win, int Cin, int Cout, int stride,
                        int pad_lo, int out_mode, const float* bias, const float* rowgroup, const void* residual,
                        int force_bn, bool im2col, cudaStream_t stream) {
  E4T_CHECK(B > 0 && Hin > 0 && Win > 0 && Cout > 0, "e4t_conv3x3: bad dims B=%d H=%d W=%d Cout=%d", B, Hin, Win, Cout);
  E4T_CHECK(Cin % 64 == 0, "e4t_conv3x3: Cin must be a multiple of 64 (got %d)", Cin);
  E4T_CHECK(stride == 1 || (stride == 2 && ((Hin % 2 == 0 && Win % 2 == 0) || (pad_lo == 1 && im2col))),
            "e4t_conv3x3: bad stride/size");
  E4T_CHECK(pad_lo == 1 || (stride == 2 && pad_lo == 0), "e4t_conv3x3: bad padding %d for stride %d", pad_lo, stride);
  const int H = (Hin + stride - 1) / stride, W = (Win + stride - 1) / stride;
  const bool wide = W > 128;
  const int img = H * W;
  int BH = 1, BB = 1;
  if (!im2col) {
    E4T_CHECK((W <= 128 && (128 % W) == 0) || (wide && W % 128 == 0),
              "e4t_conv3x3: output width must divide 128 or be a multiple of 128 (got %d)", W);
    if (wide) {
      BB = 1;
      BH = 1;
    } else if (img >= 128) {
      BB = 1;
      BH = 128 / W;
      E4T_CHECK(H % BH == 0, "e4t_conv3x3: H=%d not a multiple of tile height %d", H, BH);
    } else {
      E4T_CHECK(128 % img == 0, "e4t_conv3x3: H*W must divide 128");
      BB = 128 / img;
      BH = H;
    }
  }
  E4T_CHECK(out_mode == 0 || out_mode == 1, "e4t_conv3x3: bad out_mode");
  const int BW = wide ? 128 : W;
  GemmArgs g;
  memset(&g, 0, sizeof(g));
  g.M = B * img; g.N = Cout; g.K = Cin; g.batch = 1;
  g.conv = 1; g.H = H; g.W = W; g.BH = BH; g.BB = BB; g.cin_chunks = Cin / 64; g.cout = Cout; g.cstride = stride;
  g.cpad = pad_lo;
  g.m_tiles = cdiv(g.M, kBM);
  g.kchunks = 9 * g.cin_chunks;
  g.kper = g.kchunks; g.splits = 1;
  g.BN = pick_bn(Cout, g.m_tiles, false, force_bn, g.kchunks, residual != nullptr, false);
  g.n_tiles = cdiv(Cout, g.BN);
  g.out = out; g.out_mode = out_mode; g.ldo = Cout; g.out_bstride = 0;
  g.bias = bias; g.rowgroup = rowgroup; g.rows_per_group = img;
  g.residual = (const bf16*)residual; g.ldr = Cout; g.res_bstride = 0;
  g.alpha = 1.f;
  CUtensorMap mA, mB;
  {
    uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)Win, (uint64_t)Hin, (uint64_t)B};
    uint64_t str[3] = {(uint64_t)Cin * 2, (uint64_t)Win * Cin * 2, (uint64_t)Hin * Win * Cin * 2};
    uint32_t es[4] = {1, (uint32_t)stride, (uint32_t)stride, 1};
    if (im2col) {
      const int lower[2] = {-pad_lo, -pad_lo};
      const int upper[2] = {stride * (W - 1) - pad_lo - (Win - 1), stride * (H - 1) - pad_lo - (Hin - 1)};
      if (int e = e4t_tmap_encode_im2col(&mA, x, dims, str, lower, upper, kBK, kBM, es)) return e;
    } else {
      uint32_t box[4] = {kBK, (uint32_t)(BW * stride), (uint32_t)(BH * stride), (uint32_t)BB};
      if (int e = e4t_tmap_encode(&mA, x, 4, dims, str, box, 2, 128, stride == 1 ? nullptr : es)) return e;
    }
  }
  {
    uint64_t dims[2] = {(uint64_t)Cin, (uint64_t)9 * Cout};
    uint64_t str[1] = {(uint64_t)Cin * 2};
    uint32_t box[2] = {kBK, (uint32_t)g.BN};
    if (int e = e4t_tmap_encode(&mB, w, 2, dims, str, box, 2)) return e;
  }
  return launch_gemm(mA, mB, g, stream, im2col);
}

extern "C" int e4t_conv3x3_bf16(const void* x, const void* w, void* out, int B, int H, int W, int Cin, int Cout,
                                int out_mode, const float* bias, const float* rowgroup, const void* residual,
                                int force_bn, void* stream_) {
  return conv3x3_impl(x, w, out, B, H, W, Cin, Cout, 1, 1, out_mode, bias, rowgroup, residual, force_bn, false,
                      (cudaStream_t)stream_);
}

// e4t_conv3x3_bf16 with the A operand in TMA im2col mode: any output size (tiles span rows and images).
extern "C" int e4t_conv3x3_im2col_bf16(const void* x, const void* w, void* out, int B, int H, int W, int Cin, int Cout,
                                       int out_mode, const float* bias, const float* rowgroup, const void* residual,
                                       int force_bn, void* stream_) {
  return conv3x3_impl(x, w, out, B, H, W, Cin, Cout, 1, 1, out_mode, bias, rowgroup, residual, force_bn, true,
                      (cudaStream_t)stream_);
}

// 3x3 / stride 2 / pad 1 (diffusers Downsample2D.conv, e4t/models/unet_2d_blocks.py:801-808): x [B][H][W][Cin] ->
// out [B][ceil(H/2)][ceil(W/2)][Cout].  Even sizes: the tiled box where it covers the output size, im2col elsewhere;
// odd sizes: im2col.
extern "C" int e4t_conv3x3_s2_bf16(const void* x, const void* w, void* out, int B, int H, int W, int Cin, int Cout,
                                   const float* bias, int force_bn, void* stream_) {
  const bool odd = (H % 2) != 0 || (W % 2) != 0;
  return conv3x3_impl(x, w, out, B, H, W, Cin, Cout, 2, 1, 0, bias, nullptr, nullptr, force_bn,
                      odd || !conv_tiled_fits(H / 2, W / 2), (cudaStream_t)stream_);
}

// 3x3 / stride 2 with pad_lo zero rows / columns on the top and left: pad_lo = 1 is e4t_conv3x3_s2_bf16; pad_lo = 0 is
// diffusers' Downsample2D(padding=0) (F.pad(x, (0, 1, 0, 1)) then an unpadded stride-2 convolution; the VAE encoder).
extern "C" int e4t_conv3x3_s2p_bf16(const void* x, const void* w, void* out, int B, int H, int W, int Cin, int Cout,
                                    int pad_lo, const float* bias, int force_bn, void* stream_) {
  return conv3x3_impl(x, w, out, B, H, W, Cin, Cout, 2, pad_lo, 0, bias, nullptr, nullptr, force_bn,
                      !conv_tiled_fits(H / 2, W / 2), (cudaStream_t)stream_);
}

// 3x3 / stride 1 / pad 1 weight gradient: dw9[tap][co][ci] += sum_{b,y,x} dy[b][y][x][co] * x[b][y+ky-1][x+kx-1][ci]
// (tap = ky*3+kx; fp32 atomic accumulation, split-K over the pixels).  x NHWC bf16 [B][H][W][Cin], dy [B][H][W][Cout].
// Replaces autograd's conv2d weight gradient behind every ResnetBlock2D / Upsample2D / Downsample2D conv when the base
// UNet is trainable (tuning_e4t.py:139-146).  Cin, Cout % 64 == 0.  Each K chunk is 64 consecutive pixels: a tiled
// box of whole rows where W | 64 and H*W % 64 == 0, else an im2col-mode load (any image size; the last chunk's
// pixels past B*H*W are zero in both operands).
extern "C" int e4t_conv3x3_wgrad(const void* x, const void* dy, float* dw9, int B, int H, int W, int Cin, int Cout,
                                 void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  E4T_CHECK(Cin % 64 == 0 && Cout % 64 == 0, "e4t_conv3x3_wgrad: Cin, Cout must be multiples of 64 (%d, %d)", Cin, Cout);
  E4T_CHECK(B > 0 && H > 0 && W > 0, "e4t_conv3x3_wgrad: bad image %dx%dx%d", B, H, W);
  const bool im2col = !(W <= 64 && (64 % W) == 0 && (H * W) % 64 == 0 && H % (64 / W) == 0);
  const long long pixels = (long long)B * H * W;
  GemmArgs g;
  memset(&g, 0, sizeof(g));
  g.M = Cout; g.N = Cin; g.K = (int)pixels; g.batch = 9;
  g.a_mn = 1; g.b_mn = 1; g.a_batched = 0; g.b_batched = 1;
  g.conv = 2; g.H = H; g.W = W; g.cout = Cout; g.cstride = 1; g.cpad = 1;
  g.m_tiles = cdiv(Cout, kBM);
  g.kchunks = cdiv(pixels, kBK);
  // enough K-splits to fill the machine about twice: tiles = 9 taps x m_tiles x n_tiles x splits
  const int base_tiles = 9 * g.m_tiles * cdiv(Cin, 256);
  int splits = cdiv(2 * num_sms(), base_tiles);
  if (splits < 1) splits = 1;
  if (splits > g.kchunks) splits = g.kchunks;
  g.kper = cdiv(g.kchunks, splits);
  g.splits = cdiv(g.kchunks, g.kper);
  g.BN = Cin >= 256 ? 256 : (Cin >= 192 ? 192 : (Cin >= 128 ? 128 : 64));
  g.n_tiles = cdiv(Cin, g.BN);
  g.out = dw9; g.out_mode = 2; g.ldo = Cin; g.out_bstride = (long long)Cout * Cin;
  g.rows_per_group = 1; g.alpha = 1.f;
  CUtensorMap mA, mB;
  {
    uint64_t dims[3] = {(uint64_t)Cout, (uint64_t)pixels, 1};
    uint64_t str[2] = {(uint64_t)Cout * 2, (uint64_t)pixels * Cout * 2};
    uint32_t box[3] = {64, kBK, 1};
    if (int e = e4t_tmap_encode(&mA, dy, 3, dims, str, box, 2)) return e;
  }
  {
    uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)W, (uint64_t)H, (uint64_t)B};
    uint64_t str[3] = {(uint64_t)Cin * 2, (uint64_t)W * Cin * 2, (uint64_t)H * W * Cin * 2};
    if (im2col) {
      const int lower[2] = {-1, -1}, upper[2] = {-1, -1};   // the stride-1 pad-1 box: W x H tap-(0, 0) positions
      const uint32_t es[4] = {1, 1, 1, 1};
      if (int e = e4t_tmap_encode_im2col(&mB, x, dims, str, lower, upper, 64, kBK, es)) return e;
    } else {
      uint32_t box[4] = {64, (uint32_t)W, (uint32_t)(64 / W), 1};
      if (int e = e4t_tmap_encode(&mB, x, 4, dims, str, box, 2)) return e;
    }
  }
  return launch_gemm(mA, mB, g, stream, im2col);
}
