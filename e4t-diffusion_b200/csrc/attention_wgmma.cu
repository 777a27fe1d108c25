// e4t — warpgroup-level attention for the long non-causal self-attention of the SD-v1.4 UNet, level 0 (N = M = 4096,
// 8 heads of 40) and level 1 (N = M = 1024, 8 heads of 80), and of the SD 2.x UNet (heads of 64 at every level: 5, 10
// and 20 heads, 9216 / 2304 / 576 tokens at 768²).  wgmma.mma_async from SWIZZLE_128B shared-memory tiles
// that TMA fills, fp32 accumulators in registers.  Same function, arguments and outputs as the mma.sync kernels of
// attention.cu, which keep every other shape.
//
// Which shapes run here (attn_wgmma_shape_ok): dh = 40, 64 or 80, N and M multiples of 128 and >= 512; for dh = 64 and
// 80 also a grid of (N / 128) x H x B CTAs of at least half the device's SM count.
//
// Loading: a head slice is dh bf16 wide inside a token row.  Q/K/V/dO are described to TMA as the 4-D tensor
// (dh, H, tokens, B) with a box of 64 x 1 x rows x 1, loaded once per 64-column panel (x = 0, and x = 64 for dh = 80):
// columns >= dh are out of bounds and arrive as zeros, so a panel is rows x 128 B, swizzled, with no neighbouring head
// in the padding (dh = 64 fills its panel, no padding).  A tile is its panels one after the other.  Products over the head dim take ceil(dh / 16) k-steps,
// the fifth one (dh = 80) reading the second panel; products whose N is the head dim use an instruction of exactly
// N = dh, which reads an MN-major operand's second panel at the descriptor's leading byte offset.
//
// Forward, CTA = (128 queries, head, batch), 384 threads: warpgroup 0 is the producer (one thread issues TMA into a
// ring of K/V blocks of 128 keys), warpgroups 1 and 2 own 64 query rows each.  S = Q·Kᵀ from shared memory, online
// softmax in the exp2 domain on the accumulator registers, P re-packed in registers as the A operand of O += P·V
// (V is the MN-major B operand).  Q·Kᵀ of block j + 1 is issued before P·V of block j, and the softmax of block j + 1
// runs while P·V of block j is still in flight.
//
// Backward (single pass), CTA = (128 keys, head, batch), 384 threads: K and V stay in shared memory; warpgroups 1 and 2
// own 64 keys each and, per block of 64 queries, compute Sᵀ = K·Qᵀ and dPᵀ = V·dOᵀ from shared memory, Pᵀ and dSᵀ in
// registers, dV += Pᵀ·dO and dK += dSᵀ·Q with Pᵀ / dSᵀ as register A operands, and store dSᵀ (bf16) to shared memory.
// Warpgroup 0 issues the TMA loads of Q, dO, LSE and D (one thread) and computes dQ_block = dS·K over the CTA's 128
// keys from the stored dSᵀ (MN-major A) and K (MN-major B); the fp32 block goes to shared memory and is added to dQacc
// by one bulk tensor reduce (cp.reduce.async.bulk.tensor add), double buffered so that it overlaps the next block.
#include "attention.cuh"
#include "wgmma.cuh"

static constexpr int kWgThreads = 384;
static constexpr int kFwdStages = 3;     // K/V ring of the forward
static constexpr int kTile128 = 128 * 128;   // bytes of a 128-row panel
static constexpr int kTile64 = 64 * 128;     // bytes of a 64-row panel
static constexpr size_t kMaxSmem = 227 * 1024;

// k-step k (16 columns of the head dim) of a K-major tile whose 64-column panels are `panel` bytes apart, in
// descriptor units
__device__ __forceinline__ constexpr uint64_t kstep(int k, uint32_t panel) {
  return (uint64_t)((k / 4) * (panel >> 4) + 2 * (k % 4));
}

__device__ __forceinline__ uint8_t* align1024(uint8_t* p) {
  return p + ((1024u - (smem_u32(p) & 1023u)) & 1023u);
}

// Shared-memory layouts, used by the kernels and by the host for the launch size
template <int DH>
struct FwdSmem {
  static constexpr int P = (DH + 63) / 64;                 // 64-column panels of a tile
  static constexpr uint32_t kTile = P * kTile128;          // Q, K or V: 128 rows
  static constexpr uint32_t kStage = 2 * kTile;            // K, V
  static constexpr uint32_t kOffBar = kTile + kFwdStages * kStage;
  static constexpr size_t bytes = 1024 + kOffBar + 8 * (1 + 2 * kFwdStages);
  // leading byte offset of the MN-major V: the stride between its panels (a single panel leaves it unread)
  static constexpr uint32_t kLboV = P > 1 ? kTile128 : kTile64;
  static_assert(bytes <= kMaxSmem, "forward shared memory");
};

template <int DH>
struct BwdSmem {
  static constexpr int P = (DH + 63) / 64, BQ = 64;
  static constexpr int kStages = P > 1 ? 2 : 3;             // Q/dO ring; a third two-panel stage does not fit
  static constexpr uint32_t kKV = P * kTile128;            // K or V: 128 rows
  static constexpr uint32_t kQ = P * kTile64;              // Q or dO: 64 rows
  static constexpr uint32_t kStage = 2 * kQ;               // Q, dO
  static constexpr uint32_t kOffQ = 2 * kKV;               // after K, V
  static constexpr uint32_t kOffdS = kOffQ + kStages * kStage;   // [2][128 keys][64 queries] bf16
  static constexpr uint32_t kOffdQ = kOffdS + 2 * kTile128;      // [2][64 queries][DH] fp32
  static constexpr uint32_t kdQBytes = BQ * DH * 4;
  static constexpr uint32_t kOffL = kOffdQ + 2 * kdQBytes;       // [stages][64] LSE, [stages][64] D
  static constexpr uint32_t kOffBar = kOffL + kStages * 2 * BQ * 4;
  static constexpr size_t bytes = 1024 + kOffBar + 8 * (1 + 2 * kStages + 4);
  // leading byte offset of the MN-major K in dQ = dS·K (a single panel leaves it unread)
  static constexpr uint32_t kLboK = P > 1 ? kTile128 : kTile64;
  static_assert(kOffdQ % 128 == 0 && kdQBytes % 128 == 0 && kOffL % 16 == 0 && kOffBar % 8 == 0, "smem layout");
  static_assert(bytes <= kMaxSmem, "backward shared memory");
};

// =============================================================================================
// Forward
// =============================================================================================
// online-softmax step on a 64 x 128 accumulator tile: s becomes P (fp32), m / l the running maximum (exp2 domain) and
// row sum of this thread's two rows, alpha the factor the earlier O and l are scaled by
__device__ __forceinline__ void fwd_softmax(float (&s)[64], float (&m)[2], float (&l)[2], float (&alpha)[2], float sl2) {
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    float mx = -INFINITY;
#pragma unroll
    for (int j = 0; j < 16; ++j) mx = fmaxf(mx, fmaxf(s[4 * j + 2 * hr], s[4 * j + 2 * hr + 1]));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
    const float mnew = fmaxf(m[hr], mx * sl2);
    alpha[hr] = ex2_approx(m[hr] - mnew);
    m[hr] = mnew;
    float rs = 0.f;
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const float p = ex2_approx(fmaf(s[4 * j + 2 * hr + e], sl2, -mnew));
        s[4 * j + 2 * hr + e] = p;
        rs += p;
      }
    l[hr] = l[hr] * alpha[hr] + rs;
  }
}

// fp32 accumulator tile (64 x 8 NJ) -> bf16 A fragments of its NJ / 2 k-steps
template <int NJ>
__device__ __forceinline__ void pack_acc(const float* s, uint32_t* p) {
#pragma unroll
  for (int i = 0; i < 2 * NJ; ++i) p[i] = pack_bf16(s[2 * i], s[2 * i + 1]);
}

template <int DH>
__global__ void __launch_bounds__(kWgThreads, 1)
attn_wgmma_fwd_kernel(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapK,
                      const __grid_constant__ CUtensorMap mapV, const AttnArgs a) {
  using L = FwdSmem<DH>;
  constexpr int KS = (DH + 15) / 16, NO = DH;
  constexpr uint32_t kStage = L::kStage;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);   // [Q][stages x (K, V)], each P panels of 128 x 128 B
  uint64_t* q_bar = reinterpret_cast<uint64_t*>(smem + L::kOffBar);
  uint64_t* full_bar = q_bar + 1;
  uint64_t* empty_bar = full_bar + kFwdStages;
  const int wg = threadIdx.x >> 7;
  const int b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * 128;
  const int nblk = a.M / 128;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&mapQ);
    tma_prefetch_desc(&mapK);
    tma_prefetch_desc(&mapV);
    mbar_init(q_bar, 1);
    for (int i = 0; i < kFwdStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 256);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    setmaxnreg_dec<24>();
    if (threadIdx.x != 0) return;
    mbar_expect_tx(q_bar, L::kTile);
#pragma unroll
    for (int pn = 0; pn < L::P; ++pn) tma_load_4d(smem + pn * kTile128, &mapQ, q_bar, 64 * pn, h, q0, b);
    int s = 0;
    uint32_t ph = 0;
    for (int j = 0; j < nblk; ++j) {
      mbar_wait(&empty_bar[s], ph ^ 1u);
      uint8_t* sK = smem + L::kTile + s * kStage;
      mbar_expect_tx(&full_bar[s], kStage);
#pragma unroll
      for (int pn = 0; pn < L::P; ++pn) {
        tma_load_4d(sK + pn * kTile128, &mapK, &full_bar[s], 64 * pn, h, j * 128, b);
        tma_load_4d(sK + L::kTile + pn * kTile128, &mapV, &full_bar[s], 64 * pn, h, j * 128, b);
      }
      if (++s == kFwdStages) {
        s = 0;
        ph ^= 1u;
      }
    }
    return;
  }

  setmaxnreg_inc<240>();
  const int cw = wg - 1;   // query rows [64 cw, 64 cw + 64) of the tile
  const int lane = threadIdx.x & 31, warp = (threadIdx.x >> 5) & 3;
  const uint32_t s0 = smem_u32(smem);
  const uint64_t descQ = wgmma_desc(s0 + kTile64 * cw, 16, 1024);
  const uint64_t descK = wgmma_desc(s0 + L::kTile, 16, 1024);
  const uint64_t descV = wgmma_desc(s0 + 2 * L::kTile, L::kLboV, 1024);   // MN-major: a k-step is 16 rows of 128 B
  const float sl2 = a.scale * kLog2e;
  float s[64], o[NO / 2];
  uint32_t p[32];
  float m_r[2] = {-INFINITY, -INFINITY}, l_r[2] = {0.f, 0.f}, alpha[2];
#pragma unroll
  for (int i = 0; i < NO / 2; ++i) o[i] = 0.f;

  auto issue_qk = [&](int st) {
    const uint64_t dk = descK + (uint64_t)(st * (kStage >> 4));
#pragma unroll
    for (int k = 0; k < KS; ++k) Wgmma<128, 0, 0>::mma(s, descQ + kstep(k, kTile128), dk + kstep(k, kTile128), k > 0);
    wgmma_commit();
  };

  mbar_wait(q_bar, 0);
  mbar_wait(&full_bar[0], 0);
  wgmma_fence();
  issue_qk(0);
  wgmma_wait<0>();
  reg_fence<64>(s);
  fwd_softmax(s, m_r, l_r, alpha, sl2);
  pack_acc<16>(s, p);

  auto issue_pv = [&](int st) {
    const uint64_t dv = descV + (uint64_t)(st * (kStage >> 4));
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) WgmmaRS<NO, 1>::mma(o, p + 4 * kk, dv + (uint64_t)(kk * (2048 >> 4)), 1);
    wgmma_commit();
  };
  int st = 0;
  uint32_t ph = 0;
  for (int j = 0; j + 1 < nblk; ++j) {
    int sn = st + 1;
    uint32_t phn = ph;
    if (sn == kFwdStages) {
      sn = 0;
      phn ^= 1u;
    }
    mbar_wait(&full_bar[sn], phn);
    reg_fence<64>(s);
    reg_fence<NO / 2>(o);
    reg_fence_u32<32>(p);
    wgmma_fence();
    issue_qk(sn);
    issue_pv(st);
    wgmma_wait<1>();   // S of block j + 1; P·V of block j may still run under its softmax
    reg_fence<64>(s);
    fwd_softmax(s, m_r, l_r, alpha, sl2);
    wgmma_wait<0>();
    reg_fence<NO / 2>(o);
    reg_fence_u32<32>(p);
    mbar_arrive(&empty_bar[st]);
#pragma unroll
    for (int i = 0; i < NO / 8; ++i) {
      o[4 * i] *= alpha[0];
      o[4 * i + 1] *= alpha[0];
      o[4 * i + 2] *= alpha[1];
      o[4 * i + 3] *= alpha[1];
    }
    pack_acc<16>(s, p);
    st = sn;
    ph = phn;
  }
  reg_fence<NO / 2>(o);
  reg_fence_u32<32>(p);
  wgmma_fence();
  issue_pv(st);
  wgmma_wait<0>();
  reg_fence<NO / 2>(o);
  reg_fence_u32<32>(p);

#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    float l = l_r[hr];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const int row = q0 + 64 * cw + 16 * warp + (lane >> 2) + 8 * hr;
    const float inv = 1.f / l;
    bf16* orow = a.O + b * a.o_bs + (long long)row * a.ldo + h * DH;
#pragma unroll
    for (int dt = 0; dt < DH / 8; ++dt)
      *reinterpret_cast<uint32_t*>(orow + dt * 8 + 2 * (lane & 3)) =
          pack_bf16(o[4 * dt + 2 * hr] * inv, o[4 * dt + 2 * hr + 1] * inv);
    if ((lane & 3) == 0) a.LSE[((long long)b * a.H + h) * a.N + row] = (m_r[hr] + log2f(l)) * (1.f / kLog2e);
  }
}

// =============================================================================================
// Backward (single pass)
// =============================================================================================
template <int DH>
__global__ void __launch_bounds__(kWgThreads, 1)
attn_wgmma_bwd_kernel(const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapK,
                      const __grid_constant__ CUtensorMap mapV, const __grid_constant__ CUtensorMap mapdO,
                      const __grid_constant__ CUtensorMap mapdQ, const AttnArgs a) {
  using L = BwdSmem<DH>;
  constexpr int KS = (DH + 15) / 16, NO = DH, BQ = L::BQ, kBwdStages = L::kStages;
  constexpr uint32_t kStage = L::kStage, kOffQ = L::kOffQ, kOffdS = L::kOffdS, kOffdQ = L::kOffdQ;
  constexpr uint32_t kdQBytes = L::kdQBytes, kOffL = L::kOffL, kOffBar = L::kOffBar;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = align1024(smem_raw);
  float* sL = reinterpret_cast<float*>(smem + kOffL);
  uint64_t* kv_bar = reinterpret_cast<uint64_t*>(smem + kOffBar);
  uint64_t* full_bar = kv_bar + 1;
  uint64_t* empty_bar = full_bar + kBwdStages;
  uint64_t* ds_full = empty_bar + kBwdStages;   // [2] dSᵀ of a block stored by both key warpgroups
  uint64_t* ds_empty = ds_full + 2;             // [2] dQ product of that block retired
  const int wg = threadIdx.x >> 7;
  const int b = blockIdx.z, h = blockIdx.y, k0 = blockIdx.x * 128;
  const int lane = threadIdx.x & 31, warp = (threadIdx.x >> 5) & 3;
  const int nq = a.N / BQ;
  const long long bh = (long long)b * a.H + h;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&mapQ);
    tma_prefetch_desc(&mapK);
    tma_prefetch_desc(&mapV);
    tma_prefetch_desc(&mapdO);
    tma_prefetch_desc(&mapdQ);
    mbar_init(kv_bar, 1);
    for (int i = 0; i < kBwdStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 256);
    }
    for (int i = 0; i < 2; ++i) {
      mbar_init(&ds_full[i], 256);
      mbar_init(&ds_empty[i], 128);
    }
    fence_mbar_init();
  }
  __syncthreads();
  const uint32_t s0 = smem_u32(smem);

  if (wg == 0) {
    // ===================== loads, and dQ_block = dS·K reduced into dQacc ========================================
    setmaxnreg_dec<72>();
    auto load_block = [&](int i) {   // thread 0: Q, dO, LSE, D of query block i into slot i % stages
      const int s = i % kBwdStages;
      mbar_wait(&empty_bar[s], ((uint32_t)(i / kBwdStages) & 1u) ^ 1u);
      uint8_t* sQ = smem + kOffQ + s * kStage;
      mbar_expect_tx(&full_bar[s], kStage + 2 * BQ * 4);
#pragma unroll
      for (int pn = 0; pn < L::P; ++pn) {
        tma_load_4d(sQ + pn * kTile64, &mapQ, &full_bar[s], 64 * pn, h, i * BQ, b);
        tma_load_4d(sQ + L::kQ + pn * kTile64, &mapdO, &full_bar[s], 64 * pn, h, i * BQ, b);
      }
      bulk_load_1d(sL + s * 2 * BQ, a.LSE + bh * a.N + i * BQ, BQ * 4, &full_bar[s]);
      bulk_load_1d(sL + s * 2 * BQ + BQ, a.Dv + bh * a.N + i * BQ, BQ * 4, &full_bar[s]);
    };
    if (threadIdx.x == 0) {
      mbar_expect_tx(kv_bar, 2 * L::kKV);
#pragma unroll
      for (int pn = 0; pn < L::P; ++pn) {
        tma_load_4d(smem + pn * kTile128, &mapK, kv_bar, 64 * pn, h, k0, b);
        tma_load_4d(smem + L::kKV + pn * kTile128, &mapV, kv_bar, 64 * pn, h, k0, b);
      }
      for (int i = 0; i < kBwdStages - 1 && i < nq; ++i) load_block(i);
    }
    __syncwarp();
    const uint64_t descS = wgmma_desc(s0 + kOffdS, kTile64, 1024);   // A, MN-major: rows are keys, 64 queries wide
    const uint64_t descK = wgmma_desc(s0, L::kLboK, 1024);           // B, MN-major: rows are keys, head dim wide
    mbar_wait(kv_bar, 0);
    float dq[NO / 2];
    for (int i = 0; i < nq; ++i) {
      const int buf = i & 1;
      if (threadIdx.x == 0 && i + kBwdStages - 1 < nq) load_block(i + kBwdStages - 1);
      __syncwarp();
      mbar_wait(&ds_full[buf], (uint32_t)(i >> 1) & 1u);
      const uint64_t da = descS + (uint64_t)(buf * (kTile128 >> 4));
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 8; ++kk)
        Wgmma<NO, 1, 1>::mma(dq, da + (uint64_t)(kk * (2048 >> 4)), descK + (uint64_t)(kk * (2048 >> 4)), kk > 0);
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence<NO / 2>(dq);
      mbar_arrive(&ds_empty[buf]);
      // the reduce that read this staging buffer two blocks ago has finished reading it
      if (threadIdx.x == 0) tma_store_wait_read<1>();
      named_bar_sync(1, 128);
      float* stg = reinterpret_cast<float*>(smem + kOffdQ + buf * kdQBytes);
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        float* row = stg + (16 * warp + (lane >> 2) + 8 * hr) * DH + 2 * (lane & 3);
#pragma unroll
        for (int dt = 0; dt < DH / 8; ++dt)
          *reinterpret_cast<float2*>(row + 8 * dt) =
              make_float2(dq[4 * dt + 2 * hr] * a.scale, dq[4 * dt + 2 * hr + 1] * a.scale);
      }
      fence_proxy_async_smem();
      named_bar_sync(1, 128);
      if (threadIdx.x == 0) {
        tma_reduce_add_3d(&mapdQ, stg, h * DH, i * BQ, b);
        tma_store_commit();
      }
    }
    if (threadIdx.x == 0) tma_store_wait_all();
    return;
  }

  // ===================== warpgroup cw owns keys [k0 + 64 cw, k0 + 64 cw + 64) ===================================
  setmaxnreg_inc<216>();
  const int cw = wg - 1;
  const uint64_t descKa = wgmma_desc(s0 + kTile64 * cw, 16, 1024);              // A of Sᵀ: this warpgroup's K rows
  const uint64_t descVa = wgmma_desc(s0 + L::kKV + kTile64 * cw, 16, 1024);     // A of dPᵀ
  const uint64_t descQk = wgmma_desc(s0 + kOffQ, 16, 1024);                     // B of Sᵀ (K-major Q block)
  const uint64_t descQm = wgmma_desc(s0 + kOffQ, kTile64, 1024);                // B of dK (the same tile, MN-major)
  const float sl2 = a.scale * kLog2e;
  float st[32], dpt[32], dk[NO / 2], dv[NO / 2];
  uint32_t pp[16], ps[16];
#pragma unroll
  for (int i = 0; i < NO / 2; ++i) dk[i] = dv[i] = 0.f;
  const int r0 = 64 * cw + 16 * warp + (lane >> 2);   // this thread's key rows of the CTA tile: r0, r0 + 8
  mbar_wait(kv_bar, 0);
  for (int i = 0; i < nq; ++i) {
    const int s = i % kBwdStages, buf = i & 1;
    mbar_wait(&full_bar[s], (uint32_t)(i / kBwdStages) & 1u);
    const uint64_t so = (uint64_t)(s * (kStage >> 4));
    reg_fence<32>(st);
    reg_fence<32>(dpt);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < KS; ++k)
      Wgmma<64, 0, 0>::mma(st, descKa + kstep(k, kTile128), descQk + so + kstep(k, kTile64), k > 0);
    wgmma_commit();
#pragma unroll
    for (int k = 0; k < KS; ++k)
      Wgmma<64, 0, 0>::mma(dpt, descVa + kstep(k, kTile128), descQk + so + (L::kQ >> 4) + kstep(k, kTile64), k > 0);
    wgmma_commit();
    const float* l_s = sL + s * 2 * BQ + 2 * (lane & 3);
    wgmma_wait<1>();   // Sᵀ; the exponentials run under dPᵀ
    reg_fence<32>(st);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float2 l = *reinterpret_cast<const float2*>(l_s + 8 * j);
      const float l0 = l.x * kLog2e, l1 = l.y * kLog2e;
      st[4 * j] = ex2_approx(fmaf(st[4 * j], sl2, -l0));
      st[4 * j + 1] = ex2_approx(fmaf(st[4 * j + 1], sl2, -l1));
      st[4 * j + 2] = ex2_approx(fmaf(st[4 * j + 2], sl2, -l0));
      st[4 * j + 3] = ex2_approx(fmaf(st[4 * j + 3], sl2, -l1));
    }
    pack_acc<8>(st, pp);
    wgmma_wait<0>();
    reg_fence<32>(dpt);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float2 d = *reinterpret_cast<const float2*>(l_s + BQ + 8 * j);
      dpt[4 * j] = st[4 * j] * (dpt[4 * j] - d.x);
      dpt[4 * j + 1] = st[4 * j + 1] * (dpt[4 * j + 1] - d.y);
      dpt[4 * j + 2] = st[4 * j + 2] * (dpt[4 * j + 2] - d.x);
      dpt[4 * j + 3] = st[4 * j + 3] * (dpt[4 * j + 3] - d.y);
    }
    pack_acc<8>(dpt, ps);
    // dSᵀ rows of this warpgroup -> shared memory (swizzled rows of 64 queries) for the dQ product
    mbar_wait(&ds_empty[buf], ((uint32_t)(i >> 1) & 1u) ^ 1u);
    uint8_t* sdS = smem + kOffdS + buf * kTile128;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      *reinterpret_cast<uint32_t*>(sdS + sw128_off(r0, j) + 4 * (lane & 3)) = ps[2 * j];
      *reinterpret_cast<uint32_t*>(sdS + sw128_off(r0 + 8, j) + 4 * (lane & 3)) = ps[2 * j + 1];
    }
    fence_proxy_async_smem();
    mbar_arrive(&ds_full[buf]);
    reg_fence<NO / 2>(dk);
    reg_fence<NO / 2>(dv);
    wgmma_fence();
#pragma unroll
    for (int kq = 0; kq < 4; ++kq)
      WgmmaRS<NO, 1>::mma(dv, pp + 4 * kq, descQm + so + (uint64_t)((L::kQ >> 4) + kq * (2048 >> 4)), 1);
#pragma unroll
    for (int kq = 0; kq < 4; ++kq) WgmmaRS<NO, 1>::mma(dk, ps + 4 * kq, descQm + so + (uint64_t)(kq * (2048 >> 4)), 1);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence<NO / 2>(dk);
    reg_fence<NO / 2>(dv);
    reg_fence_u32<16>(pp);
    reg_fence_u32<16>(ps);
    mbar_arrive(&empty_bar[s]);
  }
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int key = k0 + r0 + 8 * hr;
    bf16* dkr = a.dK + b * a.dk_bs + (long long)key * a.lddk + h * DH + 2 * (lane & 3);
    bf16* dvr = a.dV + b * a.dv_bs + (long long)key * a.lddv + h * DH + 2 * (lane & 3);
#pragma unroll
    for (int dt = 0; dt < DH / 8; ++dt) {
      *reinterpret_cast<uint32_t*>(dkr + 8 * dt) = pack_bf16(dk[4 * dt + 2 * hr] * a.scale, dk[4 * dt + 2 * hr + 1] * a.scale);
      *reinterpret_cast<uint32_t*>(dvr + 8 * dt) = pack_bf16(dv[4 * dt + 2 * hr], dv[4 * dt + 2 * hr + 1]);
    }
  }
}

// =============================================================================================
// Host
// =============================================================================================
bool attn_wgmma_shape_ok(int B, int H, int N, int M, int dh) {
  if (!(dh == 40 || dh == 64 || dh == 80) || N < 512 || M < 512 || N % 128 != 0 || M % 128 != 0) return false;
  if (dh == 40) return true;
  // dh = 80: the wgmma kernels measured faster than mma.sync at every grid down to 64 CTAs (level 1 at B = 1), so the
  // boundary is not a speed one: grids below half the SM count (that one included, on 132 SMs) keep the mma.sync
  // kernels, and with them a level-1 shape on which those kernels stay checked against the switch.
  // dh = 64 takes the same rule: the wgmma kernels measured faster at every SD 2.x grid down to its smallest, 80 CTAs
  // (level 1 at 512², B = 1: forward 1.6x, backward 2.4x on an H100 SXM at 700 W; DESIGN.md §5), and every SD 2.x
  // UNet self-attention of 512 tokens or more has at least that grid, so only smaller grids stay on mma.sync
  int sms = 0, dev = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (sms <= 0) sms = 132;
  return 2LL * (N / 128) * H * B >= sms;
}

// TMA needs 16-byte aligned bases and strides; the library's callers always pass them, a caller that does not gets
// an error instead of a wrong answer
static int head_map(CUtensorMap* m, const bf16* p, const AttnArgs& a, int tokens, long long ld, long long bs, int rows) {
  E4T_CHECK(((uintptr_t)p & 15) == 0 && ld % 8 == 0 && bs % 8 == 0,
            "attention (wgmma): tensors must be 16-byte aligned with strides that are multiples of 8 elements");
  const uint64_t dims[4] = {(uint64_t)a.dh, (uint64_t)a.H, (uint64_t)tokens, (uint64_t)a.B};
  const uint64_t str[3] = {(uint64_t)a.dh * 2, (uint64_t)ld * 2, (uint64_t)bs * 2};
  const uint32_t box[4] = {64, 1, (uint32_t)rows, 1};
  return e4t_tmap_encode(m, p, 4, dims, str, box, 2);
}

int attn_wgmma_fwd(const AttnArgs& a, cudaStream_t st) {
  CUtensorMap mQ, mK, mV;
  if (int e = head_map(&mQ, a.Q, a, a.N, a.ldq, a.q_bs, 128)) return e;
  if (int e = head_map(&mK, a.K, a, a.M, a.ldk, a.k_bs, 128)) return e;
  if (int e = head_map(&mV, a.V, a, a.M, a.ldv, a.v_bs, 128)) return e;
  E4T_CHECK(a.ldo % 2 == 0 && a.o_bs % 2 == 0, "attention (wgmma): output strides must be even");
  const size_t smem = a.dh == 40 ? FwdSmem<40>::bytes : a.dh == 64 ? FwdSmem<64>::bytes : FwdSmem<80>::bytes;
  auto kernel = a.dh == 40   ? attn_wgmma_fwd_kernel<40>
                : a.dh == 64 ? attn_wgmma_fwd_kernel<64>
                             : attn_wgmma_fwd_kernel<80>;
  E4T_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kernel<<<dim3(a.N / 128, a.H, a.B), kWgThreads, smem, st>>>(mQ, mK, mV, a);
  E4T_COUNT_LAUNCH();
  E4T_LAUNCH_CHECK();
  return 0;
}

int attn_wgmma_bwd(const AttnArgs& a, cudaStream_t st) {
  CUtensorMap mQ, mK, mV, mdO, mdQ;
  if (int e = head_map(&mQ, a.Q, a, a.N, a.ldq, a.q_bs, 64)) return e;
  if (int e = head_map(&mK, a.K, a, a.M, a.ldk, a.k_bs, 128)) return e;
  if (int e = head_map(&mV, a.V, a, a.M, a.ldv, a.v_bs, 128)) return e;
  if (int e = head_map(&mdO, a.dO, a, a.N, a.lddo, a.do_bs, 64)) return e;
  {
    const uint64_t C = (uint64_t)a.H * a.dh;
    const uint64_t dims[3] = {C, (uint64_t)a.N, (uint64_t)a.B};
    const uint64_t str[2] = {C * 4, (uint64_t)a.N * C * 4};
    const uint32_t box[3] = {(uint32_t)a.dh, 64, 1};
    E4T_CHECK(((uintptr_t)a.dQacc & 15) == 0 && ((uintptr_t)a.LSE & 15) == 0 && ((uintptr_t)a.Dv & 15) == 0,
              "attention (wgmma): LSE, D and dQ scratch must be 16-byte aligned");
    if (int e = e4t_tmap_encode(&mdQ, a.dQacc, 3, dims, str, box, 4, 0)) return e;
  }
  E4T_CHECK(a.lddk % 2 == 0 && a.dk_bs % 2 == 0 && a.lddv % 2 == 0 && a.dv_bs % 2 == 0,
            "attention (wgmma): gradient strides must be even");
  const size_t smem = a.dh == 40 ? BwdSmem<40>::bytes : a.dh == 64 ? BwdSmem<64>::bytes : BwdSmem<80>::bytes;
  auto kernel = a.dh == 40   ? attn_wgmma_bwd_kernel<40>
                : a.dh == 64 ? attn_wgmma_bwd_kernel<64>
                             : attn_wgmma_bwd_kernel<80>;
  E4T_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kernel<<<dim3(a.M / 128, a.H, a.B), kWgThreads, smem, st>>>(mQ, mK, mV, mdO, mdQ, a);
  E4T_COUNT_LAUNCH();
  E4T_LAUNCH_CHECK();
  return 0;
}
