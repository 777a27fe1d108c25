// e4t — what attention.cu (mma.sync kernels, dispatch) and attention_wgmma.cu (warpgroup kernels) share.
#pragma once
#include "common.cuh"

static constexpr float kLog2e = 1.4426950408889634f;

struct AttnArgs {
  int B, H, N, M, dh;
  float scale;
  int stages, lazy, poly, p_smem;   // forward variants (attn_fwd_kernel); stages is also the Q/dO buffering of the backward
  const bf16* Q; long long ldq, q_bs;
  const bf16* K; long long ldk, k_bs;
  const bf16* V; long long ldv, v_bs;
  bf16* O; long long ldo, o_bs;
  const bf16* dO; long long lddo, do_bs;
  float* LSE;        // [B][H][N]
  const float* Dv;   // [B][H][N] rowsum(dO∘O)
  float* dQacc;      // [B][N][H*dh] fp32 (fused backward)
  bf16* dQ; long long lddq, dq_bs;
  bf16* dK; long long lddk, dk_bs;
  bf16* dV; long long lddv, dv_bs;
};

// Warpgroup (wgmma + TMA) kernels for long non-causal self-attention, csrc/attention_wgmma.cu.
// attn_wgmma_shape_ok: the shapes those kernels take (dh = 40, 64 or 80, N and M multiples of 128 and >= 512; for
// dh = 64 and 80 also a grid of (N / 128) x H x B CTAs of at least half the SM count).
bool attn_wgmma_shape_ok(int B, int H, int N, int M, int dh);
// forward: O, LSE.  backward: dK, dV, and dQ reduced into the zeroed a.dQacc (the caller converts it to bf16).
int attn_wgmma_fwd(const AttnArgs& a, cudaStream_t st);
int attn_wgmma_bwd(const AttnArgs& a, cudaStream_t st);
