"""Warpgroup (wgmma) self-attention kernels (csrc/attention_wgmma.cu) against the mma.sync kernels they replace for long
non-causal self-attention (E4T_ATTN_WGMMA=0 selects those) and against an fp32 torch reference."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _clean_env():
    os.environ.pop("E4T_ATTN_WGMMA", None)
    yield
    os.environ.pop("E4T_ATTN_WGMMA", None)


def _rel(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / (b.norm() + 1e-12)).item()


def _inputs(B, H, N, dh, seed):
    """q, k, v as column slices of one fused (B, N, 3C) projection, dq / dk / dv as slices of one gradient buffer"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    C = H * dh
    qkv = (torch.randn(B, N, 3 * C, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
    do = (torch.randn(B, N, C, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
    return qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:], do


def _run(q, k, v, do, H):
    from e4t_b200 import ops
    B, N, C = q.shape
    grads = torch.full((B, N, 3 * C), float("nan"), device="cuda", dtype=torch.bfloat16)
    o, lse = ops.attn_fwd(q, k, v, H)
    ops.attn_bwd(q, k, v, o, do, lse, H, dq=grads[..., :C], dk=grads[..., C:2 * C], dv=grads[..., 2 * C:])
    torch.cuda.synchronize()
    return o, lse, grads


def _reference(q, k, v, do, H):
    B, N, C = q.shape
    dh = C // H
    qh, kh, vh = (t.float().view(B, N, H, dh).transpose(1, 2).detach().requires_grad_() for t in (q, k, v))
    s = (qh @ kh.transpose(-1, -2)) * dh ** -0.5
    o = (s.softmax(-1) @ vh).transpose(1, 2).reshape(B, N, C)
    o.backward(do.float())
    grads = torch.cat([t.grad.transpose(1, 2).reshape(B, N, C) for t in (qh, kh, vh)], -1)
    return o.detach(), torch.logsumexp(s.detach(), -1), grads


@pytest.mark.parametrize("B,H,N,dh", [(2, 8, 4096, 40), (1, 3, 512, 40), (1, 8, 1152, 40)])
def test_wgmma_attention_matches_mma_sync_and_fp32_reference(B, H, N, dh):
    q, k, v, do = _inputs(B, H, N, dh, N + dh)
    o1, lse1, g1 = _run(q, k, v, do, H)
    os.environ["E4T_ATTN_WGMMA"] = "0"
    o0, lse0, g0 = _run(q, k, v, do, H)
    assert not torch.equal(o1, o0), "both runs took the same kernel"
    C = H * dh
    assert _rel(o1, o0) < 2e-3 and (lse1 - lse0).abs().max().item() < 1e-4
    for i, name in enumerate(("dq", "dk", "dv")):
        assert _rel(g1[..., i * C:(i + 1) * C], g0[..., i * C:(i + 1) * C]) < 2e-3, name
    oref, lse_ref, gref = _reference(q, k, v, do, H)
    assert _rel(o1, oref) < 6e-3 and (lse1 - lse_ref).abs().max().item() < 1e-3
    for i, name in enumerate(("dq", "dk", "dv")):
        assert _rel(g1[..., i * C:(i + 1) * C], gref[..., i * C:(i + 1) * C]) < 1e-2, name


@pytest.mark.parametrize("B,H,N,dh", [(1, 8, 4096 - 24, 40),    # ragged last tiles
                                      (1, 8, 384, 40),          # below the length threshold
                                      (1, 8, 1024, 80), (1, 4, 512, 64)])   # other head dims
def test_shapes_outside_the_wgmma_dispatch_keep_the_mma_sync_kernels(B, H, N, dh):
    """The forward is deterministic, so O and LSE are bit-identical when the switch changes nothing; dQ goes through
    fp32 atomics in the mma.sync backward, dK / dV do not."""
    q, k, v, do = _inputs(B, H, N, dh, N + dh)
    o1, lse1, g1 = _run(q, k, v, do, H)
    os.environ["E4T_ATTN_WGMMA"] = "0"
    o0, lse0, g0 = _run(q, k, v, do, H)
    C = H * dh
    assert torch.equal(o1, o0) and torch.equal(lse1, lse0)
    assert torch.equal(g1[..., C:], g0[..., C:])
    assert _rel(g1[..., :C], g0[..., :C]) < 2e-3
