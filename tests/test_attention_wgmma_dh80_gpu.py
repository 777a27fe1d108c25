"""The warpgroup (wgmma) self-attention kernels at dh = 80 (the level-1 self-attention of the SD-v1.4 UNet, 1024 tokens,
8 heads of 80): against the mma.sync kernels (E4T_ATTN_WGMMA=0) and an fp32 torch reference, on column slices of fused
buffers, with sinks at every key-block edge, at the grid-size boundary of the dispatch and under CUDA graph replay.

A head slice of 80 bf16 takes two 64-column TMA panels whose second one reaches columns 80..127 of the box, so the
inputs are slices of one fused buffer and the gradients are written into a NaN-filled buffer with guard columns: a read
of a neighbouring head or a write past the slice shows up as a wrong or NaN value."""
import os

import pytest
import torch

import test_attention_numerics_gpu as AN

pytestmark = pytest.mark.gpu

H80, DH = 8, 80
C = H80 * DH


@pytest.fixture(autouse=True)
def _clean_env():
    os.environ.pop("E4T_ATTN_WGMMA", None)
    yield
    os.environ.pop("E4T_ATTN_WGMMA", None)


def _rel(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / (b.norm() + 1e-12)).item()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _inputs(B, H, N, seed):
    """q, k, v as column slices of one fused (B, N, 3C) projection"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    c = H * DH
    qkv = (torch.randn(B, N, 3 * c, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
    do = (torch.randn(B, N, c, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
    return qkv[..., :c], qkv[..., c:2 * c], qkv[..., 2 * c:], do


GUARD = 8


def _run(q, k, v, do, H):
    """dq / dk / dv go into column slices of one NaN-filled (B, N, 3C + 4 GUARD) buffer, GUARD columns before, between
    and after them; returns o, lse, the three gradients and the guard columns"""
    from e4t_b200 import ops
    B, N, c = q.shape
    buf = torch.full((B, N, 3 * c + 4 * GUARD), float("nan"), device="cuda", dtype=torch.bfloat16)
    sl = [slice(GUARD + i * (c + GUARD), GUARD + i * (c + GUARD) + c) for i in range(3)]
    o, lse = ops.attn_fwd(q, k, v, H)
    ops.attn_bwd(q, k, v, o, do, lse, H, dq=buf[..., sl[0]], dk=buf[..., sl[1]], dv=buf[..., sl[2]])
    torch.cuda.synchronize()
    guard = torch.cat([buf[..., :GUARD]] + [buf[..., s.stop:s.stop + GUARD] for s in sl], -1)
    return o, lse, [buf[..., s] for s in sl], guard


def _reference(q, k, v, do, H):
    B, N, c = q.shape
    dh = c // H
    qh, kh, vh = (t.float().view(B, N, H, dh).transpose(1, 2).detach().requires_grad_() for t in (q, k, v))
    s = (qh @ kh.transpose(-1, -2)) * dh ** -0.5
    o = (s.softmax(-1) @ vh).transpose(1, 2).reshape(B, N, c)
    o.backward(do.float())
    grads = [t.grad.transpose(1, 2).reshape(B, N, c) for t in (qh, kh, vh)]
    return o.detach(), torch.logsumexp(s.detach(), -1), grads


@pytest.mark.parametrize("B,N", [(4, 1024), (16, 1024), (8, 512), (3, 1152)])
def test_dh80_wgmma_matches_mma_sync_and_fp32_reference(B, N):
    assert 2 * (N // 128) * H80 * B >= _sms(), "the shape must lie above the dispatch threshold"
    q, k, v, do = _inputs(B, H80, N, N + DH)
    o1, lse1, g1, guard1 = _run(q, k, v, do, H80)
    os.environ["E4T_ATTN_WGMMA"] = "0"
    o0, lse0, g0, _ = _run(q, k, v, do, H80)
    assert not torch.equal(o1, o0), "both runs took the same kernel"
    assert guard1.isnan().all(), "a gradient was written past its column slice"
    assert _rel(o1, o0) < 2e-3 and (lse1 - lse0).abs().max().item() < 1e-4
    for name, a, b in zip(("dq", "dk", "dv"), g1, g0):
        assert torch.isfinite(a.float()).all(), name
        assert _rel(a, b) < 2e-3, name
    oref, lse_ref, gref = _reference(q, k, v, do, H80)
    assert _rel(o1, oref) < 6e-3 and (lse1 - lse_ref).abs().max().item() < 1e-3
    for name, a, r in zip(("dq", "dk", "dv"), g1, gref):
        assert _rel(a, r) < 1e-2, name


def test_dh80_sink_at_every_128_key_block_edge():
    """A sink key at every 128-key block edge of the wgmma kernels (and key 0, M - 1) at the level-1 shape."""
    B, N = 4, 1024
    sinks, npl = AN._sinks_for(B, H80, N, 128)
    assert B * H80 >= npl
    failures = AN.run_case("self 1024 dh80 wgmma, 128-key blocks", B, N, N, H80, DH, sinks=sinks, seed=N + 128)
    assert not failures, "\n".join(failures)


def test_dh80_decoy_past_the_last_key():
    """Every image's key 0 is a shared-direction sink, so a read one key past M (image b + 1's key 0) doubles its
    weight in image b's peaked rows."""
    B, N = 3, 1024
    failures = AN.run_case("decoy 1024 dh80", B, N, N, H80, DH, sinks=[0] * (B * H80), shared_dir=True, delta=48.0,
                           seed=N + 5)
    assert not failures, "\n".join(failures)


@pytest.mark.parametrize("side", ["below", "at"])
def test_dh80_dispatch_boundary(side):
    """dh = 80 grids of fewer 128-query CTAs than half the SM count keep the mma.sync kernels (bit-identical O, LSE,
    dK, dV under the switch); a grid of half the SM count takes the wgmma kernels."""
    half = (_sms() + 1) // 2
    tiles = half - 1 if side == "below" else half
    B, H, N = 1, 1, 128 * tiles
    q, k, v, do = _inputs(B, H, N, tiles)
    o1, lse1, g1, _ = _run(q, k, v, do, H)
    os.environ["E4T_ATTN_WGMMA"] = "0"
    o0, lse0, g0, _ = _run(q, k, v, do, H)
    if side == "below":
        assert torch.equal(o1, o0) and torch.equal(lse1, lse0)
        assert torch.equal(g1[1], g0[1]) and torch.equal(g1[2], g0[2])
        assert _rel(g1[0], g0[0]) < 2e-3
    else:
        assert not torch.equal(o1, o0), "a grid of half the SM count still took the mma.sync kernel"
        assert _rel(o1, o0) < 2e-3
        for name, a, b in zip(("dq", "dk", "dv"), g1, g0):
            assert _rel(a, b) < 2e-3, name


def test_dh80_graph_replay_matches_eager():
    """Forward and backward at B = 16, level 1, captured in one CUDA graph and replayed.  dQ is an fp32 bulk-reduce
    sum whose order varies between runs, so the comparison is against the 2e-3 bound, not bitwise."""
    from e4t_b200 import ops
    B, N = 16, 1024
    q, k, v, do = _inputs(B, H80, N, 7)
    o_e, lse_e, g_e, _ = _run(q, k, v, do, H80)
    grads = torch.empty((B, N, 3 * C), device="cuda", dtype=torch.bfloat16)

    def step():
        o, lse = ops.attn_fwd(q, k, v, H80)
        ops.attn_bwd(q, k, v, o, do, lse, H80, dq=grads[..., :C], dk=grads[..., C:2 * C], dv=grads[..., 2 * C:])
        return o, lse

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        o_g, lse_g = step()
    grads.fill_(float("nan"))
    graph.replay()
    torch.cuda.synchronize()
    assert _rel(o_g, o_e) < 2e-3 and (lse_g - lse_e).abs().max().item() < 1e-4
    for i, (name, ref) in enumerate(zip(("dq", "dk", "dv"), g_e)):
        got = grads[..., i * C:(i + 1) * C]
        assert torch.isfinite(got.float()).all(), name
        assert _rel(got, ref) < 2e-3, name
