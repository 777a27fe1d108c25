"""The warpgroup (wgmma) self-attention kernels at dh = 64, the head width of every Stable Diffusion 2.x UNet level
(level 0 at 768²: 9216 tokens, 5 heads; level 1 at 768²: 2304 tokens, 10 heads; level 0 at 512²: 4096 tokens, 5 heads):
against the mma.sync kernels (E4T_ATTN_WGMMA=0) and an fp32 torch reference, on column slices of fused buffers, with
sinks at every key-block edge, at the grid-size boundary of the dispatch and under CUDA graph replay.

A head of 64 bf16 fills its 64-column TMA panel exactly, so the box has no zero padding: the inputs are slices of one
fused buffer and the gradients are written into a NaN-filled buffer with guard columns, so a read of a neighbouring head
or a write past the slice shows up as a wrong or NaN value."""
import json
import os
import subprocess
import sys
import textwrap

import pytest
import torch

import test_attention_numerics_gpu as AN
from test_attention_wgmma_dh80_gpu import GUARD, _rel, _reference

pytestmark = pytest.mark.gpu

DH = 64


@pytest.fixture(autouse=True)
def _clean_env():
    os.environ.pop("E4T_ATTN_WGMMA", None)
    yield
    os.environ.pop("E4T_ATTN_WGMMA", None)


def _inputs(B, H, N, seed):
    """q, k, v as column slices of one fused (B, N, 3C) projection"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    c = H * DH
    qkv = (torch.randn(B, N, 3 * c, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
    do = (torch.randn(B, N, c, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
    return qkv[..., :c], qkv[..., c:2 * c], qkv[..., 2 * c:], do


def _run(q, k, v, do, H):
    """dq / dk / dv go into column slices of one NaN-filled (B, N, 3C + 4 GUARD) buffer; returns o, lse, the three
    gradients and the guard columns"""
    from e4t_b200 import ops
    B, N, c = q.shape
    buf = torch.full((B, N, 3 * c + 4 * GUARD), float("nan"), device="cuda", dtype=torch.bfloat16)
    sl = [slice(GUARD + i * (c + GUARD), GUARD + i * (c + GUARD) + c) for i in range(3)]
    o, lse = ops.attn_fwd(q, k, v, H)
    ops.attn_bwd(q, k, v, o, do, lse, H, dq=buf[..., sl[0]], dk=buf[..., sl[1]], dv=buf[..., sl[2]])
    torch.cuda.synchronize()
    guard = torch.cat([buf[..., :GUARD]] + [buf[..., s.stop:s.stop + GUARD] for s in sl], -1)
    return o, lse, [buf[..., s] for s in sl], guard


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# (2, 5, 9216): level 0 at 768²; (4, 10, 2304): level 1 at 768²; (4, 5, 4096): level 0 at 512²; (1, 10, 1024): level 1
# at 512², B = 1, the smallest SD 2.x grid (80 CTAs); (3, 2, 1536): 512 < N and an odd batch
@pytest.mark.parametrize("B,H,N", [(2, 5, 9216), (4, 10, 2304), (4, 5, 4096), (1, 10, 1024), (3, 2, 1536)])
def test_dh64_wgmma_matches_mma_sync_and_fp32_reference(B, H, N):
    assert 2 * (N // 128) * H * B >= _sms(), "the shape must lie above the dispatch threshold"
    q, k, v, do = _inputs(B, H, N, N + DH + H)
    o1, lse1, g1, guard1 = _run(q, k, v, do, H)
    os.environ["E4T_ATTN_WGMMA"] = "0"
    o0, lse0, g0, _ = _run(q, k, v, do, H)
    assert not torch.equal(o1, o0), "both runs took the same kernel"
    assert guard1.isnan().all(), "a gradient was written past its column slice"
    assert _rel(o1, o0) < 2e-3 and (lse1 - lse0).abs().max().item() < 1e-4
    for name, a, b in zip(("dq", "dk", "dv"), g1, g0):
        assert torch.isfinite(a.float()).all(), name
        assert _rel(a, b) < 2e-3, name
    oref, lse_ref, gref = _reference(q, k, v, do, H)
    assert _rel(o1, oref) < 6e-3 and (lse1 - lse_ref).abs().max().item() < 1e-3
    for name, a, r in zip(("dq", "dk", "dv"), g1, gref):
        assert _rel(a, r) < 1e-2, name


def test_dh64_sink_at_every_128_key_block_edge():
    """A sink key at every 128-key block edge of the wgmma kernels (and key 0, M - 1) at the SD 2.x level-1 768²
    shape."""
    H, N = 10, 2304
    _, npl = AN._sinks_for(1, H, N, 128)
    B = -(-npl // H)                       # enough images that every placement has a head
    sinks, _ = AN._sinks_for(B, H, N, 128)
    failures = AN.run_case("self 2304 dh64 wgmma, 128-key blocks", B, N, N, H, DH, sinks=sinks, seed=N + 128)
    assert not failures, "\n".join(failures)


@pytest.mark.parametrize("side", ["below", "at"])
def test_dh64_dispatch_boundary(side):
    """dh = 64 grids of fewer 128-query CTAs than half the SM count keep the mma.sync kernels (bit-identical O, LSE,
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


def test_dh64_graph_replay_matches_eager():
    """Forward and backward at the SD 2.x level-1 768² shape, B = 4, captured in one CUDA graph and replayed.  dQ is an
    fp32 bulk-reduce sum whose order varies between runs, so the comparison is against the 2e-3 bound, not bitwise."""
    from e4t_b200 import ops
    B, H, N = 4, 10, 2304
    C = H * DH
    q, k, v, do = _inputs(B, H, N, 7)
    o_e, lse_e, g_e, _ = _run(q, k, v, do, H)
    grads = torch.empty((B, N, 3 * C), device="cuda", dtype=torch.bfloat16)

    def step():
        o, lse = ops.attn_fwd(q, k, v, H)
        ops.attn_bwd(q, k, v, o, do, lse, H, dq=grads[..., :C], dk=grads[..., C:2 * C], dv=grads[..., 2 * C:])
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


_PROFILE = textwrap.dedent("""
    import json, sys
    import torch
    from torch.profiler import ProfilerActivity, profile
    sys.path[:0] = sys.argv[1:]
    from e4t_b200 import ops
    B, H, N, C = 1, 5, 4096, 320
    g = torch.Generator(device="cuda").manual_seed(3)
    qkv = (torch.randn(B, N, 3 * C, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
    do = (torch.randn(B, N, C, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
    q, k, v = qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:]
    def run():
        o, lse = ops.attn_fwd(q, k, v, H)
        ops.attn_bwd(q, k, v, o, do, lse, H)
        torch.cuda.synchronize()
    run()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run()
    print(json.dumps(sorted({e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA})))
""")


def test_dh64_wgmma_kernels_launch():
    """The profiler sees the <64> instantiations of both warpgroup kernels, and no mma.sync attention kernel, for the
    SD 2.x level-0 512² self-attention.  It profiles in a child process, so that the process the rest of the suite runs
    in (tests/test_gemm_exact_gpu.py reads kernel names from its own profiler sessions) never had a session of it."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else [])
    r = subprocess.run(cmd + ["-c", _PROFILE, root, os.path.join(root, "e4t-diffusion_b200")], capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    names = json.loads(r.stdout.strip().splitlines()[-1])
    assert any("attn_wgmma_fwd_kernel<64>" in n for n in names), names
    assert any("attn_wgmma_bwd_kernel<64>" in n for n in names), names
    assert not any("attn_fwd_kernel" in n or "attn_bwd_kv_kernel" in n for n in names), names
