"""Token merging (ToMe) without a GPU: the fp64 oracle against a brute-force per-token restatement, the block
selection tables of SD 1.x / SD 2.x, the odd-batch rule and apply_patch's argument checks."""
import math

import pytest
import torch

from oracle import e4t_oracle as O
from oracle import tome_oracle as T


def _brute(x, h, w, r, sy, sx, pattern):
    """Per-token loops over the rules: dst per cell, best dst by cosine (first maximum in raster order), merged = the
    r largest node_max (ties to the lower raster index), merge = mean, unmerge = representative's row."""
    B, N, C = x.shape
    dst = set()
    for cy in range(h // sy):
        for cx in range(w // sx):
            k = int(pattern[cy, cx])
            dst.add((cy * sy + k // sx) * w + cx * sx + k % sx)
    dst_l = sorted(dst)
    src_l = [t for t in range(N) if t not in dst]
    plans = []
    for b in range(B):
        xb = x[b].double()
        unit = [xb[t] / max(xb[t].norm().item(), 1e-12) for t in range(N)]
        best = {}
        for i in src_l:
            bv, bj = -math.inf, None
            for j in dst_l:
                v = float(unit[i] @ unit[j])
                if v > bv:
                    bv, bj = v, j
            best[i] = (bv, bj)
        ranked = sorted(src_l, key=lambda i: (-best[i][0], i))
        merged = set(ranked[:r])
        kept = [t for t in range(N) if t not in merged]
        row = {t: p for p, t in enumerate(kept)}
        pos = [row[t] if t in row else row[best[t][1]] for t in range(N)]
        y = torch.zeros(len(kept), C, dtype=torch.float64)
        cnt = [0] * len(kept)
        for t in range(N):
            y[pos[t]] += xb[t]
            cnt[pos[t]] += 1
        y /= torch.tensor(cnt, dtype=torch.float64)[:, None]
        plans.append(dict(pos=torch.tensor(pos), merged_y=y, node_max=torch.tensor([best[i][0] for i in src_l], dtype=torch.float64),
                          node_idx=torch.tensor([best[i][1] for i in src_l])))
    return plans


@pytest.mark.parametrize("B,h,w,C,sy,sx,ratio", [(2, 8, 8, 16, 2, 2, 0.5), (3, 7, 9, 8, 2, 2, 0.3),
                                                 (2, 6, 6, 8, 1, 2, 0.4), (1, 5, 6, 12, 3, 2, 0.6)])
def test_oracle_matches_brute_force(B, h, w, C, sy, sx, ratio):
    g = torch.Generator().manual_seed(h * 100 + w)
    x = torch.randn(B, h * w, C, generator=g, dtype=torch.float64)    # continuous: no ties
    pattern = torch.randint(0, sy * sx, (h // sy, w // sx), generator=g)
    n_dst = (h // sy) * (w // sx)
    r = min(int(h * w * ratio), h * w - n_dst)
    p = T.make_plan(x, h, w, r, sy, sx, pattern)
    ref = _brute(x, h, w, r, sy, sx, pattern)
    y = T.merge(x, p)
    for b in range(B):
        assert torch.equal(p["pos"][b], ref[b]["pos"])
        assert torch.equal(p["node_idx"][b], ref[b]["node_idx"])
        torch.testing.assert_close(p["node_max"][b], ref[b]["node_max"], rtol=0, atol=1e-12)
        torch.testing.assert_close(y[b], ref[b]["merged_y"], rtol=0, atol=1e-12)
        # CSR rows: members ascending, each row's members are exactly the tokens with that pos
        ro, mem = p["row_off"][b], p["members"][b]
        for q in range(p["w"].shape[1]):
            ms = mem[ro[q]:ro[q + 1]]
            assert torch.equal(ms, torch.nonzero(p["pos"][b] == q).reshape(-1))
            assert p["w"][b, q] == 1.0 / len(ms)
    res = torch.randn(B, h * w, C, generator=g, dtype=torch.float64)
    out = T.unmerge(y, p, res)
    for b in range(B):
        torch.testing.assert_close(out[b], ref[b]["merged_y"][ref[b]["pos"]] + res[b], rtol=0, atol=1e-12)


def test_tie_rules():
    # every token equal: every cosine is 1; best dst = the first dst, merged = the r lowest src raster indices
    x = torch.ones(1, 16, 8, dtype=torch.float64)
    p = T.make_plan(x, 4, 4, 5, 2, 2)
    src = p["src_idx"]
    assert torch.equal(p["node_idx"][0], torch.full_like(src, int(p["dst_idx"][0])))
    assert torch.equal(torch.nonzero(p["merged"][0]).reshape(-1), torch.arange(5))


# ---- block selection, grid and r ---------------------------------------------------------------------------------
def _levels(cfg, H0, W0):
    """(N, H, W) of each UNet level's transformer blocks (the down-sampling convs round up)."""
    out, H, W = [], H0, W0
    for i in range(len(cfg["block_out_channels"]) - 1):
        out.append((H * W, H, W))
        H, W = (H + 1) // 2, (W + 1) // 2
    out.append((H * W, H, W))   # mid block
    return out


SD2 = dict(O.SD14_UNET, attention_head_dim=(5, 10, 20, 20), cross_attention_dim=1024)


@pytest.mark.parametrize("cfg", [O.SD14_UNET, SD2], ids=["sd1", "sd2"])
@pytest.mark.parametrize("px", [(512, 512), (768, 768), (520, 520), (520, 776), (776, 520)])
def test_block_selection_tables(cfg, px):
    H0, W0 = px[0] // 8, px[1] // 8
    table = []
    for md in (1, 2, 4, 8):
        for N, H, W in _levels(cfg, H0, W0):
            geo = T.block_geometry(H0, W0, N, 0.5, md, 2, 2)
            if geo is None:
                table.append((md, N, None))
                continue
            ds, h, w, r = geo
            assert (h, w) == (H, W), (md, N, geo)
            assert r == min(int(N * 0.5), N - (h // 2) * (w // 2))
            table.append((md, N, ds))
    # default max_downsample = 1: exactly the full-resolution level merges
    l0 = H0 * W0
    assert [n for md, n, ds in table if md == 1 and ds is not None] == [l0]
    # the level of downsample d merges from max_downsample = d on
    for md, n, ds in table:
        if ds is not None:
            assert ds <= md
    assert all(ds is not None for md, n, ds in table if md == 8)


def test_sd14_512_numbers():
    ds, h, w, r = T.block_geometry(64, 64, 4096, 0.5, 1, 2, 2)
    assert (ds, h, w, r) == (1, 64, 64, 2048)
    assert T.block_geometry(64, 64, 1024, 0.5, 1, 2, 2) is None
    assert T.block_geometry(64, 64, 1024, 0.5, 2, 2, 2) == (2, 32, 32, 512)
    # 96 x 96 latent (SD 2.x 768²): 9216 tokens, 6912 src, r = 4608
    assert T.block_geometry(96, 96, 9216, 0.5, 1, 2, 2) == (1, 96, 96, 4608)
    # odd sides: tail rows / columns are src; r is capped by the src count at high ratios
    assert T.block_geometry(65, 67, 65 * 67, 0.5, 1, 2, 2) == (1, 65, 67, 2177)
    assert T.block_geometry(65, 67, 65 * 67, 0.9, 1, 2, 2) == (1, 65, 67, 65 * 67 - 32 * 33)


def test_odd_batch_uses_the_zero_pattern():
    # the oracle's own plans: odd batch -> pattern zeros whatever the generator says
    recorded = []
    orig = T.make_plan

    def spy(x, h, w, r, sy=2, sx=2, pattern=None):
        recorded.append(pattern)
        return orig(x, h, w, r, sy, sx, pattern)

    T.make_plan = spy
    try:
        sd = O.synth_state_dict(O.unet_param_shapes(O.TINY_UNET), 5)
        for B in (1, 2):
            g = torch.Generator().manual_seed(0)
            x = torch.randn(B, 4, 16, 16)
            ehs = torch.randn(B, 77, O.TINY_UNET["cross_attention_dim"])
            recorded.clear()
            T.unet_forward(sd, O.TINY_UNET, x, torch.tensor([10] * B), ehs, generator=g)
            assert len(recorded) == 3          # down block 0 and the two attentions of the last up block
            if B == 1:
                assert all(p is None for p in recorded)
            else:
                assert all(p is not None and p.shape == (8, 8) for p in recorded)
    finally:
        T.make_plan = orig


def test_unpatched_oracle_is_unchanged():
    sd = O.synth_state_dict(O.unet_param_shapes(O.TINY_UNET), 5)
    x = torch.randn(1, 4, 16, 16)
    ehs = torch.randn(1, 77, O.TINY_UNET["cross_attention_dim"])
    a = O.unet_forward(sd, O.TINY_UNET, x, torch.tensor([10]), ehs)
    with T.patched((16, 16), ratio=0.0):
        b = O.unet_forward(sd, O.TINY_UNET, x, torch.tensor([10]), ehs)
    c = O.unet_forward(sd, O.TINY_UNET, x, torch.tensor([10]), ehs)
    assert torch.equal(a, b) and torch.equal(a, c)


# ---- apply_patch arguments ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [dict(ratio=1.0), dict(ratio=-0.1), dict(ratio=1.5), dict(max_downsample=3),
                                dict(max_downsample=0), dict(max_downsample=16), dict(sx=0), dict(sy=0),
                                dict(sx=1.5)])
def test_apply_patch_refuses(kw):
    from e4t.models.unet_2d_condition import UNet2DConditionModel
    from e4t_b200 import tome
    from e4t_b200._lib import E4TError
    unet = UNet2DConditionModel(**O.ref_unet_kwargs(O.TINY_UNET))
    with pytest.raises(E4TError):
        tome.apply_patch(unet, **kw)
    assert tome.signature(unet) is None


def test_apply_and_remove_patch_on_cpu_modules():
    from e4t.models.attention import BasicTransformerBlock
    from e4t.models.unet_2d_condition import UNet2DConditionModel
    from e4t_b200 import tome
    unet = UNet2DConditionModel(**O.ref_unet_kwargs(O.TINY_UNET))
    blocks = [m for m in unet.modules() if isinstance(m, BasicTransformerBlock)]
    assert tome.apply_patch(unet, ratio=0.0) is unet and tome.signature(unet) is None
    tome.apply_patch(unet, ratio=0.5)
    s1 = tome.signature(unet)
    assert s1 is not None and all(b._tome is unet._tome_info for b in blocks)
    tome.apply_patch(unet, ratio=0.25, use_rand=False)
    assert tome.signature(unet) not in (None, s1)
    tome.remove_patch(unet)
    assert tome.signature(unet) is None and all(b._tome is None for b in blocks)
    assert len(unet._forward_pre_hooks) == 0
    with pytest.raises(TypeError):
        tome.apply_patch(object())
