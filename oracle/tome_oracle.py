"""CPU ORACLE for token merging (ToMe) — TEST INFRASTRUCTURE ONLY.

fp64 restatement of tomesd 0.1.x's bipartite_soft_matching_random2d and of its patched diffusers BasicTransformerBlock,
with the tie rules tomesd leaves open fixed as e4t_b200/tome.py documents them (best dst: lowest raster index; merged
src: larger node_max first, then lower raster index).  tomesd is not installed: **parity unpinned**, like the
diffusers pieces of e4t_oracle.py.

A plan is a dict of int64 / fp64 CPU tensors in the layout the GPU kernels write:
  pos (B, N)          merged row of each token's representative (kept tokens in raster order)
  row_off (B, N'+1)   CSR row offsets, members (B, N) members in ascending raster order, w (B, N') = 1 / row length
`unet_forward` / `patched` run e4t_oracle's UNet with merging blocks, either matching on their own inputs or replaying
plans recorded from the GPU (e4t_b200.tome.record_plans), in call order.
"""
import contextlib
import math

import torch
import torch.nn.functional as F

from oracle import e4t_oracle as O


def block_geometry(H0, W0, N, ratio, max_downsample, sx, sy):
    """(downsample, h, w, r) of a block with N tokens under an H0 x W0 latent, or None when it does not merge."""
    ds = int(math.ceil(math.sqrt((H0 * W0) // N)))
    if ds > max_downsample:
        return None
    h, w = int(math.ceil(H0 / ds)), int(math.ceil(W0 / ds))
    n_dst = (h // sy) * (w // sx)
    return ds, h, w, (min(int(N * ratio), N - n_dst) if n_dst > 0 else 0)


def partition(h, w, sy, sx, pattern):
    """(src_idx, dst_idx): raster indices of the src and dst tokens, each in raster order.  pattern (h//sy, w//sx)."""
    hc, wc = h // sy, w // sx
    is_dst = torch.zeros(h, w, dtype=torch.bool)
    if hc > 0 and wc > 0:
        cy, cx = torch.meshgrid(torch.arange(hc), torch.arange(wc), indexing="ij")
        k = pattern.to(torch.int64).cpu()
        is_dst[cy * sy + k // sx, cx * sx + k % sx] = True
    flat = is_dst.reshape(-1)
    return torch.nonzero(~flat).reshape(-1), torch.nonzero(flat).reshape(-1)


def match(x, src_idx, dst_idx):
    """node_max (B, Ns) fp64 and node_idx (B, Ns) raster index of the best dst (first maximum in raster order)."""
    xn = x.to(torch.float64)
    xn = xn / xn.norm(dim=-1, keepdim=True).clamp_min(1e-12)
    s = xn[:, src_idx] @ xn[:, dst_idx].transpose(1, 2)
    node_max, j = s.max(dim=-1)
    return node_max, dst_idx[j]


def select(node_max, src_idx, r):
    """(B, Ns) bool: the r src tokens of each image with the largest node_max, ties to the lower raster index."""
    order = torch.sort(node_max, dim=-1, descending=True, stable=True).indices   # src ranks follow raster order
    merged = torch.zeros(node_max.shape, dtype=torch.bool)
    merged.scatter_(1, order[:, :r], True)
    return merged


def build_plan(N, src_idx, node_idx, merged):
    """The GPU layout (pos, row_off, members, w) of a selection."""
    B = merged.shape[0]
    r = int(merged[0].sum())
    pos = torch.empty(B, N, dtype=torch.int64)
    members = torch.empty(B, N, dtype=torch.int64)
    row_off = torch.empty(B, N - r + 1, dtype=torch.int64)
    w = torch.empty(B, N - r, dtype=torch.float64)
    for b in range(B):
        kept = torch.ones(N, dtype=torch.bool)
        kept[src_idx[merged[b]]] = False
        pos[b, kept] = torch.arange(N - r)
        rep = torch.arange(N)
        rep[src_idx[merged[b]]] = node_idx[b][merged[b]].to(torch.int64)
        pos[b] = pos[b, rep]
        order = torch.sort(pos[b] * N + torch.arange(N)).indices      # by row, then raster index
        members[b] = order
        counts = torch.bincount(pos[b], minlength=N - r)
        row_off[b, 0] = 0
        row_off[b, 1:] = torch.cumsum(counts, 0)
        w[b] = 1.0 / counts.to(torch.float64)
    return dict(pos=pos, row_off=row_off, members=members, w=w)


def make_plan(x, h, w, r, sy=2, sx=2, pattern=None):
    """Matching and selection of one block call on x (B, h*w, C).  pattern None: all zeros (top-left dst)."""
    if pattern is None:
        pattern = torch.zeros(h // sy, w // sx, dtype=torch.int64)
    src_idx, dst_idx = partition(h, w, sy, sx, pattern)
    node_max, node_idx = match(x, src_idx, dst_idx)
    merged = select(node_max, src_idx, r)
    p = build_plan(x.shape[1], src_idx, node_idx, merged)
    p.update(src_idx=src_idx, dst_idx=dst_idx, node_max=node_max, node_idx=node_idx, merged=merged, r=r)
    return p


def as_cpu_plan(p):
    """A plan recorded from the GPU (int32 / fp32 CUDA tensors) in the oracle's layout."""
    return dict(pos=p["pos"].cpu().long(), row_off=p["row_off"].cpu().long(), members=p["members"].cpu().long(),
                w=p["w"].cpu().double(), r=int(p["r"]))


def merge(x, plan):
    """(B, N, C) -> (B, N', C): mean over each merged row's members."""
    B, N, C = x.shape
    Nm = plan["w"].shape[1]
    out = torch.stack([torch.zeros(Nm, C, dtype=x.dtype).index_add(0, plan["pos"][b], x[b]) for b in range(B)])
    return out * plan["w"].to(x.dtype)[..., None]


def unmerge(y, plan, residual):
    """(B, N', C) -> (B, N, C): y[pos i] + residual[i]."""
    return torch.stack([y[b][plan["pos"][b]] for b in range(y.shape[0])]) + residual


def transformer_block(sd, p, x, ctx, heads, plan, merge_attn=True, merge_crossattn=False, merge_mlp=False):
    """e4t_oracle.transformer_block with tomesd's patched sub-layers."""
    C = x.shape[-1]
    ln = lambda k, t: F.layer_norm(t, (C,), sd[p + k + ".weight"], sd[p + k + ".bias"], 1e-5)

    def sub(f, t, on):
        return unmerge(f(merge(t, plan)), plan, x) if on else f(t) + x

    x = sub(lambda t: O.cross_attention(sd, p + "attn1.", t, None, heads), ln("norm1", x), merge_attn)
    x = sub(lambda t: O.cross_attention(sd, p + "attn2.", t, ctx, heads), ln("norm2", x), merge_crossattn)

    def ff(t):
        u, g = F.linear(t, sd[p + "ff.net.0.proj.weight"], sd[p + "ff.net.0.proj.bias"]).chunk(2, dim=-1)
        return F.linear(u * F.gelu(g), sd[p + "ff.net.2.weight"], sd[p + "ff.net.2.bias"])

    return sub(ff, ln("norm3", x), merge_mlp)


@contextlib.contextmanager
def patched(latent_hw, ratio=0.5, max_downsample=1, sx=2, sy=2, merge_attn=True, merge_crossattn=False,
            merge_mlp=False, plans=None, generator=None, use_rand=True):
    """Within the block, e4t_oracle's UNet (and every function built on it, such as pretrain_step) merges tokens in
    the blocks the rules select.  plans: a list of recorded plans consumed in call order; None: each block matches on
    its own input, with patterns from `generator` (zeros when use_rand is False or the batch is odd)."""
    H0, W0 = latent_hw
    queue = None if plans is None else list(plans)
    orig = O.transformer_block

    def block(sd, p, x, ctx, heads):
        geo = block_geometry(H0, W0, x.shape[1], ratio, max_downsample, sx, sy)
        if geo is None or geo[3] <= 0:
            return orig(sd, p, x, ctx, heads)
        _, h, w, r = geo
        if queue is not None:
            plan = queue.pop(0)
            assert plan["r"] == r and plan["pos"].shape == (x.shape[0], x.shape[1])
        else:
            pattern = None
            if use_rand and x.shape[0] % 2 == 0:
                pattern = torch.randint(0, sy * sx, (h // sy, w // sx), generator=generator)
            plan = make_plan(x.detach(), h, w, r, sy, sx, pattern)
        return transformer_block(sd, p, x, ctx, heads, plan, merge_attn, merge_crossattn, merge_mlp)

    O.transformer_block = block
    try:
        yield queue
    finally:
        O.transformer_block = orig


def unet_forward(sd, cfg, sample, timesteps, ehs, return_encoder_outputs=False, **tome_kw):
    """e4t_oracle.unet_forward with token merging (keyword arguments of `patched`)."""
    with patched(tuple(sample.shape[-2:]), **tome_kw):
        return O.unet_forward(sd, cfg, sample, timesteps, ehs, return_encoder_outputs)
