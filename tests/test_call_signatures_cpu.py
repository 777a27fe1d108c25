"""CPU checks of the signature-replay harness in test_call_signatures_gpu.py: its fp64 references against independent
formulations, the NaN-guarded tensor layout, and the block error measure."""
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_call_signatures_gpu as H  # noqa: E402

F64 = torch.float64


def test_attention_reference_matches_sdpa_and_autograd():
    g = torch.Generator().manual_seed(0)
    B, N, M, Hh, dh = 2, 24, 24, 3, 8
    for causal in (False, True):
        q, k, v, do = (torch.randn(B, n, Hh * dh, generator=g, dtype=F64) for n in (N, M, M, N))
        scale = dh ** -0.5
        o, lse, p = H._attn_ref_fwd(q, k, v, Hh, scale, causal)
        qr, kr, vr = (t.clone().view(B, -1, Hh, dh).transpose(1, 2).requires_grad_(True) for t in (q, k, v))
        ref = F.scaled_dot_product_attention(qr, kr, vr, is_causal=causal, scale=scale)
        ref.backward(do.view(B, N, Hh, dh).transpose(1, 2))
        assert torch.allclose(o, ref.transpose(1, 2).reshape(B, N, -1), atol=1e-12)
        s = (qr.detach() @ kr.detach().transpose(-1, -2)) * scale
        if causal:
            s = s.masked_fill(torch.ones(N, M, dtype=torch.bool).triu(1), float("-inf"))
        assert torch.allclose(lse, torch.logsumexp(s, -1), atol=1e-12)
        grads = H._attn_ref_bwd(q, k, v, o, do, p, Hh, scale)
        for got, t in zip(grads, (qr, kr, vr)):
            assert torch.allclose(got, t.grad.transpose(1, 2).reshape(B, -1, Hh * dh), atol=1e-10)


def test_conv_references_match_autograd():
    g = torch.Generator().manual_seed(1)
    Bn, Hs, W, Ci, Co = 2, 6, 8, 5, 4
    x = torch.randn(Bn, Ci, Hs, W, generator=g, dtype=F64, requires_grad=True)
    w = torch.randn(Co, Ci, 3, 3, generator=g, dtype=F64, requires_grad=True)
    y = F.conv2d(x, w, padding=1)
    dy = torch.randn_like(y)
    y.backward(dy)
    # conv_in's weight gradient: wide = dY (NHWC), narrow = x (NCHW), sgn = +1 -> acc[co][ci][tap]
    acc = _narrow(dy.permute(0, 2, 3, 1), x.detach(), 1)
    assert torch.allclose(acc, w.grad.reshape(Co, Ci, 9), atol=1e-10)
    # conv_out's: wide = X (NHWC), narrow = dY (NCHW), sgn = -1 -> acc[ci][co][tap]
    acc = _narrow(x.detach().permute(0, 2, 3, 1), dy, -1)
    assert torch.allclose(acc, w.grad.permute(1, 0, 2, 3).reshape(Ci, Co, 9), atol=1e-10)
    # Downsample2D(padding=0): bottom / right zero pad, stride 2
    xs = torch.randn(1, Ci, 6, 6, generator=g, dtype=F64)
    ref = F.conv2d(F.pad(xs, (0, 1, 0, 1)), w.detach(), stride=2)
    manual = torch.zeros(1, Co, 3, 3, dtype=F64)
    xp = F.pad(xs, (0, 1, 0, 1))
    for oy in range(3):
        for ox in range(3):
            manual[0, :, oy, ox] = torch.einsum("cij,ocij->o", xp[0, :, 2 * oy:2 * oy + 3, 2 * ox:2 * ox + 3], w.detach())
    assert torch.allclose(ref, manual, atol=1e-12)


def _narrow(wide, narrow, sgn):
    c = H.Call.__new__(H.Call)
    c.kw = dict(wide=wide, narrow=narrow, sgn=sgn)
    c.run = lambda: None
    return H.h_narrow_conv_wgrad(c)[0].ref


def test_adamw_reference_matches_torch():
    g = torch.Generator().manual_seed(2)
    p0 = torch.randn(100, generator=g, dtype=F64)
    p = p0.clone().requires_grad_(True)
    opt = torch.optim.AdamW([p], lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2)
    m, v, pr = torch.zeros(100, dtype=F64), torch.zeros(100, dtype=F64), p0.clone()
    for t in range(1, 5):
        gr = torch.randn(100, generator=g, dtype=F64)
        p.grad = gr * 0.5
        opt.step()
        pr, m, v = H._adamw_ref(pr, gr, m, v, 1e-3, 0.9, 0.999, 1e-8, 1e-2, t, 0.5)
    assert torch.allclose(pr, p.detach(), atol=1e-14, rtol=0)


def test_guarded_layout_and_outside_check():
    base = torch.empty(2, 5, 3 * 8, dtype=torch.bfloat16)[..., 8:16]          # a column slice of a fused buffer
    sp = H.spec(base)
    gt = H.Guarded(sp, device="cpu")
    assert gt.t.shape == base.shape and gt.t.stride() == base.stride()
    assert bool(gt.t.isnan().all()) and gt.outside_intact()
    gt.t.fill_(1.0)
    assert gt.outside_intact()
    gt.buf[gt.off + 8] = 2.0                                                 # one element in the gap after a row
    assert not gt.outside_intact()
    dense = H.Guarded(("T", (4, 4), (4, 1), "float32", 2), device="cpu")
    dense.t.fill_(0.0)
    assert dense.outside_intact() and dense.off == H.GUARD + 2
    dense.buf[dense.off + 16] = 0.0                                          # first element past the end
    assert not dense.outside_intact()


def test_block_error_names_the_wrong_tile():
    ref = torch.randn(512, 256, dtype=F64)
    got = ref.clone()
    got[256:384, 128:192] += 0.05 * ref.pow(2).mean().sqrt()                  # one 128 x 64 tile off by 5 %
    err = got - ref
    rms = ref.pow(2).mean().sqrt()
    glob = (err.pow(2).mean().sqrt() / rms).item()
    worst, where = H.block_errors(err, rms, 128, 64)
    assert where == (2, 2) and abs(worst - 0.05) < 1e-9 and abs(glob - 0.05 / 4) < 1e-9     # 16 tiles: diluted 4x
