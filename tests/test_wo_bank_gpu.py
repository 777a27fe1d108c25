"""The WeightOffsets bank (e4t_b200/wobank.py, wo_bank_*_kernel in csrc/elementwise.cu) against fp64, projection by
projection.

The bank runs the closed form of e4t/weightoffsets.py for every attention projection of a UNet in batched launches:
forward = factors (vx, a, vy, b, s) and W_eff = bf16(W ⊙ (1 + Δ)); backward = five reductions of G = dW_eff ⊙ W
(Ga, Gbc, G1, GTb, GTs), two column mat-vecs (dvx, dvy) and the nine parameter gradients, ADDED into the optimiser
arena's .grad views.  Each projection is found through a host-packed device table, so the banks here are built the way
engine.PretrainStep builds them: real CrossAttention modules, parameters homed in an engine.FlatAdamW arena.

Bounds.  Everything in the bank is fp32 arithmetic on fp32 inputs.  Each element is held to
    |got - ref| <= k · 2⁻²⁴ · S
where S is the same closed form evaluated on absolute values (every sum a sum of magnitudes) and k is the length of
the kernel's longest addition chain for that element plus its roundings (see _stage_k).  Two kinds of check:
  * stage: each kernel output against fp64 of the kernel's OWN inputs (the fp32 factors / reductions it read);
  * end to end: against fp64 autograd of the literal module, sum((W ⊙ (1 + wo_delta)) · dW_eff), with k the sum of the
    stage k along the element's dependency chain (first-order propagation, _e2e_k).
W_eff (bf16) may differ from the fp64 value by one bf16 rounding plus the fp32 error of Δ times |W|.  The `.v` scalar
is a backward error: its S is |g₀| + Σ|w1·dvx| + Σ|w2·dvy|.
"""
import math

import pytest
import torch

from oracle import e4t_oracle as O

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24        # unit roundoff of fp32
U16 = 2.0 ** -8         # unit roundoff of bf16
KEYS = ("v", "linear1.weight", "linear1.bias", "linear2.weight", "linear2.bias", "linear_column.weight",
        "linear_column.bias", "linear_row.weight", "linear_row.bias")     # WeightOffsets.kernel_params() order
GRADS = ("v", "w1", "b1", "w2", "b2", "Wc", "bc", "Wr", "br")
# (query_dim, cross_attention_dim, inner): self (qkv) and cross (q + kv) groups; R = C, R > C, R < C; sides that are
# multiples of 8 but not of 32 or 128; max_r (1288) and max_c (1280) come from different projections
MIXED = [(1280, None, 1280), (320, 768, 320), (640, 1024, 640), (8, None, 8), (40, 1288, 72), (1288, 8, 8),
         (200, None, 136)]


@pytest.fixture(scope="module", autouse=True)
def _keep_direct_grad_write():
    """FlatAdamW sets functional.DIRECT_GRAD_WRITE for the whole process; put it back after this file."""
    from e4t_b200 import functional as FN
    saved = FN.DIRECT_GRAD_WRITE
    yield
    FN.DIRECT_GRAD_WRITE = saved


# ---- fp64 closed form (works on values and, given absolute values, on magnitudes) ------------------------------------
def _p64(wo, absval=False):
    v, w1, b1, w2, b2, Wc, bc, Wr, br = (t.detach().double() for t in wo.kernel_params())
    p = dict(v=v, w1=w1[:, 0], b1=b1, w2=w2[:, 0], b2=b2, Wc=Wc, bc=bc, Wr=Wr, br=br)
    return {k: t.abs() for k, t in p.items()} if absval else p


def _factors(p):
    vx = p["w1"] * p["v"] + p["b1"]
    vy = p["w2"] * p["v"] + p["b2"]
    return dict(vx=vx, a=p["Wc"] @ vx, vy=vy, b=p["Wr"] @ vy, s=p["Wr"].sum(1))


def _reductions(G, a, bc, b, s):
    return dict(Ga=G @ a, Gbc=G @ bc, G1=G.sum(1), GTb=G.t() @ b, GTs=G.t() @ s)


def _matvecs(Wc, Wr, GTb, Ga):
    return dict(dvx=Wc.t() @ GTb, dvy=Wr.t() @ Ga)


def _grads(p, vx, vy, r, dvx, dvy):
    return dict(v=(p["w1"] @ dvx + p["w2"] @ dvy).reshape(1), w1=(dvx * p["v"])[:, None], b1=dvx,
                w2=(dvy * p["v"])[:, None], b2=dvy, Wc=r["GTb"][:, None] * vx[None, :], bc=r["GTs"],
                Wr=r["Ga"][:, None] * vy[None, :] + r["Gbc"][:, None], br=r["G1"])


def _magnitudes(wo, W, dWs):
    """S of every intermediate and gradient: the closed form on |parameters|, |W| and Σ|dW_eff|."""
    p = _p64(wo, absval=True)
    f = _factors(p)
    r = _reductions(W.abs() * sum(d.abs() for d in dWs), f["a"], p["bc"], f["b"], f["s"])
    mv = _matvecs(p["Wc"], p["Wr"], r["GTb"], r["Ga"])
    return f, r, mv, _grads(p, f["vx"], f["vy"], r, mv["dvx"], mv["dvy"])


def _literal(lin, wo, dW=None):
    """fp64 of the literal module: W ⊙ (1 + wo_delta) and, given dW_eff, autograd of sum(W_eff · dW_eff)."""
    sd = {k: t.detach().double().requires_grad_(dW is not None) for k, t in wo.state_dict(keep_vars=True).items()}
    W = lin.weight.detach().double()
    weff = W * (1 + O.wo_delta(sd, ""))
    if dW is None:
        return weff.detach(), None
    return weff.detach(), dict(zip(GRADS, torch.autograd.grad((weff * dW).sum(), [sd[k] for k in KEYS])))


def _stage_k(R, C):
    """Longest addition chain + roundings of every bank output, from the kernels' loop structure."""
    k = dict(vx=2, vy=2,                                    # w·v + β (fma or product + add)
             a=math.ceil(R / 32) + 5 + 2,                   # lane-strided loop, 5-level warp tree; + vx's roundings
             b=math.ceil(C / 32) + 5 + 2, s=math.ceil(C / 32) + 5,
             Ga=math.ceil(R / 32) + 5 + 1,                  # same loop over r; + the rounding of g = dW·W
             GTb=8 + math.ceil(C / 8) + 2,                  # 8 warps' shared atomics, ⌈C/8⌉ CTAs' global atomics; g, g·b
             dvx=32 + math.ceil(R / 32), dvy=32 + math.ceil(C / 32),   # 32-term fma chain, then one atomic per CTA row
             weff=6)                                        # 1 + br, b·a, +, s·bc, +, W·(...) before the bf16 rounding
    k.update(Gbc=k["Ga"], G1=k["Ga"], GTs=k["GTb"])
    # gradients: g += u·w + t is two roundings, g += d·v and g += d one or two, dv: per-thread chain over R then C,
    # a warp tree, a tree over the 8 warps and the final add
    k["grad"] = dict(Wr=2, Wc=2, w1=2, w2=2, b1=1, b2=1, bc=1, br=1,
                     v=math.ceil(R / 256) + math.ceil(C / 256) + 5 + 5 + 1)
    return k


def _e2e_k(R, C, extra=0):
    """First-order propagation: a quantity's k is its own stage k plus the largest k among its inputs.  `extra` adds
    roundings for the paths that sum two backward passes (accumulation into .grad, the two-phase exchange)."""
    k = _stage_k(R, C)
    e = dict(vx=k["vx"], vy=k["vy"], a=k["a"], b=k["b"], s=k["s"])
    e.update(Ga=k["Ga"] + e["a"] + extra, Gbc=k["Gbc"] + extra, G1=k["G1"] + extra, GTb=k["GTb"] + e["b"] + extra,
             GTs=k["GTs"] + e["s"] + extra)
    e.update(dvx=k["dvx"] + e["GTb"], dvy=k["dvy"] + e["Ga"])
    g = k["grad"]
    e["grad"] = dict(Wr=g["Wr"] + max(e["Ga"] + e["vy"], e["Gbc"]) + extra, Wc=g["Wc"] + e["GTb"] + e["vx"] + extra,
                     w1=g["w1"] + e["dvx"] + extra, b1=g["b1"] + e["dvx"] + extra, w2=g["w2"] + e["dvy"] + extra,
                     b2=g["b2"] + e["dvy"] + extra, bc=g["bc"] + e["GTs"] + extra, br=g["br"] + e["G1"] + extra,
                     v=g["v"] + max(e["dvx"], e["dvy"]) + extra)
    e["weff"] = k["weff"] + max(e["a"] + e["b"], e["s"])
    return e


# ---- the bank's layout and the checks --------------------------------------------------------------------------------
class _Proj:
    __slots__ = ("name", "lin", "wo", "R", "C", "fac", "bw", "weff", "dweff")


def _projections(bank, names):
    """Every projection of the bank with its slices: fac (vx[R] a[R] vy[C] b[C] s[C]) and bw (Ga[C] Gbc[C] G1[C]
    GTb[R] GTs[R] dvx[R] dvy[C]) in table order, W_eff / dW_eff as rows of its group's view."""
    out, fo, bo = [], 0, 0
    groups = [(m, grp) for m, grp, _ in bank.groups]
    want = [(m, grp) for m in bank.modules for grp in (("q", "kv") if m.is_cross else ("qkv",))]
    assert groups == want
    for m, group in groups:
        w_view, dw_view = bank.views[(id(m), group)]
        row = 0
        for x in group:                                       # "qkv" -> to_q, to_k, to_v
            lin, wo = getattr(m, "to_" + x), getattr(m, "wo_" + x)
            p = _Proj()
            p.name, p.lin, p.wo = names[id(lin)], lin, wo
            R, C = p.R, p.C = lin.in_features, lin.out_features
            p.fac, p.bw = (fo, fo + 2 * R + 3 * C), (bo, bo + 4 * C + 3 * R)
            p.weff, p.dweff = w_view[row:row + C], dw_view[row:row + C]
            fo, bo, row = fo + 2 * R + 3 * C, bo + 4 * C + 3 * R, row + C
            out.append(p)
    assert fo == bank.fac.numel() and bo == bank.bw.numel()
    return out


def _split(t, sizes, names):
    out, o = {}, 0
    for n, s in zip(names, sizes):
        out[n] = t[o:o + s].double()
        o += s
    return out


def _fac(bank, p):
    return _split(bank.fac[p.fac[0]:p.fac[1]], (p.R, p.R, p.C, p.C, p.C), ("vx", "a", "vy", "b", "s"))


def _bw(bank, p):
    return _split(bank.bw[p.bw[0]:p.bw[1]], (p.C, p.C, p.C, p.R, p.R, p.R, p.C),
                  ("Ga", "Gbc", "G1", "GTb", "GTs", "dvx", "dvy"))


class _Checks:
    """Collects every elementwise check; keeps each tensor's worst ratio to its bound and its relative RMS."""

    def __init__(self, title):
        self.title, self.worst, self.fails = title, {}, []

    def __call__(self, what, proj, got, ref, bound):
        got = got.detach().double().reshape(ref.shape)
        err = (got - ref).abs()
        ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)
        i = int(ratio.reshape(-1).argmax())
        r = ratio.reshape(-1)[i].item()
        if not torch.isfinite(got).all():
            r = math.inf
        rel = (err.pow(2).mean().sqrt() / ref.pow(2).mean().sqrt().clamp_min(1e-300)).item()
        w = self.worst.get(what)
        if w is None or r > w[0]:
            self.worst[what] = (r, proj, max(rel, w[2] if w else 0.0))
        else:
            self.worst[what] = (w[0], w[1], max(rel, w[2]))
        if not r <= 1.0:
            self.fails.append(f"{proj}: {what} element {i}: got {got.reshape(-1)[i].item():.9g} ref "
                              f"{ref.reshape(-1)[i].item():.9g} bound {bound.reshape(-1)[i].item():.3g} "
                              f"(ratio {r:.3g})")

    def done(self):
        print(f"\n[{self.title}] worst |got - ref| / bound per tensor (projection), relative RMS error:")
        for what in sorted(self.worst):
            r, proj, rel = self.worst[what]
            print(f"  {what:<26} {r:9.3e}  ({proj})  rel-RMS {rel:.2e}")
        assert not self.fails, f"{len(self.fails)} checks out of bound, first ones:\n" + "\n".join(self.fails[:12])


def _bound(k, mag):
    return k * U32 * mag


def _check_forward(chk, bank, projs):
    for p in projs:
        k, e = _stage_k(p.R, p.C), _e2e_k(p.R, p.C)
        got = _fac(bank, p)
        ref, mag = _factors(_p64(p.wo)), _factors(_p64(p.wo, absval=True))
        for n in ("vx", "a", "vy", "b", "s"):                               # k: _stage_k (inputs are parameters)
            chk(f"fwd {n}", p.name, got[n], ref[n], _bound(k[n], mag[n]))
        W = p.lin.weight.detach().double()
        pp = _p64(p.wo)
        # stage: the kernel's own fp32 a, b, s; k = 6 roundings, then one bf16 rounding of the value
        own = W * (1 + pp["br"][:, None] + got["b"][:, None] * got["a"][None, :] + got["s"][:, None] * pp["bc"][None, :])
        own_mag = W.abs() * (1 + pp["br"].abs()[:, None] + (got["b"][:, None] * got["a"][None, :]).abs()
                             + (got["s"][:, None] * pp["bc"][None, :]).abs())
        chk("fwd W_eff (stage)", p.name, p.weff, own, U16 * own.abs() + (1 + U16) * _bound(k["weff"], own_mag))
        # end to end: the literal module; the fp32 error of Δ (_e2e_k) times |W|, then one bf16 rounding
        lit, _ = _literal(p.lin, p.wo)
        lit_mag = W.abs() * (1 + pp["br"].abs()[:, None] + mag["b"][:, None] * mag["a"][None, :]
                             + mag["s"][:, None] * pp["bc"].abs()[None, :])
        chk("fwd W_eff (e2e)", p.name, p.weff, lit, U16 * lit.abs() + (1 + U16) * _bound(e["weff"], lit_mag))


def _grad_views(p):
    return dict(zip(GRADS, (q.grad for q in p.wo.kernel_params())))


def _check_backward(chk, bank, projs, g_before, dWs, extra=0, reductions_are_kernel_outputs=True):
    """After a backward: bw and the nine gradients of every projection.  g_before: {name: [9 fp64 grads]} read before
    the backward (stage reference); dWs: {name: [dW_eff, ...]} whose sum the end-to-end reference differentiates."""
    for p in projs:
        k, e = _stage_k(p.R, p.C), _e2e_k(p.R, p.C, extra)
        pp, pa = _p64(p.wo), _p64(p.wo, absval=True)
        W = p.lin.weight.detach().double()
        fac, bw = _fac(bank, p), _bw(bank, p)
        # stage 1: the five reductions from the dW_eff the kernel read and its own fp32 a, b, s
        if reductions_are_kernel_outputs:
            dW = p.dweff.double()
            ref = _reductions(dW * W, fac["a"], pp["bc"], fac["b"], fac["s"])
            mag = _reductions((dW * W).abs(), fac["a"].abs(), pa["bc"], fac["b"].abs(), fac["s"].abs())
            for n in ref:                                                     # k: Ga/Gbc/G1 ⌈R/32⌉+6, GTb/GTs 8+⌈C/8⌉+2
                chk(f"bwd {n} (stage)", p.name, bw[n], ref[n], _bound(k[n], mag[n]))
        # stage 2: dvx = Wcᵀ GTb, dvy = Wrᵀ Ga from the kernel's own reductions; k = 32 + ⌈n/32⌉
        ref = _matvecs(pp["Wc"], pp["Wr"], bw["GTb"], bw["Ga"])
        mag = _matvecs(pa["Wc"], pa["Wr"], bw["GTb"].abs(), bw["Ga"].abs())
        for n in ref:
            chk(f"bwd {n} (stage)", p.name, bw[n], ref[n], _bound(k[n], mag[n]))
        # stage 3: the gradients from the kernel's own vx, vy, reductions, dvx, dvy, added to what .grad held
        got = _grad_views(p)
        gb = g_before[p.name]
        ref = _grads(pp, fac["vx"], fac["vy"], bw, bw["dvx"], bw["dvy"])
        mag = _grads(pa, fac["vx"].abs(), fac["vy"].abs(), {n: t.abs() for n, t in bw.items()}, bw["dvx"].abs(),
                     bw["dvy"].abs())
        for n, g0 in zip(GRADS, gb):                                           # k: _stage_k()["grad"]
            chk(f"grad {n} (stage)", p.name, got[n], g0 + ref[n], _bound(k["grad"][n], g0.abs() + mag[n]))
        # end to end: fp64 autograd of the literal module, summed over the dW_eff's; k: _e2e_k
        dsum = sum(d.double() for d in dWs[p.name])
        _, ref = _literal(p.lin, p.wo, dsum)
        f_m, r_m, mv_m, g_m = _magnitudes(p.wo, W, [d.double() for d in dWs[p.name]])
        for n, g0 in zip(GRADS, gb):
            chk(f"grad {n} (e2e)", p.name, got[n], g0 + ref[n], _bound(e["grad"][n], g0.abs() + g_m[n]))
        if reductions_are_kernel_outputs and len(dWs[p.name]) == 1:
            f = _factors(pp)
            ref = _reductions(dsum * W, f["a"], pp["bc"], f["b"], f["s"])
            ref.update(_matvecs(pp["Wc"], pp["Wr"], ref["GTb"], ref["Ga"]))
            for n in ("Ga", "Gbc", "G1", "GTb", "GTs"):
                chk(f"bwd {n} (e2e)", p.name, bw[n], ref[n], _bound(e[n], r_m[n]))
            for n in ("dvx", "dvy"):
                chk(f"bwd {n} (e2e)", p.name, bw[n], ref[n], _bound(e[n], mv_m[n]))


def _snapshot(projs):
    return {p.name: [g.detach().double().clone() for g in _grad_views(p).values()] for p in projs}


def _wo_mask(opt, bank):
    mask = torch.zeros(opt.grad.numel(), dtype=torch.bool, device=opt.grad.device)
    for q in bank.params:
        o = (q.grad.data_ptr() - opt.grad.data_ptr()) // 4
        mask[o:o + q.numel()] = True
    return mask


def _check_neighbours(opt, mask, g0):
    """Every arena element outside the WeightOffsets gradients (other parameters, padding) is bit-identical to g₀."""
    got, want = opt.grad.view(torch.int32)[~mask], g0.view(torch.int32)[~mask]
    assert got.numel() > 0 and torch.equal(got, want), f"{int((got != want).sum())} arena elements outside the " \
                                                        f"WeightOffsets gradients changed"


def _dweff_patterns(bank, projs, seed):
    """Two dW_eff: N(0, 1), and u·wᵀ + noise per projection (large row and column means, so G1 / GTs do not cancel
    where W has a mean)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    gauss = torch.randn(bank.dweff.shape, device="cuda", generator=g)
    mean = torch.empty_like(bank.dweff)
    o = 0
    for p in projs:
        u = 1 + 0.3 * torch.randn(p.C, device="cuda", generator=g)
        w = 1 + 0.3 * torch.randn(p.R, device="cuda", generator=g)
        mean[o:o + p.C * p.R] = (u[:, None] * w[None, :] + 0.5 * torch.randn(p.C, p.R, device="cuda", generator=g)).reshape(-1)
        o += p.C * p.R
    return gauss, mean


def _per_proj(projs, flat):
    """{name: [dW_eff slice]} of a flat dW_eff laid out like bank.dweff (the projections in table order)."""
    out, o = {}, 0
    for p in projs:
        out[p.name] = [flat[o:o + p.C * p.R].view(p.C, p.R)]
        o += p.C * p.R
    return out


def _backward(bank, dweff):
    bank.dweff.copy_(dweff)
    bank._launch_backward()
    torch.cuda.synchronize()


def _names(root):
    from e4t.models.cross_attention import CrossAttention
    names = {}
    for n, m in root.named_modules():
        if isinstance(m, CrossAttention):
            for s in ("to_q", "to_k", "to_v"):
                names[id(getattr(m, s))] = f"{n}.{s}"
    return names


def _arena_bank(root, extra_params):
    """FlatAdamW over every WeightOffsets parameter with `extra_params` interleaved as arena neighbours, and a WOBank
    over every CrossAttention module of `root` — as engine.PretrainStep builds them."""
    from e4t.models.cross_attention import CrossAttention
    from e4t_b200.engine import FlatAdamW
    from e4t_b200.wobank import WOBank
    attns = [m for m in root.modules() if isinstance(m, CrossAttention)]
    params, extra = [], list(extra_params)
    for i, m in enumerate(attns):
        for wo in (m.wo_q, m.wo_k, m.wo_v):
            params += list(wo.kernel_params())
        if i < len(extra):
            params.append(extra[i])
    for p in root.parameters():
        p.requires_grad_(False)
    for p in params:
        p.requires_grad_(True)
    opt = FlatAdamW(params, lr=1e-3)
    return opt, WOBank(attns), attns


# ---- 1. mixed shapes -------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def mixed():
    from e4t.models.cross_attention import CrossAttention
    torch.manual_seed(0)
    mods = torch.nn.ModuleList(CrossAttention(query_dim=q, cross_attention_dim=x, heads=1, dim_head=n)
                               for q, x, n in MIXED)
    g = torch.Generator().manual_seed(1234)

    def uni(shape, lo, hi):
        return lo + (hi - lo) * torch.rand(shape, generator=g)

    with torch.no_grad():      # Δ = O(1): v in [0.5, 2], a, b, s = O(1), biases O(0.1-1); W with a positive mean
        for m in mods:
            for lin in (m.to_q, m.to_k, m.to_v):
                lin.weight.copy_(uni(lin.weight.shape, -0.5, 1.0))
            for wo in (m.wo_q, m.wo_k, m.wo_v):
                R, C = wo.linear_column.weight.shape[0], wo.linear_row.weight.shape[0]
                wo.v.copy_(uni((1,), 0.5, 2.0))
                wo.linear1.weight.copy_(uni((R, 1), -1, 1)); wo.linear1.bias.copy_(uni((R,), -0.5, 0.5))
                wo.linear2.weight.copy_(uni((C, 1), -1, 1)); wo.linear2.bias.copy_(uni((C,), -0.5, 0.5))
                wo.linear_column.weight.copy_(uni((R, R), -1, 1) * math.sqrt(3 / R))
                wo.linear_column.bias.copy_(uni((R,), -0.5, 0.5))
                wo.linear_row.weight.copy_(uni((C, C), -1, 1) * math.sqrt(3 / C))
                wo.linear_row.bias.copy_(uni((C,), -0.5, 0.5))
    mods.cuda()
    opt, bank, attns = _arena_bank(mods, [m.to_out[0].weight for m in mods])
    assert bank.max_r == 1288 and bank.max_c == 1280
    projs = _projections(bank, _names(mods))
    assert len(projs) == 21 and {(p.R, p.C) for p in projs} >= {(40, 72), (1288, 72), (1288, 8)}
    yield mods, opt, bank, projs
    del mods, opt, bank, projs
    torch.cuda.empty_cache()


def test_mixed_forward_factors_weff_and_determinism(mixed):
    from e4t_b200.wobank import WOBank
    mods, opt, bank, projs = mixed
    bank._launch_forward()
    torch.cuda.synchronize()
    chk = _Checks("mixed shapes, forward")
    _check_forward(chk, bank, projs)
    first = bank.weff.clone()
    bank._launch_forward()
    rev = WOBank(list(mods)[::-1])
    rev._launch_forward()
    torch.cuda.synchronize()
    assert torch.equal(bank.weff.view(torch.int16), first.view(torch.int16)), "W_eff changed between two forwards"
    for key, (w, _) in bank.views.items():       # the forward has no atomics: any order gives the same bits
        assert torch.equal(rev.views[key][0].view(torch.int16), w.view(torch.int16)), key
    chk.done()


def test_mixed_backward_accumulates_into_grad_and_leaves_neighbours(mixed):
    mods, opt, bank, projs = mixed
    bank._launch_forward()
    gen = torch.Generator(device="cuda").manual_seed(7)
    g0 = torch.randn(opt.grad.shape, device="cuda", generator=gen)        # finite: the kernels read-modify-write
    opt.grad.copy_(g0)
    mask = _wo_mask(opt, bank)
    gauss, mean = _dweff_patterns(bank, projs, 11)
    chk = _Checks("mixed shapes, backward")
    before = _snapshot(projs)
    _backward(bank, gauss)
    _check_backward(chk, bank, projs, before, _per_proj(projs, gauss))
    _check_neighbours(opt, mask, g0)
    # accumulation: no zeroing in between -> g₀ + ref(gauss) + ref(mean); the memset re-zeroes dvx / dvy
    mid = _snapshot(projs)
    _backward(bank, mean)
    _check_backward(chk, bank, projs, mid, _per_proj(projs, mean))
    # the accumulated result against g₀ + ref₁ + ref₂ directly; extra = 1: the second pass adds once more
    d1, d2 = _per_proj(projs, gauss), _per_proj(projs, mean)
    chk2 = _Checks("mixed shapes, two backwards accumulated")
    for p in projs:
        e = _e2e_k(p.R, p.C, extra=1)
        W = p.lin.weight.detach().double()
        _, r1 = _literal(p.lin, p.wo, d1[p.name][0].double())
        _, r2 = _literal(p.lin, p.wo, d2[p.name][0].double())
        g_m = _magnitudes(p.wo, W, [d1[p.name][0].double(), d2[p.name][0].double()])[3]
        got = _grad_views(p)
        for n, g00 in zip(GRADS, before[p.name]):
            chk2(f"grad {n} (g0+ref1+ref2)", p.name, got[n], g00 + r1[n] + r2[n],
                 _bound(e["grad"][n], g00.abs() + g_m[n]))
    _check_neighbours(opt, mask, g0)
    chk.done()
    chk2.done()


def test_mixed_two_phase_exchange_matches_fp64_of_the_summed_dweff(mixed):
    """The data-parallel path: reduce on each "rank's" dW_eff, sum the bw buffers (what the all-reduce leaves), apply."""
    from ctypes import c_int, c_longlong
    from e4t_b200 import _lib
    from e4t_b200._lib import ptr, stream
    mods, opt, bank, projs = mixed
    bank._launch_forward()
    gen = torch.Generator(device="cuda").manual_seed(8)
    g0 = torch.randn(opt.grad.shape, device="cuda", generator=gen)
    opt.grad.copy_(g0)
    mask = _wo_mask(opt, bank)
    d1, d2 = _dweff_patterns(bank, projs, 12)
    n, mr, mc = c_int(len(bank.projs)), c_int(bank.max_r), c_int(bank.max_c)
    bws = []
    for d in (d1, d2):
        bank.dweff.copy_(d)
        _lib.call("e4t_wo_bank_bwd_reduce", ptr(bank._table), n, mr, mc, ptr(bank.bw), c_longlong(bank.bw.numel()),
                  stream())
        bws.append(bank.bw.clone())
    bank.bw.copy_(bws[0] + bws[1])
    before = _snapshot(projs)
    _lib.call("e4t_wo_bank_bwd_apply", ptr(bank._table), n, mr, mc, stream())
    torch.cuda.synchronize()
    chk = _Checks("mixed shapes, two-phase exchange")
    dws = {k: v1 + v2 for (k, v1), (_, v2) in zip(_per_proj(projs, d1).items(), _per_proj(projs, d2).items())}
    _check_backward(chk, bank, projs, before, dws, extra=1, reductions_are_kernel_outputs=False)
    _check_neighbours(opt, mask, g0)
    chk.done()


def test_mixed_base_weight_gradient_for_tuning(mixed):
    """Tuning trains the base projection weights too: _BankFn returns dW = dW_eff ⊙ (1 + Δ) for them."""
    from e4t_b200.wobank import _BankFn
    mods, opt, bank, projs = mixed
    ws = [lin.weight for lin, _ in bank.projs]
    tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        for w in ws:
            w.requires_grad_(True)
        token = _BankFn.apply(bank, *bank.params, *ws)
        gauss, _ = _dweff_patterns(bank, projs, 13)
        bank.dweff.copy_(gauss)
        dws = torch.autograd.grad(token, ws, torch.ones_like(token))
        torch.cuda.synchronize()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32
        for w in ws:
            w.requires_grad_(False)
    chk = _Checks("mixed shapes, base-weight gradient")
    for p, got in zip(projs, dws):
        pp = _p64(p.wo)
        dW = p.dweff.double()
        f_m = _factors(_p64(p.wo, absval=True))
        ref = dW * (1 + O.wo_delta({k: t.detach().double() for k, t in p.wo.state_dict().items()}, ""))
        mag = dW.abs() * (1 + pp["br"].abs()[:, None] + f_m["b"][:, None] * f_m["a"][None, :]
                          + f_m["s"][:, None] * pp["bc"].abs()[None, :])
        # Δ is WeightOffsets.forward() in torch fp32: mat-vecs of unknown summation order (worst case n roundings for
        # R- and C-term sums) after vx / vy (2), then b·a, s·bc, two adds, 1 + Δ and the product with dW_eff (6)
        chk("base dW", p.name, got, ref, _bound((p.R + 2) + (p.C + 2) + 6, mag))
    chk.done()


# ---- 2. SD-v1.4 UNet ---------------------------------------------------------------------------------------------------
def test_sd14_bank_all_864_tensors():
    from e4t.models.unet_2d_condition import UNet2DConditionModel
    from e4t.models.cross_attention import CrossAttention
    unet = UNet2DConditionModel(**O.ref_unet_kwargs(O.SD14_UNET))
    unet.load_state_dict(O.synth_state_dict(O.unet_param_shapes(O.SD14_UNET), 3), strict=True)
    unet.cuda()
    attns = [m for m in unet.modules() if isinstance(m, CrossAttention)]
    opt, bank, _ = _arena_bank(unet, [m.to_out[0].weight for m in attns])
    projs = _projections(bank, _names(unet))
    assert len(projs) == 96 and len(bank.params) == 864
    bank._launch_forward()
    torch.cuda.synchronize()
    chk = _Checks("SD-v1.4, forward")
    _check_forward(chk, bank, projs)
    # the per-projection path (ops.wo_factors + ops.wo_weff) runs the same fp32 expressions in the same order
    with torch.no_grad():
        for m, group, _ in bank.groups:
            w_ref, _ = m.effective_weights(group)
            assert torch.equal(bank.views[(id(m), group)][0].view(torch.int16), w_ref.view(torch.int16)), group
    chk.done()
    gen = torch.Generator(device="cuda").manual_seed(5)
    g0 = torch.randn(opt.grad.shape, device="cuda", generator=gen)
    opt.grad.copy_(g0)
    mask = _wo_mask(opt, bank)
    gauss, mean = _dweff_patterns(bank, projs, 6)
    chk = _Checks("SD-v1.4, backward + accumulation")
    before = _snapshot(projs)
    _backward(bank, gauss)
    _check_backward(chk, bank, projs, before, _per_proj(projs, gauss))
    _check_neighbours(opt, mask, g0)
    mid = _snapshot(projs)
    _backward(bank, mean)
    _check_backward(chk, bank, projs, mid, _per_proj(projs, mean))
    _check_neighbours(opt, mask, g0)
    chk.done()
    del unet, opt, bank, projs, attns
    torch.cuda.empty_cache()


# ---- 3. dW_eff from a real step ----------------------------------------------------------------------------------------
def test_bank_backward_of_a_real_tiny_step():
    """One PretrainStep forward_loss + backward: dW_eff is accumulated by the split-K GEMMs of both UNet passes before
    _BankFn's backward runs; the WeightOffsets gradients (from zero) must be the fp64 closed form of that dW_eff."""
    from e4t.encoder import E4TEncoder
    from e4t.models.modeling_clip import CLIPTextConfig, CLIPTextModel
    from e4t.models.unet_2d_condition import UNet2DConditionModel
    from e4t_b200.engine import PretrainStep
    ucfg, vcfg, tcfg = O.TINY_UNET, O.VIT_TINY, O.CLIP_TEXT_TINY
    fd = O.pooled_feature_dim(ucfg)
    unet = UNet2DConditionModel(**O.ref_unet_kwargs(ucfg))
    unet.load_state_dict(O.synth_state_dict(O.unet_param_shapes(ucfg), 1), strict=True)
    enc = E4TEncoder(arch="ViT-tiny-test", word_embedding_dim=tcfg["width"], n_odd_layers=129, unet_feature_dim=fd)
    enc.load_state_dict(O.synth_state_dict(O.encoder_param_shapes(vcfg, fd, tcfg["width"], 129), 2), strict=True)
    text = CLIPTextModel(CLIPTextConfig(vocab_size=tcfg["vocab"], hidden_size=tcfg["width"],
                                        intermediate_size=tcfg["mlp"], num_hidden_layers=tcfg["layers"],
                                        num_attention_heads=tcfg["heads"]))
    text.load_state_dict(O.synth_state_dict(O.text_param_shapes(tcfg), 3), strict=True)
    step = PretrainStep(unet.cuda(), enc.cuda(), text.cuda(), O.PLACEHOLDER_ID, class_token_id=320, lr=1e-3,
                        weight_dtype=torch.float32)
    bank = step.wo_bank
    projs = _projections(bank, _names(unet))
    before = _snapshot(projs)
    assert all(float(g.abs().max()) == 0 for gs in before.values() for g in gs)
    batch = O.synth_batch(2, seed=42, latent_hw=16, image_hw=64)
    out = step.forward_loss({k: v.cuda() for k, v in batch.items()})
    out["loss"].backward()
    torch.cuda.synchronize()
    dweff = bank.dweff.clone()
    assert float(dweff.abs().max()) > 0
    chk = _Checks("tiny PretrainStep, dW_eff of both UNet passes")
    _check_backward(chk, bank, projs, before, _per_proj(projs, dweff))
    chk.done()
