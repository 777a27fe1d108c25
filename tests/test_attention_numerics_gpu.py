"""Attention at peaked scores: a sink key Δ = 8, 24 or 48 nats above the rest of a row, at every block edge of the
kernel that runs, against fp64.

Every other attention test draws q and k from randn at a scale near 1: the scaled logits have a standard deviation of
0.25 to 1, so the online softmax's running max hardly moves after the first key block, its rescale factor stays near 1,
and the backward never sees one key holding nearly all of a row's mass.  Trained checkpoints do produce such rows
(attention sinks on the BOS key, high-norm ViT tokens).  The generator here builds them, keeps half the query rows of
each (image, head) flat so that every gradient keeps a real-signal scale, and checks O, the LSE, dQ, dK and dV with
the measures of test_call_signatures_gpu.py (RMS error over the tensor, over each 64-row block) plus a per-row check:
each query row of dQ and each key row of dK / dV within 4x the op's bound of that row's own fp64 RMS, for rows whose
derived error (the fp32 arithmetic of S, P and dP - D and the bf16 rounding of P and dS, `reference`) is below half
that bound.  O is held elementwise and the LSE per row to bounds derived the same way, so weight wrongly given to keys
far below a row's max (an exp2 argument clamped at -20, a key read past the end) fails them.
"""
import math
import os

import pytest
import torch

import test_call_signatures_gpu as H

pytestmark = pytest.mark.gpu

F64 = torch.float64
DELTAS = (8.0, 24.0, 48.0)
SIGMAS = (1.0, 3.0, 6.0)
U32 = 2.0 ** -24
B_O, B_GRAD = 6e-3, 1e-2                   # the replay's bounds: O, gradients


# ---------------------------------------------------------------------------------------------------------------------
# the score generator
# ---------------------------------------------------------------------------------------------------------------------
def peaked_qk(B, N, M, heads, dh, scale, g, sinks=None, mode="sink", shared_dir=False, delta=None):
    """fp32 q (B, N, heads*dh) and k (B, M, heads*dh) for scale·q·kᵀ with, per (image, head) slot i:
      * every q and k orthogonal to a unit direction d (drawn per slot, or per head with shared_dir) except as below,
        so a flat row's logits have a spread of about σ = SIGMAS[(i // 3) % 3] nats;
      * mode "sink": key sinks[i] (default: a random key) is δ·d, and each even query row gets + γ·d, so its logit on
        the sink is s·γ·δ = Δ + (that row's largest other logit), Δ = DELTAS[i % 3] (or `delta`); the odd rows stay
        flat;
      * mode "rise" / "fall": every key gets + c_j·d with c_j rising (falling) linearly over the row, so the even rows'
        logits climb by 8 nats per 128 keys over a row: the running max rises in every block (its rescale factor is
        e^-8 or less) or, falling, every block after the first underflows.
    Returns q, k, the peaked-row mask (N,) and the per-slot sink list."""
    C = heads * dh
    dev = "cuda"
    nd = heads if shared_dir else B * heads
    d = torch.randn(nd, dh, generator=g, device=dev)
    d = d / d.norm(dim=-1, keepdim=True)
    d = d.view(1, heads, dh).expand(B, heads, dh) if shared_dir else d.view(B, heads, dh)
    sig = torch.tensor([SIGMAS[(i // 3) % 3] for i in range(B * heads)], device=dev).view(B, 1, heads, 1)
    a = sig.sqrt() * dh ** -0.25 / scale ** 0.5     # q, k ~ N(0, a²): scale·q·k has a standard deviation of σ

    def perp(t):
        t = t * a
        return t - (t * d[:, None]).sum(-1, keepdim=True) * d[:, None]

    q = perp(torch.randn(B, N, heads, dh, generator=g, device=dev))
    k = perp(torch.randn(B, M, heads, dh, generator=g, device=dev))
    peaked = torch.arange(N, device=dev) % 2 == 0
    if sinks is None:
        sinks = torch.randint(0, M, (B * heads,), generator=g, device=dev).tolist()
    if mode == "sink":
        for i in range(B * heads):
            b, h = divmod(i, heads)
            # γ per row: Δ (+ 0.5 for the bf16 rounding of q and k) above that row's largest other logit
            dl = (delta or DELTAS[i % 3]) + 0.5
            mx = ((q[b, peaked, h] @ k[b, :, h].T) * scale).max(1).values
            dlt = math.sqrt((dl + mx.max().item()) / scale)
            k[b, sinks[i], h] = dlt * d[b, h]
            q[b, peaked, h] += ((dl + mx) / (scale * dlt))[:, None] * d[b, h]
    else:
        L = 8.0 * M / 128 + 8.0
        gd = math.sqrt(L / scale)
        c = torch.linspace(0.0, 1.0, M, device=dev)
        if mode == "fall":
            c = c.flip(0)
        k += gd * c.view(1, M, 1, 1) * d[:, None]
        q[:, peaked] += gd * d[:, None]
    return q.reshape(B, N, C), k.reshape(B, M, C), peaked, sinks


def achieved(q16, k16, heads, scale, peaked, sinks, causal=False, rows=64):
    """(min Δ, σ range) reached by the bf16 values over the first `rows` peaked and flat rows of every slot, in fp64."""
    B, N, C = q16.shape
    dh = C // heads
    pi = peaked.nonzero().flatten()[:rows]
    fi = (~peaked).nonzero().flatten()[:rows]
    dmin, sig = math.inf, []
    for b in range(B):
        qh = q16[b].double().view(N, heads, dh).transpose(0, 1)
        kh = k16[b].double().view(-1, heads, dh).transpose(0, 1)
        for h in range(heads):
            j = sinks[b * heads + h]
            sp = (qh[h, pi] @ kh[h].T) * scale
            sf = (qh[h, fi] @ kh[h].T) * scale
            if causal:
                sp = sp.masked_fill(torch.arange(sp.shape[1], device=sp.device)[None] > pi[:, None], -math.inf)
                sf = sf.masked_fill(torch.arange(sf.shape[1], device=sf.device)[None] > fi[:, None], -math.inf)
                ok = pi >= j
                if not bool(ok.any()):
                    continue
                sp = sp[ok]
            others = torch.cat([sp[:, :j], sp[:, j + 1:]], 1)
            dmin = min(dmin, (sp[:, j] - others.max(1).values).min().item())
            fin = sf[torch.isfinite(sf)]
            sig.append(fin.std().item())
    return dmin, (min(sig), max(sig))


# ---------------------------------------------------------------------------------------------------------------------
# fp64 reference and the derived bounds
# ---------------------------------------------------------------------------------------------------------------------
UB = 2.0 ** -9        # relative rounding of a bf16 operand the kernels feed to the tensor cores (P, dS)


def ulp_bf16(r):
    e = torch.floor(torch.log2(r.abs().clamp_min(2.0 ** -126)))
    return torch.exp2(e - 7)


def reference(q, k, v, do, heads, scale, causal):
    """fp64 o, lse and, given do, dq, dk, dv per image, with bounds derived from the arithmetic the kernels do:

    * P's relative error: S = scale·Q·Kᵀ is a dh-long fp32 dot product, at most u32·(dh + 1)·scale·Σ|q·k| nats off;
      the exp2 argument s - m and the stored LSE add u32·2|lse|, ex2 / lg2 2^-21:  δp_ij.
    * O (elementwise): P rounded to bf16 (UB) and M-long fp32 sums (M·u32) on P·|V|, δp on P·|V|, the output's bf16
      rounding (1 ulp): o_bound = ulp(o) + 2·((UB + M·u32)·(P|V|) + (P·δp)|V|).
    * LSE (per row): lse_bound = 2·(Σ_j P_ij δp_ij + M·u32 + 2^-21).
    * dS_ij = P_ij (dP_ij - D_i) is off by e_ij = P_ij·(ε_ij + δp_ij |dP_ij - D_i|), ε_ij = u32·(|dP| + |D| +
      (dh + 1)·(Σ|dO·V| + Σ|dO·O|)) (the dh-long fp32 dot products dP and D), and is rounded to bf16 (UB).  Per row, as
      an RMS over the row's elements (|t| = a row's per-element RMS): dQ row i gets scale·Σ_j e_ij |k_j| (D_i and the
      row's LSE are shared by the row, so its errors add up) + scale·UB·sqrt(Σ_j dS_ij² |k_j|²); dK row j
      scale·sqrt(Σ_i e_ij² |q_i|²) + scale·UB·sqrt(Σ_i dS_ij² |q_i|²) (rows independent); dV row j
      sqrt(Σ_i (P_ij δp_ij)² |dO_i|²) + UB·sqrt(Σ_i P_ij² |dO_i|²).
    Returns (o, lse, dq, dk, dv), (o_bound, lse_bound), {"dq", "dk", "dv": per-row noise (B, rows, heads)}."""
    B, N, C = q.shape
    M = k.shape[1]
    dh = C // heads
    z = lambda *s: torch.empty(*s, dtype=F64, device="cuda")
    o_r, lse_r, ob, lb = z(B, N, C), z(B, heads, N), z(B, N, C), z(B, heads, N)
    grads, noise = None, None
    if do is not None:
        grads = [z(B, N, C), z(B, M, C), z(B, M, C)]
        noise = {"dq": z(B, N, heads), "dk": z(B, M, heads), "dv": z(B, M, heads)}
    hv = lambda t: t.reshape(1, -1, heads, dh).transpose(1, 2)          # (1, H, T, dh)
    rms = lambda t: t.pow(2).mean(-1, keepdim=True).sqrt()                 # (1, H, T, 1)
    tr = lambda t: t[0, :, :, 0].T                                         # (T, H)
    for b in range(B):
        qd, kd, vd = (H._d(t[b:b + 1]) for t in (q, k, v))
        o, lse, p = H._attn_ref_fwd(qd, kd, vd, heads, scale, causal)
        o_r[b], lse_r[b] = o[0], lse[0]
        qh, kh, vh = hv(qd), hv(kd), hv(vd)
        dp_ = U32 * (scale * (dh + 1) * (qh.abs() @ kh.abs().transpose(-1, -2)) + 2 * lse.abs()[..., None]) + 2.0 ** -21
        pdp = p * dp_
        del dp_
        va = vh.abs()
        obh = ulp_bf16(hv(o)) + 2 * ((UB + M * U32) * (p @ va) + pdp @ va)
        ob[b] = obh.transpose(1, 2).reshape(N, C)
        lb[b] = (2 * (pdp.sum(-1) + M * U32 + 2.0 ** -21))[0]
        if do is not None:
            o16 = o.to(torch.bfloat16).double()                            # the backward is given bf16 O
            dod = H._d(do[b:b + 1])
            gq, gk, gv = H._attn_ref_bwd(qd, kd, vd, o16, dod, p, heads, scale)
            grads[0][b], grads[1][b], grads[2][b] = gq[0], gk[0], gv[0]
            doh, oh = hv(dod), hv(o16)
            dp = doh @ vh.transpose(-1, -2)
            D = (doh * oh).sum(-1, keepdim=True)
            eps = U32 * (dp.abs() + D.abs() + (dh + 1) * (doh.abs() @ va.transpose(-1, -2)
                                                          + (doh * oh).abs().sum(-1, keepdim=True)))
            e = p * eps + pdp * (dp - D).abs()
            del eps
            ds2 = (p * (dp - D)).pow(2)
            qr, kr, dor = rms(qh), rms(kh), rms(doh)
            noise["dq"][b] = tr(scale * (e @ kr + UB * (ds2 @ kr.pow(2)).sqrt()))
            noise["dk"][b] = tr(scale * ((e.pow(2).transpose(-1, -2) @ qr.pow(2)).sqrt()
                                         + UB * (ds2.transpose(-1, -2) @ qr.pow(2)).sqrt()))
            noise["dv"][b] = tr((pdp.pow(2).transpose(-1, -2) @ dor.pow(2)).sqrt()
                                + UB * (p.pow(2).transpose(-1, -2) @ dor.pow(2)).sqrt())
            del e, ds2, dp, D
        del o, lse, p, pdp, va
    return (o_r, lse_r) + (tuple(grads) if grads else ()), (ob, lb), noise


def elementwise(got, ref, bound):
    """(worst |got - ref| / bound, flat index of the worst); non-finite got counts as infinitely far."""
    r = (got.double() - ref).abs() / bound
    r = torch.where(torch.isfinite(r), r, torch.full_like(r, math.inf)).reshape(-1)
    i = int(r.argmax())
    return r[i].item(), i


def row_error(got, ref, heads, noise, bound):
    """Worst per-(token, head) RMS error relative to that row's own ref RMS, over the rows whose derived noise is below
    half the per-row bound (LOCAL x bound) of their RMS; the number of such rows and the (flat row, head) of the
    worst."""
    dh = got.shape[-1] // heads
    e = (got.double() - ref).reshape(-1, heads, dh).pow(2).mean(-1).sqrt()
    r = ref.reshape(-1, heads, dh).pow(2).mean(-1).sqrt()
    m = noise.reshape(-1, heads) < H.LOCAL * bound / 2 * r
    rel = torch.where(m, e / r.clamp_min(1e-300), torch.zeros_like(e))
    rel = torch.where(torch.isfinite(rel), rel, torch.full_like(rel, math.inf))
    i = int(rel.argmax())
    return rel.max().item(), int(m.sum()), divmod(i, heads)


# ---------------------------------------------------------------------------------------------------------------------
# one case
# ---------------------------------------------------------------------------------------------------------------------
def placements(M, kb):
    """key 0, the last and first keys around every kb-key boundary, the first key of the last block, and M - 1"""
    s = {0, M - 1, (M - 1) // kb * kb}
    for e in range(kb, M, kb):
        s |= {e - 1, e}
    return sorted(s)


def run_case(label, B, N, M, heads, dh, *, causal=False, small=False, mode="sink", sinks=None, shared_dir=False,
             delta=None, seed=0):
    """O elementwise and the LSE per row against their derived bounds (reference()), and dQ / dK / dV against the
    replay's tensor and block bounds plus the per-row bound.  The sink keys' V rows are zero, so a peaked row's O is
    made only of the keys far below its max: weight wrongly given to them shows up against an O near 0."""
    from e4t_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(seed)
    scale = dh ** -0.5
    q, k, peaked, sinks = peaked_qk(B, N, M, heads, dh, scale, g, sinks=sinks, mode=mode, shared_dir=shared_dir,
                                    delta=delta)
    q, k = q.to(torch.bfloat16), k.to(torch.bfloat16)
    v = torch.randn(B, M, heads * dh, generator=g, device="cuda").to(torch.bfloat16)
    if mode == "sink":
        for i, j in enumerate(sinks):
            b, h = divmod(i, heads)
            v[b, j, h * dh:(h + 1) * dh] = 0
    do = torch.randn(B, N, heads * dh, generator=g, device="cuda").to(torch.bfloat16)
    (o_ref, lse_ref, dq_ref, dk_ref, dv_ref), (o_bound, lse_bound), noise = reference(q, k, v, do, heads, scale,
                                                                                      causal)
    if small:
        o, lse = ops.attn_small_fwd(q, k, v, heads, causal=causal)
    else:
        o, lse = ops.attn_fwd(q, k, v, heads)
    # the backward gets the reference O (bf16) and LSE, so it is checked on its own
    o16, lse32 = o_ref.to(torch.bfloat16), lse_ref.float()
    dq, dk, dv = ops.attn_bwd(q, k, v, o16, do, lse32, heads, causal=causal)
    torch.cuda.synchronize()
    if mode == "sink":
        dmin, sig = achieved(q, k, heads, scale, peaked, sinks, causal)
        reached = f"Δ ≥ {dmin:.1f} nats, flat-row σ {sig[0]:.2f} to {sig[1]:.2f}"
    else:
        reached = f"{mode} ramp of {8.0 * M / 128 + 8.0:.0f} nats"
    failures = []
    lw, li = elementwise(lse, lse_ref, lse_bound)
    ow, oi = elementwise(o, o_ref, o_bound)
    print(f"[{label}] {reached}; lse worst {lw:.2f}x its per-row bound (at most {lse_bound.max().item():.1e}), "
          f"o worst {ow:.2f}x its elementwise bound")
    if lw > 1:
        failures.append(f"lse (image, head, query) {divmod(li, N)}: {lw:.2f}x its derived bound "
                        f"{lse_bound.reshape(-1)[li].item():.2e}")
    if ow > 1:
        failures.append(f"o element {divmod(oi, heads * dh)}: {ow:.2f}x its derived bound "
                        f"{o_bound.reshape(-1)[oi].item():.2e}")
    for name, got, ref, bound in (("o", o, o_ref, B_O), ("dq", dq, dq_ref, B_GRAD), ("dk", dk, dk_ref, B_GRAD),
                                  ("dv", dv, dv_ref, B_GRAD)):
        finite, glob, worst, where = H.evaluate(H.Check(name, got, ref, bound, block=(64, dh)))
        line = (f"[{label}] {name}: global {glob / bound:.2f}x, worst 64-row block {worst / bound:.2f}x the bound "
                f"(at {where})")
        if not finite:
            failures.append(f"{name} not finite")
        if glob > bound or worst > H.LOCAL * bound:
            failures.append(f"{name}: global {glob:.2e}, block {worst:.2e} at {where} (bound {bound})")
        if name != "o":
            rw, nrows, at = row_error(got, ref, heads, noise[name], bound)
            line += f", worst row {rw / bound:.2f}x over the {nrows} of {got.numel() // dh} rows above their noise (at {at})"
            if rw > H.LOCAL * bound:
                failures.append(f"{name}: row (token, head) {at} error {rw:.2e} > {H.LOCAL * bound:.1e}")
        print(line)
    return failures


@pytest.fixture(autouse=True)
def _clean_env():
    os.environ.pop("E4T_ATTN_WGMMA", None)
    yield
    os.environ.pop("E4T_ATTN_WGMMA", None)


def _sinks_for(B, heads, M, kb):
    pl = placements(M, kb)
    return [pl[i % len(pl)] for i in range(B * heads)], len(pl)


# (label, B, N, M, heads, dh, key-block size of the kernel that runs, E4T_ATTN_WGMMA)
SHAPES = [
    ("self 4096 dh40 wgmma", 8, 4096, 4096, 8, 40, 128, None),
    ("self 4096 dh40 mma.sync", 16, 4096, 4096, 8, 40, 64, "0"),
    ("self 5184 dh40 (576² level 0)", 21, 5184, 5184, 8, 40, 64, None),
    ("ViT-H 257 dh80", 1, 257, 257, 16, 80, 64, None),
    ("cross 4096x77 dh40", 1, 4096, 77, 8, 40, 64, None),
    ("cross 256x77 dh160", 1, 256, 77, 8, 160, 64, None),
    ("self 1024 dh80", 4, 1024, 1024, 8, 80, 64, None),
]


@pytest.mark.parametrize("shape", SHAPES, ids=[s[0] for s in SHAPES])
def test_sink_at_every_block_edge(shape):
    label, B, N, M, heads, dh, kb, wg = shape
    if wg is not None:
        os.environ["E4T_ATTN_WGMMA"] = wg
    sinks, npl = _sinks_for(B, heads, M, kb)
    assert B * heads >= npl, f"{label}: {B * heads} slots for {npl} sink placements"
    failures = run_case(label, B, N, M, heads, dh, sinks=sinks, seed=N + M + dh)
    assert not failures, "\n".join(failures)


def test_text_tower_causal():
    """77² x 12 x 64, causal: attn_small_fwd and the causal fused backward (CLIP text tower); key 0 (the BOS sink every
    query sees) and the other block edges."""
    sinks, _ = _sinks_for(8, 12, 77, 64)
    sinks = [0 if i % 2 == 0 else s for i, s in enumerate(sinks)]
    failures = run_case("text 77 causal dh64", 8, 77, 77, 12, 64, causal=True, small=True, sinks=sinks, seed=77)
    assert not failures, "\n".join(failures)


@pytest.mark.parametrize("mode", ["rise", "fall"])
@pytest.mark.parametrize("wg", [None, "0"], ids=["default", "mma_sync"])
def test_ramp(mode, wg):
    """Logits rising with the key index (the running max moves in every key block, alpha <= e^-8 each time), and
    falling (every block after the first underflows)."""
    if wg is not None:
        os.environ["E4T_ATTN_WGMMA"] = wg
    failures = run_case(f"4096 {mode} ramp {wg or 'default'}", 2, 4096, 4096, 8, 40, mode=mode, seed=3)
    failures += run_case(f"5184 {mode} ramp {wg or 'default'}", 1, 5184, 5184, 8, 40, mode=mode, seed=4)
    assert not failures, "\n".join(failures)


@pytest.mark.parametrize("shape", [("4096 wgmma", 4096, None), ("4096 mma.sync", 4096, "0"), ("5184", 5184, None),
                                   ("257 dh80", 257, None)], ids=lambda s: s[0])
def test_decoy_past_the_last_key(shape):
    """Every image's key 0 is a Δ = 48 sink on a direction its head shares with the other images, so a read of one key
    past M (image b + 1's key 0) doubles the sink's weight in image b's peaked rows: a wrong row, not a 1/M error."""
    label, M, wg = shape
    if wg is not None:
        os.environ["E4T_ATTN_WGMMA"] = wg
    heads, dh = (16, 80) if M == 257 else (8, 40)
    B = 3
    failures = run_case(f"decoy {label}", B, M, M, heads, dh, sinks=[0] * (B * heads), shared_dir=True, delta=48.0,
                        seed=M + 5)
    assert not failures, "\n".join(failures)
