"""The wgmma GEMM engine (csrc/gemm.cu), every kernel it instantiates, bit for bit and element by element.

The engine's control flow and addressing do not depend on the data, so the cases here choose data whose right answer
is known exactly, and any wrong element anywhere fails.

Exact cases.  Operands are bf16 integers in {-2..2}; bias, row-group addend, residual and the seeded start of an
accumulating call are integers; alpha is 1, 0.5, -2 or 0.25.  The generator asserts that for every output the sum of
magnitudes, |alpha|·Σ|a||b| plus every addend, stays below 2²² (so below 2²⁴ after alpha's two fraction bits).  Then
every product and every partial sum is an integer (or a quarter) that fp32 holds exactly, in any order and under any
rounding mode, split-K atomics included.  So an fp32 output must equal the fp64 reference exactly, and a bf16 output
must equal the fp64 reference rounded to fp32 and then to bf16 (round to nearest even).  Every case runs twice and
the two results must be bitwise equal; a case marked `plain` also runs with E4T_GEMM_EPI_PLAIN=0 (the register
epilogue) and must match the staged result bit for bit.  Hardware premise: the H100's bf16 wgmma accumulates
integer-valued fp32 sums below 2²⁴ exactly.  The published tensor-core models (exact products, aligned and truncated
additions) imply it; these cases measure it: on an H100 80GB HBM3 (700 W) every case matched, sums of magnitudes
above 10⁴ and K up to 8192 included, so the cap stays 2²².

Memory.  Every tensor sits in a buffer that is NaN everywhere else: guard bands before and after, row-pitch gaps and
batch-stride gaps.  Outputs start NaN (an accumulating call's output starts at its integer seed), and while a call
runs, the torch.empty / empty_like / zeros that ops uses return views into such buffers.  After every call the bits
outside each logical extent, and every input's bits, must be unchanged; a read of padding poisons the result, an
unwritten element stays NaN, and a write past N, past M or into a gap is seen.

Coverage rule.  `dispatch()` restates the host dispatch of launch_gemm, conv3x3_impl and e4t_conv3x3_wgrad: which
instantiation (BN, AMN, BMN, IM2COL, RES_TMA) and which epilogue a case reaches.  The CPU test
test_exact_matrix_covers_every_kernel asserts that the exact cases reach every one of the 47 instantiations in every
output mode it can receive, and each GPU case asserts, from the kernel name torch.profiler records, that the library
launched the instantiation the restatement predicts.  A new tile width or epilogue fails the CPU test until cases for
it exist.

Real-valued cases (precision, which integer data cannot see).  randn operands, fractional fp32 bias and row-group
values, a bf16 residual and alpha = 0.7.  With S = |A|·|B|ᵀ (fp64) and T = |alpha|·S + |bias| + |rowgroup| +
|residual| (+ |seed| when accumulating), each element must satisfy
    fp32: |got - ref| <= |alpha|·2K·2⁻²⁴·S + k_e·2⁻²⁴·T
    bf16: the fp32 bound E plus 2⁻⁸·(|ref| + E)
2K: at most one fp32 ulp of the running magnitude per accumulation step; k_e: one rounding per epilogue operation
(alpha, each addend, each atomic add of a split).  The epilogues round every product and sum separately (no FFMA in
the engine's SASS), so the staged and register epilogues must also agree bit for bit at alpha = 0.7.
"""
import re

import pytest
import torch
import torch.nn.functional as F

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
NAN = float("nan")
GUARD = 64                 # NaN elements before and after every buffer (128 / 256 bytes: keeps 16-byte alignment)
SMS = 132                  # H100 SXM: the engine's pick_bn / auto_splits size rounds by it
U32 = 2.0 ** -24
KMAJ = (64, 96, 128, 160, 192, 224, 256)   # tile widths of K-major B
MNMAJ = (64, 128, 192, 256)                # MN-major B
M_TAILS = (1, 63, 64, 65, 127, 129, 1000)  # 65: 1 row for the second MMA warpgroup; 63, 64, 129: none; 1000: 40
K_TAILS = (8, 72, 520, 1232)


def _cdiv(a, b):
    return -(-a // b)


def _up(a, b):
    return _cdiv(a, b) * b


# ---------------------------------------------------------------------------------------------------------------------
# host dispatch, restated (csrc/gemm.cu: pick_bn, auto_splits, launch_gemm, e4t_gemm_bf16, conv3x3_impl,
# e4t_conv3x3_s2*_bf16, e4t_conv3x3_wgrad)
# ---------------------------------------------------------------------------------------------------------------------
def pick_bn(N, mtb, b_mn, force_bn, kper=16, residual=False, atomic=False):
    """(BN, cost) as pick_bn chooses it."""
    if force_bn > 0:
        return force_bn, 0.0
    best, best_cost = 0, 1e30
    for bn in range(256, 63, -(64 if b_mn else 32)):
        rounds = float(_cdiv(_cdiv(N, bn) * mtb, SMS))
        cost = rounds * (kper * (160.0 + 3.9 * bn) + (600.0 + 12.0 * bn * (2.0 if residual else 1.0)
                                                      * (4.0 if atomic else 1.0)))
        if cost < best_cost - 1e-6:
            best, best_cost = bn, cost
    return best, best_cost


def auto_splits(N, mtb, b_mn, kchunks):
    best, best_cost = 1, 1e30
    for sp in range(1, min(kchunks, 64) + 1):
        kper = _cdiv(kchunks, sp)
        if _cdiv(kchunks, kper) != sp:
            continue
        c = pick_bn(N, mtb * sp, b_mn, 0, kper, False, True)[1]
        if c < best_cost - 1e-6:
            best, best_cost = sp, c
    return best


def epilogue(mode, N, batch, ldo, obs, mis_bytes, plain):
    """'bf16' / 'f32' / 'add' (staged, TMA store or reduce-add), or the register epilogue 'reg-<mode>[-pair|-scalar]'."""
    esz = 2 if mode == "bf16" else 4
    if (not plain and mis_bytes % 16 == 0 and N * esz % 16 == 0 and ldo * esz % 16 == 0 and ldo >= N
            and (batch == 1 or (obs > 0 and obs * esz % 16 == 0))):
        return mode
    if mode == "add":
        return "reg-add"
    pair = ldo % 2 == 0 and (batch == 1 or obs % 2 == 0) and mis_bytes % (2 * esz) == 0
    return f"reg-{mode}-" + ("pair" if pair else "scalar")


def conv_tiled_fits(H, W):
    if W > 128:
        return W % 128 == 0
    if 128 % W:
        return False
    return H % (128 // W) == 0 if H * W >= 128 else 128 % (H * W) == 0


class Case:
    """One call: kind 'gemm' / 'conv' / 'wgrad' and its parameters (see the constructors below)."""

    def __init__(self, name, kind, **p):
        self.name, self.kind, self.p = name, kind, p

    def __getattr__(self, k):
        try:
            return self.__dict__["p"][k]
        except KeyError:
            raise AttributeError(k) from None

    def __repr__(self):
        return self.name

    def dispatch(self, plain=False):
        """((AMN, BMN, IM2COL, RES_TMA), BN, epilogue) the call reaches."""
        if self.kind == "gemm":
            return self._gemm_dispatch(plain)
        if self.kind == "conv":
            return self._conv_dispatch(plain)
        H, W, Cin, Cout = self.H, self.W, self.Cin, self.Cout
        im2col = not (W <= 64 and 64 % W == 0 and H * W % 64 == 0 and H % (64 // W) == 0)
        bn = 256 if Cin >= 256 else 192 if Cin >= 192 else 128 if Cin >= 128 else 64
        return (1, 1, int(im2col), 0), bn, epilogue("add", Cin, 9, Cin, Cout * Cin, 0, plain)

    def _gemm_dispatch(self, plain):
        M, N, K, mode = self.M, self.N, self.K, self.mode
        batch = self.bt or 1
        kchunks, m_tiles = _cdiv(K, 64), _cdiv(M, 128)
        splits = self.splits
        addends = self.bias or self.rpg or self.res is not None
        if splits == 0 and mode == "add" and self.force_bn <= 0 and not addends:
            splits = auto_splits(N, m_tiles * batch, self.b_mn, kchunks)
        splits = max(1, min(splits, kchunks))
        kper = _cdiv(kchunks, splits)
        splits = _cdiv(kchunks, kper)
        bn = pick_bn(N, m_tiles * batch * splits, self.b_mn, self.force_bn, kper, self.res is not None,
                     mode == "add")[0]
        lay = self.layout()
        esz = 2 if mode == "bf16" else 4
        epi = epilogue(mode, N, batch, lay["ldo"], lay["obs"], lay["out_mis"] * esz, plain)
        res_tma = False
        if epi == "bf16" and self.res is not None and not self.a_mn and not self.b_mn:
            ldr, rbs, rmis = lay["ldr"], lay["rbs"], lay["res_mis"]
            res_tma = rmis * 2 % 16 == 0 and ldr * 2 % 16 == 0 and ldr >= N and (
                batch == 1 or (rbs > 0 and rbs * 2 % 16 == 0))
        return (int(self.a_mn), int(self.b_mn), 0, int(res_tma)), bn, epi

    def _conv_dispatch(self, plain):
        s = 2 if self.entry == "conv3x3_s2" else 1
        H, W = _cdiv(self.H, s), _cdiv(self.W, s)
        if self.entry == "conv3x3":
            im2col = False
        elif self.entry == "conv3x3_im2col":
            im2col = True
        else:
            odd = self.pad_lo == 1 and (self.H % 2 or self.W % 2)
            im2col = bool(odd) or not conv_tiled_fits(self.H // 2, self.W // 2)
        Cout = self.Cout
        bn = pick_bn(Cout, _cdiv(self.B * H * W, 128), False, self.force_bn, 9 * self.Cin // 64,
                     self.res is not None, False)[0]
        epi = epilogue(self.mode, Cout, 1, Cout, 0, 0, plain)
        res_tma = epi == "bf16" and self.res is not None and Cout * 2 % 16 == 0
        return (0, 0, int(im2col), int(res_tma)), bn, epi

    def layout(self):
        """Row pitches, batch strides and base offsets (elements) of a gemm case's tensors."""
        M, N, K, bt = self.M, self.N, self.K, self.bt
        lay = dict(lda=_up(M if self.a_mn else K, 8) + self.lda_pad, ldb=_up(N if self.b_mn else K, 8) + self.ldb_pad,
                   ldo=_up(N, self.ldo_align) + self.ldo_pad, out_mis=self.out_mis, ldr=0, rbs=0, res_mis=0)
        lay["obs"] = M * lay["ldo"] + self.bpad if bt else 0
        if self.res is not None:
            lay["ldr"] = _up(N, 8) + (72 if self.res == "slice" else 0)
            lay["res_mis"] = {"slice": 16, "mis": 4}.get(self.res, 0)
            lay["rbs"] = M * lay["ldr"] + self.bpad if bt and self.res != "shared" else 0
        return lay


def G(name, M, N, K, *, a_mn=False, b_mn=False, mode="bf16", bt=0, a3=True, b3=True, lda_pad=0, ldb_pad=0, bpad=0,
      ldo_align=None, ldo_pad=0, out_mis=0, bias=True, rpg=None, res=None, alpha=1.0, splits=1,
      force_bn=0, plain=False, acc_calls=1, big=None):
    """A gemm case.  res: None, 'tma' (dense pitch, aligned), 'slice' (column slice of a wider buffer), 'mis' (8 bytes
    off 16: read from global memory), 'shared' (2-D residual of a batched call).  big: fp32-sized addends (up to 4095,
    not bf16-representable) instead of small ones; default for fp32 outputs, where they cannot hide an error."""
    if ldo_align is None:
        ldo_align = 8 if mode == "bf16" else 4
    return Case(name, "gemm", M=M, N=N, K=K, a_mn=a_mn, b_mn=b_mn, mode=mode, bt=bt, a3=a3, b3=b3, lda_pad=lda_pad,
                ldb_pad=ldb_pad, bpad=bpad, ldo_align=ldo_align, ldo_pad=ldo_pad, out_mis=out_mis,
                bias=bias, rpg=rpg, res=res, alpha=alpha, splits=splits, force_bn=force_bn, plain=plain,
                acc_calls=acc_calls, big=(mode != "bf16") if big is None else big)


def C(name, entry, B, H, W, Cin, Cout, *, mode="bf16", bias=True, temb=False, res=None, force_bn=0, plain=False,
      pad_lo=1, big=None):
    return Case(name, "conv", entry=entry, B=B, H=H, W=W, Cin=Cin, Cout=Cout, mode=mode, bias=bias, temb=temb,
                res=res, force_bn=force_bn, plain=plain, pad_lo=pad_lo, big=(mode != "bf16") if big is None else big)


def Wg(name, B, H, W, Cin, Cout, *, plain=False):
    return Case(name, "wgrad", B=B, H=H, W=W, Cin=Cin, Cout=Cout, plain=plain, mode="add", big=False)


# ---------------------------------------------------------------------------------------------------------------------
# the exact case matrix
# ---------------------------------------------------------------------------------------------------------------------
ALPHAS = (1.0, 0.5, -2.0, 0.25)
SPLITS = (1, 3, 2, 7)


def _n_tail(bn, i, mode="bf16"):
    """N not a multiple of 32 or BN (of 8 either, for fp32 outputs), as the staged epilogue takes it: below BN, 8 (4)
    columns past a whole tile, a partial second and third tile."""
    return (bn - 24, bn + 8, 2 * bn + 40, 3 * bn - 56)[i % 4] - (0 if mode == "bf16" else 4)


def exact_cases():
    cs = []
    # every width of the four gemm instantiation families in every output mode; M, N and K tails, padded pitches
    for (a_mn, b_mn), widths in (((0, 0), KMAJ), ((1, 0), KMAJ), ((0, 1), MNMAJ), ((1, 1), MNMAJ)):
        for i, bn in enumerate(widths):
            for j, mode in enumerate(("bf16", "f32", "add")):
                t = i + 2 * j
                M, N, K = M_TAILS[t % 7], _n_tail(bn, i + j, mode), K_TAILS[(i + j) % 4]
                res = None if mode == "bf16" and not (a_mn or b_mn) else ("tma", "slice", "mis", None)[t % 4]
                splits = SPLITS[t % 4] if mode == "add" else 1
                add = splits == 1        # split-K takes no addends
                cs.append(G(f"gemm_a{a_mn}b{b_mn}_bn{bn}_{mode}_M{M}N{N}K{K}", M, N, K, a_mn=a_mn, b_mn=b_mn,
                            mode=mode, lda_pad=8 * (t % 3), ldb_pad=16 * ((t + 1) % 2), ldo_pad=8 * (t % 2),
                            bias=add, rpg=(1, 7, 100, 256, M, None)[t % 6] if add else None, res=res if add else None,
                            alpha=ALPHAS[t % 4], splits=splits, force_bn=bn,
                            plain=(a_mn, b_mn) == (0, 0) or i == 0, big=(mode != "bf16") or i % 2 == 1))
        # odd N below BN with a padded pitch: the row does not end on 16 bytes, so the register epilogue (pair stores
        # and the scalar last column)
        for j, mode in enumerate(("bf16", "f32")):
            bn = widths[-1 - j]
            N = bn - 5 - 2 * j
            cs.append(G(f"gemm_a{a_mn}b{b_mn}_oddN_{mode}_M1000N{N}", 1000, N, 520, a_mn=a_mn, b_mn=b_mn, mode=mode,
                        ldo_pad=8, rpg=7, res="mis", alpha=0.5, force_bn=bn, big=True))
    # the TMA-loaded residual (RES_TMA), every width: dense and column-slice residuals
    for i, bn in enumerate(KMAJ):
        M, N, K = M_TAILS[(i + 3) % 7], _n_tail(bn, i + 1), K_TAILS[i % 4]
        cs.append(G(f"gemm_restma_bn{bn}_M{M}N{N}K{K}", M, N, K, res=("tma", "slice")[i % 2], rpg=(7, 100, M)[i % 3],
                    alpha=ALPHAS[i % 4], force_bn=bn, plain=True, big=i % 2 == 0, lda_pad=8 * (i % 2)))
    # register epilogue reached through the output address: 8 bytes off 16 (pair stores), 2 bytes off (scalar
    # stores), an odd fp32 pitch (scalar), an accumulating output 8 bytes off (atomics)
    cs += [
        G("gemm_reg_bf16_8B", 1000, 328, 520, out_mis=4, force_bn=128, res="mis", rpg=7, big=True),
        G("gemm_reg_bf16_2B", 129, 201, 72, out_mis=1, force_bn=96, rpg=100, big=True),
        G("gemm_reg_f32_8B", 1000, 200, 520, mode="f32", out_mis=2, force_bn=64, res="tma", rpg=7),
        G("gemm_reg_f32_oddpitch", 65, 199, 72, mode="f32", ldo_align=1, force_bn=224, rpg=7, alpha=-2.0),
        G("gemm_reg_add_8B", 127, 136, 1232, mode="add", out_mis=2, splits=3, bias=False, force_bn=160),
        G("gemm_reg_mn_bf16_2B", 1000, 136, 520, a_mn=True, b_mn=True, out_mis=1, force_bn=128, big=True),
        G("gemm_reg_mn_f32_8B", 63, 320, 72, b_mn=True, mode="f32", out_mis=2, force_bn=192, res="mis"),
    ]
    # batched: both operands, a shared 2-D B, a shared 2-D A; output / residual / operand batch strides with gaps
    cs += [
        G("gemm_batched_both_restma", 520, 320, 256, bt=3, bpad=64, res="tma", rpg=100, force_bn=160, plain=True,
          big=True),
        G("gemm_batched_both_f32", 200, 76, 72, bt=2, bpad=8, mode="f32", res="slice", force_bn=96, plain=True),
        G("gemm_batched_sharedB_mn", 129, 200, 520, bt=3, b3=False, a_mn=True, bpad=16, mode="f32", force_bn=64,
          plain=True),
        G("gemm_batched_sharedA_mn", 65, 256, 72, bt=2, a3=False, b_mn=True, bpad=8, res="shared", force_bn=256,
          plain=True),
        G("gemm_batched_add", 64, 192, 1232, bt=2, a_mn=True, b_mn=True, bpad=32, mode="add", splits=3, bias=False,
          force_bn=192),
    ]
    # split-K: auto_splits (weight-gradient shape), two accumulating calls into a seeded output; natural pick_bn
    cs += [
        G("gemm_auto_splits", 320, 640, 8192, a_mn=True, b_mn=True, mode="add", splits=0, bias=False),
        G("gemm_acc_twice", 1000, 320, 520, mode="add", splits=3, acc_calls=2, bias=False, force_bn=224, plain=True),
        G("gemm_acc_twice_addends", 1000, 320, 520, mode="add", acc_calls=2, rpg=256, res="slice", force_bn=96),
        G("gemm_pick_bn_ff", 2048, 1280, 640, res="tma", big=True),
    ]
    # launch size: one tile; many tiles per CTA (ring and residual-barrier phases wrap)
    cs += [
        G("gemm_one_tile", 128, 128, 64, force_bn=128, plain=True),
        G("gemm_many_tiles_restma", 65536, 320, 72, res="tma", rpg=4096, big=True),
        G("gemm_many_tiles_f32", 65536, 320, 72, mode="f32", rpg=256, force_bn=64),
    ]
    # convolutions: tiled and im2col loads (tiles spanning rows and images), every width with and without residual,
    # Cout not a multiple of BN, temb row-group across image boundaries inside a tile, stride 2 with pad 1 / 0
    couts = {64: 96, 96: 160, 128: 200, 160: 168, 192: 320, 224: 232, 256: 320}
    for i, bn in enumerate(KMAJ):
        B, H, W = ((2, 24, 40), (3, 9, 13))[i % 2]
        cin = (64, 128)[i % 2]
        cs.append(C(f"conv_im2col_bn{bn}_{B}x{H}x{W}", "conv3x3_im2col", B, H, W, cin, couts[bn], temb=True,
                    force_bn=bn, plain=i < 2, big=i % 2 == 1))
        cs.append(C(f"conv_im2col_f32_bn{bn}_{B}x{H}x{W}", "conv3x3_im2col", B, H, W, cin, couts[bn], mode="f32",
                    temb=i % 2 == 0, res="r" if i % 3 == 0 else None, force_bn=bn))
        cs.append(C(f"conv_im2col_restma_bn{bn}_{B}x{W}x{H}", "conv3x3_im2col", B, W, H, cin, couts[bn], temb=True,
                    res="r", force_bn=bn, plain=i == 3, big=i % 2 == 0))
    cs += [
        C("conv_tiled_32x32_cout96", "conv3x3", 2, 32, 32, 64, 96, temb=True, force_bn=64, plain=True),
        C("conv_tiled_8x8_imgs_per_tile", "conv3x3", 3, 8, 8, 128, 320, mode="f32", temb=True, force_bn=256),
        C("conv_tiled_restma_16x16", "conv3x3", 2, 16, 16, 64, 192, temb=True, res="r", big=True),
        C("conv_tiled_wide_4x256", "conv3x3", 1, 4, 256, 64, 64, res="r", force_bn=64),
        C("conv_s2_even_16x16", "conv3x3_s2", 2, 16, 16, 64, 96, force_bn=64, big=True),
        C("conv_s2_odd_9x13", "conv3x3_s2", 2, 9, 13, 128, 320, force_bn=256),
        C("conv_s2_odd_even_9x16", "conv3x3_s2", 1, 9, 16, 64, 128),
        C("conv_s2_pad0_16x16", "conv3x3_s2", 2, 16, 16, 64, 192, pad_lo=0, force_bn=192, big=True),
        C("conv_s2_pad0_24x40", "conv3x3_s2", 1, 24, 40, 128, 160, pad_lo=0, force_bn=160),
    ]
    # weight gradients: tiled (8x8, 16x16, 64x64) and im2col (odd, 24 x 40); Cin 64 / 128 / 192 / 320 gives BN 64 /
    # 128 / 192 / 256 (320: an N tail), Cout 64 / 192 / 320 gives M tails
    cs += [
        Wg("wgrad_tiled_8x8", 2, 8, 8, 64, 192),
        Wg("wgrad_tiled_16x16", 1, 16, 16, 128, 320, plain=True),
        Wg("wgrad_tiled_64x64", 1, 64, 64, 320, 64),
        Wg("wgrad_im2col_9x13_cin64", 3, 9, 13, 64, 320),
        Wg("wgrad_im2col_24x40_cin128", 2, 24, 40, 128, 64, plain=True),
        Wg("wgrad_im2col_9x13_cin192", 1, 9, 13, 192, 192),
        Wg("wgrad_im2col_24x40_cin320", 1, 24, 40, 320, 320),
    ]
    return cs


EXACT = exact_cases()


def instantiations():
    """The 47 kernels gemm.cu builds: launch_gemm_bn's template families and their widths."""
    fams = {(0, 0, 0, 0): KMAJ, (0, 0, 0, 1): KMAJ, (0, 0, 1, 0): KMAJ, (0, 0, 1, 1): KMAJ, (1, 0, 0, 0): KMAJ,
            (0, 1, 0, 0): MNMAJ, (1, 1, 0, 0): MNMAJ, (1, 1, 1, 0): MNMAJ}
    return {(f, bn) for f, ws in fams.items() for bn in ws}


def staged_modes(fam):
    """Output modes the staged epilogue of a family receives: RES_TMA only bf16; the im2col weight gradient only the
    fp32 reduce-add; the im2col forward convolution bf16 / fp32; the gemm families all three."""
    if fam[3]:
        return {"bf16"}
    if fam == (1, 1, 1, 0):
        return {"add"}
    if fam[2]:
        return {"bf16", "f32"}
    return {"bf16", "f32", "add"}


REG_MODES = {"reg-bf16-pair", "reg-bf16-scalar", "reg-f32-pair", "reg-f32-scalar", "reg-add"}


def test_exact_matrix_covers_every_kernel():
    """CPU: the exact cases reach all 47 instantiations in every staged output mode each receives, the register
    epilogue at every K-major width and in every family that has one, and every register store kind through the
    output address alone."""
    reached, natural = {}, set()
    for c in EXACT:
        fam, bn, epi = c.dispatch()
        reached.setdefault((fam, bn), set()).add(epi)
        if epi.startswith("reg-"):
            natural.add(epi)
        if c.plain:
            pfam, pbn, pepi = c.dispatch(plain=True)
            reached.setdefault((pfam, pbn), set()).add(pepi)
    want = instantiations()
    assert len(want) == 47
    assert set(reached) <= want, sorted(set(reached) - want)
    assert not want - set(reached), f"instantiations without a case: {sorted(want - set(reached))}"
    for (fam, bn), epis in sorted(reached.items()):
        missing = staged_modes(fam) - epis
        assert not missing, f"{fam} BN={bn}: no case in staged mode(s) {sorted(missing)}"
        if fam == (0, 0, 0, 0):
            assert epis & REG_MODES, f"K-major BN={bn}: no register-epilogue case"
    for fam in {f for f, _ in want if not f[3]}:
        assert any(reached[(f, bn)] & REG_MODES for f, bn in reached if f == fam), f"{fam}: no register epilogue"
    assert natural == REG_MODES, f"register stores never reached through the output address: {REG_MODES - natural}"
    print(f"[coverage] {len(EXACT)} exact cases reach {len(reached)} / 47 instantiations")


# ---------------------------------------------------------------------------------------------------------------------
# guarded memory
# ---------------------------------------------------------------------------------------------------------------------
class Guarded:
    """A strided view into a NaN buffer; snap() records every bit, intact() compares (everything, or only what lies
    outside the view)."""

    def __init__(self, shape, stride, dtype, mis=0, device="cuda"):
        self.off = GUARD + mis
        span = 1 + sum((s - 1) * st for s, st in zip(shape, stride))
        self.buf = torch.full((self.off + span + GUARD,), NAN, dtype=dtype, device=device)
        self.t = self.buf.as_strided(tuple(shape), tuple(stride), self.off)
        self.outside = torch.ones(self.buf.shape, dtype=torch.bool, device=device)
        self.outside.as_strided(tuple(shape), tuple(stride), self.off).fill_(False)
        self.snap()

    @classmethod
    def dense(cls, shape, dtype, device="cuda"):
        stride, s = [], 1
        for d in reversed(shape):
            stride.insert(0, s)
            s *= d
        return cls(shape, stride, dtype, device=device)

    def bits(self):
        return self.buf.view(torch.int16 if self.buf.element_size() == 2 else torch.int32)

    def snap(self):
        self.before = self.bits().clone()

    def intact(self, everything=False):
        b, a = self.bits(), self.before
        return torch.equal(b, a) if everything else torch.equal(b[self.outside], a[self.outside])


class _Poison:
    """Stands in for `torch` inside ops while a call runs: empty / empty_like / zeros return views into NaN-guarded
    buffers (empty: NaN inside too), recorded in `made`."""

    def __init__(self, real):
        self._real, self.made = real, []

    def __getattr__(self, n):
        return getattr(self._real, n)

    def _new(self, shape, dtype, fill):
        g = Guarded.dense(tuple(shape), dtype or F32)
        if fill is not None:
            g.t.fill_(fill)
            g.snap()
        self.made.append(g)
        return g.t

    @staticmethod
    def _shape(size):
        return size[0] if len(size) == 1 and isinstance(size[0], (tuple, list, torch.Size)) else size

    def empty(self, *size, dtype=None, device=None, **kw):
        return self._new(self._shape(size), dtype, None)

    def empty_like(self, t, dtype=None, **kw):
        return self._new(t.shape, dtype or t.dtype, None)

    def zeros(self, *size, dtype=None, device=None, **kw):
        return self._new(self._shape(size), dtype, 0.0)


def _kernel(names):
    """(AMN, BMN, IM2COL, RES_TMA), BN of the engine kernels in a list of profiled kernel names."""
    found = set()
    for n in names:
        m = re.search(r"e4t_gemm_kernel<\s*(\d+),\s*(\d+),\s*(\d+),\s*(\w+),\s*(\w+)\s*>", n)
        if m:
            b = [int(m.group(i)) for i in (2, 3)] + [int(m.group(i) in ("true", "1")) for i in (4, 5)]
            found.add((tuple(b), int(m.group(1))))
    return found


def _run(fn, monkeypatch, plain=False, profile=False):
    """fn() with ops' allocations poisoned; (result, poisoned allocations, engine kernels launched or None)."""
    from e4t_b200 import ops
    if plain:
        monkeypatch.setenv("E4T_GEMM_EPI_PLAIN", "0")
    else:
        monkeypatch.delenv("E4T_GEMM_EPI_PLAIN", raising=False)
    real = ops.torch
    ops.torch = p = _Poison(real)
    kern = None
    try:
        if profile:
            from torch.profiler import ProfilerActivity
            with torch.profiler.profile(activities=[ProfilerActivity.CUDA]) as prof:
                r = fn()
                torch.cuda.synchronize()
            kern = _kernel(e.name for e in prof.events())
        else:
            r = fn()
        torch.cuda.synchronize()
    finally:
        ops.torch = real
        monkeypatch.delenv("E4T_GEMM_EPI_PLAIN", raising=False)
    return r, p.made, kern


# ---------------------------------------------------------------------------------------------------------------------
# building a case's tensors and its fp64 reference
# ---------------------------------------------------------------------------------------------------------------------
class Data:
    """Integer ('int') or real-valued ('real') fills; `abs` collects the magnitude sum for the exactness check."""

    def __init__(self, kind, seed, big):
        self.kind, self.big = kind, big
        self.g = torch.Generator(device="cuda").manual_seed(seed)

    def operand(self, t, scale=1.0):
        if self.kind == "int":
            t.copy_(torch.randint(-2, 3, t.shape, generator=self.g, device="cuda"))
        else:
            t.copy_(torch.randn(t.shape, generator=self.g, device="cuda") * scale)

    def addend(self, t):
        if self.kind == "int":
            hi = (2048 if t.dtype == BF16 else 4095) if self.big else 8
            t.copy_(torch.randint(-hi, hi + 1, t.shape, generator=self.g, device="cuda"))
        else:
            t.copy_(torch.randn(t.shape, generator=self.g, device="cuda"))


def _d(t):
    return t.detach().to(F64)


def build_gemm(c, data, scale=1.0):
    """Guarded tensors, the ops.gemm call and its fp64 reference and magnitude sums (|alpha|·S, T)."""
    lay = c.layout()
    M, N, K, bt = c.M, c.N, c.K, c.bt
    tens = {}

    def operand(rows, cols, ld, batched):
        if bt and batched:
            g = Guarded((bt, rows, cols), (rows * ld + c.bpad, ld, 1), BF16)
        else:
            g = Guarded((rows, cols), (ld, 1), BF16)
        data.operand(g.t, scale)
        return g

    tens["A"] = operand(*((K, M) if c.a_mn else (M, K)), lay["lda"], c.a3)
    tens["B"] = operand(*((K, N) if c.b_mn else (N, K)), lay["ldb"], c.b3)
    odt = BF16 if c.mode == "bf16" else F32
    oshape = (bt, M, N) if bt else (M, N)
    ostride = (lay["obs"], lay["ldo"], 1) if bt else (lay["ldo"], 1)
    tens["out"] = Guarded(oshape, ostride, odt, mis=lay["out_mis"])
    kw = dict(a_mn=bool(c.a_mn), b_mn=bool(c.b_mn), alpha=c.alpha, splits=c.splits, force_bn=c.force_bn)
    if c.bias:
        tens["bias"] = Guarded((N,), (1,), F32)
        data.addend(tens["bias"].t)
    if c.rpg:
        tens["rowgroup"] = Guarded((_cdiv(M, c.rpg), N), (N, 1), F32)
        data.addend(tens["rowgroup"].t)
        kw["rows_per_group"] = c.rpg
    if c.res is not None:
        if bt and c.res != "shared":
            tens["residual"] = Guarded((bt, M, N), (lay["rbs"], lay["ldr"], 1), BF16, mis=lay["res_mis"])
        else:
            tens["residual"] = Guarded((M, N), (lay["ldr"], 1), BF16, mis=lay["res_mis"])
        data.addend(tens["residual"].t)
    for k in ("bias", "rowgroup", "residual"):
        if k in tens:
            kw[k] = tens[k].t
    if c.mode == "add":
        data.addend(tens["out"].t)
        kw["accumulate"] = True
    out = tens["out"]
    out.snap()
    for t in tens.values():
        t.snap()
    seed_bits = out.bits().clone()

    A, B = _d(tens["A"].t), _d(tens["B"].t)
    A = A.transpose(-1, -2) if c.a_mn else A
    B = B if c.b_mn else B.transpose(-1, -2)
    prod, mag = A @ B, A.abs() @ B.abs()
    ref, T = c.alpha * prod, abs(c.alpha) * mag
    rows = torch.arange(M, device="cuda")
    for k, v in (("bias", lambda t: t), ("rowgroup", lambda t: t[rows // max(c.rpg or 1, 1)]),
                 ("residual", lambda t: t)):
        if k in tens:
            a = v(_d(tens[k].t))
            ref, T = ref + a, T + a.abs()
    ref = ref.expand(oshape)
    T = T.expand(oshape)
    if c.mode == "add":
        init = _d(out.t)
        ref, T = init + c.acc_calls * ref, init.abs() + c.acc_calls * T
    fn_kw = dict(kw, out=out.t)

    def call():
        from e4t_b200 import ops
        out.bits().copy_(seed_bits)
        for _ in range(c.acc_calls):
            ops.gemm(tens["A"].t, tens["B"].t, **fn_kw)
        return out.t.clone()
    return call, tens, ref, T, abs(c.alpha) * mag.expand(oshape)


def build_conv(c, data, scale=1.0):
    from e4t_b200 import ops
    tens = {}
    s = 2 if c.entry == "conv3x3_s2" else 1
    Ho, Wo = _cdiv(c.H, s), _cdiv(c.W, s)
    tens["x"] = Guarded.dense((c.B, c.H, c.W, c.Cin), BF16)
    tens["w9"] = Guarded.dense((9, c.Cout, c.Cin), BF16)
    data.operand(tens["x"].t, scale)
    data.operand(tens["w9"].t, scale)
    kw = dict(force_bn=c.force_bn)
    if c.bias:
        tens["bias"] = Guarded.dense((c.Cout,), F32)
        data.addend(tens["bias"].t)
    if c.temb:
        tens["rowgroup"] = Guarded.dense((c.B, c.Cout), F32)
        data.addend(tens["rowgroup"].t)
    if c.res:
        tens["residual"] = Guarded.dense((c.B, Ho, Wo, c.Cout), BF16)
        data.addend(tens["residual"].t)
    for k in ("bias", "rowgroup", "residual"):
        if k in tens:
            kw[k] = tens[k].t
    for t in tens.values():
        t.snap()
    x = _d(tens["x"].t).permute(0, 3, 1, 2)
    w = _d(tens["w9"].t).view(3, 3, c.Cout, c.Cin).permute(2, 3, 0, 1)
    if c.entry == "conv3x3_s2" and c.pad_lo == 0:
        conv = lambda x_, w_: F.conv2d(F.pad(x_, (0, 1, 0, 1)), w_, stride=2)     # noqa: E731
    else:
        conv = lambda x_, w_: F.conv2d(x_, w_, stride=s, padding=1)               # noqa: E731
    ref, T = conv(x, w).permute(0, 2, 3, 1), conv(x.abs(), w.abs()).permute(0, 2, 3, 1)
    mag = T.clone()
    if "bias" in tens:
        ref, T = ref + _d(tens["bias"].t), T + _d(tens["bias"].t).abs()
    if "rowgroup" in tens:
        r = _d(tens["rowgroup"].t)[:, None, None, :]
        ref, T = ref + r, T + r.abs()
    if "residual" in tens:
        ref, T = ref + _d(tens["residual"].t), T + _d(tens["residual"].t).abs()
    if c.entry == "conv3x3_s2":
        kw.pop("rowgroup", None)
        kw.pop("residual", None)
        call = lambda: ops.conv3x3_s2(tens["x"].t, tens["w9"].t, pad_lo=c.pad_lo, **kw)    # noqa: E731
    else:
        fn = getattr(ops, c.entry)
        call = lambda: fn(tens["x"].t, tens["w9"].t, out_dtype=BF16 if c.mode == "bf16" else F32, **kw)  # noqa: E731
    return call, tens, ref, T, mag


def build_wgrad(c, data):
    from e4t_b200 import ops
    tens = {"x": Guarded.dense((c.B, c.H, c.W, c.Cin), BF16), "dy": Guarded.dense((c.B, c.H, c.W, c.Cout), BF16)}
    data.operand(tens["x"].t)
    data.operand(tens["dy"].t)
    for t in tens.values():
        t.snap()
    x, dy = _d(tens["x"].t).permute(0, 3, 1, 2), _d(tens["dy"].t).permute(0, 3, 1, 2)
    shape = (c.Cout, c.Cin, 3, 3)
    ref = torch.nn.grad.conv2d_weight(x, shape, dy, padding=1).permute(2, 3, 0, 1).reshape(9, c.Cout, c.Cin)
    T = torch.nn.grad.conv2d_weight(x.abs(), shape, dy.abs(), padding=1).permute(2, 3, 0, 1).reshape(9, c.Cout, c.Cin)
    return lambda: ops.conv3x3_wgrad(tens["x"].t, tens["dy"].t), tens, ref, T, T


def build(c, data, scale=1.0):
    if c.kind == "gemm":
        return build_gemm(c, data, scale)
    if c.kind == "conv":
        return build_conv(c, data, scale)
    return build_wgrad(c, data)


def _seed(c):
    return sum(map(ord, c.name)) * 7919 % (1 << 31)


def _run_checked(c, call, tens, monkeypatch, plain=False, profile=False):
    """One call; asserts every input unchanged and every output's outside intact.  Returns (result, kernels)."""
    r, made, kern = _run(call, monkeypatch, plain=plain, profile=profile)
    for name, t in tens.items():
        assert t.intact(everything=name != "out"), f"{c.name}{' plain' if plain else ''}: {name} written " \
                                                   f"{'outside its extent' if name == 'out' else ''}"
    for t in made:
        assert t.intact(), f"{c.name}{' plain' if plain else ''}: output written past its allocation"
    return r.clone(), kern


def _first_mismatch(got, want):
    bad = (got.double() != want.double()) | ~torch.isfinite(got.double())
    idx = tuple(int(i) for i in bad.nonzero()[0])
    return f"{int(bad.sum())} of {bad.numel()} elements differ; first at {idx}: got {got[idx].item()}, " \
           f"want {want[idx].item()}"


@pytest.mark.gpu
@pytest.mark.parametrize("case", EXACT, ids=lambda c: c.name)
def test_exact(case, monkeypatch):
    c = case
    call, tens, ref, T, _ = build(c, Data("int", _seed(c), c.big))
    cap = T.max().item() * 4
    assert cap < 2 ** 24, f"{c.name}: magnitude {cap} reaches 2^24, the sums are not exact"
    want = ref.to(F32)
    if c.mode == "bf16":
        want = want.to(BF16)
    got, kern = _run_checked(c, call, tens, monkeypatch, profile=True)
    fam, bn, epi = c.dispatch()
    assert kern == {(fam, bn)}, f"{c.name}: launched {kern}, the restated dispatch says {(fam, bn)} ({epi})"
    assert got.shape == want.shape and got.dtype == want.dtype
    assert torch.equal(got, want) and bool(torch.isfinite(got).all()), f"{c.name} ({epi}): " + _first_mismatch(got, want)
    again, _ = _run_checked(c, call, tens, monkeypatch)
    assert torch.equal(_bits(again), _bits(got)), f"{c.name}: second run differs"
    if c.plain:
        reg, _ = _run_checked(c, call, tens, monkeypatch, plain=True)
        assert torch.equal(_bits(reg), _bits(got)), \
            f"{c.name} ({c.dispatch(plain=True)[2]} vs staged): " + _first_mismatch(reg, got)


def _bits(t):
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


# ---------------------------------------------------------------------------------------------------------------------
# real-valued cases: per-element fp64 bounds
# ---------------------------------------------------------------------------------------------------------------------
def real_cases():
    cs = []
    modes = ("bf16", "f32", "add")
    for (a_mn, b_mn), widths in (((0, 0), KMAJ), ((1, 0), KMAJ), ((0, 1), MNMAJ), ((1, 1), MNMAJ)):
        for i, bn in enumerate(widths):
            mode = modes[(i + a_mn + 2 * b_mn) % 3]
            M, N, K = (1000, 129, 520, 65)[i % 4], _n_tail(bn, i, mode), (1232, 520, 72)[i % 3]
            kmaj_bf16 = mode == "bf16" and not (a_mn or b_mn)
            cs.append(G(f"real_a{a_mn}b{b_mn}_bn{bn}_{mode}", M, N, K, a_mn=a_mn, b_mn=b_mn, mode=mode,
                        rpg=(7, 100)[i % 2], res=("mis" if kmaj_bf16 and i % 2 else "tma"), alpha=0.7, force_bn=bn,
                        plain=True, lda_pad=8 * (i % 2)))
    for bn in (96, 224):
        cs.append(G(f"real_restma_bn{bn}", 1000, 2 * bn + 17, 1232, res="slice", rpg=100, alpha=0.7, force_bn=bn,
                    plain=True))
    # addends that a bf16 round trip would move by >= 100x the bound: K = 64, operands scaled by 2^-6, |bias| ~ 1
    cs += [
        G("real_addends_f32", 1000, 328, 64, mode="f32", rpg=7, res="tma", alpha=0.7, force_bn=128, plain=True),
        G("real_addends_f32_mn", 129, 320, 64, a_mn=True, b_mn=True, mode="f32", rpg=100, res="mis", alpha=0.7,
          force_bn=64, plain=True),
        G("real_split_add", 1000, 200, 1232, mode="add", splits=3, bias=False, alpha=0.7, force_bn=96),
        G("real_oddN_bf16", 1000, 251, 520, ldo_pad=8, rpg=7, res="mis", alpha=0.7, force_bn=256, plain=True),
        C("real_conv_im2col_f32", "conv3x3_im2col", 2, 24, 40, 128, 200, mode="f32", temb=True, res="r",
          force_bn=128, plain=True),
        C("real_conv_im2col_restma", "conv3x3_im2col", 3, 9, 13, 64, 320, temb=True, res="r", force_bn=256,
          plain=True),
        Wg("real_wgrad_im2col", 2, 24, 40, 320, 192),
    ]
    return cs


REAL = real_cases()


@pytest.mark.gpu
@pytest.mark.parametrize("case", REAL, ids=lambda c: c.name)
def test_real_bound(case, monkeypatch):
    c = case
    scale = 2.0 ** -6 if c.name.startswith("real_addends") else 1.0
    call, tens, ref, T, aS = build(c, Data("real", _seed(c), True), scale)
    got, _ = _run_checked(c, call, tens, monkeypatch)
    K = c.K if c.kind == "gemm" else 9 * c.Cin if c.kind == "conv" else c.B * c.H * c.W
    splits = 1
    if c.kind == "gemm" and c.mode == "add":
        splits = c.splits
    elif c.kind == "wgrad":
        splits = 64      # e4t_conv3x3_wgrad's split count is at most 2 x SMs / base tiles; 64 bounds it here
    alpha_op = 1 if (c.kind == "gemm" and c.alpha != 1.0) else 0
    addends = sum(k in tens for k in ("bias", "rowgroup", "residual"))
    k_acc = 2 * K                                                        # one fp32 ulp per accumulation step
    k_epi = alpha_op + addends + (splits if c.mode == "add" else 0)     # one rounding per epilogue operation
    E = k_acc * U32 * aS + k_epi * U32 * T
    bound = E + (2.0 ** -8 * (ref.abs() + E) if c.mode == "bf16" else 0)
    err = (got.double() - ref).abs()
    assert bool(torch.isfinite(got).all()), f"{c.name}: non-finite output"
    ratio = (err / bound.clamp_min(1e-300)).max().item()
    print(f"[real] {c.name}: k_acc = 2K = {k_acc}, k_epi = {k_epi}: worst |err| / bound = {ratio:.3f}")
    assert ratio <= 1.0, f"{c.name}: worst error {ratio:.2f} x the bound at " \
                         f"{tuple(int(i) for i in (err / bound).flatten().argmax().unsqueeze(0))}"
    if c.plain:
        reg, _ = _run_checked(c, call, tens, monkeypatch, plain=True)
        assert torch.equal(_bits(reg), _bits(got)), f"{c.name}: register epilogue differs from staged at alpha 0.7: " \
                                                    + _first_mismatch(reg, got)


# ---------------------------------------------------------------------------------------------------------------------
# argument checks: ops.gemm's shape checks (CPU tensors: they raise before any pointer is taken) and the library's
# own refusals
# ---------------------------------------------------------------------------------------------------------------------
def _cpu(*shape, dtype=BF16):
    return torch.zeros(shape, dtype=dtype)


@pytest.mark.parametrize("what,kw", [
    ("out 2-D for a batched call", dict(A=_cpu(2, 64, 32), B=_cpu(48, 32), out=_cpu(64, 48))),
    ("out too few rows", dict(A=_cpu(64, 32), B=_cpu(48, 32), out=_cpu(63, 48))),
    ("out too few columns", dict(A=_cpu(64, 32), B=_cpu(48, 32), out=_cpu(64, 40, dtype=F32))),
    ("out batch short", dict(A=_cpu(3, 64, 32), B=_cpu(48, 32), out=_cpu(2, 64, 48))),
    ("accumulate out short", dict(A=_cpu(32, 64), B=_cpu(32, 48), a_mn=True, b_mn=True, out=_cpu(48, 48, dtype=F32),
                                  accumulate=True)),
    ("residual short", dict(A=_cpu(64, 32), B=_cpu(48, 32), residual=_cpu(64, 47))),
    ("residual batch short", dict(A=_cpu(3, 64, 32), B=_cpu(48, 32), residual=_cpu(2, 64, 48))),
    ("bias length", dict(A=_cpu(64, 32), B=_cpu(48, 32), bias=_cpu(40, dtype=F32))),
    ("rowgroup rows", dict(A=_cpu(64, 32), B=_cpu(48, 32), rowgroup=_cpu(2, 48, dtype=F32), rows_per_group=7)),
    ("rowgroup columns", dict(A=_cpu(64, 32), B=_cpu(48, 32), rowgroup=_cpu(10, 40, dtype=F32), rows_per_group=7)),
    ("operand batches disagree", dict(A=_cpu(2, 64, 32), B=_cpu(3, 48, 32))),
])
def test_gemm_shape_checks(what, kw):
    from e4t_b200 import ops
    kw = dict(kw)
    A, B = kw.pop("A"), kw.pop("B")
    with pytest.raises(ValueError, match="gemm: "):
        ops.gemm(A, B, **kw)


@pytest.mark.parametrize("kw", [
    dict(A=_cpu(2, 64, 32), B=_cpu(48, 32), out=_cpu(2, 64, 48)),
    dict(A=_cpu(64, 32), B=_cpu(2, 48, 32), residual=_cpu(64, 48)),
    dict(A=_cpu(2, 64, 32), B=_cpu(2, 32, 48), b_mn=True, residual=_cpu(2, 64, 48), bias=_cpu(48, dtype=F32)),
    dict(A=_cpu(64, 32), B=_cpu(48, 32), rowgroup=_cpu(10, 48, dtype=F32), rows_per_group=7),
    dict(A=_cpu(32, 64), B=_cpu(32, 48), a_mn=True, b_mn=True, out=_cpu(64, 48, dtype=F32), accumulate=True),
], ids=["batched_out", "shared_residual", "batched_residual_bias", "rowgroup", "accumulate"])
def test_gemm_shape_checks_accept(kw):
    """Well-formed calls pass the checks and reach the library, which refuses CPU tensors."""
    from e4t_b200 import _lib, ops
    kw = dict(kw)
    A, B = kw.pop("A"), kw.pop("B")
    with pytest.raises(_lib.E4TError, match="CUDA tensors"):
        ops.gemm(A, B, **kw)


def _gpu(*shape, dtype=BF16):
    return torch.zeros(shape, dtype=dtype, device="cuda")


@pytest.mark.gpu
@pytest.mark.parametrize("what", ["lda % 8", "misaligned operand", "split-K without accumulate", "split-K with a bias",
                                  "force_bn 96 with MN-major B", "conv Cin % 64", "pad 0 at an odd side"])
def test_library_refusals(what):
    from e4t_b200 import _lib, ops
    expect = {"lda % 8": "multiples of 8", "misaligned operand": "16-byte aligned",
              "split-K without accumulate": "split-K requires", "split-K with a bias": "once per split",
              "force_bn 96 with MN-major B": "BN",
              "conv Cin % 64": "Cin must be a multiple of 64", "pad 0 at an odd side": "bad stride/size"}[what]
    with pytest.raises(_lib.E4TError, match=re.escape(expect)):
        if what == "lda % 8":
            ops.gemm(_gpu(64, 36)[:, :32], _gpu(48, 32))
        elif what == "misaligned operand":
            ops.gemm(_gpu(64 * 32 + 8).view(-1)[1:1 + 64 * 32].view(64, 32), _gpu(48, 32))
        elif what == "split-K without accumulate":
            ops.gemm(_gpu(64, 256), _gpu(48, 256), out_dtype=F32, splits=2)
        elif what == "split-K with a bias":
            ops.gemm(_gpu(64, 256), _gpu(48, 256), out=_gpu(64, 48, dtype=F32), accumulate=True, splits=2,
                     bias=_gpu(48, dtype=F32))
        elif what == "force_bn 96 with MN-major B":
            ops.gemm(_gpu(64, 64), _gpu(64, 96), b_mn=True, force_bn=96)
        elif what == "conv Cin % 64":
            ops.conv3x3(_gpu(1, 8, 8, 32), _gpu(9, 64, 32))
        else:
            ops.conv3x3_s2(_gpu(1, 9, 16, 64), _gpu(9, 64, 64), pad_lo=0)
        torch.cuda.synchronize()
