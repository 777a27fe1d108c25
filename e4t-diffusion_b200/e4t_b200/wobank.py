"""WeightOffsets bank: all WeightOffsets projections of a UNet (96 for SD-v1.4) handled by batched kernels.

Per optimisation step the reference evaluates `WeightOffsets.forward` 192 times (e4t/weightoffsets.py:14-23 called
from cross_attention.py:506,516,518 in both UNet passes).  The bank runs the closed form for every projection in
TWO launches (factors, W ⊙ (1+Δ)) at the start of a step, lets every projection GEMM accumulate its weight gradient
straight into one fp32 buffer, and produces all 864 parameter gradients in FOUR launches at the end of backward.

Requires an arena optimiser (engine.FlatAdamW): gradients are written directly into the parameters' `.grad` views.
"""
import ctypes

import torch

from . import _lib
from . import functional as FN
from ._lib import c_int, c_ll, c_void_p, ptr, stream


class _WOProj(ctypes.Structure):
    _fields_ = ([(n, c_void_p) for n in ("W", "v", "w1", "b1", "w2", "b2", "Wc", "bc", "Wr", "br", "fac", "bw", "weff",
                                         "dweff", "dv", "dw1", "db1", "dw2", "db2", "dWc", "dbc", "dWr", "dbr")]
                + [("R", c_int), ("C", c_int)])


class _BankFn(torch.autograd.Function):
    """forward: factors + W_eff for every projection; backward (runs after every projection's dX/dW GEMM, because they
    all take `token` as an input): all WeightOffsets parameter gradients, accumulated into the arena `.grad` views.
    Inputs: the 864 WeightOffsets parameters, then the 96 base projection weights — their gradient
    dW = dW_eff ⊙ (1 + Δ) (SURVEY.md App. A) is returned only when they require grad (tuning_e4t.py trains them)."""

    @staticmethod
    def forward(ctx, bank, *tensors):
        ctx.bank = bank
        bank._launch_forward()
        return torch.zeros(1, device=bank.device, dtype=torch.float32)

    @staticmethod
    def backward(ctx, _dtoken):
        FN.WO_EPOCH += 1
        bank = ctx.bank
        bank._launch_backward()
        n = len(bank.params)
        base = []
        for i, ((lin, wo), off) in enumerate(zip(bank.projs, bank._offsets)):
            if ctx.needs_input_grad[1 + n + i]:
                C, R = lin.out_features, lin.in_features
                with torch.no_grad():
                    base.append(bank.dweff[off:off + C * R].view(C, R) * (1.0 + wo()))
            else:
                base.append(None)
        return (None,) * (1 + n) + tuple(base)


class WOBank:
    def __init__(self, attn_modules):
        self.modules = list(attn_modules)
        assert self.modules
        # the kernels read W, a, bc, vx, vy and the .grad rows as float4 (W_eff stores as 4 bf16) at offsets that are
        # multiples of R or C, and the projection GEMMs need leading dimensions R and C that are multiples of 8
        for i, m in enumerate(self.modules):
            for name in ("to_q", "to_k", "to_v"):
                lin = getattr(m, name)
                if lin.in_features % 8 or lin.out_features % 8:
                    raise ValueError(f"WOBank: attention module {i} ({type(m).__name__}), {name}: {lin.in_features} "
                                     f"in- and {lin.out_features} out-features; the WeightOffsets bank needs both to "
                                     f"be multiples of 8")
        self.device = self.modules[0].to_q.weight.device
        self.groups = []      # (module, group name, [(linear, wo), ...])
        for m in self.modules:
            if m.to_k.in_features == m.to_q.in_features and not m.is_cross:
                self.groups.append((m, "qkv", [(m.to_q, m.wo_q), (m.to_k, m.wo_k), (m.to_v, m.wo_v)]))
            else:
                self.groups.append((m, "q", [(m.to_q, m.wo_q)]))
                self.groups.append((m, "kv", [(m.to_k, m.wo_k), (m.to_v, m.wo_v)]))
        self.projs = [pr for _, _, g in self.groups for pr in g]
        self.params = [p for _, wo in self.projs for p in wo.kernel_params()]
        total = sum(l.weight.numel() for l, _ in self.projs)
        self.weff = torch.empty(total, device=self.device, dtype=torch.bfloat16)
        self.dweff = torch.zeros(total, device=self.device, dtype=torch.float32)
        nf = sum(2 * l.in_features + 3 * l.out_features for l, _ in self.projs)
        nb = sum(4 * l.out_features + 3 * l.in_features for l, _ in self.projs)
        self.fac = torch.empty(nf, device=self.device, dtype=torch.float32)
        self.bw = torch.zeros(nb, device=self.device, dtype=torch.float32)
        self.max_r = max(l.in_features for l, _ in self.projs)
        self.max_c = max(l.out_features for l, _ in self.projs)
        # views handed to the attention modules: (W_eff (ΣC,R) bf16, dW_eff (ΣC,R) fp32) per group
        self.views = {}
        off = 0
        self._offsets = []
        for m, name, g in self.groups:
            R = g[0][0].in_features
            Ct = sum(l.out_features for l, _ in g)
            self.views[(id(m), name)] = (self.weff[off:off + Ct * R].view(Ct, R), self.dweff[off:off + Ct * R].view(Ct, R))
            for l, _ in g:
                self._offsets.append(off)
                off += l.weight.numel()
        self._sig = None
        self._table = None
        self._token = None
        self._key = None
        self.dp_group = None      # set by engine.PretrainStep under data parallelism: exchange the G reductions (see _launch_backward)
        assert _lib.load().e4t_wo_bank_record_size() == ctypes.sizeof(_WOProj)
        for m in self.modules:      # any (partial) load_state_dict invalidates the cached W_eff
            m.register_load_state_dict_post_hook(lambda mod, keys: FN.bump_param_epoch())

    # ---- device table -------------------------------------------------------------------------------------------
    def _signature(self):
        return tuple(p.data_ptr() for p in self.params) + tuple(l.weight.data_ptr() for l, _ in self.projs)

    def _build_table(self):
        recs = (_WOProj * len(self.projs))()
        fo = bo = 0
        for i, ((lin, wo), off) in enumerate(zip(self.projs, self._offsets)):
            R, C = lin.in_features, lin.out_features
            ps = wo.kernel_params()
            for q in ps:
                if q.grad is None or not getattr(q, "_e4t_arena", False):
                    raise RuntimeError("WOBank needs arena-homed parameters with .grad views (engine.FlatAdamW)")
            r = recs[i]
            r.W = lin.weight.data_ptr()
            r.v, r.w1, r.b1, r.w2, r.b2, r.Wc, r.bc, r.Wr, r.br = (q.data_ptr() for q in ps)
            r.dv, r.dw1, r.db1, r.dw2, r.db2, r.dWc, r.dbc, r.dWr, r.dbr = (q.grad.data_ptr() for q in ps)
            r.fac = self.fac.data_ptr() + 4 * fo
            r.bw = self.bw.data_ptr() + 4 * bo
            r.weff = self.weff.data_ptr() + 2 * off
            r.dweff = self.dweff.data_ptr() + 4 * off
            r.R, r.C = R, C
            fo += 2 * R + 3 * C
            bo += 4 * C + 3 * R
        raw = bytes(recs)
        self._table = torch.frombuffer(bytearray(raw), dtype=torch.uint8).to(self.device)
        self._sig = self._signature()

    def _launch_forward(self):
        if self._sig != self._signature():
            self._build_table()
        self.dweff.zero_()
        _lib.call("e4t_wo_bank_fwd", ptr(self._table), c_int(len(self.projs)), c_int(self.max_r), c_int(self.max_c),
                  stream())

    def _launch_backward(self):
        if self.dp_group is None:
            _lib.call("e4t_wo_bank_bwd", ptr(self._table), c_int(len(self.projs)), c_int(self.max_r), c_int(self.max_c),
                      ptr(self.bw), c_ll(self.bw.numel()), stream())
            return
        # data parallel (engine.PretrainStep): exchange the five G reductions of every projection (~2 MB) instead of the
        # 573 MB of WeightOffsets parameter gradients they expand to — every later step of the backward is linear in
        # them with rank-identical coefficients, so each rank then accumulates the SUM over ranks into its .grad views
        # (SURVEY.md App. A; the 1/world average is folded into the optimiser like for the rest of the arena)
        import torch.distributed as dist
        _lib.call("e4t_wo_bank_bwd_reduce", ptr(self._table), c_int(len(self.projs)), c_int(self.max_r),
                  c_int(self.max_c), ptr(self.bw), c_ll(self.bw.numel()), stream())
        dist.all_reduce(self.bw, op=dist.ReduceOp.SUM, group=None if self.dp_group is True else self.dp_group)
        _lib.call("e4t_wo_bank_bwd_apply", ptr(self._table), c_int(len(self.projs)), c_int(self.max_r),
                  c_int(self.max_c), stream())

    # ---- per-step access ------------------------------------------------------------------------------------------
    def get(self, module, group):
        """(W_eff view, dW_eff accumulation view, autograd token) for one attention module's projection group."""
        grad_on = torch.is_grad_enabled()
        # no-grad calls (sampling at log steps, inference) rebuild W_eff once per UNet forward: a CUDA-graph replay
        # or a partial load_state_dict moves the parameters without telling this cache (ADVICE r1)
        key = (FN.PARAM_EPOCH, FN.WO_EPOCH if grad_on else -1, grad_on, 0 if grad_on else FN.NOGRAD_FWD_EPOCH,
               tuple(p._version for p in self.params[:9]))
        if self._key != key:
            if grad_on:
                self._token = _BankFn.apply(self, *self.params, *[l.weight for l, _ in self.projs])
            else:
                self._launch_forward()
                self._token = None
            self._key = key
        w, dw = self.views[(id(module), group)]
        return w, dw, self._token

    def drop_autograd_refs(self):
        self._token = None
        self._key = None
