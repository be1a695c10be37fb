"""Precision model of the tensor-core kernels: a float64 restatement of tc_loss_grad_kernel (csrc/tc_kernel.cu, "narrow",
hidden widths <= 64) and tw_loss_grad_kernel (csrc/tc_wide_kernel.cu, "wide", 128-wide layers) that rounds to bf16 at
exactly the points where the kernels round, so that a kernel can be held to fp32-grade tolerances against it.

Modes:
  exact     no rounding at all: the float64 loss / gradient of the same program (equals the oracle, DESIGN section 3)
  tc_bf16   narrow kernel, PINN_MODE_TC_BF16
  tc_split  narrow kernel, PINN_MODE_TC_SPLIT (forward operands hi + lo)
  tw_bf16   wide kernel (bf16 operands; the planner's pass split)

Rounding points (checked against the kernels' code):
  narrow  tensor-layer weights and every hidden activation tile of every channel are bf16 hi (+ lo = bf16(v - hi) in
          split mode); the forward product is hi*hi (split: hi*hi + hi*lo + lo*hi); the first layer is fp32; the last layer
          dots the unrounded activations.  Reverse: pre-activations recomputed as W_hi * H_hi (+ fp32 bias); Zbar stored as
          hi; dgrad Zbar_hi * W_hi; wgrad sum_c Zbar_hi^T H_hi; bias sum_p Zbar_hi[0]; last-layer weight gradient
          H_hi^T (ubar_hi + ubar_lo), bias fp32.  Layer 0 reverse: fp32 without tensor layers; otherwise Zbar^0 channels
          0..n1 as hi against the coordinates' hi (+ their lo when n2 > 0).
  wide    weights and activation tiles hi only; the reverse sweep reads the forward's fp32 pre-activations (which equal
          W_hi * H_hi + b); the coordinates' lo enters the layer-0 weight gradient when n1 <= 2.
Everything else is float64 here (fp32 in the kernels).  The residual program is interpreted from the term's op list,
with autograd for the tap / theta.p adjoints; the networks' forward and reverse sweeps are written out by hand.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional

import numpy as np
import torch

from neuralpde_jl_b200 import engine as E

MODES = ("exact", "tc_bf16", "tc_split", "tw_bf16")
TC_MAX_C, TW_MAX_C, TC_MAX_TL = 5, 4, 6
# (n1, n2) channel structures the tensor-core dispatch accepts (plan.cu check_tc_terms; (4, 0) not on the wide kernel)
TC_KEYS = {(0, 0), (1, 0), (2, 0), (3, 0), (4, 0), (1, 1), (2, 1), (3, 1), (2, 2)}


def _dispatch_set(kernel: str, max_c: int):
    """(kernel, n1, n2, pure, ak) of every instantiation of PINN_TC_DISPATCH with at most max_c channels."""
    out = set()
    for n1, n2 in TC_KEYS:
        if 1 + n1 + n2 > max_c or (kernel == "tw" and (n1, n2) == (4, 0)):
            continue
        for pure in ((True, False) if n2 > 0 and n1 >= 2 else (True,)):
            for ak in (0, 1):
                out.add((kernel, n1, n2, pure, ak))
    return out


NARROW_DISPATCH = _dispatch_set("tc", TC_MAX_C)
WIDE_DISPATCH = _dispatch_set("tw", TW_MAX_C)


# ---- bf16 rounding (__floats2bfloat162_rn: fp32 -> bf16, round to nearest even) ----------------------------------
def bf16(v) -> np.ndarray:
    """float64 values of bf16(fp32(v)), round to nearest even."""
    f = np.asarray(v, dtype=np.float64).astype(np.float32)
    b = f.reshape(-1).view(np.uint32).astype(np.uint64)
    b = (b + 0x7FFF + ((b >> 16) & 1)) & 0xFFFF0000
    return b.astype(np.uint32).view(np.float32).astype(np.float64).reshape(f.shape)


def split(v):
    """(hi, lo) with hi = bf16(v), lo = bf16(v - hi), v taken in fp32 (store_half)."""
    f = np.asarray(v, dtype=np.float64).astype(np.float32).astype(np.float64)
    hi = bf16(f)
    return hi, bf16(f - hi)


# ---- activations: value and three derivatives (act_eval) ----------------------------------------------------------
def act_derivs(name: str, z: np.ndarray):
    if name == "identity":
        return z, np.ones_like(z), np.zeros_like(z), np.zeros_like(z)
    if name == "tanh":
        t = np.tanh(z)
        s = 1 - t * t
        return t, s, -2 * t * s, s * (6 * t * t - 2)
    g = 1 / (1 + np.exp(-z))
    g1 = g * (1 - g)
    g2 = g1 * (1 - 2 * g)
    g3 = g1 * (1 - 6 * g1)
    if name == "sigmoid":
        return g, g1, g2, g3
    if name == "softplus":
        return np.logaddexp(0, z), g, g1, g2
    if name == "swish":
        return z * g, g + z * g1, 2 * g1 + z * g2, 3 * g2 + z * g3
    if name == "sin":
        s, c = np.sin(z), np.cos(z)
        return s, c, -s, -c
    raise ValueError(name)


# ---- channel planning (plan.cu: plan_channels, canonical_order, plan_taps, split_passes) -------------------------
@dataclass
class Slot:
    net: int
    rows: List[int]
    dir1: List[int] = field(default_factory=list)
    pairs: List[tuple] = field(default_factory=list)    # (a, b), indices into dir1, a <= b
    pure: bool = True

    @property
    def n1(self):
        return len(self.dir1)

    @property
    def n2(self):
        return len(self.pairs)

    @property
    def C(self):
        return 1 + self.n1 + self.n2


def plan_term(tm: E.TermSpec, nets: List[E.NetSpec]):
    """Slots of a term (networks in order of first tap, canonical channel order) and each tap's (slot, channel)."""
    slot_of: Dict[int, int] = {}
    slots: List[Slot] = []
    for tp in tm.taps:
        if tp.net not in slot_of:
            slot_of[tp.net] = len(slots)
            rows = tm.net_rows[tp.net] if tm.net_rows is not None and tp.net < len(tm.net_rows) \
                and tm.net_rows[tp.net] is not None else list(range(nets[tp.net].dims[0]))
            slots.append(Slot(tp.net, list(rows)))
    for tp in tm.taps:
        ch = slots[slot_of[tp.net]]
        if tp.order > 2:
            raise ValueError("the tensor-core model propagates derivatives up to order 2")
        for q in range(tp.order):
            if tp.dirs[q] not in ch.dir1:
                ch.dir1.append(tp.dirs[q])
    for tp in tm.taps:
        if tp.order == 2:
            ch = slots[slot_of[tp.net]]
            a, b = sorted((ch.dir1.index(tp.dirs[0]), ch.dir1.index(tp.dirs[1])))
            if (a, b) not in ch.pairs:
                ch.pairs.append((a, b))
    for ch in slots:                       # canonical_order: directions with a pure second derivative first
        order = []
        for a, b in ch.pairs:
            if a == b and a not in order:
                order.append(a)
        npure = len(order)
        order += [j for j in range(ch.n1) if j not in order]
        inv = {o: i for i, o in enumerate(order)}
        ch.dir1 = [ch.dir1[o] for o in order]
        ch.pairs = [tuple(sorted((inv[a], inv[b]))) for a, b in ch.pairs]
        ch.pure = npure == ch.n2
        if ch.pure:
            ch.pairs = [(q, q) for q in range(ch.n2)]
    taps = []
    for tp in tm.taps:
        s = slot_of[tp.net]
        ch = slots[s]
        if tp.order == 0:
            c = 0
        elif tp.order == 1:
            c = 1 + ch.dir1.index(tp.dirs[0])
        else:
            c = 1 + ch.n1 + ch.pairs.index(tuple(sorted((ch.dir1.index(tp.dirs[0]), ch.dir1.index(tp.dirs[1])))))
        taps.append((s, c))
    return slots, taps


def split_passes(slots: List[Slot], taps):
    """Wide kernel: a network with more than 4 channels runs in several passes (first fit over the directions, a
    direction with a pure second derivative costs 2 channels); each pass has the value channel."""
    if all(ch.C <= TW_MAX_C for ch in slots):
        return slots, taps
    new: List[Slot] = []
    first_new, where = [], {}
    for s, ch in enumerate(slots):
        first_new.append(len(new))
        if ch.C <= TW_MAX_C:
            for j in range(ch.n1):
                where[s, j] = (len(new), j)
            new.append(ch)
            continue
        if not ch.pure:
            raise ValueError("the wide kernel splits only pure second derivatives into passes")
        placed = [False] * ch.n1
        while not all(placed):
            g = Slot(ch.net, ch.rows)
            cost = 0
            for j in range(ch.n1):
                cj = 2 if j < ch.n2 else 1
                if placed[j] or cost + cj > TW_MAX_C - 1:
                    continue
                placed[j] = True
                cost += cj
                where[s, j] = (len(new), g.n1)
                g.dir1.append(ch.dir1[j])
                if j < ch.n2:
                    g.pairs.append((g.n2, g.n2))
            new.append(g)
    out = []
    for s, c in taps:
        n1 = slots[s].n1
        if c == 0:
            out.append((first_new[s], 0))
        elif c <= n1:
            ns, pos = where[s, c - 1]
            out.append((ns, 1 + pos))
        else:
            ns, pos = where[s, c - 1 - n1]
            out.append((ns, 1 + new[ns].n1 + pos))
    return new, out


# ---- channel chain rule (chain_fwd / chain_bwd in tc_common.cuh), vectorised over [channel][neuron][point] ----------
def chain_fwd(act: str, ch: Slot, z: np.ndarray) -> np.ndarray:
    a, d1, d2, _ = act_derivs(act, z[0])
    h = np.empty_like(z)
    h[0] = a
    for i in range(ch.n1):
        h[1 + i] = d1 * z[1 + i]
    for s, (pa, pb) in enumerate(ch.pairs):
        h[1 + ch.n1 + s] = d1 * z[1 + ch.n1 + s] + d2 * z[1 + pa] * z[1 + pb]
    return h


def chain_bwd(act: str, ch: Slot, z: np.ndarray, hb: np.ndarray) -> np.ndarray:
    _, d1, d2, d3 = act_derivs(act, z[0])
    zb = np.empty_like(z)
    acc0 = d1 * hb[0]
    for i in range(ch.n1):
        acc0 = acc0 + d2 * z[1 + i] * hb[1 + i]
        zb[1 + i] = d1 * hb[1 + i]
    for s, (pa, pb) in enumerate(ch.pairs):
        g = hb[1 + ch.n1 + s]
        za, zbb = z[1 + pa], z[1 + pb]
        acc0 = acc0 + (d2 * z[1 + ch.n1 + s] + d3 * za * zbb) * g
        zb[1 + pa] += d2 * zbb * g
        zb[1 + pb] += d2 * za * g
        zb[1 + ch.n1 + s] = d1 * g
    zb[0] = acc0
    return zb


# ---- residual program (run_program in ffma_kernel.cuh) -----------------------------------------------------------
def run_program(prog, X: torch.Tensor, taps: List[torch.Tensor], params: torch.Tensor) -> torch.Tensor:
    n = X.shape[1]
    v: List[torch.Tensor] = []
    for ins in prog:
        op, a, b, imm = (list(ins) + [0, 0, 0.0])[:4]
        if op == "const":
            r = torch.full((n,), float(imm), dtype=torch.float64)
        elif op == "coord":
            r = X[a]
        elif op == "tap":
            r = taps[a]
        elif op == "param":
            r = params[a].expand(n)
        elif op in ("add", "sub", "mul", "div", "pow"):
            x, y = v[a], v[b]
            r = {"add": x + y, "sub": x - y, "mul": x * y}[op] if op in ("add", "sub", "mul") else \
                (x / y if op == "div" else torch.pow(x, y))
        elif op == "neg":
            r = -v[a]
        elif op == "powi":
            r = v[a] ** int(imm)
        else:
            r = {"sin": torch.sin, "cos": torch.cos, "exp": torch.exp, "log": torch.log, "tanh": torch.tanh,
                 "sqrt": torch.sqrt, "abs": torch.abs}[op](v[a])
        v.append(r)
    return v[-1]


# ---- the model ---------------------------------------------------------------------------------------------------
@dataclass
class Result:
    total: float
    terms: np.ndarray
    grad: Optional[np.ndarray]
    resid: List[np.ndarray]


@dataclass
class Floor:
    """TcModel.noise_floor: relative change of the total, of each term loss and of the whole gradient; absolute change
    of each term's residuals (max over points) and of each gradient block (L2 norm, by TcModel.blocks name)."""
    total: float
    terms: np.ndarray
    resid: List[float]
    grad: float
    blocks: Dict[str, float]


class TcModel:
    """Model of one problem: ``spec`` is the engine's ProblemSpec, ``points[t]`` term t's (dim, N) point matrix as
    uploaded (hoisted rows included), ``qw[t]`` its quadrature weights (None: unweighted)."""

    def __init__(self, spec: E.ProblemSpec, points, qw=None, mode: str = "exact", chunk: int = 8192):
        if mode not in MODES:
            raise ValueError(mode)
        self.spec, self.mode, self.chunk = spec, mode, chunk
        self.points = [np.asarray(p, dtype=np.float64) for p in points]
        self.qw = [None if w is None else np.asarray(w, dtype=np.float64) for w in (qw or [None] * len(points))]
        nets = spec.nets
        self.wide = any(d > 64 for n in nets for d in n.dims[1:-1])
        self.plans = []
        for tm in spec.terms:
            slots, taps = plan_term(tm, nets)
            if mode == "tw_bf16":
                slots, taps = split_passes(slots, taps)
            self.plans.append((slots, taps))
        self.offsets = []
        for n in nets:
            offs, o = [], n.theta_offset
            for l in range(len(n.acts)):
                offs.append((o, o + n.dims[l] * n.dims[l + 1]))
                o += n.dims[l] * n.dims[l + 1] + n.dims[l + 1]
            self.offsets.append(offs)

    # (kernel, n1, n2, pure, ak) of every (term, slot) -- what PINN_TC_DISPATCH instantiates for this problem
    def dispatch_keys(self):
        kernel = "tw" if self.wide else "tc"
        out = set()
        for slots, _ in self.plans:
            for ch in slots:
                acts = self.spec.nets[ch.net].acts
                ak = int(all(a == "tanh" for a in acts[:-1]))
                out.add((kernel, ch.n1, ch.n2, bool(ch.pure), ak))
        return out

    def blocks(self):
        """(name, slice) of every layer's W and b and of theta.p."""
        out = []
        for k, offs in enumerate(self.offsets):
            n = self.spec.nets[k]
            for l, (w, b) in enumerate(offs):
                out.append(("net%d.W%d" % (k, l), slice(w, b)))
                out.append(("net%d.b%d" % (k, l), slice(b, b + n.dims[l + 1])))
        if self.spec.n_params:
            out.append(("p", slice(self.spec.param_offset, self.spec.param_offset + self.spec.n_params)))
        return out

    def noise_floor(self, theta, eps: float = 1e-7, draws: int = 4, seed: int = 0, want_grad: bool = False,
                    base: Optional[Result] = None) -> Floor:
        """How far fp32-level differences can move this mode's result through its bf16 rounding points: the largest
        change over `draws` evaluations in which every hidden activation moves by eps (normal, absolute: the accuracy of
        the kernels' approximate tanh) and every reverse-sweep adjoint by eps relative, before they are rounded.  A
        residual that is small against its inputs, or a deep bf16 network, turns such a difference into flipped
        roundings; the rounding is discontinuous, so no fp32-grade bound holds below this floor.  `base`: the
        unperturbed result at theta, if already evaluated (with a gradient when want_grad)."""
        if base is None:
            base = self.evaluate(theta, want_grad=want_grad)
        fl = Floor(0.0, np.zeros(len(base.terms)), [0.0] * len(base.resid), 0.0,
                   {name: 0.0 for name, _ in self.blocks()} if want_grad else {})
        self._rng = np.random.default_rng(seed)
        try:
            for _ in range(draws):
                self._eps = eps
                p = self.evaluate(theta, want_grad=want_grad)
                fl.total = max(fl.total, abs(p.total - base.total) / abs(base.total))
                fl.terms = np.maximum(fl.terms, np.abs(p.terms - base.terms) / np.abs(base.terms))
                fl.resid = [max(a, float(np.max(np.abs(r - r0)))) for a, r, r0 in zip(fl.resid, p.resid, base.resid)]
                if want_grad:
                    d = p.grad - base.grad
                    fl.grad = max(fl.grad, float(np.linalg.norm(d) / np.linalg.norm(base.grad)))
                    for name, sl in self.blocks():
                        fl.blocks[name] = max(fl.blocks[name], float(np.linalg.norm(d[sl])))
        finally:
            self._eps = 0.0
        return fl

    _eps = 0.0

    def _noisy(self, h):
        return h + self._eps * self._rng.standard_normal(h.shape) if self._eps else h

    def _noisy_rel(self, v):
        return v * (1 + self._eps * self._rng.standard_normal(v.shape)) if self._eps else v

    # -- rounding helpers of the mode ----------------------------------------------------------------------------
    def _hi(self, v):
        return v if self.mode == "exact" else bf16(v)

    def _params(self, theta, k):
        n = self.spec.nets[k]
        Ws, bs = [], []
        for l, (w, b) in enumerate(self.offsets[k]):
            Ws.append(theta[w:b].reshape(n.dims[l], n.dims[l + 1]).T)
            bs.append(theta[b:b + n.dims[l + 1]])
        return Ws, bs

    def _forward(self, theta, ch: Slot, X):
        n = self.spec.nets[ch.net]
        Ws, bs = self._params(theta, ch.net)
        acts, L = n.acts, len(n.acts)
        x = X[ch.rows]
        z = np.zeros((ch.C, n.dims[1], x.shape[1]))
        z[0] = Ws[0] @ x + bs[0][:, None]
        for j, d in enumerate(ch.dir1):
            z[1 + j] = Ws[0][:, d][:, None]
        zs, hs = [z], [self._noisy(chain_fwd(acts[0], ch, z))]
        for l in range(1, L - 1):
            h = hs[-1]
            if self.mode == "tc_split":
                hh, hl = split(h)
                wh, wl = split(Ws[l])
                acc = np.matmul(wh, hh) + np.matmul(wl, hh) + np.matmul(wh, hl)
            else:
                acc = np.matmul(self._hi(Ws[l]), self._hi(h))
            acc[0] += bs[l][:, None]
            zs.append(acc)
            hs.append(self._noisy(chain_fwd(acts[l], ch, acc)))
        u = np.einsum("o,con->cn", Ws[L - 1][0], hs[-1])
        u[0] += bs[L - 1][0]
        return dict(x=x, z=zs, h=hs, u=u)

    def _backward(self, theta, ch: Slot, rec, ub, grad):
        n = self.spec.nets[ch.net]
        Ws, bs = self._params(theta, ch.net)
        acts, L, TL = n.acts, len(n.acts), len(n.acts) - 2
        offs = self.offsets[ch.net]
        exact = self.mode == "exact"
        hL = rec["h"][-1]
        ubr = ub if exact else sum(split(ub))
        w, b = offs[L - 1]
        grad[w:b] += np.einsum("con,cn->o", self._hi(hL), ubr)
        grad[b] += ub[0].sum()
        hb = Ws[L - 1][0][None, :, None] * ub[:, None, :]
        for l in range(TL, 0, -1):
            Hin = self._hi(rec["h"][l - 1])
            if exact:
                z = rec["z"][l]
            else:                       # narrow: recompute from the hi tiles; wide: the stashed forward value (the same)
                z = np.matmul(bf16(Ws[l]), Hin)
                z[0] += bs[l][:, None]
            Zb = self._hi(self._noisy_rel(chain_bwd(acts[l], ch, z, hb)))
            w, b = offs[l]
            grad[w:b] += np.einsum("con,ckn->ok", Zb, Hin).T.ravel()
            grad[b:b + n.dims[l + 1]] += Zb[0].sum(-1)
            hb = np.matmul(self._hi(Ws[l]).T, Zb)
        zb = self._noisy_rel(chain_bwd(acts[0], ch, rec["z"][0], hb))
        x = rec["x"]
        if exact or TL == 0:
            Z, xr = zb, x
        else:
            Z = bf16(zb[:1 + ch.n1])
            xh, xl = split(x)
            lo = ch.n2 > 0 if self.mode != "tw_bf16" else ch.n1 <= 2
            xr = xh + xl if lo else xh
        gW = Z[0] @ xr.T
        for j, d in enumerate(ch.dir1):
            gW[:, d] += Z[1 + j].sum(-1)
        w, b = offs[0]
        grad[w:b] += gW.T.ravel()
        grad[b:b + n.dims[1]] += Z[0].sum(-1)

    def evaluate(self, theta, weights=None, want_grad: bool = True) -> Result:
        """Total, term losses, gradient (want_grad) and per-point residuals of every term at theta (used as given:
        pass theta rounded to fp32 for a comparison with an fp32 engine)."""
        spec = self.spec
        theta = np.asarray(theta, dtype=np.float64)
        grad = np.zeros(spec.n_theta) if want_grad else None
        wts = np.ones(len(spec.terms)) if weights is None else np.asarray(weights, dtype=np.float64)
        terms, resid = [], []
        p0, npar = spec.param_offset, spec.n_params
        for t, tm in enumerate(spec.terms):
            slots, taps = self.plans[t]
            X = self.points[t]
            N = X.shape[1]
            weighted = tm.reduction == E.REDUCE_WSUM
            scale = tm.scale if weighted else 1.0 / N
            seed = scale * wts[t]
            acc, rs = 0.0, []
            for c0 in range(0, N, self.chunk):
                Xc = X[:, c0:c0 + self.chunk]
                qc = self.qw[t][c0:c0 + self.chunk] if weighted else np.ones(Xc.shape[1])
                recs = [self._forward(theta, ch, Xc) for ch in slots]
                tv = [torch.tensor(recs[s]["u"][c], requires_grad=want_grad) for s, c in taps]
                pv = torch.tensor(theta[p0:p0 + npar], requires_grad=want_grad and npar > 0)
                r = run_program(tm.prog, torch.as_tensor(Xc), tv, pv)
                S = (torch.as_tensor(qc) * r * r).sum()
                acc += float(S.detach())
                rs.append(r.detach().numpy().copy())
                if want_grad:
                    gs = torch.autograd.grad(S * seed, tv + ([pv] if npar else []), allow_unused=True)
                    if npar and gs[-1] is not None:
                        grad[p0:p0 + npar] += gs[-1].numpy()
                    ubs = [np.zeros((ch.C, Xc.shape[1])) for ch in slots]
                    for (s, c), g in zip(taps, gs[:len(taps)]):
                        if g is not None:
                            ubs[s][c] += g.numpy()
                    for ch, rec, ub in zip(slots, recs, ubs):
                        self._backward(theta, ch, rec, ub, grad)
            terms.append(scale * acc)
            resid.append(np.concatenate(rs))
        terms = np.array(terms)
        return Result(float(np.dot(wts, terms)), terms, grad, resid)


# ---- capturing what symbolic_discretize gives the engine ------------------------------------------------------------
class SpecRecorder:
    """Stand-in for ``Engine`` that keeps the ProblemSpec and the uploaded point matrices (no GPU needed)."""

    def __init__(self, spec: E.ProblemSpec):
        self.spec = spec
        self.np_dtype = np.float64 if spec.dtype in ("float64", "f64") else np.float32
        self.n_terms, self.n_theta = len(spec.terms), int(spec.n_theta)
        self.points: Dict[int, np.ndarray] = {}
        self.qw: Dict[int, Optional[np.ndarray]] = {}

    def set_points_host(self, term, pts, weights=None, stream=0):
        self.points[term] = np.array(pts, dtype=self.np_dtype)
        self.qw[term] = None if weights is None else np.array(weights, dtype=self.np_dtype)

    def set_global_count(self, term, n):
        pass

    def model(self, mode: str, **kw) -> TcModel:
        n = len(self.spec.terms)
        return TcModel(self.spec, [self.points[t] for t in range(n)], [self.qw.get(t) for t in range(n)], mode, **kw)


class RecordingEngine(E.Engine):
    """The real engine, recording the uploaded point matrices the same way."""

    def __init__(self, spec):
        super().__init__(spec)
        self.points, self.qw = {}, {}

    def set_points_host(self, term, pts, weights=None, stream=0):
        SpecRecorder.set_points_host(self, term, pts, weights)
        super().set_points_host(term, pts, weights, stream)

    model = SpecRecorder.model
