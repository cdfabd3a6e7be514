"""float64 restatement of the two fused MoE autograd nodes of ``xtuner_b200/fused.py`` (``FusedMoEFunction`` behind
``fused_moe``, ``FusedMoEBlockFunction`` behind ``fused_moe_block``), stage by stage in the forward and end to end in
the backward.  Test infrastructure only; nothing under ``xtuner_b200/`` imports it.  Plain torch on whatever device the
operands are on.

It adds only the composition: every kernel it passes through has its own reference module, and each stage is checked
with that module's check (``gemm_reference``, ``swiglu_fp8_reference``, ``norm_combine_reference``,
``router_reference``).

Forward, stage-local.  Each stage's input is the node's own saved tensor (:func:`from_autograd` reads them from
``out.grad_fn``), so a stage is checked exactly where its kernel has an exact restatement and within that kernel's
bound elsewhere: the block's rstd (``rstd_rel``) and x (bit for bit given rstd); logits (``gate_bound`` of the kernel
the node runs: the tensor-core gate of the one-launch gate + route, or xtb_gate_logits); router_weights (the expf
bound); ids, topk_weights and tokens_per_expert (``check_greedy_exact``, or the replayed ids and the restated weights);
x_perm and row_id_map (an exact stable gather); h and y (the grouped-GEMM bound); a (SwiGLU, exact or a near tie of
silu); out (bit for bit, ``combine``).

Backward, end to end.  One float64 chain from the saved forward tensors and the incoming gradients through every stage
of the node's backward, rounded to bf16 where the node stores bf16 (g_comb, g_y, g_a, ds, g_h, g_xp, g_x_gate, the
dispatch sum, g_x), with a first-order bound carried beside every value.  For a value v of the chain with bound B
(|kernel - v| <= B elementwise):

  * a reduction of length n in fp32 adds gamma-type accumulation error on S = sum |a| |b|: the grouped GEMMs
    max(2^-16, n 2^-27) S (one fp32 rounding per 16-deep wgmma step, ``gemm_reference``), the router and gate
    reductions the gamma(n) of their reference modules;
  * a linear stage carries the upstream bound through |d out / d in|: a GEMM through |W| (B_out += B_in |W|), the
    SwiGLU backward through |u| (ds), |s| (grad_u) and |sigmoid F| (grad_g), the router backward through the magnitude
    of its own Jacobian, the dispatch sum by adding;
  * a bf16 store where the chain rounds too: kernel and chain round values at most B apart, so they store the same bf16
    value unless the chain's value lies within B of a rounding midpoint; there the bound becomes
    B + |v - bf16(v)| + u (|v| + B) (u = 2^-8, plus 2^-134 for the subnormal step) and 0 elsewhere (:func:`store`);
  * the float64 reference carries its own rounding: 2^-40 |v| is added to every bound (REF_SLACK), far below any
    fp32 error and enough that an exact bf16 midpoint in the chain does not fail on the last bit of the checker's
    own float64 arithmetic;
  * an output the node stores in bf16 is checked with ``check_near_tie`` against the unrounded chain value: correctly
    rounded, or one ulp off only where the value lies within tau B of the midpoint between its two bf16 neighbours.

Checks on the gradients: g_y is exact (``act_grad``), g_tw carries the ``prob_grad_ref`` bound, g_w2 is stage-local
(exact g_y, the saved a, the grouped-GEMM accumulation bound), the residual gradient is g_out bit for bit; g_w13,
g_x / g_h, g_gate_w and g_norm_w are held to the propagated bound times one tau per quantity (:data:`TAU`): fp32
outputs as |got - ref| <= tau B, bf16 outputs as above.  No fraction of elements may miss and no row is left out.

Router backward (:func:`router_bwd_ref`): float64 autograd through softmax / sigmoid of the node's own fp32 logits,
the gather at the node's ids (replayed ids may repeat), the normalisation and the scaling.  Bound: the arithmetic
gamma(4K + 16 + E/32 + 5) on A, the magnitude of the Jacobian applied to |g| (A = p (gp + sum gp p) for softmax,
gp p (1 - p) for sigmoid, gp the magnitude of the gradient reaching p); the router_weights' own relative error rho
(``greedy_ref`` plus (4K + 8) u for topk_weights) times 5 A (softmax) or 3 A + 8u gp p (sigmoid); and g_tw's bound
carried through the same magnitudes.

Loss: sum(out^2) must be within 1e-4 relative of the same sum over a float64 forward at the node's ids that rounds
to bf16 only where the reference's eager composition does (:func:`forward64` with ``rounded``), from 2^14 output
elements on; :func:`check_loss` says why not against a wholly unrounded forward and not below that size.
:func:`backward_reference` with ``fw`` = the unrounded forward runs the same chain with no rounding: the CPU test
holds it to float64 autograd through ``oracle.moe_oracle``.

Tightness.  Every bound is a worst case over summation orders and signs, so its ratio to the real error depends on
how much of it is the final bf16 rounding (g_w13, g_x, g_h, h, y: ratios near 1 on an H100) and how much is fp32
accumulation, where real errors are random in sign and grow like the square root of what the bound adds up.  Three
stay far below 1 for that reason and cannot be tightened without restating the kernels' exact summation order, which
would make the chain an emulation rather than a reference: g_gate_w sums over T tokens the worst case of each token's
router gradient, whose largest part is ``prob_grad_ref``'s gamma(8 ceil(H/256) + 6) on g_tw; g_norm_w is
``g_norm_w_ref``'s gamma over the per-CTA token chains; the fallback's x and g_h assume a serial fp32 reduction over H
because torch does not document the order of its rms_norm reduction.

The fused-norm block rounds x once, bf16(h rstd w) with the fp32 weight; the composed path for other H
(``F.rms_norm`` with the weight cast to bf16, then ``fused_moe``) is checked against its own restatement
(``fallback``), with torch's reductions bounded by gamma(H + 32) and its weight gradient rounded to bf16 as autograd's
cast back does.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, Optional, Tuple

import torch

from tests import gemm_reference as G
from tests import norm_combine_reference as NC
from tests import router_reference as R
from tests import swiglu_fp8_reference as SW

U = 2.0 ** -8  # bf16 unit roundoff
U32 = 2.0 ** -24
TINY = 2.0 ** -134  # half the smallest bf16 subnormal step
LOSS_REL = 1e-4
LOSS_MIN_TERMS = 1 << 14  # the loss is compared from this many output elements on (check_loss)
REF_SLACK = 2.0 ** -40  # relative: the float64 reference's own arithmetic (and the checker's), next to fp32's 2^-24
# one tau per checked gradient (|got - ref| <= tau * bound): the bounds are worst-case, so 1 everywhere
TAU = {"g_x": 1.0, "g_h": 1.0, "g_w13": 1.0, "g_w2": 1.0, "g_gate_w": 1.0, "g_norm_w": 1.0}
BF16_GRADS = ("g_x", "g_h", "g_w13", "g_w2")  # stored in bf16 by the node (g_gate_w too for a bf16 gate parameter)

SAVED = {
    "moe": ("x", "gate_w", "w13", "w2", "rw", "tw", "ids", "rmap", "tpe", "x_perm", "h", "a", "y"),
    "block": ("h_in", "norm_w", "rstd", "x", "gate_w", "w13", "w2", "rw", "tw", "ids", "rmap", "tpe", "x_perm", "h",
              "a", "y"),
}


@dataclass
class Node:
    """One run of a node: ``kind`` is ``moe`` (FusedMoEFunction), ``block`` (FusedMoEBlockFunction) or ``fallback``
    (the block's composition for H outside the fused norm: F.rms_norm, then FusedMoEFunction with residual h).  ``t``
    holds the saved tensors under the names of :data:`SAVED` (w13 as [E, 2I, H], w2 as [E, H, I]) plus ``out``,
    ``logits``, ``residual`` and for ``fallback`` ``h_in`` and ``norm_w``."""

    kind: str
    t: Dict[str, Optional[torch.Tensor]]
    K: int
    norm: bool
    scaling: float
    hf: float
    scoring: str
    eps: float = 1e-6

    @property
    def counts(self):
        return [int(c) for c in self.t["tpe"].tolist()]

    @property
    def residual(self):
        return self.t["h_in"] if self.kind in ("block", "fallback") else self.t["residual"]


def node_of(t: torch.Tensor):
    """The fused node behind ``t``: ``t.grad_fn`` or the first node up its graph that carries the node's ``cfg``."""
    todo, seen = [t.grad_fn], set()
    while todo:
        fn = todo.pop(0)
        if fn is None or id(fn) in seen:
            continue
        seen.add(id(fn))
        if hasattr(fn, "cfg") and "FusedMoE" in type(fn).__name__:
            return fn
        todo.extend(f for f, _ in fn.next_functions)
    raise AssertionError("no fused MoE node behind this tensor")


def from_autograd(out, logits, *, kind="moe", residual=None, h_in=None, norm_w=None, eps=1e-6) -> Node:
    """Reads the saved tensors and the configuration of the node that produced ``out`` (before its backward ran)."""
    fn = node_of(out)
    block = "Block" in type(fn).__name__
    assert block == (kind == "block"), f"{kind}: the graph holds {type(fn).__name__}"
    names = SAVED["block" if block else "moe"]
    t = dict(zip(names, fn.saved_tensors))
    E = t["gate_w"].shape[0]
    I = t["a"].shape[1]
    H = t["x"].shape[1]
    t["w13"] = t["w13"].view(E, 2 * I, H)
    t["w2"] = t["w2"].view(E, H, I)
    t["out"] = out.detach().reshape(-1, H)
    t["logits"] = logits.detach()
    t["residual"] = None if residual is None else residual.detach().reshape(-1, H)
    if kind == "fallback":
        t["h_in"], t["norm_w"] = h_in.detach().reshape(-1, H), norm_w.detach()
    if block:
        K, norm, scaling, hf, scoring = fn.cfg
    else:
        K, norm, scaling, hf, scoring, has_res = fn.cfg
        assert has_res == (residual is not None or kind == "fallback")
    return Node(kind, t, K, norm, scaling, hf, "sigmoid" if scoring == 1 else "softmax", eps)


def one_launch(T: int, H: int, E: int, K: int) -> bool:
    """Whether the node computes gate and route in xtb_gate_route_dispatch (the tensor-core gate)."""
    return E <= 8 and K <= 8 and H % 128 == 0 and H <= 4096


# ---- bounds ----------------------------------------------------------------------------------------------------------


def acc(n: int) -> float:
    """fp32 accumulation of an n-long grouped-GEMM reduction, on S (module docstring)."""
    return max(G.TAU, n * 2.0 ** -27)


def store(v: torch.Tensor, B: torch.Tensor, pure: bool = False) -> Tuple[torch.Tensor, torch.Tensor]:
    """``(bf16(v) as float64, bound)`` of a bf16 store where kernel and chain round values at most B apart."""
    if pure:
        return v, B
    B = B + REF_SLACK * v.abs()
    r = SW.bf16_round(v).double()
    m, e = torch.frexp(r)
    step = torch.pow(2.0, (e - 8).double()).clamp_min(2.0 ** -133)
    step = torch.where(r == 0, torch.full_like(r, 2.0 ** -133), step)
    inward = torch.where((m.abs() == 0.5) & (step > 2.0 ** -133), step / 2, step) / 2
    sgn = torch.where(r < 0, -1.0, 1.0)
    d = (v - r) * sgn  # signed distance from r, away from zero positive
    safe = (B < step / 2 - d) & (B < inward + d) & torch.isfinite(v)
    return r, torch.where(safe, torch.zeros_like(B), B + (v - r).abs() + U * (v.abs() + B) + TINY)


def _per_expert(kind, a, b, counts, Ba=None):
    """float64 grouped product with S and, with ``Ba``, the upstream bound carried through |b|."""
    if kind == "tn":
        out = torch.zeros((len(counts), a.shape[1], b.shape[1]), dtype=torch.float64, device=a.device)
    else:
        n_out = b.shape[1] if kind == "nt" else b.shape[2]
        out = torch.zeros((a.shape[0], n_out), dtype=torch.float64, device=a.device)
    S, P = torch.zeros_like(out), torch.zeros_like(out)
    o = G.offsets(counts)
    for e, sel, ref, s in G.products(kind, a, b, counts):
        out[sel], S[sel] = ref, s
        if Ba is not None:
            if kind == "tn":
                P[sel] = Ba[o[e] : o[e + 1]].T @ b[o[e] : o[e + 1]].double().abs()
            else:
                w = b[e].double().abs()
                P[sel] = Ba[sel] @ (w.T if kind == "nt" else w)
    return out, S, P


# ---- forward ---------------------------------------------------------------------------------------------------------


def permutation(ids: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """``(sorted flat index per permuted row, row_id_map)``: rows by expert, stable in the token-major flat index."""
    flat = ids.reshape(-1)
    order = torch.argsort(flat, stable=True)
    rmap = torch.empty_like(order)
    rmap[order] = torch.arange(order.numel(), device=ids.device)
    return order, rmap.to(torch.int32)


def _first_bad(bad: torch.Tensor, what: str, got, want):
    i = tuple(int(v) for v in bad.nonzero()[0])
    raise AssertionError(f"{what}: {int(bad.sum())} elements differ; first at {i}: got {got[i].tolist()!r}, "
                         f"want {want[i].tolist()!r}")


def check_forward(node: Node, replay: Optional[torch.Tensor] = None) -> Dict[str, float]:
    """Every forward stage against its kernel's reference, from the node's own saved inputs; returns worst ratios."""
    t, K = node.t, node.K
    T, H = t["x"].shape
    E = t["gate_w"].shape[0]
    r: Dict[str, float] = {}
    if node.kind == "block":
        h, rstd = t["h_in"], t["rstd"]
        want = NC.rstd_ref(h, node.eps)
        r["rstd"] = NC.check_bound(rstd, want, NC.rstd_rel(H) * want, "rstd")
        NC.assert_bits_equal(t["x"], NC.rmsnorm_x(h, rstd, t["norm_w"]), "x (fused norm)")
    elif node.kind == "fallback":
        x64, xb = fallback_x_ref(t["h_in"], t["norm_w"], node.eps)
        r["x (rms_norm fallback)"] = NC.check_near_tie(t["x"], x64, xb, "x (rms_norm fallback)")[0]
    lg64, S = R.gate_ref(t["x"], t["gate_w"], None)
    gk = "mma" if one_launch(T, H, E, K) else R.gate_kernel(T, H, E)
    r[f"logits ({gk})"] = R.check_bound(t["logits"], lg64, R.gate_bound(gk, H, S), "logits")
    p64, pb = R.greedy_ref(t["logits"], node.scoring)
    r["router_weights"] = R.check_bound(t["rw"], p64, pb, "router_weights")
    if replay is None:
        R.check_greedy_exact(t["rw"], t["tw"], t["ids"], t["tpe"], K, node.norm, node.scaling, "routing")
        # ids equal to float64 wherever the float64 values decide them (logit error carried into p: 2 p max|dz|)
        q64, qb = R.greedy_ref(lg64, node.scoring)
        qb = qb + 2 * q64 * R.gate_bound(gk, H, S).amax(-1, keepdim=True)
        dec = R.decided_rows(q64, qb, K)
        ids64 = R.topk_rounds(q64, K)
        bad = (t["ids"] != ids64).any(-1) & dec
        if bool(bad.any()):
            _first_bad(bad[:, None].expand(-1, K), "ids on decided rows", t["ids"], ids64)
    else:
        if not torch.equal(t["ids"], replay.reshape(T, K)):
            _first_bad(t["ids"] != replay.reshape(T, K), "replayed ids", t["ids"], replay.reshape(T, K))
        want = R.topk_weights_restated(t["rw"], t["ids"], node.norm, node.scaling)
        bad = (t["tw"].view(torch.int32) != want.view(torch.int32)) & ~((t["tw"] == 0) & (want == 0))
        if bool(bad.any()):
            _first_bad(bad, "topk_weights (replay)", t["tw"], want)
        assert torch.equal(t["tpe"], torch.bincount(t["ids"].reshape(-1), minlength=E)), "tokens_per_expert"
    order, rmap = permutation(t["ids"])
    if not torch.equal(t["rmap"], rmap):
        _first_bad(t["rmap"] != rmap, "row_id_map", t["rmap"], rmap)
    NC.assert_bits_equal(t["x_perm"], t["x"][order // K], "x_perm")
    c = node.counts
    r["h"] = G.check_bound(t["h"], "nt", t["x_perm"], t["w13"], c, what="h")
    SW.check_swiglu_fwd(t["h"], t["a"], "a")
    r["y"] = G.check_bound(t["y"], "nt", t["a"], t["w2"], c, what="y")
    NC.assert_bits_equal(t["out"], NC.combine(t["y"], t["rmap"], t["tw"], node.residual, node.hf, K), "out")
    return r


def fallback_x_ref(h: torch.Tensor, w: torch.Tensor, eps: float) -> Tuple[torch.Tensor, torch.Tensor]:
    """``(x, bound)`` of F.rms_norm(h, w.to(bf16), eps): h rstd bf16(w) in float64, torch's fp32 reductions within
    gamma(H + 32) / 2 on rstd, rsqrt 4u, two products."""
    H = h.shape[1]
    x = h.double() * NC.rstd_ref(h, eps)[:, None] * w.to(torch.bfloat16).double()
    return x, (R.gamma(H + 32) / 2 + 8 * U32) * 1.01 * x.abs()


def forward64(inp: Dict[str, torch.Tensor], ids: torch.Tensor, K: int, norm: bool, scaling: float, hf: float,
              scoring: str, eps: float = 1e-6, rounded: bool = False) -> Dict[str, torch.Tensor]:
    """The node's forward in float64, routed at ``ids``: ``inp`` holds x (or h_in and norm_w), gate_w, w13 [E, 2I, H],
    w2 [E, H, I] and residual (or None).  ``rounded``: round to bf16 where the reference's eager composition stores
    bf16 (x, h, silu, a, y, the combined sum, its hidden_factor product, out), in float64 between those points;
    otherwise no rounding at all."""
    rn = (lambda v: SW.bf16_round(v).double()) if rounded else (lambda v: v)  # noqa: E731
    f = {k: (v.double() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in inp.items()}
    if "h_in" in f:
        f["rstd"] = torch.rsqrt(f["h_in"].square().mean(-1) + eps)
        f["x"] = rn(f["h_in"] * f["rstd"][:, None] * f["norm_w"])
        f["residual"] = f["h_in"]
    x, E = f["x"], f["gate_w"].shape[0]
    f["logits"] = x @ f["gate_w"].T
    f["rw"] = torch.softmax(f["logits"], -1) if scoring == "softmax" else torch.sigmoid(f["logits"])
    w = f["rw"].gather(1, ids)
    if norm:
        w = w / w.sum(-1, keepdim=True)
    f["tw"] = w * scaling
    f["ids"] = ids
    f["tpe"] = torch.bincount(ids.reshape(-1), minlength=E)
    order, f["rmap"] = permutation(ids)
    f["x_perm"] = x[order // K]
    c = [int(v) for v in f["tpe"].tolist()]
    f["h"] = rn(_per_expert("nt", f["x_perm"], f["w13"], c)[0])
    I = f["h"].shape[1] // 2
    g = f["h"][:, :I]
    f["a"] = rn(rn(g * torch.sigmoid(g)) * f["h"][:, I:])
    f["y"] = rn(_per_expert("nt", f["a"], f["w2"], c)[0])
    yk = f["y"][f["rmap"].long()].view(x.shape[0], K, -1)
    f["out"] = rn(rn((yk * f["tw"][..., None]).sum(1)) * hf)
    if f.get("residual") is not None:
        f["out"] = rn(f["out"] + f["residual"])
    return f


def check_loss(out: torch.Tensor, ref: torch.Tensor) -> Optional[float]:
    """The squared-output loss sum(out^2) against ``forward64(..., rounded=True)``, relative to that sum; returns the
    relative difference (asserted <= 1e-4).  Its terms do not cancel, so a systematic error shows at full size (a 1 %
    scale of out moves it by 2e-2).  The reference it is held to rounds where the reference's eager composition rounds:
    the node keeps those roundings, and they are not unbiased (a = bf16(bf16(silu(g)) u) sits about 1e-4 below
    silu(g) u on average), so against an unrounded forward a correct node would miss the bar by a few 1e-4.  Where the
    node and the reference round an intermediate to neighbouring bf16 values (a near tie), every output of that row
    moves by about one ulp; over a few hundred elements (T = 1) one such row alone is 2e-4 of the sum, so below
    LOSS_MIN_TERMS elements the bar is not a property of a correct node and None is returned."""
    if out.numel() < LOSS_MIN_TERMS:
        return None
    a = out.double().square().sum()
    b = ref.square().sum()
    rel = float((a - b).abs() / b.clamp_min(1e-300))
    assert rel <= LOSS_REL, f"loss sum(out^2): {float(a)!r} against float64 {float(b)!r} (relative {rel:.3g})"
    return rel


# ---- backward --------------------------------------------------------------------------------------------------------


def router_bwd_ref(logits, ids, K, scoring, norm, scaling, g_tw, B_tw, g_rw, g_lg, pure=False):
    """``(grad_logits, bound)`` in float64 (module docstring)."""
    T, E = logits.shape
    ld = logits.double().detach().requires_grad_(True)
    with torch.enable_grad():
        p = torch.softmax(ld, -1) if scoring == "softmax" else torch.sigmoid(ld)
        w = p.gather(1, ids)
        if norm:
            w = w / w.sum(-1, keepdim=True)
        loss = (w * scaling * g_tw).sum()
        if g_rw is not None:
            loss = loss + (p * g_rw.double()).sum()
        (gl,) = torch.autograd.grad(loss, ld)
    if g_lg is not None:
        gl = gl + g_lg.double()
    if pure:
        return gl, torch.zeros_like(gl)
    pd = p.detach()
    sel = pd.gather(1, ids)
    s = sel.sum(-1, keepdim=True) if norm else torch.ones_like(sel[:, :1])

    def grad_p(gt):  # the magnitude of the gradient reaching router_weights from |g_tw|
        gt = gt.abs()
        c = abs(scaling) * (gt + ((gt * sel / s).sum(-1, keepdim=True) if norm else 0.0)) / s
        return torch.zeros_like(pd).scatter_add(1, ids, c)

    def jac(gp):
        if scoring == "softmax":
            return pd * (gp + (gp * pd).sum(-1, keepdim=True))
        return gp * pd * (1 - pd)

    gp = grad_p(g_tw) + (g_rw.double().abs() if g_rw is not None else 0.0)
    A = jac(gp)
    glg = g_lg.double().abs() if g_lg is not None else 0.0
    _, pb = R.greedy_ref(logits, scoring)
    rel = torch.where(pd > 0, (pb - 2.0 ** -149) / pd.clamp_min(1e-300), torch.zeros_like(pd))
    rho = rel.amax(-1, keepdim=True) + (4 * K + 8) * U32
    perr = 5 * rho * A if scoring == "softmax" else 3 * rho * A + 8 * U32 * gp * pd
    bound = R.gamma(4 * K + 16 + E // 32 + 5) * (A + glg) + perr + jac(grad_p(B_tw)) + 2.0 ** -140
    return gl, bound


def backward_reference(node: Node, g_out, g_logits=None, g_rw=None, fw=None
                       ) -> Dict[str, Tuple[torch.Tensor, torch.Tensor]]:
    """``{name: (float64 reference, bound)}`` for every gradient the node returns.  With ``fw`` (:func:`forward64`) the
    chain runs on those float64 forward values with no rounding and the bounds are 0."""
    pure = fw is not None
    t = fw if pure else node.t
    K, hf = node.K, node.hf
    x, gw, w13, w2 = t["x"], t["gate_w"], t["w13"], t["w2"]
    T, H = x.shape
    E, I = gw.shape[0], w2.shape[2]
    M = T * K
    rmap, c = t["rmap"], [int(v) for v in t["tpe"].tolist()]
    tw, y, h, a, x_perm = t["tw"], t["y"], t["h"], t["a"], t["x_perm"]
    dev = x.device
    z = lambda shape: torch.zeros(shape, dtype=torch.float64, device=dev)  # noqa: E731
    res: Dict[str, Tuple[torch.Tensor, torch.Tensor]] = {}

    # combine backward: g_comb = g_out hf, g_y = g_comb p, g_tw = sum_h g_comb y
    if pure:
        g_comb = g_out.double() * hf
        g_y = z((M, H))
        flat = rmap.long()
        g_y[flat] = (g_comb[:, None, :] * tw.double()[..., None]).reshape(M, H)
        g_tw = (g_comb[:, None, :] * y[flat].view(T, K, H)).sum(-1)
        B_tw = torch.zeros_like(g_tw)
    else:
        g_comb = g_out if hf == 1.0 else (g_out.float() * hf).to(torch.bfloat16)
        g_y = NC.act_grad(g_comb, rmap, tw, K, M)[0]
        g_tw, B_tw = NC.prob_grad_ref(g_comb, y, rmap, K)
    g_y = g_y.double()

    # w2 backward: g_a = g_y w2 (nn), g_w2 = g_y^T a (tn, stage-local)
    p, S, _ = _per_expert("nn", g_y, w2, c)
    g_a, B_a = store(p, acc(H) * S, pure)
    o = G.offsets(c)
    tn_acc = torch.tensor([acc(o[e + 1] - o[e]) for e in range(E)], dtype=torch.float64, device=dev)[:, None, None]
    p, S, _ = _per_expert("tn", g_y, a, c)
    res["g_w2"] = (p, tn_acc * S)

    # SwiGLU backward: grad_u = g_a s, ds = g_a u, grad_g = ds sigmoid (1 + g (1 - sigmoid))
    g, u = h[:, :I], h[:, I:]
    if pure:
        sig = torch.sigmoid(g)
        gu, B_gu = g_a * g * sig, z((M, I))
        ds = g_a * u
        gg, B_gg = ds * sig * (1 + g * (1 - sig)), z((M, I))
    else:
        s, alt, tie = SW.s_candidates(g)
        sd = s.double()
        gu, B_gu = store(g_a * sd, B_a * sd.abs() + torch.where(tie, g_a.abs() * (alt.double() - sd).abs(), 0.0))
        ud = u.double()
        ds, B_ds = store(g_a * ud, B_a * ud.abs())
        p, e_k = SW.grad_g_ref(g, ds)
        sig = SW.sigmoid_ref(g)[0]
        gg, B_gg = store(p, e_k + B_ds * (sig * (1 + g.double() * (1 - sig))).abs())
    g_h, B_h = torch.cat([gg, gu], 1), torch.cat([B_gg, B_gu], 1)

    # w13 backward: g_xp = g_h w13 (nn), g_w13 = g_h^T x_perm (tn)
    p, S, P = _per_expert("nn", g_h, w13, c, B_h)
    g_xp, B_xp = store(p, P + acc(2 * I) * S, pure)
    p, S, P = _per_expert("tn", g_h, x_perm, c, B_h)
    res["g_w13"] = (p, P + tn_acc * S)

    # router and gate backward
    gl, B_l = router_bwd_ref(t["logits"], t["ids"], K, node.scoring, node.norm, node.scaling, g_tw, B_tw, g_rw,
                             g_logits, pure)
    xd, gwd = x.double(), gw.double()
    depth = T + 64 if E > 16 else -(-T // 132) + 8 + 512
    res["g_gate_w"] = (gl.T @ xd, B_l.T @ xd.abs() + R.gamma(depth) * (gl.abs().T @ xd.abs()))
    g_xg, B_xg = store(gl @ gwd, B_l @ gwd.abs() + R.gamma(E + 2) * (gl.abs() @ gwd.abs()), pure)

    # dispatch backward: bf16(bf16(sum_k g_xp[row(t, k)]) + g_x_gate)
    rows = rmap.long().view(T, K)
    s1 = g_xp[rows].sum(1)
    s1, B_s1 = store(s1, B_xp[rows].sum(1) + R.gamma(K) * g_xp[rows].abs().sum(1), pure)
    if node.kind == "moe":
        res["g_x"] = (s1 + g_xg, B_s1 + B_xg)
        if node.residual is not None:
            res["g_res"] = (g_out.double(), z((T, H)))
        return res

    # the block: RMSNorm backward of the bf16 g_x, then + g_out
    gx, B_gx = store(s1 + g_xg, B_s1 + B_xg, pure)
    hd = t["h_in"].double()
    if pure:
        rstd, nw = t["rstd"], t["norm_w"]
    elif node.kind == "block":
        rstd, nw = t["rstd"].double(), t["norm_w"].double()
    else:
        rstd, nw = NC.rstd_ref(t["h_in"], node.eps), t["norm_w"].to(torch.bfloat16).double()
    r = rstd[:, None]
    wg = gx * nw
    cc = (wg * hd).sum(-1, keepdim=True) * r * r / H
    p = (wg - hd * cc) * r
    Sg = r * (wg.abs() + hd.abs() * r * r * (wg * hd).abs().sum(-1, keepdim=True) / H)
    prop = r * (nw.abs() * B_gx + hd.abs() * r * r * (nw.abs() * B_gx * hd.abs()).sum(-1, keepdim=True) / H)
    tn = hd * r * gx  # terms of g_norm_w
    if node.kind == "fallback":
        rho_r = R.gamma(H + 32) / 2 + 4 * U32
        e_k = (R.gamma(H + 32) + 3 * rho_r) * Sg
        e_w = (R.gamma(T + 32) + rho_r) * tn.abs().sum(0)
    else:
        e_k = R.gamma(NC.G_H_ROUNDINGS) * Sg
        e_w = R.gamma(NC.gnw_depth(T, 264)) * tn.abs().sum(0)
    gh1, B_gh1 = store(p, e_k + prop, pure)
    res["g_h"] = (gh1 + g_out.double(), B_gh1)
    res["g_norm_w"] = (tn.sum(0), e_w + (hd.abs() * r * B_gx).sum(0))
    return res


def check_backward(node: Node, grads: Dict[str, torch.Tensor], g_out, g_logits=None, g_rw=None,
                   gate_bf16: bool = False) -> Dict[str, float]:
    """The node's gradients against :func:`backward_reference`; ``grads`` maps g_x / g_h, g_res, g_gate_w, g_w13, g_w2,
    g_norm_w to what autograd returned (g_norm_w may be None: the weight did not require grad).  ``gate_bf16``: the
    gate parameter is bf16, so its gradient went through autograd's cast back to bf16 (as the fallback's norm weight
    gradient does).  Returns the worst ratio per quantity."""
    ref = backward_reference(node, g_out, g_logits, g_rw)
    H = node.t["x"].shape[1]
    out: Dict[str, float] = {}
    if "g_res" in ref:
        NC.assert_bits_equal(grads["g_res"].reshape(-1, H), g_out, "g_residual")
    bf = set(BF16_GRADS) | ({"g_gate_w"} if gate_bf16 else set()) | ({"g_norm_w"} if node.kind == "fallback" else set())
    for name in ("g_w2", "g_w13", "g_x", "g_h", "g_gate_w", "g_norm_w"):
        if name not in ref or grads.get(name) is None:
            continue
        v, b = ref[name]
        got = grads[name].reshape(v.shape)
        b = TAU[name] * b + REF_SLACK * v.abs()
        if name in bf:
            out[name] = NC.check_near_tie(got, v, b, name)[0]
        else:
            out[name] = NC.check_bound(got, v, b, name)
    return out
