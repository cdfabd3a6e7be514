"""Lane-level model of ``csrc/gate_mma.cu`` (the tensor-core gate inside ``xtb_gate_route_dispatch``).  The CUDA kernel
cannot run in the CPU suite; this re-states its index arithmetic line by line — weight split into bf16 planes in B-fragment order,
per-lane 16-byte loads of x, the K permutation inside a 32-column block, the PTX fragment layout of
mma.sync.m16n8k16 (row.col, bf16), the K-quarter reduction and the output mapping — and checks that the result is
``x.float() @ w.T``.  It guards the mapping, not the hardware: the kernel's own tests are
tests/test_gpu_router_edges.py::test_fused_gate_logits and ::test_fused_gate_route_equals_router_on_its_own_logits."""
import numpy as np
import pytest
import torch

TOK, KQ = 32, 4


def bf16_round(v: np.ndarray) -> np.ndarray:
    return torch.from_numpy(v.astype(np.float32)).to(torch.bfloat16).float().numpy()


def mma_m16n8k16(c, a, b):
    """c[lane][4] += A @ B with the PTX fragment layout.  a: [32 lanes][4 regs][2 halves], b: [32][2][2]."""
    A = np.zeros((16, 16), np.float32)
    B = np.zeros((16, 8), np.float32)
    for lane in range(32):
        g, t = lane >> 2, lane & 3
        A[g, 2 * t : 2 * t + 2] = a[lane, 0]
        A[g + 8, 2 * t : 2 * t + 2] = a[lane, 1]
        A[g, 2 * t + 8 : 2 * t + 10] = a[lane, 2]
        A[g + 8, 2 * t + 8 : 2 * t + 10] = a[lane, 3]
        B[2 * t : 2 * t + 2, g] = b[lane, 0]
        B[2 * t + 8 : 2 * t + 10, g] = b[lane, 1]
    C = A.astype(np.float64) @ B.astype(np.float64)
    for lane in range(32):
        g, t = lane >> 2, lane & 3
        c[lane, 0] += C[g, 2 * t]
        c[lane, 1] += C[g, 2 * t + 1]
        c[lane, 2] += C[g + 8, 2 * t]
        c[lane, 3] += C[g + 8, 2 * t + 1]


@pytest.mark.parametrize("T,H,E", [(70, 256, 5), (33, 128, 8)])
def test_gate_mma_index_model(T, H, E):
    rng = np.random.default_rng(T)
    x = bf16_round(rng.standard_normal((T, H)))
    w = rng.standard_normal((E, H)).astype(np.float32) * 0.1
    n_steps = H // 32
    # ---- planes[p][step][lane][8] as the kernel fills them ------------------------------------------------
    planes = np.zeros((3, n_steps, 32, 8), np.float32)
    for step in range(n_steps):
        for ln in range(32):
            g, t = ln >> 2, ln & 3
            v = w[g, step * 32 + t * 8 : step * 32 + t * 8 + 8] if g < E else np.zeros(8, np.float32)
            hi = bf16_round(v)
            mid = bf16_round(v - hi)
            lo = bf16_round(v - hi - mid)
            planes[0, step, ln], planes[1, step, ln], planes[2, step, ln] = hi, mid, lo
    np.testing.assert_allclose(planes.sum(0).reshape(n_steps, 8, 4, 8)[:, :E].transpose(1, 0, 2, 3).reshape(E, H), w, rtol=2e-7, atol=0)

    logits = np.full((T, E), np.nan, np.float64)
    q_steps = n_steps // KQ
    for blk in range((T + TOK - 1) // TOK):
        red = np.zeros((2, KQ, 16, 8), np.float64)
        for warp in range(8):
            tg, kq = warp & 1, warp >> 1
            row0 = blk * TOK + tg * 16
            step0 = kq * q_steps
            c = np.zeros((32, 4), np.float64)
            for s in range(q_steps):
                step = step0 + s
                va = np.zeros((32, 8), np.float32)
                vb = np.zeros((32, 8), np.float32)
                for lane in range(32):
                    g, t = lane >> 2, lane & 3
                    ra, rb = min(row0 + g, T - 1), min(row0 + g + 8, T - 1)
                    col = step0 * 32 + t * 8 + s * 32
                    va[lane] = x[ra, col : col + 8]
                    vb[lane] = x[rb, col : col + 8]
                for p in (2, 1, 0):
                    wf = planes[p, step]  # [lane][8]: words x,y,z,w = element pairs (0,1)(2,3)(4,5)(6,7)
                    for half in range(2):  # first mma: words x,y ; second: words z,w
                        o = 4 * half
                        a = np.stack([va[:, o : o + 2], vb[:, o : o + 2], va[:, o + 2 : o + 4], vb[:, o + 2 : o + 4]], axis=1)
                        b = np.stack([wf[:, o : o + 2], wf[:, o + 2 : o + 4]], axis=1)
                        mma_m16n8k16(c, a, b)
            for lane in range(32):
                g, t = lane >> 2, lane & 3
                red[tg, kq, g, 2 * t], red[tg, kq, g, 2 * t + 1] = c[lane, 0], c[lane, 1]
                red[tg, kq, g + 8, 2 * t], red[tg, kq, g + 8, 2 * t + 1] = c[lane, 2], c[lane, 3]
        for tg in range(2):
            for r in range(16):
                token = blk * TOK + tg * 16 + r
                if token < T:
                    logits[token] = red[tg, :, r, :E].sum(0)
    ref = x.astype(np.float64) @ w.astype(np.float64).T
    assert not np.isnan(logits).any()
    np.testing.assert_allclose(logits, ref, rtol=1e-6, atol=1e-6)


def _greedy_route_token(lg, E, K, scoring, norm_topk, scaling):
    """``greedy_route_token<1, 8>`` of csrc/greedy_router.cuh (the router of the one-launch gate+router kernel), statement
    by statement (float32 arithmetic).  With one lane per token the group shuffles are empty and the kernel's two
    selection masks, ``taken`` (this lane's experts) and ``used`` (the token's), are one."""
    f32 = np.float32
    p = np.full(8, -np.inf, f32)
    p[:E] = lg[:E]
    m = p.max()
    if scoring == 0:
        s = f32(0)
        for j in range(8):
            p[j] = np.exp(p[j] - m, dtype=f32) if j < E else f32(0)
            s = f32(s + p[j])
        p = (p / s).astype(f32)
    else:
        for j in range(8):
            p[j] = f32(1) / (f32(1) + np.exp(-p[j], dtype=f32)) if j < E else -np.inf
    used, total = 0, f32(0)
    wv, se = np.zeros(K, f32), np.zeros(K, np.int64)
    for k in range(K):
        bv, be = -np.inf, 0x7FFFFFFF
        for j in range(8):
            if not (used >> j) & 1 and j < E and p[j] > bv:
                bv, be = p[j], j
        if be < 0 or be >= E:  # NaN rows: the lowest index not selected yet
            be, bv = next(e for e in range(E) if not (used >> e) & 1), f32(0)
        used |= 1 << be
        wv[k], se[k] = bv, be
        total = f32(total + bv)
    for k in range(K):
        v = wv[k]
        if norm_topk:
            v = f32(v / total)
        if scaling != 1.0:
            v = f32(v * f32(scaling))
        wv[k] = v
    return p, wv, se


@pytest.mark.parametrize("E,K,scoring,norm,scaling", [(8, 2, "softmax", True, 1.0), (5, 3, "softmax", False, 2.0), (8, 1, "sigmoid", True, 1.0),
                                                     (4, 2, "sigmoid", False, 1.5)])
def test_route_token_model_matches_oracle_router(E, K, scoring, norm, scaling):
    """The per-token router of the one-launch gate+router kernel and its ballot histogram vs the oracle's greedy router."""
    from oracle import moe_oracle as O

    T = 70
    lg = torch.randn(T, E, generator=torch.Generator().manual_seed(E * 10 + K)) * 2
    ref = O.greedy_router(lg, K, norm, scaling, scoring)
    ids = np.zeros((T, K), np.int64)
    with np.errstate(over="ignore", invalid="ignore"):
        for t in range(T):
            p, wv, se = _greedy_route_token(np.pad(lg[t].numpy(), (0, 8 - E)), E, K, 0 if scoring == "softmax" else 1, norm, scaling)
            ids[t] = se
            np.testing.assert_allclose(p[:E], ref["router_weights"][t].numpy(), rtol=2e-6, atol=1e-7)
            np.testing.assert_allclose(wv, ref["topk_weights"][t].numpy(), rtol=2e-6, atol=1e-7)
    assert np.array_equal(ids, ref["topk_ids"].numpy())
    # chunk histograms by ballots: counts[c][e] = #(token, k) of the 32-token chunk c routed to expert e
    n_chunks = (T + 31) // 32
    counts = np.zeros((n_chunks, E), np.int64)
    for c in range(n_chunks):
        for k in range(K):
            for e in range(E):
                ballot = [(c * 32 + lane < T) and ids[min(c * 32 + lane, T - 1), k] == e for lane in range(32)]
                counts[c, e] += sum(ballot)
    assert np.array_equal(counts.sum(0), ref["topkens_per_expert"].numpy())


def test_route_token_model_nan_fallback_after_a_gap():
    """A row whose NaN experts run the top-k out of comparable scores after a gap in the selected ids: the fallback takes
    the lowest id not selected yet (1), not the round number (2).  Written out by hand: torch.topk, and so the oracle,
    ranks NaN first."""
    f32 = np.float32
    lg = np.array([3, np.nan, 2, np.nan, 0, 0, 0, 0], f32)
    with np.errstate(invalid="ignore"):
        p, wv, se = _greedy_route_token(lg, 4, 3, 1, True, 1.0)
    s3, s2 = f32(1) / (f32(1) + np.exp(f32(-3))), f32(1) / (f32(1) + np.exp(f32(-2)))
    assert se.tolist() == [0, 2, 1]
    np.testing.assert_array_equal(p[[0, 2]], [s3, s2])
    assert np.isnan(p[[1, 3]]).all()
    np.testing.assert_array_equal(wv, [s3 / f32(s3 + s2), s2 / f32(s3 + s2), 0])
