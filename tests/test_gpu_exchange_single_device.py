"""The peer-exchange kernels (csrc/comm.cu) and the expert-parallel pulls (csrc/ep.cu) on ONE device, against the
references of tests/exchange_reference.py.

Every kernel here takes a device table of per-rank base pointers and reads or writes through it with ordinary global
loads and stores, so W buffers on one GPU stand in for W ranks and the same machine code runs with the same addressing.
Every buffer sits in a NaN-filled arena with guard bytes around it (R.SimWorld), and every output must leave them alone.
Copies are compared bit for bit; a NaN is compared by position only (the CUDA cast gives 0x7FFF, torch 0x7FC0).

* xtb_a2a_pull: both directions of a2a_plan for W in {1, 2, 3, 4, 8, 16}, Ulysses [1, S, Hq, 128] bf16 shapes forward and
  inverse, 3-D and 5-D shapes with outer = 1 and mid = 1, fp32 and int8 elements, rows of 16, 48 and 14336 bytes; totals
  below, at and above one grid-stride step; the round trip is the identity; refusals.
* xtb_allgather_push: bf16 and fp32 shards (every fp32 special class), W in {1, 2, 3, 8}, n = 8, a vector tail, >= 4 waves.
* xtb_reduce_scatter_pull / xtb_allreduce_pull_f32: W = 1 .. 8 and 16 (the 4-wide rank batches and their tails), scales
  1, 1/W, 2^-3, exact and random inputs: bit-equal to the exact restatement and within the float64 bound.
* xtb_ep_write_header, xtb_ep_pull_to_experts / xtb_ep_pull_to_sources: W in {1, 2, 4, 8, 16} x E in {W, 8W, 256, 1024}
  under five loads, first-use and reuse paths, capacity, m_rows and refusals; the EP exchange end to end against ep = 1.
* xtb_peer_memcpy_batch (a refused batch copies nothing) and xtb_peer_barrier at world = 1 and its refusals only: a
  barrier with world > 1 waits for peers that do not exist on one device, so this file never launches one.
* One a2a and one EP case whose addresses pass 2^31 bytes.
"""
import contextlib
import ctypes

import numpy as np
import pytest
import torch

from tests import exchange_reference as R
from tests.gpu_harness import XTB_ERR_INVALID, Worst, sm_count
from xtuner_b200._capi import check, current_stream, ensure_init, ptr

pytestmark = pytest.mark.gpu

WORST = Worst("exchange_single_device")  # in random mode
PEAK = {}


@contextlib.contextmanager
def _peaks():
    yield
    for k, v in sorted(PEAK.items()):
        print(f"exchange_single_device: peak memory {k}: {v / 2**30:.2f} GiB")


_report = WORST.fixture(_peaks)


def _t(x):
    return torch.as_tensor(x, device="cuda")


# ---- xtb_a2a_pull ------------------------------------------------------------------------------------------------------

# (name, shape for world W, dtype, scatter_dim, gather_dim)
A2A_CASES = [
    ("ulysses_fwd_h32", lambda W: (1, 64, 32, 128), torch.bfloat16, 2, 1),
    ("ulysses_inv_h32", lambda W: (1, 64 * W, 32 // W, 128), torch.bfloat16, 1, 2),
    ("ulysses_fwd_h8", lambda W: (1, 32, 8, 128), torch.bfloat16, 2, 1),
    ("ulysses_inv_h8", lambda W: (1, 32 * W, 8 // W, 128), torch.bfloat16, 1, 2),
    ("ulysses_fwd_h24", lambda W: (2, 16, 24, 128), torch.bfloat16, 2, 1),
    ("ulysses_inv_h24", lambda W: (2, 16 * W, 24 // W, 128), torch.bfloat16, 1, 2),
    ("3d_f32_lo", lambda W: (3 * W, 5, 12), torch.float32, 0, 1),
    ("3d_f32_hi", lambda W: (5, 2 * W, 12), torch.float32, 1, 0),
    ("5d_i8_outer1_mid1_row48", lambda W: (1, 2 * W, 1, 3, 16), torch.int8, 1, 3),
    ("5d_i8_outer1_mid1_hi", lambda W: (1, 3, 1, 2 * W, 16), torch.int8, 3, 1),
    ("5d_f32", lambda W: (2, W, 3, 4, 8), torch.float32, 1, 3),
    ("5d_f32_hi", lambda W: (2, 3, 3, 2 * W, 4), torch.float32, 3, 1),
    ("row16", lambda W: (4 * W, 4), torch.float32, 0, 1),
    ("row14336", lambda W: (2 * W, 7168), torch.bfloat16, 0, 1),
    ("row14336_mid3", lambda W: (1, 2 * W, 3, 7168), torch.bfloat16, 1, 3),
]
A2A_WORLDS = [1, 2, 3, 4, 8, 16]


def _a2a_params():
    from xtuner_b200.comm import a2a_plan

    out = []
    for name, shape_fn, dtype, s, g in A2A_CASES:
        for W in A2A_WORLDS:
            if name.startswith("ulysses_inv") and int(name.split("_h")[1]) % W:
                continue
            shape = shape_fn(W)
            es = torch.tensor([], dtype=dtype).element_size()
            if shape[s] % W or a2a_plan(shape, s, g, W, 0, es).row_bytes % 16:
                continue
            out.append(pytest.param(shape, dtype, s, g, W, id=f"{name}-W{W}"))
    return out


def _a2a_args(plan):
    return (plan.n_o, plan.n_x, plan.n_m, plan.row_bytes, plan.src_stride_o, plan.src_stride_x, plan.src_stride_m,
            plan.src_base, plan.dst_stride_o, plan.dst_stride_x, plan.dst_stride_m, plan.dst_peer_stride)


def _run_a2a(inputs, s, g, what):
    """Every simulated rank pulls its share of every input; returns the W outputs after checking them and the guards."""
    from xtuner_b200.comm import a2a_plan

    W, shape, dtype = len(inputs), tuple(inputs[0].shape), inputs[0].dtype
    es = inputs[0].element_size()
    nbytes = inputs[0].numel() * es
    world = R.SimWorld(W, nbytes)
    for r in range(W):
        world.buf(r, dtype, shape).copy_(inputs[r])
    outs = []
    for r in range(W):
        plan = a2a_plan(shape, s, g, W, r, es)
        o = R.guarded(nbytes)
        check(ensure_init().xtb_a2a_pull(world.table.data_ptr(), o.ptr(0), r, W, *_a2a_args(plan), current_stream()),
              "xtb_a2a_pull")
        outs.append((o, plan))
    torch.cuda.synchronize()
    got = []
    for r, (o, plan) in enumerate(outs):
        t = o.buf(0, dtype, plan.out_shape)
        R.assert_bits_equal(t, R.a2a(inputs, s, g, r), f"{what}: rank {r}")
        assert o.guards_intact(), f"{what}: rank {r} wrote outside its output"
        got.append(t)
    assert world.guards_intact(), f"{what}: an input guard changed"
    return got


@pytest.mark.parametrize("shape,dtype,s,g,W", _a2a_params())
def test_a2a_pull_matches_reference_and_round_trips(shape, dtype, s, g, W):
    es = torch.tensor([], dtype=dtype).element_size()
    nbytes = int(np.prod(shape)) * es
    inputs = [R.labels(nbytes, r).view(dtype).view(shape) for r in range(W)]
    mid = _run_a2a(inputs, s, g, f"a2a {shape} s={s} g={g}")
    back = _run_a2a([m.clone() for m in mid], g, s, "inverse")
    for r in range(W):
        R.assert_bits_equal(back[r], inputs[r], f"round trip rank {r}")


@pytest.mark.parametrize("W", [2, 3])
@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_a2a_pull_grid_stride_step(W, delta):
    """16-byte rows, so the total is the row count: one grid-stride step of a source's blocks is per_src * 256 * 8
    vectors, per_src capped at 2 * SMs / W.  Totals just below, at and just above one full step."""
    cap = max(1, 2 * sm_count() // W)
    total = cap * 256 * 8 + delta
    inputs = [R.labels(W * total * 16, r).view(torch.int16).view(W * total, 8) for r in range(W)]
    _run_a2a(inputs, 0, 1, f"a2a total={total}")


def test_a2a_pull_refusals():
    from xtuner_b200.comm import a2a_plan

    lib, W = ensure_init(), 2
    shape = (2 * W, 64)
    world = R.SimWorld(W, 2 * W * 64 * 2)
    o = R.guarded(2 * W * 64 * 2)
    args = list(_a2a_args(a2a_plan(shape, 0, 1, W, 1, 2)))
    names = ["row_bytes", "src_stride_o", "src_stride_x", "src_stride_m", "src_base", "dst_stride_o", "dst_stride_x",
             "dst_stride_m", "dst_peer_stride"]
    n0 = lib.xtb_launch_count()
    for k, name in enumerate(names):
        bad = list(args)
        bad[3 + k] += 8
        rc = lib.xtb_a2a_pull(world.table.data_ptr(), o.ptr(0), 1, W, *bad, current_stream())
        assert rc == XTB_ERR_INVALID, f"{name} not a multiple of 16 was accepted"
    assert lib.xtb_a2a_pull(world.table.data_ptr(), o.ptr(0), 1, W, *args[:3], 0, *args[4:],
                            current_stream()) == XTB_ERR_INVALID
    assert lib.xtb_launch_count() == n0
    torch.cuda.synchronize()
    assert bool((o.arena == R.FILL32).all())


# ---- xtb_allgather_push ------------------------------------------------------------------------------------------------


def _ag_n(kind):
    return {"8": 8, "tail": 8 * (3 * 2048 + 5), "waves": 8 * (4 * 2 * sm_count() * 256 + 3)}[kind]


@pytest.mark.parametrize("W", [1, 2, 3, 8])
@pytest.mark.parametrize("f32", [True, False], ids=["f32", "bf16"])
@pytest.mark.parametrize("kind", ["8", "tail", "waves"])
def test_allgather_push(W, f32, kind):
    lib, n = ensure_init(), _ag_n(kind)
    shards = [R.f32_specials(n, seed=r) for r in range(W)]
    if not f32:
        shards = [x.to(torch.bfloat16) for x in shards]
    outs = R.SimWorld(W, W * n * 2)
    for r in range(W):
        check(lib.xtb_allgather_push(shards[r].data_ptr(), outs.table.data_ptr(), r, W, n, int(f32), current_stream()),
              "xtb_allgather_push")
    torch.cuda.synchronize()
    want = R.allgather(shards)
    for d in range(W):
        R.assert_bits_equal(outs.buf(d, torch.bfloat16), want, f"all-gather output of rank {d}")
    assert outs.guards_intact(), "all-gather wrote outside an output"


# ---- xtb_reduce_scatter_pull / xtb_allreduce_pull_f32 ------------------------------------------------------------------


def _scales(W):
    return [1.0, float(np.float32(1.0 / W)), 0.125]


@pytest.mark.parametrize("W", [1, 2, 3, 4, 5, 6, 7, 8, 16])
@pytest.mark.parametrize("out_f32", [True, False], ids=["f32out", "bf16out"])
@pytest.mark.parametrize("mode", ["exact", "random"])
def test_reduce_scatter_pull(W, out_f32, mode):
    lib, n = ensure_init(), 8 * 4099
    x = R.rank_values(W, W * n, mode, seed=100 * W + out_f32)
    world = R.SimWorld(W, W * n * 2)
    for r in range(W):
        world.buf(r, torch.bfloat16).copy_(x[r])
    es = 4 if out_f32 else 2
    for scale in _scales(W):
        outs = []
        for me in range(W):
            o = R.guarded(n * es)
            check(lib.xtb_reduce_scatter_pull(world.table.data_ptr(), o.ptr(0), me, W, n, scale, int(out_f32),
                                              current_stream()), "xtb_reduce_scatter_pull")
            outs.append(o)
        torch.cuda.synchronize()
        for me, o in enumerate(outs):
            got = o.buf(0, torch.float32 if out_f32 else torch.bfloat16)
            what = f"reduce-scatter W={W} rank {me} scale {scale}"
            R.assert_bits_equal(got, R.reduce_scatter(x, me, scale, out_f32), what)
            ref64, S = R.sum_ref64(x, me, scale)
            ratio = R.assert_within(got, ref64, R.rs_bound(ref64, S, W, scale, out_f32), what + " (fp64)")
            if mode == "exact":
                exact = ref64.float() if out_f32 else R.bf16_rne(ref64.float())
                R.assert_bits_equal(got, exact, what + " (exact sum)")
            else:
                WORST.note(f"reduce_scatter {'f32' if out_f32 else 'bf16'} out", ratio)
            assert o.guards_intact(), what + ": wrote outside its output"
    assert world.guards_intact()


@pytest.mark.parametrize("W", list(range(1, 17)))
@pytest.mark.parametrize("mode", ["exact", "random"])
def test_allreduce_pull_f32(W, mode):
    lib, n = ensure_init(), 4 * 8195
    x = R.rank_values(W, n, mode, seed=7 * W, dtype=torch.float32)
    world = R.SimWorld(W, n * 4)
    for r in range(W):
        world.buf(r, torch.float32).copy_(x[r])
    scale = float(np.float32(1.0 / W))
    outs = []
    for me in range(W):
        o = R.guarded(n * 4)
        check(lib.xtb_allreduce_pull_f32(world.table.data_ptr(), o.ptr(0), me, W, n, scale, current_stream()),
              "xtb_allreduce_pull_f32")
        outs.append(o)
    torch.cuda.synchronize()
    want = R.allreduce(x, scale)
    ref64, S = R.sum_ref64(x, 0, scale, shard=False)
    for me, o in enumerate(outs):
        got = o.buf(0, torch.float32)
        R.assert_bits_equal(got, want, f"all-reduce W={W} rank {me}")
        R.assert_bits_equal(got, outs[0].buf(0, torch.float32), f"all-reduce W={W}: rank {me} differs from rank 0")
        ratio = R.assert_within(got, ref64, R.rs_bound(ref64, S, W, scale, True), "all-reduce fp64")
        if mode == "exact":
            R.assert_bits_equal(got, ref64.float(), "all-reduce exact sum")
        else:
            WORST.note("allreduce f32", ratio)
        assert o.guards_intact()


# ---- expert-parallel exchange ------------------------------------------------------------------------------------------


@pytest.mark.parametrize("E", [1, 8, 256, 257, 1024])
def test_ep_write_header(E):
    tpe = torch.randint(0, 2**31 - 1, (E,), dtype=torch.int64, device="cuda")
    tpe[0] = 2**31 - 1
    o = R.guarded(4 * E)
    check(ensure_init().xtb_ep_write_header(tpe.data_ptr(), o.ptr(0), E, current_stream()), "xtb_ep_write_header")
    torch.cuda.synchronize()
    assert torch.equal(o.buf(0, torch.int32), tpe.to(torch.int32))
    assert o.guards_intact()


class _EP:
    """W source-major staging buffers (header written by xtb_ep_write_header, then the labelled rows) of one count table."""

    def __init__(self, cnt, row_bytes, rows=None):
        self.cnt, self.rb = cnt, row_bytes
        self.W, self.E = cnt.shape
        self.El = self.E // self.W
        self.hdr = R.ep_hdr_bytes(self.E)
        self.words = row_bytes // 4
        self.rows = rows if rows is not None else R.ep_rows(cnt, row_bytes)
        self.M = [len(r) for r in self.rows]
        self.src = R.SimWorld(self.W, self.hdr + max(max(self.M), 1) * row_bytes)
        self.cnt_dev = _t(cnt.astype(np.int32))
        self.te_all = [R.ep_to_experts(cnt, d) for d in range(self.W)]
        for s in range(self.W):
            tpe = _t(cnt[s].astype(np.int64))
            check(ensure_init().xtb_ep_write_header(tpe.data_ptr(), self.src.ptr(s), self.E, current_stream()),
                  "xtb_ep_write_header")
            torch.cuda.synchronize()
            if self.M[s]:
                self.src.bytes(s)[self.hdr : self.hdr + self.M[s] * row_bytes].copy_(self.rows[s].view(torch.uint8).view(-1))

    def owners(self, cap):
        return R.SimWorld(self.W, self.hdr + max(cap, 1) * self.rb)

    def owner_rows(self, own, d):
        return own.bytes(d)[self.hdr :].view(torch.int32).view(-1, self.words)

    def to_experts(self, own, d, cap, first=True, status_init=(-1, 0)):
        """pull for owner d into own's buffer d; returns (cnt_all_out, tpe_local, status) of the first-use path."""
        lib = ensure_init()
        cnt_out = torch.full((self.W * self.E,), -7, dtype=torch.int32, device="cuda") if first else None
        tpe = torch.full((self.El,), -7, dtype=torch.int64, device="cuda") if first else None
        status = torch.tensor(status_init, dtype=torch.int32, device="cuda") if first else None
        check(lib.xtb_ep_pull_to_experts(self.src.table.data_ptr(), None if first else self.cnt_dev.data_ptr(),
                                         ptr(cnt_out), own.ptr(d, self.hdr), ptr(tpe), ptr(status), d, self.W, self.E,
                                         self.rb, self.hdr, cap, current_stream()), "xtb_ep_pull_to_experts")
        return cnt_out, tpe, status

    def to_sources(self, own, s, cap, m_rows):
        out = R.guarded(max(self.M[s], 1) * self.rb)
        check(ensure_init().xtb_ep_pull_to_sources(own.table.data_ptr(), self.cnt_dev.data_ptr(), out.ptr(0), s, self.W,
                                                   self.E, self.rb, self.hdr, cap, m_rows, current_stream()),
              "xtb_ep_pull_to_sources")
        return out

    def check_first_use(self, d, cnt_out, tpe, status, cap):
        total = len(self.te_all[d])
        assert torch.equal(cnt_out, self.cnt_dev.view(-1)), f"owner {d}: cnt_all_out differs from the headers"
        want_tpe = self.cnt[:, d * self.El : (d + 1) * self.El].sum(0)
        assert tpe.tolist() == want_tpe.tolist(), f"owner {d}: tokens_per_expert_local"
        assert status.tolist() == [total, int(total > cap)], f"owner {d}: status {status.tolist()}, total {total}, cap {cap}"


EP_ROW_BYTES = [16, 48, 4096, 14336]
EP_GRID = [(W, E) for W in (1, 2, 4, 8, 16) for E in sorted({W, 8 * W, 256, 1024})]
EP_LOADS = ["uniform", "zipf", "holes", "empty_rank", "one_owner"]


def _pick_row_bytes(cnt, pref, budget=48 << 20):
    W = cnt.shape[0]
    most = max(int(cnt.sum(0).reshape(W, -1).sum(1).max()), int(cnt.sum(1).max()), 1)
    fits = [rb for rb in EP_ROW_BYTES if 2 * W * most * rb <= budget]
    return pref if pref in fits else max(fits)


@pytest.mark.parametrize("load", EP_LOADS)
@pytest.mark.parametrize("W,E", EP_GRID)
def test_ep_pulls_match_reference(W, E, load):
    seed = 1000 * W + E + EP_LOADS.index(load)
    cnt = R.ep_counts(W, E, load, seed)
    ep = _EP(cnt, _pick_row_bytes(cnt, EP_ROW_BYTES[seed % 4]))
    cap = max(len(t) for t in ep.te_all)
    own, own2 = ep.owners(cap), ep.owners(cap)
    firsts = [ep.to_experts(own, d, cap) for d in range(W)]
    for d in range(W):
        ep.to_experts(own2, d, cap, first=False)  # reuse path: counts from cnt_all_in
    torch.cuda.synchronize()
    owner_rows = [ep.owner_rows(own, d) for d in range(W)]
    for d in range(W):
        what = f"W={W} E={E} {load} rb={ep.rb} owner {d}"
        R.check_to_experts(owner_rows[d][:cap], ep.rows, cnt, d, cap, what)
        ep.check_first_use(d, *firsts[d], cap)
        assert torch.equal(ep.owner_rows(own2, d), owner_rows[d]), what + ": reuse path differs from first use"
    assert own.guards_intact() and own2.guards_intact() and ep.src.guards_intact()
    backs = [ep.to_sources(own, s, cap, ep.M[s]) for s in range(W)]
    torch.cuda.synchronize()
    for s in range(W):
        got = backs[s].bytes(0).view(torch.int32).view(-1, ep.words)
        R.check_to_sources(got, owner_rows, cnt, s, cap, ep.M[s], f"W={W} E={E} {load} source {s}", ep.te_all)
        R.assert_rows_equal(got[: ep.M[s]], ep.rows[s], f"round trip of source {s}")
        assert backs[s].guards_intact()


def test_ep_pull_more_rows_than_warps():
    """one owner receives more rows than the 2 * SMs * 8 warps of the grid (and rows of 48 bytes: no 8-vector batch)"""
    W, E = 2, 8
    n_warps = 2 * sm_count() * 8
    cnt = np.zeros((W, E), dtype=np.int64)
    cnt[:, 4:] = (n_warps + 37) // 4
    ep = _EP(cnt, 48)
    cap = len(ep.te_all[1])
    assert cap > n_warps
    own = ep.owners(cap)
    f = ep.to_experts(own, 1, cap)
    torch.cuda.synchronize()
    R.check_to_experts(ep.owner_rows(own, 1)[:cap], ep.rows, cnt, 1, cap, "owner 1")
    ep.check_first_use(1, *f, cap)
    for s in range(W):
        b = ep.to_sources(own, s, cap, ep.M[s])
        torch.cuda.synchronize()
        R.assert_rows_equal(b.bytes(0).view(torch.int32).view(-1, 12)[: ep.M[s]], ep.rows[s], f"round trip {s}")


def test_ep_capacity_and_m_rows():
    W, E = 4, 16
    cnt = R.ep_counts(W, E, "uniform", seed=5, rows_per_rank=200)
    ep = _EP(cnt, 4096)
    total = [len(t) for t in ep.te_all]
    assert min(total) > 8
    for cap_of in (lambda t: t - 5, lambda t: 0, lambda t: t, lambda t: t + 3):
        caps = [cap_of(t) for t in total]
        cap = min(caps)  # one capacity for every rank, as the dispatcher uses
        own = ep.owners(max(total) + 3)
        firsts = [ep.to_experts(own, d, cap) for d in range(W)]
        torch.cuda.synchronize()
        owner_rows = [ep.owner_rows(own, d) for d in range(W)]
        for d in range(W):
            R.check_to_experts(owner_rows[d], ep.rows, cnt, d, cap, f"owner {d} cap {cap}")
            ep.check_first_use(d, *firsts[d], cap)
        # the way back leaves every row whose source lies past the capacity untouched; m_rows below the row count
        for s in range(W):
            for m_rows in (ep.M[s], ep.M[s] - 7, 0):
                b = ep.to_sources(own, s, cap, m_rows)
                torch.cuda.synchronize()
                got = b.bytes(0).view(torch.int32).view(-1, ep.words)
                R.check_to_sources(got, owner_rows, cnt, s, cap, m_rows, f"source {s} cap {cap} m_rows {m_rows}", ep.te_all)
                assert b.guards_intact()
        assert own.guards_intact()


def test_ep_refusals():
    lib = ensure_init()
    cnt = np.ones((2, 8), dtype=np.int64)
    ep = _EP(cnt, 16)
    own = ep.owners(16)
    table, cd, dst = ep.src.table.data_ptr(), ep.cnt_dev.data_ptr(), own.ptr(0, ep.hdr)

    def te(world=2, E=8, rb=16, hdr=256, cin=cd, cout=None, rank=0):
        return lib.xtb_ep_pull_to_experts(table, cin, cout, dst, None, None, rank, world, E, rb, hdr, 16,
                                          current_stream())

    def ts(world=2, E=8, rb=16, hdr=256, rank=0):
        return lib.xtb_ep_pull_to_sources(table, cd, dst, rank, world, E, rb, hdr, 16, 8, current_stream())

    n0 = lib.xtb_launch_count()
    for f in (te, ts):
        assert f(world=17, E=34) == XTB_ERR_INVALID, "W > 16"
        assert f(world=16, E=1040) == XTB_ERR_INVALID, "E > 1024"
        assert f(world=3, E=8) == XTB_ERR_INVALID, "E not divisible by W"
        assert f(world=1, E=1025) == XTB_ERR_INVALID, "E > 1024"
        assert f(E=8, hdr=16) == XTB_ERR_INVALID, "header shorter than 4 E"
        assert f(E=1024, hdr=4080) == XTB_ERR_INVALID, "header shorter than 4 E"
        assert f(rb=24) == XTB_ERR_INVALID, "row_bytes not a multiple of 16"
        assert f(rb=0) == XTB_ERR_INVALID
        assert f(rank=2) == XTB_ERR_INVALID
    assert te(cin=None, cout=None) == XTB_ERR_INVALID, "neither cnt_all_in nor cnt_all_out"
    assert lib.xtb_launch_count() == n0
    torch.cuda.synchronize()
    assert bool((own.arena == R.FILL32).all())


def test_ep_end_to_end_matches_ep1():
    """W simulated ranks with their own tokens and top-k ids: permute -> header -> pull to experts -> the grouped expert
    MLP on each owner's rows -> pull to sources -> unpermute, forward and backward through the same pulls, against the
    ep = 1 path on the concatenated tokens.  The owners see every expert's rows in the ep = 1 order, and the grouped GEMMs
    are per-row deterministic, so every result must be bit-identical."""
    from xtuner_b200 import ops

    W, E, K, H, I = 4, 16, 2, 256, 128
    El = E // W
    g = torch.Generator(device="cuda").manual_seed(11)
    T = [96 + 32 * s for s in range(W)]
    xs = [torch.randn(t, H, generator=g, device="cuda").to(torch.bfloat16) for t in T]
    ids = [torch.rand(t, E, generator=g, device="cuda").topk(K, dim=1).indices.to(torch.int32) for t in T]
    ps = [torch.rand(t, K, generator=g, device="cuda") for t in T]
    gos = [torch.randn(t, H, generator=g, device="cuda").to(torch.bfloat16) for t in T]
    w13 = (torch.randn(E, 2 * I, H, generator=g, device="cuda") * H**-0.5).to(torch.bfloat16)
    w2 = (torch.randn(E, H, I, generator=g, device="cuda") * I**-0.5).to(torch.bfloat16)

    def experts(xp, tpe, a, b):
        return ops.group_gemm(ops.swiglu(ops.group_gemm(xp, a, tpe)), b, tpe)

    # ep = 1
    x1 = torch.cat(xs).requires_grad_(True)
    w13_1, w2_1 = w13.clone().requires_grad_(True), w2.clone().requires_grad_(True)
    xp, rmap, _, tpe = ops.permute(x1, torch.cat(ids), n_experts=E, return_extra=True)
    ref = ops.unpermute(experts(xp, tpe, w13_1, w2_1), rmap, torch.cat(ps))
    g_x1, g_w13_1, g_w2_1 = torch.autograd.grad(ref, (x1, w13_1, w2_1), torch.cat(gos))

    # ep = W on one device
    lib, rb = ensure_init(), 2 * H
    hdr = R.ep_hdr_bytes(E)
    x_s = [x.clone().requires_grad_(True) for x in xs]
    perm = [ops.permute(x_s[s], ids[s], n_experts=E, return_extra=True) for s in range(W)]
    cnt = np.stack([perm[s][3].cpu().numpy() for s in range(W)])
    M = [int(c.sum()) for c in cnt]
    n_own = [int(cnt[:, d * El : (d + 1) * El].sum()) for d in range(W)]
    cap = sum(M)
    cnt_dev = _t(cnt.astype(np.int32))

    def stage(tensors, header_tpe=None):
        wld = R.SimWorld(W, hdr + max(max(len(t) for t in tensors), 1) * rb)
        for r, t in enumerate(tensors):
            if header_tpe is not None:
                check(lib.xtb_ep_write_header(header_tpe[r].data_ptr(), wld.ptr(r), E, current_stream()),
                      "xtb_ep_write_header")
            if len(t):
                wld.bytes(r)[hdr : hdr + len(t) * rb].copy_(t.detach().contiguous().view(torch.uint8).view(-1))
        return wld

    def pull_to_experts(src, first):
        own = R.SimWorld(W, hdr + cap * rb)
        tpes, cnt_out = [], torch.empty(W * E, dtype=torch.int32, device="cuda")
        for d in range(W):
            tl = torch.empty(El, dtype=torch.int64, device="cuda")
            check(lib.xtb_ep_pull_to_experts(src.table.data_ptr(), None if first else cnt_dev.data_ptr(),
                                             cnt_out.data_ptr() if first else None, own.ptr(d, hdr), tl.data_ptr(),
                                             None, d, W, E, rb, hdr, cap, current_stream()), "xtb_ep_pull_to_experts")
            tpes.append(tl)
        rows = [own.bytes(d)[hdr : hdr + n_own[d] * rb].view(torch.bfloat16).view(-1, H) for d in range(W)]
        return rows, tpes

    def pull_to_sources(own):
        outs = []
        for s in range(W):
            o = torch.empty(M[s], H, dtype=torch.bfloat16, device="cuda")
            check(lib.xtb_ep_pull_to_sources(own.table.data_ptr(), cnt_dev.data_ptr(), o.data_ptr(), s, W, E, rb, hdr,
                                             cap, M[s], current_stream()), "xtb_ep_pull_to_sources")
            outs.append(o)
        return outs

    rows, tpes = pull_to_experts(stage([p[0] for p in perm], [p[3] for p in perm]), first=True)
    assert [int(t.sum()) for t in tpes] == n_own
    e_d = [r.clone().requires_grad_(True) for r in rows]
    w13_d = [w13[d * El : (d + 1) * El].clone().requires_grad_(True) for d in range(W)]
    w2_d = [w2[d * El : (d + 1) * El].clone().requires_grad_(True) for d in range(W)]
    y_d = [experts(e_d[d], tpes[d], w13_d[d], w2_d[d]) for d in range(W)]
    b_s = [b.requires_grad_(True) for b in pull_to_sources(stage(y_d))]
    out_s = [ops.unpermute(b_s[s], perm[s][1], ps[s]) for s in range(W)]
    R.assert_bits_equal(torch.cat(out_s), ref, "EP forward vs ep = 1")

    g_b = [torch.autograd.grad(out_s[s], b_s[s], gos[s])[0] for s in range(W)]
    g_y, _ = pull_to_experts(stage(g_b), first=False)  # the backward of the return trip: the reuse path
    grads = [torch.autograd.grad(y_d[d], (e_d[d], w13_d[d], w2_d[d]), g_y[d]) for d in range(W)]
    g_xp = pull_to_sources(stage([gr[0] for gr in grads]))
    g_x = [torch.autograd.grad(perm[s][0], x_s[s], g_xp[s])[0] for s in range(W)]
    R.assert_bits_equal(torch.cat(g_x), g_x1, "EP input gradient vs ep = 1")
    R.assert_bits_equal(torch.cat([gr[1] for gr in grads]), g_w13_1, "EP w13 gradient vs ep = 1")
    R.assert_bits_equal(torch.cat([gr[2] for gr in grads]), g_w2_1, "EP w2 gradient vs ep = 1")


# ---- xtb_peer_memcpy_batch ---------------------------------------------------------------------------------------------


def _batch(dsts, srcs, nbytes):
    n = len(dsts)
    return ((ctypes.c_void_p * max(n, 1))(*dsts), (ctypes.c_void_p * max(n, 1))(*srcs), (ctypes.c_int64 * max(n, 1))(*nbytes))


def test_peer_memcpy_batch():
    lib = ensure_init()
    sizes = [1, 3, 17, 4097, 0, 65535]
    src = R.labels(1 << 20, 3)
    dst = R.guarded(1 << 20)
    offs = [0, 4096, 8192, 12288, 20480, 24576]
    d_ptrs = [dst.ptr(0, o) for o in offs] + [src.data_ptr()]
    s_ptrs = [src.data_ptr() + o + 5 for o in offs] + [src.data_ptr()]  # the last entry has dst == src: skipped
    nb = sizes + [64]
    check(lib.xtb_peer_memcpy_batch(*_batch(d_ptrs, s_ptrs, nb), len(nb), current_stream()), "xtb_peer_memcpy_batch")
    torch.cuda.synchronize()
    want = torch.full((1 << 20,), 0, dtype=torch.uint8, device="cuda")
    want.view(torch.int32).fill_(R.FILL32)
    for o, n in zip(offs, sizes):
        want[o : o + n] = src[o + 5 : o + 5 + n]
    assert torch.equal(dst.bytes(0), want), "a copy landed wrong or past its byte count"
    assert dst.guards_intact()
    assert torch.equal(src, R.labels(1 << 20, 3))
    # n = 0, n = 4096 accepted, n = 4097 refused
    assert lib.xtb_peer_memcpy_batch(*_batch([], [], []), 0, current_stream()) == 0
    d4 = R.guarded(4096)
    d_ptrs = [d4.ptr(0, i) for i in range(4096)]
    s_ptrs = [src.data_ptr() + 4095 - i for i in range(4096)]
    check(lib.xtb_peer_memcpy_batch(*_batch(d_ptrs, s_ptrs, [1] * 4096), 4096, current_stream()), "4096 entries")
    torch.cuda.synchronize()
    assert torch.equal(d4.bytes(0), src[:4096].flip(0))
    assert lib.xtb_peer_memcpy_batch(*_batch(d_ptrs + d_ptrs[:1], s_ptrs + s_ptrs[:1], [1] * 4097), 4097,
                                     current_stream()) == XTB_ERR_INVALID


@pytest.mark.parametrize("bad", ["null_dst", "null_src", "negative"])
def test_peer_memcpy_batch_refuses_before_copying(bad):
    """A batch with a bad second entry is refused and copies nothing, not even the good first entry."""
    lib = ensure_init()
    src = R.labels(4096, 1)
    d0, d1 = R.guarded(4096), R.guarded(4096)
    dsts = [d0.ptr(0), None if bad == "null_dst" else d1.ptr(0)]
    srcs = [src.data_ptr(), None if bad == "null_src" else src.data_ptr()]
    nb = [4096, -1 if bad == "negative" else 4096]
    assert lib.xtb_peer_memcpy_batch(*_batch(dsts, srcs, nb), 2, current_stream()) == XTB_ERR_INVALID
    torch.cuda.synchronize()
    assert bool((d0.arena == R.FILL32).all()), "the first entry of a refused batch was copied"
    assert bool((d1.arena == R.FILL32).all())


# ---- xtb_peer_barrier: world = 1 and refusals only ----------------------------------------------------------------------


def test_peer_barrier_world1_and_refusals():
    lib = ensure_init()
    pads = torch.zeros(64, dtype=torch.int32, device="cuda")
    table = torch.tensor([pads.data_ptr()], dtype=torch.int64, device="cuda")
    n0 = lib.xtb_launch_count()
    # world = 1: nothing to wait for, nothing launched
    assert lib.xtb_peer_barrier(table.data_ptr(), 0, 1, 0, current_stream()) == 0
    assert lib.xtb_peer_barrier(table.data_ptr(), 0, 1, 5, current_stream()) == 0
    assert lib.xtb_launch_count() == n0
    assert lib.xtb_peer_barrier(None, 0, 1, 0, current_stream()) == XTB_ERR_INVALID  # null table
    assert lib.xtb_peer_barrier(table.data_ptr(), 0, 0, 0, current_stream()) == XTB_ERR_INVALID  # world 0
    assert lib.xtb_peer_barrier(table.data_ptr(), 1, 1, 0, current_stream()) == XTB_ERR_INVALID  # rank >= world
    assert lib.xtb_peer_barrier(table.data_ptr(), -1, 1, 0, current_stream()) == XTB_ERR_INVALID
    assert lib.xtb_peer_barrier(table.data_ptr(), 0, 1, -1, current_stream()) == XTB_ERR_INVALID  # negative channel
    assert lib.xtb_launch_count() == n0
    torch.cuda.synchronize()
    assert bool((pads == 0).all())


# ---- 64-bit addressing -------------------------------------------------------------------------------------------------


def _chunks(n, step):
    return [(i, min(n, i + step)) for i in range(0, n, step)]


def test_a2a_pull_past_2g():
    """[S, 8, 128] int16 inputs with S = 2^20 + 64 (2 GiB + 128 KiB), scatter on the heads, gather on the sequence, W = 2.
    Both table entries point at one input (the addressing is what is under test); rank 1's output passes 2^31 bytes."""
    from xtuner_b200.comm import a2a_plan

    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    W, S = 2, (1 << 20) + 64
    shape = (S, 8, 128)
    inp = torch.arange(S * 8 * 128 // 2, dtype=torch.int32, device="cuda").view(torch.int16).view(shape)
    table = torch.tensor([inp.data_ptr()] * W, dtype=torch.int64, device="cuda")
    plan = a2a_plan(shape, 1, 0, W, 1, 2)
    nbytes = inp.numel() * 2
    assert nbytes > 2**31
    o = R.guarded(nbytes)
    check(ensure_init().xtb_a2a_pull(table.data_ptr(), o.ptr(0), 1, W, *_a2a_args(plan), current_stream()),
          "xtb_a2a_pull")
    torch.cuda.synchronize()
    out = o.buf(0, torch.int16, plan.out_shape)
    assert plan.out_shape == (W * S, 4, 128)
    for src in range(W):
        for a, b in _chunks(S, 1 << 17):
            assert torch.equal(out[src * S + a : src * S + b], inp[a:b, 4:8]), f"rows {a}..{b} of source {src}"
    assert o.guards_intact()
    PEAK["a2a past 2^31"] = torch.cuda.max_memory_allocated()
    assert PEAK["a2a past 2^31"] < 10 * 2**30


def test_ep_pulls_past_2g():
    """W = 2, E = 2, rows of 14336 bytes, every row routed to expert 0 (owner 0).  Both table entries point at one source
    buffer of R rows (1 GiB), so owner 0 receives 2R rows and writes past 2^31 bytes; rank 1's way back reads past it."""
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    lib, W, E, rb = ensure_init(), 2, 2, 14336
    words, hdr = rb // 4, R.ep_hdr_bytes(E)
    Rr = (1 << 30) // rb + 101
    assert 2 * Rr * rb > 2**31
    src = torch.empty(hdr // 4 + Rr * words, dtype=torch.int32, device="cuda")
    src[: hdr // 4] = 0
    src[0] = Rr
    rows = src[hdr // 4 :].view(Rr, words)
    for a, b in _chunks(Rr, 8192):
        r = torch.arange(a, b, dtype=torch.int32, device="cuda")[:, None]
        rows[a:b] = r * 4099 + torch.arange(words, dtype=torch.int32, device="cuda")[None, :]
    table = torch.tensor([src.data_ptr()] * W, dtype=torch.int64, device="cuda")
    own = torch.full((hdr // 4 + 2 * Rr * words + 64,), R.FILL32, dtype=torch.int32, device="cuda")
    own_table = torch.tensor([own.data_ptr()] * W, dtype=torch.int64, device="cuda")
    cnt_out = torch.empty(W * E, dtype=torch.int32, device="cuda")
    status = torch.tensor([-1, 0], dtype=torch.int32, device="cuda")
    check(lib.xtb_ep_pull_to_experts(table.data_ptr(), None, cnt_out.data_ptr(), own.data_ptr() + hdr, None,
                                     status.data_ptr(), 0, W, E, rb, hdr, 2 * Rr, current_stream()),
          "xtb_ep_pull_to_experts")
    torch.cuda.synchronize()
    assert cnt_out.tolist() == [Rr, 0, Rr, 0] and status.tolist() == [2 * Rr, 0]
    got = own[hdr // 4 :]
    for half in range(2):
        for a, b in _chunks(Rr, 8192):
            assert torch.equal(got[(half * Rr + a) * words : (half * Rr + b) * words].view(-1, words), rows[a:b]), \
                f"expert-major rows {half * Rr + a}..{half * Rr + b}"
    assert bool((got[2 * Rr * words :] == R.FILL32).all())
    del got
    back = torch.full((Rr * words + 64,), R.FILL32, dtype=torch.int32, device="cuda")
    cnt_dev = _t(np.array([[Rr, 0], [Rr, 0]], dtype=np.int32))
    check(lib.xtb_ep_pull_to_sources(own_table.data_ptr(), cnt_dev.data_ptr(), back.data_ptr(), 1, W, E, rb, hdr,
                                     2 * Rr, Rr, current_stream()), "xtb_ep_pull_to_sources")
    torch.cuda.synchronize()
    for a, b in _chunks(Rr, 8192):
        assert torch.equal(back[a * words : b * words].view(-1, words), rows[a:b]), f"returned rows {a}..{b}"
    assert bool((back[Rr * words :] == R.FILL32).all())
    PEAK["EP past 2^31"] = torch.cuda.max_memory_allocated()
    assert PEAK["EP past 2^31"] < 10 * 2**30
