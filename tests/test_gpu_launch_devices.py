"""Kernels that take more shared memory than a launch gets by default, launched on two GPUs from one process.

By default a kernel may take 48 KB of shared memory, static and dynamic together.  CUDA keeps a kernel's raised limit
per device, so every kernel that needs more has to be opted in again on each device it runs on.  Each test below calls
one family of entries first on cuda:0 and then on cuda:1, with the same seeded inputs and at shapes where every launch
needs more than 48 KB, and asserts status 0, untouched guard rows and bit-equal outputs on the two devices.  The
expert-parallel pull kernels need peers and are left to the exchange tests."""
import pytest
import torch

from tests.gpu_harness import Guarded
from xtuner_b200._capi import check, current_stream, ensure_init, ptr

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def two_devices():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    p0, p1 = (torch.cuda.get_device_properties(d) for d in (0, 1))
    if (p0.name, p0.multi_processor_count) != (p1.name, p1.multi_processor_count):
        pytest.skip("the two GPUs differ; grid sizes, and so reduction orders, follow the SM count")


def _rand(shape, seed, dev, dtype=torch.bfloat16):
    return torch.randn(shape, generator=torch.Generator().manual_seed(seed)).to(dtype).to(dev)


def _bits(t):
    return t.view({torch.bfloat16: torch.int16, torch.float32: torch.int32}.get(t.dtype, t.dtype))


def _same_on_both_devices(run):
    """run(dev) -> {name: output tensor}, called with `dev` current; asserts the two devices' outputs are bit-equal."""
    outs = []
    for dev in ("cuda:0", "cuda:1"):
        with torch.cuda.device(dev):
            got = run(dev)
            torch.cuda.synchronize()
        outs.append({k: v.cpu() for k, v in got.items()})
    for k in outs[0]:
        assert torch.equal(_bits(outs[0][k]), _bits(outs[1][k])), f"{k}: cuda:1 differs from cuda:0"


@pytest.mark.parametrize("wide", [False, True], ids=["128-column-tiles", "256-column-tiles"])
def test_group_gemms(wide):
    """xtb_group_gemm_nt, _nt_swiglu, _nn, _tn and _tn_pair; N, Kd % 256 (I % 128 for the SwiGLU) picks the tile"""
    n, inter = (512, 256) if wide else (384, 192)
    counts = [100, 0, 37, 163]
    E, M = len(counts), sum(counts)

    def run(dev):
        lib = ensure_init()
        tpe = torch.tensor(counts, dtype=torch.int64, device=dev)
        x, dy, dy2 = _rand((M, n), 1, dev), _rand((M, n), 2, dev), _rand((M, 256), 3, dev)
        w, w13 = _rand((E, n, n), 4, dev), _rand((E, 2 * inter, n), 5, dev)
        nt, nn = Guarded(M, n, torch.bfloat16, dev), Guarded(M, n, torch.bfloat16, dev)
        h, a = Guarded(M, 2 * inter, torch.bfloat16, dev), Guarded(M, inter, torch.bfloat16, dev)
        tn, pa, pb = (Guarded(E * r, n, torch.bfloat16, dev) for r in (n, n, 256))
        st = current_stream()
        check(lib.xtb_group_gemm_nt(ptr(x), ptr(w), ptr(tpe), M, n, n, E, ptr(nt.v), st), "xtb_group_gemm_nt")
        check(lib.xtb_group_gemm_nt_swiglu(ptr(x), ptr(w13), ptr(tpe), M, inter, n, E, ptr(h.v), ptr(a.v), st),
              "xtb_group_gemm_nt_swiglu")
        check(lib.xtb_group_gemm_nn(ptr(dy), ptr(w), ptr(tpe), M, n, n, E, ptr(nn.v), st), "xtb_group_gemm_nn")
        check(lib.xtb_group_gemm_tn(ptr(dy), ptr(x), ptr(tpe), M, n, n, E, ptr(tn.v), st), "xtb_group_gemm_tn")
        check(lib.xtb_group_gemm_tn_pair(ptr(dy), ptr(x), n, n, ptr(pa.v), ptr(dy2), ptr(x), 256, n, ptr(pb.v),
                                         ptr(tpe), M, E, st), "xtb_group_gemm_tn_pair")
        return {name: g.check(name) for name, g in
                dict(nt=nt, nt_swiglu_h=h, nt_swiglu_a=a, nn=nn, tn=tn, tn_pair_a=pa, tn_pair_b=pb).items()}

    _same_on_both_devices(run)


@pytest.mark.parametrize("H", [1024, 2048])
def test_gate_route_dispatch(H):
    """the fused gate-route kernel's planes take 48 H bytes of dynamic shared memory on top of its static 5 KB: H = 1024
    needs exactly 48 KB of dynamic memory, H = 2048 96 KB"""
    T, E, K = 300, 8, 2

    def run(dev):
        lib = ensure_init()
        x, w = _rand((T, H), 6, dev), _rand((E, H), 7, dev, torch.float32)
        lg, rw = Guarded(T, E, torch.float32, dev), Guarded(T, E, torch.float32, dev)
        tw = Guarded(T, K, torch.float32, dev)
        ids, i32 = Guarded(T, K, torch.int64, dev), Guarded(T, K, torch.int32, dev)
        tpe = torch.full((E,), -1, dtype=torch.int64, device=dev)
        ws = torch.zeros(int(lib.xtb_moe_permute_workspace_bytes(T, K, E)), dtype=torch.uint8, device=dev)
        check(lib.xtb_gate_route_dispatch(ptr(x), ptr(w), T, H, E, K, 0, 1, 1.0, ptr(lg.v), ptr(rw.v), ptr(tw.v),
                                          ptr(ids.v), ptr(i32.v), ptr(tpe), ptr(ws), current_stream()),
              "xtb_gate_route_dispatch")
        return dict(logits=lg.check("logits"), rw=rw.check("rw"), tw=tw.check("tw"), ids=ids.check("ids"),
                    i32=i32.check("i32"), tpe=tpe, ws=ws)

    _same_on_both_devices(run)


def test_moe_permute_bulk():
    """the bulk-copy row gather stages 8 rows: 8 KB rows (H = 4096 bf16) need 65 KB"""
    T, K, E, H = 300, 2, 8, 4096

    def run(dev):
        lib = ensure_init()
        x = _rand((T, H), 8, dev)
        ids = torch.randint(0, E, (T, K), generator=torch.Generator().manual_seed(9), dtype=torch.int32).to(dev)
        perm, rmap = Guarded(T * K, H, torch.bfloat16, dev), Guarded(T * K, 1, torch.int32, dev)
        idx = Guarded(T * K, 1, torch.int64, dev)
        tpe = torch.full((E,), -1, dtype=torch.int64, device=dev)
        ws = torch.zeros(int(lib.xtb_moe_permute_workspace_bytes(T, K, E)), dtype=torch.uint8, device=dev)
        check(lib.xtb_moe_permute(ptr(x), ptr(ids), T, K, E, H * 2, ptr(perm.v), ptr(rmap.v), ptr(idx.v), ptr(tpe),
                                  ptr(ws), current_stream()), "xtb_moe_permute")
        return dict(permuted=perm.check("permuted"), row_id_map=rmap.check("row_id_map"),
                    sorted_indices=idx.check("sorted_indices"), tpe=tpe)

    _same_on_both_devices(run)


@pytest.mark.parametrize("K", [2, 8])
def test_dispatch_bwd_rmsnorm(K):
    """the pipelined kernel stages two token groups: 80 KB at K = 2, 88 KB at K = 8"""
    T, H = 300, 2048

    def run(dev):
        lib = ensure_init()
        g_xp = _rand((T * K, H), 10, dev)
        gate, h, g_res = _rand((T, H), 11, dev), _rand((T, H), 12, dev), _rand((T, H), 13, dev)
        rmap = torch.randperm(T * K, generator=torch.Generator().manual_seed(14)).to(torch.int32).to(dev)
        rstd = _rand((T,), 15, dev, torch.float32).abs() + 0.5
        w = _rand((H,), 16, dev, torch.float32)
        g_h, g_nw = Guarded(T, H, torch.bfloat16, dev), Guarded(1, H, torch.float32, dev)
        ws = torch.empty(int(lib.xtb_moe_dispatch_bwd_rmsnorm_workspace_bytes(T, H)), dtype=torch.uint8, device=dev)
        check(lib.xtb_moe_dispatch_bwd_rmsnorm(ptr(g_xp), ptr(rmap), ptr(gate), ptr(h), ptr(rstd), ptr(w), ptr(g_res),
                                               T, K, H, ptr(g_h.v), ptr(g_nw.v), ptr(ws), current_stream()),
              "xtb_moe_dispatch_bwd_rmsnorm")
        return dict(g_h=g_h.check("g_h"), g_norm_w=g_nw.check("g_norm_w"))

    _same_on_both_devices(run)


@pytest.mark.parametrize("E", [8, 16])
def test_gate_logits(E):
    """the small-E gate keeps the fp32 weight in shared memory: E H 4 bytes, 64 KB at E = 8, 128 KB at E = 16"""
    T, H = 300, 2048

    def run(dev):
        x, w, b = _rand((T, H), 17, dev), _rand((E, H), 18, dev, torch.float32), _rand((E,), 19, dev, torch.float32)
        lg = Guarded(T, E, torch.float32, dev)
        check(ensure_init().xtb_gate_logits(ptr(x), ptr(w), ptr(b), ptr(lg.v), T, H, E, current_stream()),
              "xtb_gate_logits")
        return dict(logits=lg.check("logits"))

    _same_on_both_devices(run)


def test_rmsnorm_gate():
    """the fused norm and gate keep both weights in shared memory: (E + 1) H 4 bytes, 72 KB at E = 8, H = 2048"""
    T, H, E = 300, 2048, 8

    def run(dev):
        h, w, gw = _rand((T, H), 20, dev), _rand((H,), 21, dev, torch.float32), _rand((E, H), 22, dev, torch.float32)
        x, rstd = Guarded(T, H, torch.bfloat16, dev), Guarded(T, 1, torch.float32, dev)
        lg = Guarded(T, E, torch.float32, dev)
        check(ensure_init().xtb_rmsnorm_gate(ptr(h), ptr(w), ptr(gw), 1e-6, T, H, E, ptr(x.v), ptr(rstd.v), ptr(lg.v),
                                             current_stream()), "xtb_rmsnorm_gate")
        return dict(x=x.check("x"), rstd=rstd.check("rstd"), logits=lg.check("logits"))

    _same_on_both_devices(run)
