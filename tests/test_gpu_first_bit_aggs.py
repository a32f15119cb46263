"""`-m gpu`: FIRST and BIT_AND / BIT_OR / BIT_XOR on the device, checked against the reference semantics applied to the
oracle's scan rows (tests/first_bit_ref.py), with every other aggregate of a plan checked against the oracle itself.
Covers generic and plan-specialised kernels, host- and device-resident sources, forward and backward scans, 1 and 3
blocks, the hand-over between the lean kernel and the list-mode general kernel, two shards merged through
b2_exec_agg_word_ops, and the growth-and-redo of the HBM group table."""
import ctypes as C
import os

import pytest
import torch

import kvfmt
import scenarios as sc
from first_bit_ref import I64, LONG, REAL, U64, UNS, Spec, bits, scenario_specs, select_cases, select_region
from test_gpu_parity import _gen_block, _source
from tikv_b200 import dist as bd
from tikv_b200 import ffi
from tikv_b200.executor import BatchExecutor, DagHandler, DeviceRegion
from tikv_b200.plan import ColumnDef, Plan, col, const_int, lt

pytestmark = pytest.mark.gpu

JITS = [ffi.JIT_OFF, ffi.JIT_SYNC]
JIT_IDS = ["aot", "jit"]


def _run(spec, ranges, region, jit, ctx):
    got = DagHandler(spec.plan(), ranges, region, jit=jit).handle_request()
    return spec.check(got, ranges, region._host if isinstance(region, DeviceRegion) else region, ctx)


@pytest.fixture(scope="module")
def dirty_regions():
    return {n: sc.dirty_region(21, n_keys=1500).build(read_ts=sc.READ_TS, n_write_blocks=n) for n in (1, 3)}


@pytest.mark.parametrize("jit", JITS, ids=JIT_IDS)
@pytest.mark.parametrize("desc", [False, True], ids=["fwd", "bwd"])
@pytest.mark.parametrize("blocks", [1, 3])
def test_scenarios_match_reference(blocks, desc, jit, dirty_regions):
    host = dirty_regions[blocks]
    dev = DeviceRegion(host)
    for name, spec in scenario_specs(desc):
        for ranges, rname in ((sc.WHOLE, "whole"), (sc.split_ranges(), "split")):
            for region, where in ((host, "host"), (dev, "device")):
                _run(spec, ranges, region, jit, f"{name}/{rname}/{where}/b{blocks}/{'bwd' if desc else 'fwd'}/{jit}")


# ---- hand-made regions: edge values and the lean / list-mode hand-over ------------------------------------------------

COLS = [ColumnDef(100, pk_handle=True), ColumnDef(1), ColumnDef(2), ColumnDef(3, unsigned=True), ColumnDef(4, tp=ffi.TP_DOUBLE)]
H, A, B, U, R = range(5)


def _region(rows, locked=lambda h: False, n_write_blocks=1):
    """rows: dicts {column offset: value}; `locked(h)` puts a Lock and a Rollback record above row h, which makes the
    lean kernel hand that row over to the general kernel (list mode)."""
    kinds = {A: "int", B: "int", U: "uint", R: "f64"}
    r = kvfmt.Region()
    for h, row in enumerate(rows):
        key = kvfmt.row_key(sc.TABLE, h)
        r.put(key, kvfmt.row_v2([(c, row.get(c), k) for c, k in kinds.items() if c in row]), 10, 20)
        if locked(h):
            r.lock_rec(key, 30, 31, last_change=(20, 1))
            r.rollback(key, 50)
    return r.build(read_ts=sc.READ_TS, n_write_blocks=n_write_blocks)


def _edge_rows(n):
    edge_i = [None, -1, -(1 << 63), (1 << 63) - 1, 0, 1]
    edge_u = [None, U64, 1 << 63, 0, 1]
    edge_r = [None, -0.0, 0.0, float("nan"), -1.5, 5e-324, float("inf")]
    return [{A: i % 9, B: edge_i[(i // 9) % len(edge_i)], U: edge_u[(i // 7) % len(edge_u)], R: edge_r[(i // 5) % len(edge_r)]} for i in range(n)]


def _edge_specs(desc):
    S = lambda aggs, by=(): Spec(sc.TABLE, COLS, aggs, by, (), desc)
    return [("edge_nokey", S([("first", B, I64), ("first", U, UNS), ("first", R, REAL), ("bit_and", B, I64), ("bit_or", U, UNS), ("bit_xor", B, I64)])),
            ("edge_key", S([("first", B, I64), ("first", R, REAL), ("bit_and", U, UNS), ("bit_xor", B, I64), ("sum", B, I64)], [(A, I64)])),
            ("edge_real_key", S([("first", B, I64), ("bit_or", B, I64)], [(R, REAL)])),
            ("edge_two_keys", S([("first", R, REAL), ("bit_and", B, I64)], [(A, I64), (R, REAL)]))]


@pytest.mark.parametrize("jit", JITS, ids=JIT_IDS)
@pytest.mark.parametrize("desc", [False, True], ids=["fwd", "bwd"])
def test_edge_values(desc, jit):
    """NULL first rows, -0.0 and NaN kept as their bits, INT64_MIN, -1 and 2^64-1 through every state."""
    host = _region(_edge_rows(2000), n_write_blocks=3)
    for name, spec in _edge_specs(desc):
        for region, where in ((host, "host"), (DeviceRegion(host), "device")):
            _run(spec, sc.WHOLE, region, jit, f"{name}/{where}/{desc}/{jit}")


@pytest.mark.parametrize("first_locked", [True, False], ids=["first_row_list_mode", "first_row_lean"])
@pytest.mark.parametrize("desc", [False, True], ids=["fwd", "bwd"])
def test_lean_and_list_mode_hand_over(first_locked, desc):
    """Rows of one group committed by both kernels of a unit: the first row (in scan order) of each group by the list-mode
    general kernel and the later ones by the lean kernel, or the reverse.  Both compute the same FIRST key rule."""
    n, groups = 3000, 37
    rows = [{A: h % groups, B: h * 3 - 5000, U: (h * 0x9E3779B97F4A7C15) & U64, R: float(h) - 0.5} for h in range(n)]
    first_h = set(range(n - groups, n)) if desc else set(range(groups))
    host = _region(rows, locked=lambda h: (h in first_h) == first_locked)
    for name, spec in (("key", Spec(sc.TABLE, COLS, [("first", B, I64), ("first", R, REAL), ("bit_xor", U, UNS), ("count", B, I64)], [(A, I64)], (), desc)),
                       ("nokey", Spec(sc.TABLE, COLS, [("first", B, I64), ("bit_or", B, I64), ("first", U, UNS)], (), (), desc))):
        for region in (host, DeviceRegion(host)):
            with BatchExecutor(spec.plan(), sc.WHOLE, region, jit=ffi.JIT_SYNC) as ex:
                r = ex.next_batch(1 << 30)
                assert r.error is None and r.is_drained
                st = ex.collect_exec_stats()
            assert st.jit_launches >= 2 * st.num_iterations, (st.jit_launches, st.num_iterations)  # a lean and a general launch per unit

            class Res:
                status = 0
                rows = r.rows
            exp = spec.check(Res, sc.WHOLE, host, f"{name}/{first_locked}/{desc}")
            if name == "key":
                for k, v in exp.items():  # the first row of group g is h = g (forward) or the last h with h % groups == g
                    g = k[0][1]
                    h = g if not desc else max(x for x in range(n) if x % groups == g)
                    assert v[0] == bits(h * 3 - 5000)


def test_first_row_in_a_later_unit():
    """Backward scan over three blocks: each group's first row (in scan order) lies in the last unit, which is committed
    after the units holding the group's other rows; forward scans give the mirror case for the earliest block."""
    rows = [{A: h % 11, B: h, R: -float(h)} for h in range(3000)]
    host = _region(rows, n_write_blocks=3)
    for desc in (False, True):
        spec = Spec(sc.TABLE, COLS, [("first", B, I64), ("first", R, REAL), ("bit_and", B, I64)], [(A, I64)], (), desc)
        for jit in JITS:
            for region in (host, DeviceRegion(host)):
                exp = _run(spec, sc.WHOLE, region, jit, f"{desc}/{jit}")
        for k, v in exp.items():
            g = k[0][1]
            assert v[0] == bits(max(h for h in range(3000) if h % 11 == g) if desc else g)


def _shard_rows(lo, hi):
    return [(h, {A: h % 13, B: None if h % 17 == 0 else h * 7 - 9000, U: (h * 0x9E3779B97F4A7C15) & U64, R: None if h % 19 == 0 else h / 4 - 300.0})
            for h in range(lo, hi)]


def _handle_region(rows, n_write_blocks=1):
    kinds = {A: "int", B: "int", U: "uint", R: "f64"}
    r = kvfmt.Region()
    for h, row in rows:
        r.put(kvfmt.row_key(sc.TABLE, h), kvfmt.row_v2([(c, row.get(c), k) for c, k in kinds.items()]), 10, 20)
    return r.build(read_ts=sc.READ_TS, n_write_blocks=n_write_blocks)


N_SHARD = 1500
SHARD_AGGS = [("count", B, I64), ("first", B, I64), ("bit_and", B, I64), ("bit_or", U, UNS), ("bit_xor", B, I64), ("first", R, REAL)]


def _shard_worker(rank, world, port, desc, q):
    import os
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        # each rank's region holds only its own rows, so entry numbers restart at 0 on every rank: FIRST keys of
        # different ranks do not compare, and only the part-order rule of the merge gives the right answer
        dev = DeviceRegion(_handle_region(_shard_rows(rank * N_SHARD, (rank + 1) * N_SHARD)))
        spec = Spec(sc.TABLE, COLS, SHARD_AGGS, [(A, I64)], (), desc)
        with BatchExecutor(spec.plan(), sc.WHOLE, dev) as ex:
            r = ex.next_batch(1 << 30)
            assert r.error is None and r.is_drained
            keys, nul, acc = (t.cpu() for t in bd.agg_partials_as_tensors(ex, 0))
            ops = bd.agg_word_ops(ex)
        k, n, a = bd.merge_agg_partials(keys, nul, acc, word_ops=ops, desc=desc)
        got = {}
        for i in range(k.shape[0]):
            w = [int(x) & U64 for x in a[i]]
            f1 = None if w[2] == 0 or w[2] & 1 else ("i", w[3])
            f2 = None if w[8] == 0 or w[8] & 1 else ("f", w[9])
            got[(bits(int(k[i])),)] = [("i", w[0]), f1, ("i", ~w[4] & U64), ("i", w[5]), ("i", w[6]), f2]
        whole = _handle_region(_shard_rows(0, world * N_SHARD))
        exp = spec.expected(sc.WHOLE, whole)
        layout = ops == [ffi.MERGE_ADD, ffi.MERGE_ADD, ffi.MERGE_FIRST_KEY, ffi.MERGE_FIRST_VALUE, ffi.MERGE_OR, ffi.MERGE_OR, ffi.MERGE_XOR,
                         ffi.MERGE_ADD, ffi.MERGE_FIRST_KEY, ffi.MERGE_FIRST_VALUE]
        q.put((rank, bool(layout and got == exp and len(exp) == 13)))
    except Exception as e:  # reported to the parent, which fails the test
        q.put((rank, repr(e)[:500]))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("desc", [False, True], ids=["fwd", "bwd"])
def test_two_ranks_merge_through_word_ops(desc):
    """Two ranks, each with its own region and its own request on the GPU; their device-resident partial tables, merged
    with b2_exec_agg_word_ops over gloo, equal the whole-table result (FIRST from the first rank in scan order)."""
    import socket
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_shard_worker, args=(r, 2, port, desc, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=300) for _ in range(2))
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    assert res == [(0, True), (1, True)], res


@pytest.mark.parametrize("desc", [False, True], ids=["fwd", "bwd"])
def test_reference_select_cases(desc):
    """test_select.rs test_aggr_first / test_aggr_bit_ops (name restated as an INT column): the reference's expected rows."""
    for name, rows, spec, want in select_cases(desc):
        host = select_region(rows)
        for jit in JITS:
            for region in (host, DeviceRegion(host)):
                got = DagHandler(spec.plan(), sc.WHOLE, region, jit=jit).handle_request()
                assert got.status == 0 and spec.got(got) == want, (name, jit)


def test_growth_and_redo_with_first():
    """9 M rows in 4.5 M groups of two rows (key = handle DIV 2): the first HBM table overflows, grows and the request
    runs again.  Forward, FIRST(handle) of group g is 2g; backward it is 2g + 1; BIT_XOR(handle) is 1 for every group."""
    from tikv_b200.plan import int_divide
    n_rows, n_cols = 9_000_000, 4
    g, blk = _gen_block(n_rows, n_cols, 2, 11, [0, 0, 0, 0], [0, 37, 0, 0], None, first_handle=0)
    try:
        dev = _source([blk.block], ffi.LOC_DEVICE)
        columns = [ColumnDef(100, pk_handle=True)] + [ColumnDef(i + 1) for i in range(n_cols)]
        for desc in (False, True):
            plan = Plan().table_scan(sc.TABLE, columns, desc=desc).aggregation(
                [("first", col(0)), ("count", const_int(1)), ("bit_xor", col(0))], group_by=[int_divide(col(0), const_int(2))]).build()
            r = DagHandler(plan, sc.WHOLE, dev).handle_request()
            assert r.status == 0, r.message
            assert r.n_rows == n_rows // 2
            f, cnt, x, key = r.columns
            assert all(c == 2 for c in cnt) and all(v == 1 for v in x)
            assert all(fv == 2 * kv + (1 if desc else 0) for fv, kv in zip(f, key))
            assert sum(key) == (n_rows // 2) * (n_rows // 2 - 1) // 2
    finally:
        ffi.lib().b2_gen_destroy(g)


@pytest.fixture(scope="module", autouse=True)
def _warm_plans():
    """Compile the plan-specialised kernels of this file's plans on all host cores before its first test (NVRTC only; a
    shape already in the on-disk cache costs nothing)."""
    import threading
    plans = [spec.plan() for desc in (False, True) for _, spec in scenario_specs(desc) + _edge_specs(desc)]
    plans += [spec.plan() for desc in (False, True) for _, _, spec, _ in select_cases(desc)]
    plans += [Spec(sc.TABLE, COLS, [("first", B, I64), ("first", R, REAL), ("bit_xor", U, UNS), ("count", B, I64)], [(A, I64)], (), d).plan() for d in (False, True)]
    plans += [Spec(sc.TABLE, COLS, [("first", B, I64), ("bit_or", B, I64), ("first", U, UNS)], (), (), d).plan() for d in (False, True)]
    plans += [Spec(sc.TABLE, COLS, [("first", B, I64), ("first", R, REAL), ("bit_and", B, I64)], [(A, I64)], (), d).plan() for d in (False, True)]
    sem = threading.Semaphore(os.cpu_count() or 4)

    def one(p):
        with sem:
            ffi.lib().b2_plan_precompile(C.byref(p.c), C.byref(C.c_int32(0)))
    ths = [threading.Thread(target=one, args=(p,)) for p in plans]
    [t.start() for t in ths]
    [t.join() for t in ths]
    yield
