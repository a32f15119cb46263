"""`-m "not gpu"`: FIRST and BIT_AND / BIT_OR / BIT_XOR without a GPU: the reference semantics the GPU tests check against
(known answers from the reference's own tests), the plans the device path accepts and refuses, the new entry point, the
tipb numbers, and the multi-rank merge of the new states over two gloo ranks."""
import ctypes as C
import os
import socket
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from first_bit_ref import U64, fold

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    from tikv_b200 import ffi
    return ffi.lib()


def test_aggregate_numbers_follow_tipb():
    """b2_aggr_desc.kind carries tipb::ExprType unchanged.  tipb is not vendored, so the aggregate numbers of
    expression.proto are restated here by name."""
    from tikv_b200 import ffi
    tipb = {"Count": 3001, "Sum": 3002, "Avg": 3003, "Min": 3004, "Max": 3005, "First": 3006, "GroupConcat": 3007,
            "Agg_BitAnd": 3008, "Agg_BitOr": 3009, "Agg_BitXor": 3010}
    ours = {"Count": ffi.AGG_COUNT, "Sum": ffi.AGG_SUM, "Avg": ffi.AGG_AVG, "Min": ffi.AGG_MIN, "Max": ffi.AGG_MAX, "First": ffi.AGG_FIRST,
            "Agg_BitAnd": ffi.AGG_BIT_AND, "Agg_BitOr": ffi.AGG_BIT_OR, "Agg_BitXor": ffi.AGG_BIT_XOR}
    for k, v in ours.items():
        assert tipb[k] == v, k
    hdr = ffi._header_enum("B2_AGG_")
    assert {k: v for k, v in hdr.items()} == {"COUNT": 3001, "SUM": 3002, "AVG": 3003, "MIN": 3004, "MAX": 3005, "FIRST": 3006,
                                               "BIT_AND": 3008, "BIT_OR": 3009, "BIT_XOR": 3010}
    assert ffi._header_enum("B2_MERGE_") == {"ADD": 0, "MAX": 1, "OR": 2, "XOR": 3, "FIRST_KEY": 4, "FIRST_VALUE": 5}
    assert (ffi.MERGE_ADD, ffi.MERGE_MAX, ffi.MERGE_OR, ffi.MERGE_XOR, ffi.MERGE_FIRST_KEY, ffi.MERGE_FIRST_VALUE) == (0, 1, 2, 3, 4, 5)


def test_bit_op_known_answers():
    """impl_bit_op.rs test_bit_and / test_bit_or / test_bit_xor (each step of those sequences) and test_integration."""
    # test_bit_and: !0, NULL -> !0, 7, 4, 4 x10 + NULL x7 -> 4, 7 then [1, NULL, 1] -> 1, then 2 -> 0
    seq = []
    assert fold("bit_and", seq) == U64
    seq.append(None); assert fold("bit_and", seq) == U64
    seq.append(7); assert fold("bit_and", seq) == 7
    seq.append(4); assert fold("bit_and", seq) == 4
    seq += [4] * 10 + [None] * 7; assert fold("bit_and", seq) == 4
    assert fold("bit_and", [7, 1, None, 1]) == 1 and fold("bit_and", [7, 1, None, 1, 2]) == 0
    # test_bit_or: 0, NULL -> 0, 1, 5, 8 x10 + NULL x7 -> 13, [2, 2, NULL, 1] -> 15, 2 -> 15, -1 -> !0
    seq = []
    assert fold("bit_or", seq) == 0
    for v, want in ((None, 0), (1, 1), (4, 5)):
        seq.append(v); assert fold("bit_or", seq) == want
    seq += [8] * 10 + [None] * 7; assert fold("bit_or", seq) == 13
    seq += [2, 2, None, 1]; assert fold("bit_or", seq) == 15
    seq.append(2); assert fold("bit_or", seq) == 15
    seq.append(-1); assert fold("bit_or", seq) == U64
    # test_bit_xor: 0, NULL -> 0, 1, 5 -> 4, 8 x9 + NULL x7 -> 12, 9 x10 -> 12, [2, 2, NULL, 1] -> 13, 2 -> 15
    seq = []
    assert fold("bit_xor", seq) == 0
    for v, want in ((None, 0), (1, 1), (5, 4)):
        seq.append(v); assert fold("bit_xor", seq) == want
    seq += [8] * 9 + [None] * 7; assert fold("bit_xor", seq) == 12
    seq += [9] * 10; assert fold("bit_xor", seq) == 12
    seq += [2, 2, None, 1]; assert fold("bit_xor", seq) == 13
    seq.append(2); assert fold("bit_xor", seq) == 15
    # test_integration: rows [6, 3, 4, 5, 1, 2] of [1000, 1, 23, 42, NULL, 99, -1, 1000]
    col = [1000, 1, 23, 42, None, 99, -1, 1000]
    vals = [col[i] for i in (6, 3, 4, 5, 1, 2)]
    assert (fold("bit_and", vals), fold("bit_or", vals), fold("bit_xor", vals)) == (0, 0xFFFF_FFFF_FFFF_FFFF, 18446744073709551520)


def test_first_known_answers():
    """impl_first.rs test_update / test_update_vector: the first row's value is the answer, a NULL one too."""
    assert fold("first", []) is None
    assert fold("first", [None, 1, 2]) is None
    assert fold("first", [1, None, 2]) == 1
    assert fold("first", [-0.0, 0.0]) == 0.0 and str(fold("first", [-0.0, 0.0])) == "-0.0"


def _check(lib, plan):
    return lib.b2_check_supported(C.byref(plan.c)), lib.b2_last_error_message()


def test_check_supported(lib):
    from tikv_b200 import ffi
    from tikv_b200.plan import ColumnDef, Plan, col, const_int
    cols = [ColumnDef(1, pk_handle=True), ColumnDef(2), ColumnDef(3, unsigned=True), ColumnDef(4, tp=ffi.TP_DOUBLE),
            ColumnDef(5, tp=ffi.TP_VARCHAR), ColumnDef(6, tp=ffi.TP_NEWDECIMAL), ColumnDef(7, tp=ffi.TP_DATETIME), ColumnDef(8, tp=ffi.TP_DURATION)]
    scan = lambda: Plan().table_scan(5, cols)
    ok = [[("first", col(1))], [("first", col(3, tp=ffi.TP_DOUBLE))], [("first", col(2, unsigned=True)), ("sum", col(1))],
          [("bit_and", col(1)), ("bit_or", col(2, unsigned=True)), ("bit_xor", col(1))],
          [("count", const_int(1)), ("first", col(1)), ("max", col(1)), ("first", col(3, tp=ffi.TP_DOUBLE))]]
    for aggs in ok:
        for gb in ([], [col(1)], [col(3, tp=ffi.TP_DOUBLE)], [col(1), col(2, unsigned=True), col(0)]):
            rc, msg = _check(lib, scan().aggregation(aggs, group_by=gb).build())
            assert rc == ffi.B2_OK, (aggs, msg)
    first = b"FIRST over a bytes / JSON / decimal / date-time / duration value"
    bits = b"BIT_AND / BIT_OR / BIT_XOR over a bytes / JSON / decimal / date-time / duration value"
    bad = [(("first", col(4, tp=ffi.TP_VARCHAR)), first), (("first", col(5, tp=ffi.TP_NEWDECIMAL)), first),
           (("first", col(6, tp=ffi.TP_DATETIME)), first), (("first", col(7, tp=ffi.TP_DURATION)), first),
           (("first", col(4, tp=ffi.TP_JSON)), first),
           (("bit_and", col(3, tp=ffi.TP_DOUBLE)), b"over a Real value"), (("bit_or", col(3, tp=ffi.TP_DOUBLE)), b"over a Real value"),
           (("bit_xor", col(3, tp=ffi.TP_DOUBLE)), b"over a Real value"), (("bit_xor", col(4, tp=ffi.TP_VARCHAR)), bits),
           (("bit_and", col(5, tp=ffi.TP_NEWDECIMAL)), bits), (("bit_or", col(6, tp=ffi.TP_DATETIME)), bits)]
    for agg, why in bad:
        rc, msg = _check(lib, scan().aggregation([agg]).build())
        assert rc == ffi.B2_ERR_UNSUPPORTED and why in msg, (agg, msg)
    # FIRST's pair sits at an even word: 71 words of Real SUM + FIRST still fit, the state limit still holds
    rc, msg = _check(lib, scan().aggregation([("sum", col(3, tp=ffi.TP_DOUBLE)), ("avg", col(3, tp=ffi.TP_DOUBLE)), ("first", col(1))]).build())
    assert rc == ffi.B2_OK, msg
    rc, msg = _check(lib, scan().aggregation([("sum", col(3, tp=ffi.TP_DOUBLE))] * 2 + [("first", col(1))] * 6).build())
    assert rc == ffi.B2_ERR_UNSUPPORTED and b"aggregate state too large" in msg


def test_word_ops_entry_point(lib):
    from tikv_b200 import ffi
    assert "b2_exec_agg_word_ops" in ffi.EXPORTED_SYMBOLS and hasattr(lib, "b2_exec_agg_word_ops")
    n = C.c_uint32(4)
    ops = (C.c_uint8 * 4)()
    assert lib.b2_exec_agg_word_ops(None, ops, C.byref(n)) == ffi.B2_ERR_INVALID_ARG


# ---- two gloo ranks: the partial FIRST / BIT_* states of each rank's shard merge to the whole-table answer ------------

def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _i64(v):
    v &= U64
    return v - (1 << 64) if v >= (1 << 63) else v


def _first_key(entry, desc, is_null):  # b2_device.h first_agg_key
    r62 = (1 << 62) - 1
    r = r62 - entry if desc else entry
    return (1 << 63) | ((r62 - r) << 1) | (1 if is_null else 0)


# state words: FIRST(c2) [0, 1] | BIT_AND(c2) [2] | BIT_OR(c1) [3] | BIT_XOR(c1) [4] | COUNT [5]
def _states(rows, desc):
    """The device state of each group of `rows` (forward scan order: (group, c2, c1)) as the kernels build it."""
    st = {}
    for i, (g, f, x) in enumerate(rows):
        s = st.setdefault(g, [0] * 6)
        k = _first_key(i, desc, f is None)
        if k > s[0]:
            s[0], s[1] = k, (f or 0) & U64
        s[2] |= (~f & U64) if f is not None else 0
        s[3] |= (x & U64) if x is not None else 0
        s[4] ^= (x & U64) if x is not None else 0
        s[5] += 1
    return st


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import kvfmt
    import orc
    import scenarios as sc
    from tikv_b200 import dist as bd
    from tikv_b200 import ffi
    from tikv_b200.plan import Plan

    region = sc.dirty_region(11, n_keys=500).build(read_ts=sc.READ_TS)
    cuts = [-1000, 600, 5000]
    ops = [ffi.MERGE_FIRST_KEY, ffi.MERGE_FIRST_VALUE, ffi.MERGE_OR, ffi.MERGE_OR, ffi.MERGE_XOR, ffi.MERGE_ADD]

    def rows_of(ranges):
        res = orc.dag_handle(Plan().table_scan(sc.TABLE, sc.COLUMNS).build(), ranges, region)
        return [(r[sc.C6], r[sc.C2], r[sc.C1]) for r in res.rows()]

    ok = []
    for desc in (False, True):
        mine = rows_of([kvfmt.table_range(sc.TABLE, cuts[rank], cuts[rank + 1])])
        st = _states(mine, desc)
        if rank == 0:
            st[1000] = [_first_key(0, desc, False), 5, ~5 & U64, 0, 0, 1]  # a group rank 1 does not have
        else:
            st[2000] = [_first_key(3, desc, True), 0, 0, 0, 0, 2]  # a FIRST whose value is NULL, BIT_AND over NULLs only
        keys = torch.tensor(sorted(st), dtype=torch.int64)
        acc = torch.tensor([[_i64(w) for w in st[g]] for g in sorted(st)], dtype=torch.int64)
        k, n, a = bd.merge_agg_partials(keys, torch.zeros(len(st), dtype=torch.bool), acc, word_ops=ops, desc=desc)
        got = {}
        for i in range(k.shape[0]):
            w = [int(x) & U64 for x in a[i]]
            first = None if w[0] == 0 or w[0] & 1 else w[1]
            got[int(k[i])] = (first, ~w[2] & U64, w[3], w[4], w[5])
        whole = rows_of(sc.WHOLE)
        if desc:
            whole = whole[::-1]
        exp = {}
        for g in sorted({r[0] for r in whole}):
            grp = [r for r in whole if r[0] == g]
            f = fold("first", [r[1] for r in grp])
            exp[g] = (None if f is None else f & U64, fold("bit_and", [r[1] for r in grp]), fold("bit_or", [r[2] for r in grp]),
                      fold("bit_xor", [r[2] for r in grp]), len(grp))
        exp[1000] = (5, 5, 0, 0, 1)
        exp[2000] = (None, U64, 0, 0, 2)
        ok.append(got == exp and len(exp) > 10)
    q.put((rank, ok))
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_merge_of_first_and_bit_states():
    """FIRST forward and backward (the earliest / latest part holding the group wins), a group only one part holds, a
    FIRST whose value is NULL, and BIT_AND's all-NULL identity (-1 as u64)."""
    import subprocess
    subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle")])
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=120) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert res == [(0, [True, True]), (1, [True, True])], res


def test_merge_word_ops_single_process():
    """Inside one part the larger nonzero FIRST key wins; OR / XOR words reduce with their op."""
    sys.path.insert(0, ROOT)
    from tikv_b200 import dist as bd
    from tikv_b200 import ffi
    ops = [ffi.MERGE_FIRST_KEY, ffi.MERGE_FIRST_VALUE, ffi.MERGE_XOR, ffi.MERGE_OR]
    keys = torch.tensor([1, 1, 2], dtype=torch.int64)
    acc = torch.tensor([[_i64(_first_key(9, False, False)), 7, 3, 1 << 62], [0, 0, 5, -(1 << 63)], [_i64(_first_key(2, False, True)), 0, -1, 0]], dtype=torch.int64)
    k, n, a = bd.merge_agg_partials(keys, torch.zeros(3, dtype=torch.bool), acc, word_ops=ops)
    rows = {int(k[i]): [int(x) for x in a[i]] for i in range(k.shape[0])}
    assert rows[1] == [_i64(_first_key(9, False, False)), 7, 6, -(1 << 63) | (1 << 62)]
    assert rows[2] == [_i64(_first_key(2, False, True)), 0, -1, 0]
    # without word_ops the words stay additive, as before
    k, n, a = bd.merge_agg_partials(keys, torch.zeros(3, dtype=torch.bool), acc)
    assert int(a[0, 2]) == 8
