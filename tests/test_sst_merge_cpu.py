"""`-m "not gpu"`: the merging read of b2_sst_merge without a GPU.  Generated LSM shapes of 1-12 runs: the CPU oracle
(tests/sst_merge_oracle.cpp over the oracle's block iterator) against the pure-Python model and the known answer; the
verdicts for other value types, unsorted runs and stored seqs under a global seqno; the device's per-entry rules
(tikv_b200/csrc/sst_merge.h) built for the CPU under AddressSanitizer against the model; the new stats struct against its
ctypes mirror."""
import ctypes as C
import os
import random
import subprocess

import pytest

import sstmerge as m
from tikv_b200 import ffi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def target_kvs(seed, n):
    """distinct user keys of 0-40 bytes over a small alphabet (shared prefixes, keys that prefix others), none ending in
    0x00 / 0x01 (the generator's noise keys extend target keys with those bytes)"""
    rng = random.Random(seed)
    keys = set()
    while len(keys) < n:
        k = bytes(rng.choice(b"ab\x02\xff") for _ in range(rng.randrange(0, 40)))
        if not k or k[-1] > 1:
            keys.add(k)
    return [(k, bytes(rng.randrange(256) for _ in range(rng.randrange(0, 30)))) for k in sorted(keys)]


def with_trailers(runs, seed):
    rng = random.Random(seed)
    out = []
    for r in runs:
        tl = rng.choice([0, 5])
        data, offs = m.build_run(r, trailer_len=tl, block_size=rng.choice([64, 512, 4096]), restart_interval=rng.choice([1, 3, 16]))
        out.append((data, offs, tl))
    return out


SHAPES = [(seed, 1 + seed % 12) for seed in range(36)]


@pytest.mark.parametrize("seed,n_runs", SHAPES)
def test_oracle_equals_model_and_known_answer(seed, n_runs):
    kvs = target_kvs(seed, 150)
    runs, gs, snap = m.derive_runs(kvs, seed, n_runs)
    got, counts = m.model(runs, snap, gs)
    assert got == kvs
    assert counts["n_in"] == counts["n_out"] + counts["n_invisible"] + counts["n_hidden"] + counts["n_deletions"]
    rc, okvs, ocounts = m.oracle_merge(with_trailers(runs, seed), snap, gs)
    assert rc == 0 and okvs == kvs and ocounts == counts
    if n_runs >= 4:
        assert m.features(runs, gs, snap) == m.ALL_FEATURES, m.ALL_FEATURES - m.features(runs, gs, snap)


def test_every_shape_is_generated():
    f = set()
    for seed, n in SHAPES:
        runs, gs, snap = m.derive_runs(target_kvs(seed, 150), seed, n)
        f |= m.features(runs, gs, snap)
    assert f == m.ALL_FEATURES


def test_snapshot_edges():
    """an entry at exactly the snapshot is visible, one above is not; snapshot 0 sees only seq-0 entries"""
    runs = [[(b"a", 10, m.VALUE, b"new"), (b"b", 11, m.DELETION, b"")], [(b"a", 0, m.VALUE, b"old"), (b"b", 0, m.VALUE, b"b0")]]
    for snap, exp in ((10, [(b"a", b"new"), (b"b", b"b0")]), (11, [(b"a", b"new")]), (9, [(b"a", b"old"), (b"b", b"b0")]), (0, [(b"a", b"old"), (b"b", b"b0")])):
        assert m.model(runs, snap)[0] == exp
        assert m.oracle_merge([m.build_run(r) for r in runs], snap)[:2] == (0, exp)
    assert m.oracle_merge([], 5)[:2] == (0, [])
    assert m.oracle_merge([m.build_run([])], 5)[:2] == (0, [])


def test_verdicts():
    ok = [(b"a", 5, m.VALUE, b"x"), (b"b", 5, m.VALUE, b"y")]
    for t in (m.MERGE, m.BLOB_INDEX, 0x0F, 0xFF):
        assert m.oracle_merge([m.build_run(ok), m.build_run([(b"a", 3, t, b"m")])], 10)[0] == 2
    # unsorted: user keys descending, a footer ascending within one user key, a duplicate internal key
    for bad in ([(b"b", 5, 1, b""), (b"a", 5, 1, b"")], [(b"a", 3, 1, b""), (b"a", 5, 1, b"")], [(b"a", 5, 1, b""), (b"a", 5, 1, b"")]):
        assert m.oracle_merge([m.build_run(ok), m.build_run(bad, sort=False)], 10)[0] == 1
    # a stored seq other than 0 under a global seqno
    assert m.oracle_merge([m.build_run([(b"a", 0, 1, b"")]), m.build_run(ok)], 10, [7, 0])[0] == 0
    assert m.oracle_merge([m.build_run(ok), m.build_run([(b"a", 0, 1, b"")])], 10, [7, 0])[0] == 1
    # a key shorter than its footer
    short = m.FlatBlock([(b"a" * 7, b"v")])
    import sstfmt
    assert m.oracle_merge([sstfmt.build(short, key_suffix_len=0)], 10)[0] == 1
    # an unsupported type wins over a corrupted run, as on the device (the larger code)
    assert m.oracle_merge([m.build_run([(b"b", 5, 1, b""), (b"a", 5, m.MERGE, b"")], sort=False)], 10)[0] == 2


def staged(runs):
    return [[k for k, _ in m.run_kvs(r)] for r in runs]


@pytest.mark.parametrize("seed,n_runs", SHAPES[:18])
def test_device_rules_on_the_cpu_match_the_model(seed, n_runs):
    kvs = target_kvs(seed, 120)
    runs, gs, snap = m.derive_runs(kvs, seed, n_runs)
    for s in (snap, snap // 2, 0, m.MAX_SEQ):
        st, pairs = m.emul(staged(runs), s, gs)
        assert st == 0
        flat = [(u, v, t) for run in runs for u, _, t, v in run]
        out = [(flat[i][0], flat[i][1]) for i, v in pairs if v == 1]
        exp, counts = m.model(runs, s, gs)
        assert out == exp
        assert [sum(v == k for _, v in pairs) for k in (0, 1, 2, 3)] == [counts["n_invisible"], counts["n_out"], counts["n_deletions"], counts["n_hidden"]]


def test_device_rules_verdicts_on_the_cpu():
    ok = [m.ikey(b"a", 5, 1), m.ikey(b"b", 5, 1)]
    assert m.emul([ok, [m.ikey(b"a", 3, m.MERGE)]], 10)[0] == 2
    assert m.emul([ok, [m.ikey(b"b", 5, 1), m.ikey(b"a", 5, 1)]], 10)[0] == 1
    assert m.emul([ok, [m.ikey(b"a", 3, 1), m.ikey(b"a", 5, 1)]], 10)[0] == 1
    assert m.emul([ok, [m.ikey(b"a", 5, 1), m.ikey(b"a", 5, 1)]], 10)[0] == 1
    assert m.emul([ok, [m.ikey(b"a", 1, 1)]], 10, [0, 7])[0] == 1
    assert m.emul([ok, [m.ikey(b"a", 0, 1)]], 10, [0, 7])[0] == 0
    assert m.emul([ok, [b"a" * 7]], 10)[0] == 1
    assert m.emul([[b""]], 10)[0] == 1
    # ties: the run listed first wins an equal (user key, footer) pair
    st, pairs = m.emul([[m.ikey(b"a", 5, 1)], [m.ikey(b"a", 5, 1)]], 10)
    assert st == 0 and pairs == [(0, 1), (1, 3)]


def test_merge_stats_struct_matches_its_ctypes_mirror(tmp_path):
    """b2_sst_merge_stats of include/b2_copr.h against ffi.SstMergeStats: size and every field's offset, from a C program
    compiled against the header"""
    import re
    header = open(os.path.join(ROOT, "include", "b2_copr.h")).read()
    mm = re.search(r"typedef struct b2_sst_merge_stats \{(.*?)\} b2_sst_merge_stats;", header, re.S)
    body = re.sub(r"/\*.*?\*/", "", mm.group(1), flags=re.S)
    names = [part.strip().split()[-1] for d in body.split(";") if d.strip() for part in d.split(",")]
    assert names == [f[0] for f in ffi.SstMergeStats._fields_]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(['#include <stdio.h>', '#include <stddef.h>', '#include "b2_copr.h"', 'int main(void) {',
                              '  printf("%zu", sizeof(b2_sst_merge_stats));'] + [f'  printf(" %zu", offsetof(b2_sst_merge_stats, {n}));' for n in names]
                             + ['  return 0;', '}']))
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-std=c11", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)], text=True).split()]
    assert got == [C.sizeof(ffi.SstMergeStats)] + [getattr(ffi.SstMergeStats, n).offset for n in names]
