"""Sorted runs of one LSM snapshot for the b2_sst_merge tests: a generator whose answer is known, a pure-Python model of
the merging read, and ctypes access to the CPU oracle (tests/sst_merge_oracle.cpp) and to the host build of the
device's per-entry rules (tests/sst_merge_emul.cpp).  TEST INFRASTRUCTURE."""
import ctypes as C
import os
import random
import struct
import subprocess
import tempfile

import numpy as np

import sstfmt
from sstlz4 import BUILD, ROOT, _built
from tikv_b200 import ffi

DELETION, VALUE, MERGE, SINGLE_DELETION, BLOB_INDEX = 0, 1, 2, 7, 0x11
MAX_SEQ = (1 << 56) - 1
ORACLE_SRC = os.path.join(ROOT, "tests", "sst_merge_oracle.cpp")
EMUL_SRC = os.path.join(ROOT, "tests", "sst_merge_emul.cpp")
RULES_HDR = os.path.join(ROOT, "tikv_b200", "csrc", "sst_merge.h")
ORC_SST = os.path.join(ROOT, "oracle", "orc_sst.h")
_lib = None


def ikey(user, seq, typ):
    return user + struct.pack("<Q", seq << 8 | typ)


class FlatBlock:
    """a host b2_cf_block over (key, value) pairs in the order given (kvfmt.HostBlock sorts its keys bytewise, which is
    not the internal-key order of keys that end in a footer)"""

    def __init__(self, kvs):
        self.kvs = list(kvs)
        ko, vo = np.zeros(len(kvs) + 1, dtype=np.uint32), np.zeros(len(kvs) + 1, dtype=np.uint32)
        ko[1:] = np.cumsum([len(k) for k, _ in kvs]) if kvs else []
        vo[1:] = np.cumsum([len(v) for _, v in kvs]) if kvs else []
        self.keys = np.frombuffer(b"".join(k for k, _ in kvs) + b"\0" * 32, dtype=np.uint8).copy()
        self.vals = np.frombuffer(b"".join(v for _, v in kvs) + b"\0" * 32, dtype=np.uint8).copy()
        self.key_offs, self.val_offs = ko, vo
        self.c = ffi.CfBlock()
        self.c.keys, self.c.key_offs, self.c.vals, self.c.val_offs, self.c.n = (self.keys.ctypes.data, ko.ctypes.data, self.vals.ctypes.data,
                                                                                vo.ctypes.data, len(kvs))


def run_kvs(entries):
    """[(user, seq, type, value)] -> [(internal key, value)] in internal-key order"""
    return [(ikey(u, s, t), v) for u, s, t, v in sorted(entries, key=lambda e: (e[0], -(e[1] << 8 | e[2])))]


def build_run(entries, trailer_len=5, block_size=1024, sort=True, **opts):
    """one run's data blocks: the keys passed to the block builder already end in their footer (key_suffix_len 0)"""
    kvs = run_kvs(entries) if sort else [(ikey(u, s, t), v) for u, s, t, v in entries]
    return sstfmt.build(FlatBlock(kvs), key_suffix_len=0, trailer_len=trailer_len, block_size=block_size, **opts)


# ---- the model: sort by (user key, -footer, run index), then the first visible entry of each user key ----
def model(runs, snapshot, global_seqs=None):
    """runs: [[(user, seq, type, value)]] newest first -> ([(user key, value)], counts)"""
    gs = global_seqs or [0] * len(runs)
    allv = sorted(((u, -((gs[r] or s) << 8 | t), r, i, gs[r] or s, t, v) for r, run in enumerate(runs) for i, (u, s, t, v) in enumerate(run_order(run))))
    out, c = [], dict(n_in=len(allv), n_out=0, n_invisible=0, n_hidden=0, n_deletions=0)
    prev_user, seen = None, False
    for u, _, _, _, s, t, v in allv:
        if u != prev_user:
            prev_user, seen = u, False
        if s > snapshot:
            c["n_invisible"] += 1
        elif seen:
            c["n_hidden"] += 1
        else:
            seen = True
            if t == VALUE:
                out.append((u, v))
                c["n_out"] += 1
            else:
                c["n_deletions"] += 1
    return out, c


def run_order(run):
    return sorted(run, key=lambda e: (e[0], -(e[1] << 8 | e[2])))


# ---- a known answer: runs derived from a visible state plus noise that must not change it ----
def derive_runs(kvs, seed, n_runs, long_noise=False):
    """(runs newest first, global_seqs, snapshot) whose merging read at `snapshot` is exactly `kvs` (sorted, distinct
    user keys).  Run n-1 is the bottommost (seq 0); run 1 is an ingested file (global seqno) when n >= 3; run n-2 is
    empty when n >= 4; run 0, the newest, straddles the snapshot.  Noise: older versions under the visible one (in older
    runs and in the same run), deletions under it, puts and deletions above the snapshot, deleted keys with the put they
    delete below them, keys that exist only above the snapshot, and equal (user key, footer) pairs whose copy in the run
    listed later carries another value."""
    rng = random.Random(seed)
    B = 1 << 20
    snap = B * n_runs + B // 2
    runs = [dict() for _ in range(n_runs)]  # (user, seq, type) -> value
    gs = [0] * n_runs
    ingested = 1 if n_runs >= 3 else None
    empty = n_runs - 2 if n_runs >= 4 else None
    if ingested is not None:
        gs[ingested] = B * (n_runs - ingested) + rng.randrange(1, B // 2)
    bottom = n_runs - 1 if n_runs >= 2 else None

    def seq_in(r, lo=1, hi=None):  # a sequence number of run r below hi, above lo
        if r == bottom:
            return 0
        if r == ingested:
            return gs[r]
        band_lo = B * (n_runs - r)
        top = band_lo + (B // 2 if r == 0 else B - 1)
        lo_, hi_ = max(band_lo, lo), min(top, hi if hi is not None else top)
        return rng.randrange(lo_, hi_ + 1) if hi_ >= lo_ else None

    def put(r, u, s, t, v):
        if s is None or (u, s, t) in runs[r] or (r == ingested and any(k[0] == u for k in runs[r])):
            return False
        runs[r][(u, s, t)] = v
        return True

    live = [r for r in range(n_runs) if r != empty]
    rnd = lambda: bytes(rng.randrange(256) for _ in range(rng.randrange(0, 12)))  # noqa: E731
    for u, v in kvs:
        while True:  # the visible put
            r = rng.choice(live + [bottom] * 3 if bottom is not None else live)
            s = seq_in(r)
            if s is not None and s <= snap and put(r, u, s, VALUE, v):
                break
        x = rng.random()
        older = [q for q in live if q >= r and (q != bottom or r != bottom) and q != ingested]
        if x < 0.25 and older:  # shadowed put (same run or an older one)
            q = rng.choice(older)
            put(q, u, seq_in(q, hi=s - 1) if q != r else (rng.randrange(max(1, s - 1000), s) if s > 1 and r != bottom and r != ingested else None), VALUE, rnd())
        elif x < 0.35 and older:  # a deletion under the visible put
            q = rng.choice(older)
            put(q, u, seq_in(q, hi=s - 1) if q != r else None, rng.choice([DELETION, SINGLE_DELETION]), b"")
        elif x < 0.45:  # above the snapshot: a newer put or a deletion over the visible key
            put(0, u, rng.randrange(snap + 1, snap + B // 2), rng.choice([VALUE, DELETION, SINGLE_DELETION]), rnd())
        elif x < 0.52 and r != ingested:  # the same (user key, footer) in a run listed later, with another value
            later = [q for q in live if q > r and q != bottom and q != ingested]
            earlier = [q for q in live if q < r and q != ingested]
            if r != bottom and later:
                put(rng.choice(later), u, s, VALUE, v + b"~stale")
            elif r == bottom and earlier and put(rng.choice(earlier), u, 0, VALUE, v):  # (a seq-0 entry above the bottom run)
                runs[r][(u, 0, VALUE)] = v + b"~stale"
        y = rng.random()
        if y < 0.12:  # a deleted key: tombstone above an older put
            d = u + b"\x00" + (b"L" * 140 if long_noise and rng.random() < 0.3 else b"")
            rt = rng.choice(live)
            st = seq_in(rt)
            if st is not None and st <= snap and put(rt, d, st, rng.choice([DELETION, SINGLE_DELETION]), b""):
                olds = [q for q in live if q >= rt and q != ingested and (q != bottom or rt != bottom)]
                if olds:
                    q = rng.choice(olds)
                    put(q, d, seq_in(q, hi=st - 1) if q != rt else (rng.randrange(max(1, st - 1000), st) if st > 1 and rt not in (bottom, ingested) else None), VALUE, rnd())
        elif y < 0.18:  # a key that exists only above the snapshot
            put(0, u + b"\x01" + (b"N" * 150 if long_noise and rng.random() < 0.3 else b""), rng.randrange(snap + 1, snap + B // 2), VALUE, rnd())
    out = [[(u, 0 if r == ingested else s, t, v) for (u, s, t), v in runs[r].items()] for r in range(n_runs)]
    return [run_order(x) for x in out], gs, snap


def features(runs, gs, snap):
    """which of the shapes the merge must handle a generated LSM holds"""
    f = set()
    eff = [[(u, gs[r] or s, t) for u, s, t, _ in run] for r, run in enumerate(runs)]
    by_user = {}
    for r, run in enumerate(eff):
        for u, s, t in run:
            by_user.setdefault(u, []).append((s, t, r))
        users = [u for u, _, _ in run]
        if len(set(users)) < len(users):
            f.add("versions_in_one_run")
        if not run:
            f.add("empty_run")
        if run and gs[r] == 0 and all(s == 0 for _, s, _ in run):
            f.add("seq0_run")
        if gs[r]:
            f.add("global_seqno")
    for u, vs in by_user.items():
        vs.sort(key=lambda e: -(e[0] << 8 | e[1]))
        vis = [e for e in vs if e[0] <= snap]
        if len([e for e in vis if e[1] == VALUE]) > 1 and vis[0][1] == VALUE:
            f.add("shadowed_put")
        if vis and vis[0][1] == DELETION:
            f.add("deletion")
        if vis and vis[0][1] == SINGLE_DELETION:
            f.add("single_deletion")
        above = [e for e in vs if e[0] > snap]
        if above and not vis and any(e[1] == VALUE for e in above):
            f.add("new_key_above_snapshot")
        if above and vis and vis[0][1] == VALUE:
            if any(e[1] in (DELETION, SINGLE_DELETION) for e in above):
                f.add("deletion_above_visible")
            if any(e[1] == VALUE for e in above):
                f.add("put_above_visible")
        if len({(s, t) for s, t, _ in vs}) < len(vs):
            f.add("equal_pair_across_runs")
    return f


ALL_FEATURES = {"versions_in_one_run", "empty_run", "seq0_run", "global_seqno", "shadowed_put", "deletion", "single_deletion", "new_key_above_snapshot",
                "deletion_above_visible", "put_above_visible", "equal_pair_across_runs"}


# ---- the oracle ----
def lib():
    global _lib
    if _lib is None:
        so = _built(os.path.join(BUILD, "libsstmerge.so"), [ORACLE_SRC, ORC_SST], ["g++", "-O2", "-std=c++17", "-fPIC", "-shared", ORACLE_SRC])
        L = C.CDLL(so)
        vp, u32, u64 = C.c_void_p, C.c_uint32, C.c_uint64
        L.orc_sst_merge.argtypes = [vp, vp, vp, vp, vp, u32, u32, u64, C.POINTER(vp)]
        L.orc_sst_merge.restype = C.c_int
        L.orc_sst_merge_result.argtypes = [vp] + [C.POINTER(vp)] * 4 + [C.POINTER(u32), vp]
        L.orc_sst_merge_free.argtypes = [vp]
        _lib = L
    return _lib


def oracle_merge(built, snapshot, global_seqs=None, key_prefix_len=1):
    """built: [(data, offs) or (data, offs, trailer_len)] -> (status 0 / 1 corrupted / 2 unsupported, [(key, value)], counts)"""
    L = lib()
    n = len(built)
    bufs = [np.frombuffer(bytes(b[0]) + b"\0" * 16, dtype=np.uint8) for b in built]
    offs = [np.asarray(b[1], dtype=np.uint64) for b in built]
    data_p = (C.c_void_p * max(n, 1))(*[b.ctypes.data for b in bufs])
    offs_p = (C.c_void_p * max(n, 1))(*[o.ctypes.data for o in offs])
    nb = (C.c_uint32 * max(n, 1))(*[len(o) - 1 for o in offs])
    tl = (C.c_uint32 * max(n, 1))(*[b[2] if len(b) > 2 else 5 for b in built])
    gs = (C.c_uint64 * max(n, 1))(*(global_seqs or [0] * n))
    h = C.c_void_p()
    rc = L.orc_sst_merge(data_p, offs_p, nb, tl, gs, n, key_prefix_len, snapshot, C.byref(h))
    kvs, counts = [], {}
    if rc == 0:
        p = [C.c_void_p() for _ in range(4)]
        cnt = (C.c_uint64 * 5)()
        m = C.c_uint32()
        L.orc_sst_merge_result(h, *[C.byref(x) for x in p], C.byref(m), cnt)
        blk = ffi.CfBlock()
        blk.keys, blk.key_offs, blk.vals, blk.val_offs, blk.n = p[0].value, p[1].value, p[2].value, p[3].value, m.value
        kvs = sstfmt.flat_kvs(blk)
        counts = dict(zip(("n_in", "n_out", "n_invisible", "n_hidden", "n_deletions"), list(cnt)))
    L.orc_sst_merge_free(h)
    return rc, kvs, counts


# ---- the device's per-entry rules, built for the CPU ----
def emul(runs_keys, snapshot, global_seqs=None):
    """runs_keys: [[internal key bytes]] as staged (prefix dropped) -> (status, [(id, verdict)] in merged order)"""
    exe = _built(os.path.join(BUILD, "sst_merge_emul"), [EMUL_SRC, RULES_HDR],
                 ["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", EMUL_SRC])
    gs = global_seqs or [0] * len(runs_keys)
    parts = [struct.pack("<IQ", len(runs_keys), snapshot)]
    for r, keys in enumerate(runs_keys):
        parts.append(struct.pack("<QI", gs[r], len(keys)))
        parts += [struct.pack("<I", len(k)) + k for k in keys]
    with tempfile.TemporaryDirectory() as td:
        cin, cout = os.path.join(td, "case"), os.path.join(td, "result")
        with open(cin, "wb") as f:
            f.write(b"".join(parts))
        subprocess.check_call([exe, cin, cout])
        res = open(cout, "rb").read()
    st = struct.unpack_from("<I", res)[0]
    pairs = [struct.unpack_from("<II", res, 4 + 8 * i) for i in range((len(res) - 4) // 8)]
    return st, pairs


# ---- a bench-sized LSM split on the device (torch) ----
def as_tensor(ptr, n, dtype):
    """a copy of n elements at a device address"""
    import torch

    class Dev:
        __cuda_array_interface__ = dict(shape=(n,), typestr={torch.uint8: "|u1", torch.int32: "<i4"}[dtype], data=(int(ptr), False), version=3)
    return torch.as_tensor(Dev(), device="cuda").clone()


STALE = b"stale"


def device_run(keys, koff, vals, voff, parts):
    """one run as a device-resident flat block whose keys end in their footer, in internal-key order.  parts: (row
    indices, ext: the key is row key + 0x00, seq, type, value: True = the row's, False = STALE, None = empty)"""
    import torch
    cols = {k: [] for k in ("sel", "ext", "foot", "vk")}
    for sel, ext, seq, typ, val in parts:
        k = len(sel)
        cols["sel"].append(sel)
        cols["ext"].append(torch.full((k,), int(ext), dtype=torch.long, device="cuda"))
        seq = seq if torch.is_tensor(seq) else torch.full((k,), seq, dtype=torch.long, device="cuda")
        cols["foot"].append(seq * 256 + typ)
        if typ != 1:
            vk = torch.zeros(k, dtype=torch.long, device="cuda")
        else:
            vk = torch.where(val, 1, 2) if torch.is_tensor(val) else torch.full((k,), 1 if val else 2, dtype=torch.long, device="cuda")
        cols["vk"].append(vk)
    sel, ext, foot, vk = (torch.cat(cols[c]) for c in ("sel", "ext", "foot", "vk"))
    o = torch.sort(-foot, stable=True).indices  # footer descending, then the key ascending (stable)
    o = o[torch.sort(sel[o] * 2 + ext[o], stable=True).indices]
    sel, ext, foot, vk = sel[o], ext[o], foot[o], vk[o]
    m_ = len(sel)
    ul = koff[sel + 1] - koff[sel]
    klen = ul + ext + 8
    ko = torch.zeros(m_ + 1, dtype=torch.long, device="cuda")
    ko[1:] = torch.cumsum(klen, 0)
    e = torch.repeat_interleave(torch.arange(m_, device="cuda"), klen)
    j = torch.arange(int(ko[-1]), device="cuda") - ko[e]
    u = ul[e]
    body = keys[(koff[sel][e] + torch.minimum(j, u - 1).clamp(min=0))].long()
    fb = (foot[e] >> (8 * (j - u - ext[e]).clamp(min=0, max=7))) & 0xFF
    kb = torch.where(j < u, body, torch.where((ext[e] == 1) & (j == u), 0, fb)).to(torch.uint8)
    stale = torch.tensor(list(STALE), dtype=torch.uint8, device="cuda")
    vl = torch.where(vk == 1, voff[sel + 1] - voff[sel], torch.where(vk == 2, len(STALE), 0))
    vo = torch.zeros(m_ + 1, dtype=torch.long, device="cuda")
    vo[1:] = torch.cumsum(vl, 0)
    e = torch.repeat_interleave(torch.arange(m_, device="cuda"), vl)
    j = torch.arange(int(vo[-1]), device="cuda") - vo[e]
    vb = torch.where(vk[e] == 1, vals[(voff[sel][e] + j).clamp(max=len(vals) - 1)], stale[j.clamp(max=len(STALE) - 1)])
    pad = lambda t: torch.cat([t, torch.zeros(32, dtype=torch.uint8, device="cuda")])  # noqa: E731
    return pad(kb), ko.to(torch.int32), pad(vb.to(torch.uint8)), vo.to(torch.int32), m_


def device_lsm(blk, n_l0=4):
    """a generated block (b2_gen_block: distinct keys of one length, so key + 0x00 sorts right after key) split on the
    device into the runs of a live store, newest first: n_l0 (3 or 4) small L0 runs, an L5 run and a bottom run at seq 0.
    The merging read at the returned snapshot is exactly the block.  Each run is (keys, koff, vals, voff, n) in HBM,
    keys ending in their footer (encode with key_suffix_len 0)."""
    import torch
    n = blk.block.n
    keys = as_tensor(blk.block.keys, blk.key_bytes, torch.uint8)
    koff = as_tensor(blk.block.key_offs, n + 1, torch.int32).long()
    vals = as_tensor(blk.block.vals, blk.val_bytes, torch.uint8)
    voff = as_tensor(blk.block.val_offs, n + 1, torch.int32).long()
    i = torch.arange(n, device="cuda")
    snap = 5000
    l5 = i[i % 10 == 3]
    l5, new = i[i % 10 == 3], i % 50 == 7
    shadow = (i % 53 == 9) if n_l0 == 4 else torch.zeros_like(new)
    runs = [
        [(i[i % 100 == 3], False, 3000, 1, True), (i[i % 17 == 5], False, snap + 10, 1, False)],   # puts over L5's; puts above the snapshot
        [(i[i % 29 == 1], False, snap + 5, 0, None), (i[new], False, 3500, 1, True)],              # deletions above the snapshot; new keys
        [(i[i % 31 == 2], False, snap + 3, 7, None), (i[i % 37 == 4], True, snap + 8, 1, False)],  # single deletions and new keys above it
        [(i[shadow], False, 3200, 1, True)],                                                        # puts over the bottom's
        [(l5, False, 1000 + l5 % 7, 1, l5 % 100 != 3), (i[i % 13 == 0], True, 1001, 0, None)],     # L5: puts over the bottom's; tombstones
        [(i[~new], False, 0, 1, (i[~new] % 10 != 3) & ~shadow[~new]), (i[i % 13 == 0], True, 0, 1, False)],  # bottom, and the puts deleted above
    ]
    if n_l0 == 3:
        del runs[3]
    return [device_run(keys, koff, vals, voff, ps) for ps in runs], snap
