"""A plain reference for TopN over generated and hand-built tables: no GPU and no project code in the loop.

gen_rows restates the device region generator (kernels.cu b2_gen_create: gen_mix, gen_row_kind, gen_value and the
versions it writes per row) in numpy; expected_topn / topn_indices are the exact TopN of rows in scan order, under the
device's documented total order (b2_device.h TopItem / item_less): sort key by sort key, NULL before any value, signed,
unsigned or Real compares (-0.0 == 0.0), each key reversed for DESC, and the remaining ties to the row scanned first.
That is stricter than the reference's heap, which keeps an arbitrary one of rows tied at the cut.
"""
import numpy as np

MASK = (1 << 64) - 1
_U = np.uint64

# engine.cu run_topn: the first chunk of a request holds 16 tiles of TILE entries (kernels.cuh TILE), and every later
# chunk about 7x the entries scanned before it; a chunk that would leave less than half a chunk behind takes the rest
TILE = 256


def chunk_bounds(e_lo, e_hi, seeded_rows=0):
    """Chunk boundaries of one unit (its CF_WRITE entries [e_lo, e_hi)) after `seeded_rows` entries of earlier units:
    ([c_lo, ...], seeded_rows after the unit)."""
    starts, c_lo = [], e_lo
    while c_lo < e_hi:
        want = max(16 * TILE, 7 * seeded_rows)
        c_hi = e_hi if e_hi - c_lo <= want + want // 2 else c_lo + want
        starts.append(c_lo)
        seeded_rows += c_hi - c_lo
        c_lo = c_hi
    return starts, seeded_rows


def mix64(x):
    """The scalar finaliser (Python ints)."""
    x ^= x >> 33; x = (x * 0xff51afd7ed558ccd) & MASK; x ^= x >> 33; x = (x * 0xc4ceb9fe1a85ec53) & MASK; x ^= x >> 33
    return x


def gen_mix_scalar(seed, handle, salt):
    return mix64((seed & MASK) ^ ((handle * 0x9E3779B97F4A7C15) & MASK) ^ (((salt + 1) * 0xBF58476D1CE4E5B9) & MASK))


def gen_mix(seed, handles, salt):
    """gen_mix over a uint64 array of handles (two's complement bits of the i64 handle)."""
    with np.errstate(over="ignore"):
        x = _U(seed & MASK) ^ (handles * _U(0x9E3779B97F4A7C15)) ^ _U(((salt + 1) * 0xBF58476D1CE4E5B9) & MASK)
        x ^= x >> _U(33); x *= _U(0xff51afd7ed558ccd); x ^= x >> _U(33); x *= _U(0xc4ceb9fe1a85ec53); x ^= x >> _U(33)
    return x


# gen_row_kind: 0 plain Put, 1 three versions (one newer than the read ts, the visible salt-0 Put, an older one),
# 2 Delete over an older Put (no visible row), 3 Lock record over the visible Put
ENTRIES_PER_KIND = np.array([1, 3, 2, 2], dtype=np.int64)


def gen_rows(spec, blocks):
    """Visible rows of the generated blocks, in key order.

    spec: dict(n_cols, seed, lo=None, rng=None, nulls=None, extra=0, delete=0, lockrec=0) as b2_gen_spec (col_lo,
    col_range, null_per_million, *_per_million); blocks: [(first_handle, n_rows)], one per generated block.
    Returns dict(handle=int64[n], vals=int64[n, n_cols], null=bool[n, n_cols], entry=int64[n], block=int64[n],
    n_entries=[per block]): `entry` is the index of the row's first CF_WRITE entry inside its block."""
    n_cols, seed = spec["n_cols"], spec["seed"]
    lo, rng, nulls = spec.get("lo"), spec.get("rng"), spec.get("nulls")
    extra, delete, lockrec = spec.get("extra", 0), spec.get("delete", 0), spec.get("lockrec", 0)
    out = dict(handle=[], vals=[], null=[], entry=[], block=[], n_entries=[])
    for b, (first, n) in enumerate(blocks):
        h = (np.arange(n, dtype=np.int64) + first).astype(np.uint64)
        r = gen_mix(seed, h, 1000) % _U(1000000)
        kind = np.where(r < extra, 1, np.where(r < extra + delete, 2, np.where(r < extra + delete + lockrec, 3, 0)))
        ents = ENTRIES_PER_KIND[kind]
        first_entry = np.concatenate(([0], np.cumsum(ents)[:-1]))
        vals = np.empty((n, n_cols), dtype=np.int64)
        null = np.zeros((n, n_cols), dtype=bool)
        for c in range(n_cols):
            if nulls is not None and nulls[c]:
                null[:, c] = gen_mix(seed, h, 500 + c) % _U(1000000) < _U(nulls[c])
            x = gen_mix(seed, h, c)  # (version salt 0: the visible Put)
            if rng is not None and rng[c]:
                with np.errstate(over="ignore"):
                    x = _U(lo[c] & MASK) + x % _U(rng[c])
            vals[:, c] = x.view(np.int64)
        vals[null] = 0
        keep = kind != 2
        out["handle"].append(h.view(np.int64)[keep]); out["vals"].append(vals[keep]); out["null"].append(null[keep])
        out["entry"].append(first_entry[keep]); out["block"].append(np.full(int(keep.sum()), b, dtype=np.int64))
        out["n_entries"].append(int(ents.sum()))
    for k in ("handle", "vals", "null", "entry", "block"):
        out[k] = np.concatenate(out[k])
    return out


def topn_indices(keys, limit, desc_scan=False):
    """Indices (into rows in key order) of the top `limit` rows, best first.

    keys: [(values, null_mask, desc)] per sort key, values an int64, uint64 or float64 array (NaN is not a value: the
    caller has made it NULL).  A backward scan meets the rows in reverse key order, so its ties go to the larger key."""
    n = len(keys[0][0])
    pos = np.arange(n, dtype=np.int64)
    lex = [-pos if desc_scan else pos]  # np.lexsort: the last key is the primary one
    for v, null, desc in reversed(keys):
        v = np.asarray(v)
        null = np.zeros(n, dtype=bool) if null is None else np.asarray(null, dtype=bool)
        if v.dtype == np.float64:
            assert not np.isnan(v[~null]).any(), "NaN is NULL: pass it in the null mask"
            v = np.where(null, 0.0, v) + 0.0  # (-0.0 + 0.0 is 0.0)
            v = -v if desc else v
        else:
            v = np.where(null, v.dtype.type(0), v)
            v = ~v if desc else v  # order-reversing on int64 and uint64 alike, without overflow
        lex += [v, null if desc else ~null]  # NULL first; DESC puts it last
    return np.lexsort(lex)[:limit]


def _key_array(rows, key):
    get, desc, kind = key
    vals = [get(r) if callable(get) else r[get] for r in rows]
    null = np.array([v is None or (kind == "real" and v != v) for v in vals], dtype=bool)
    dt = {"int": np.int64, "uint": np.uint64, "real": np.float64}[kind]
    if kind == "uint":
        vals = [None if m else v & MASK for v, m in zip(vals, null)]  # (results carry an unsigned column's bits as i64)
    return np.array([0 if m else v for v, m in zip(vals, null)], dtype=dt), null, desc


def expected_topn(rows, keys, limit, desc_scan=False):
    """TopN of `rows` (tuples, in key order; None is NULL): keys = [(column index or function of the row, desc, kind)]
    with kind "int", "uint" or "real".  Returns the chosen rows, best first."""
    rows = list(rows)
    if not rows or limit == 0:
        return []
    return [rows[i] for i in topn_indices([_key_array(rows, k) for k in keys], limit, desc_scan)]
