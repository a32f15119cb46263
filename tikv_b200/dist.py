"""Multi-GPU layer: one process per GPU, regions sharded statically, no data-path collective.

The reference never exchanges data between regions inside TiKV: every region returns *partial* results and TiDB
merges them (endpoint.rs:697-775 fans store-batched tasks out one region at a time).  Here each rank scans its own
regions on its own GPU; the only exchange is the final merge of those partial results, done with `torch.distributed`
(NCCL over NVLink on GPUs, gloo in the CPU tests):

  hash aggregation : all_gather of the compact partial tables (group key, additive accumulator words) + re-aggregation
  TopN             : all_gather of each rank's top-N rows + final selection
  checksum         : all_gather of the u64 partial CRCs + XOR (NCCL has no XOR reduction), all_reduce(SUM) of the counts

All merge functions take plain torch tensors, so they run unchanged on CPU tensors under gloo.  The aggregation merge of
CUDA tensors re-aggregates the gathered rows in one native call (b2_agg_merge: a sort-based group-by on the device that
gives the torch path's result bit for bit); CPU tensors take that torch path.
"""
import torch
import torch.distributed as dist

SIGN = -(1 << 63)


def shard_blocks(n_blocks, world, rank):
    """Static region -> GPU assignment: contiguous runs keep every rank's key space ordered."""
    per, rem = divmod(n_blocks, world)
    lo = rank * per + min(rank, rem)
    return list(range(lo, lo + per + (1 if rank < rem else 0)))


def _world():
    return dist.get_world_size() if dist.is_initialized() else 1


def _all_gather_var(t):
    """all_gather of tensors whose first dimension differs per rank (pad to the max, then trim)."""
    world = _world()
    if world == 1:
        return [t]
    n = torch.tensor([t.shape[0]], dtype=torch.int64, device=t.device)
    sizes = [torch.zeros_like(n) for _ in range(world)]
    dist.all_gather(sizes, n)
    m = int(max(int(s.item()) for s in sizes))
    pad = torch.zeros((m,) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
    pad[: t.shape[0]] = t
    out = [torch.zeros_like(pad) for _ in range(world)]
    dist.all_gather(out, pad)
    return [o[: int(s.item())] for o, s in zip(out, sizes)]


# ---- hash aggregation -------------------------------------------------------------------------------------------
F64_ACC_DIGITS = 66  # b2_device.h: exact Real sums are 66 carry-save 32-bit digits (bit 0 = 2^-1074)


def f64_acc_digits(x):
    """The accumulator words of one finite double (what f64_acc_add adds), as python ints."""
    import struct
    bits = struct.unpack("<Q", struct.pack("<d", float(x)))[0]
    m, e = bits & ((1 << 52) - 1), (bits >> 52) & 0x7FF
    if e:
        m |= 1 << 52
    else:
        e = 1
    v = (-m if bits >> 63 else m) << (e - 1)
    sign = -1 if v < 0 else 1
    v = abs(v)
    return [sign * ((v >> (32 * i)) & 0xFFFFFFFF) for i in range(F64_ACC_DIGITS)]


def f64_acc_value(words):
    """Correctly rounded double of an accumulator (f64_acc_round), via exact rational arithmetic."""
    from fractions import Fraction
    total = 0
    for i, w in enumerate(words):
        w = int(w)
        if w >= 1 << 63:
            w -= 1 << 64
        total += w << (32 * i)
    return float(Fraction(total, 1 << 1074))


def merge_agg_partials(keys, key_null, acc, real_words=(), max_words=(), word_ops=None, desc=False):
    """Final merge of partial aggregation tables.

    keys: int64[n] group-key bits, key_null: bool[n], acc: int64[n, W] additive accumulator words (b2_agg_partials).
    Grouped by K > 1 expressions (b2_agg_partials.key_words): keys is int64[n, K] and key_null the per-group NULL mask
    (integer, bit q = q-th expression); the result has the same shapes.
    `max_words` lists the word indices that merge by unsigned maximum (the MAX / MIN extremum keys,
    b2_agg_partials.max_word_mask); every other word is additive: counts, the 32-bit limb sums of integer SUMs and the
    digits of exact Real SUMs (`real_words` is only for callers that still carry plain f64 words).  Returns (keys, key_null, acc) with one row per group,
    sorted as torch.unique sorts (NULL mask, key words).
    Integer words are summed exactly (two's-complement wraparound is impossible below 2^32 rows per group).
    `word_ops` (agg_word_ops: one ffi.MERGE_* per word) adds the FIRST / BIT_* states: OR and XOR words reduce with their
    op; a FIRST pair is taken from the earliest gathered part (rank order, the order of shard_blocks' contiguous runs)
    holding a nonzero key, or the latest when the scan is `desc`; keys are compared only inside one part.
    CUDA tensors merge on the device in one call (b2_agg_merge); CPU tensors and `real_words` merge with torch ops."""
    multi = keys.dim() == 2
    kw = keys.shape[1] if multi else 1
    if keys.is_cuda and not real_words:
        if _world() == 1:  # nothing to gather: the native merge reads the three tables as they are
            return _merge_native(keys.view(-1, kw), key_null, acc, [keys.shape[0]], multi, max_words, word_ops, desc)
        parts = _all_gather_var(torch.cat([keys.view(-1, kw), key_null.to(torch.int64).view(-1, 1), acc], dim=1))
        allp = torch.cat(parts, dim=0)
        return _merge_native(allp[:, :kw], allp[:, kw], allp[:, kw + 1:], [p.shape[0] for p in parts], multi, max_words, word_ops, desc)
    parts = _all_gather_var(torch.cat([keys.view(-1, kw), key_null.to(torch.int64).view(-1, 1), acc], dim=1))
    return _merge_gathered_torch(parts, kw, multi, real_words, max_words, word_ops, desc)


def _merge_native(keys, key_null, acc, part_sizes, multi, max_words=(), word_ops=None, desc=False):
    """merge_agg_partials on the CUDA device of the rows: b2_agg_merge on the current stream, one call.  keys: int64[n, K]
    and acc: int64[n, W], rows may be strided (views into gathered rows); key_null: bool or integer NULL masks [n];
    part_sizes: rows of each gathered part, in rank order."""
    import ctypes as C
    from . import ffi
    if keys.stride(1) != 1:
        keys = keys.contiguous()
    if acc.shape[1] and acc.stride(1) != 1:
        acc = acc.contiguous()
    if key_null.dtype not in (torch.bool, torch.uint8) or not key_null.is_contiguous():
        key_null = key_null.to(torch.uint8).contiguous()  # masks are below 2^K <= 16
    n, kw, aw = keys.shape[0], keys.shape[1], acc.shape[1]
    ops = list(word_ops) if word_ops is not None else [ffi.MERGE_ADD] * aw
    for w in max_words:
        ops[w] = ffi.MERGE_MAX
    offs = [0]
    for m in part_sizes:
        offs.append(offs[-1] + m)
    out_k = torch.empty((n, kw) if multi else (n,), dtype=torch.int64, device=keys.device)
    out_n = torch.empty(n, dtype=torch.uint8, device=keys.device)
    out_a = torch.empty((n, aw), dtype=torch.int64, device=keys.device)
    ng = C.c_uint64()
    L = ffi.lib()
    rc = L.b2_agg_merge(keys.device.index, torch.cuda.current_stream(keys.device).cuda_stream, n, kw, aw,
                        keys.data_ptr(), keys.stride(0), key_null.data_ptr(), acc.data_ptr(), acc.stride(0) if aw else 0,
                        (C.c_uint64 * len(offs))(*offs), len(part_sizes), (C.c_uint8 * max(1, aw))(*ops), int(bool(desc)),
                        out_k.data_ptr(), out_n.data_ptr(), out_a.data_ptr(), C.byref(ng))
    if rc != 0:
        raise RuntimeError("b2_agg_merge: " + L.b2_last_error_message().decode())
    g = ng.value
    return out_k[:g], (out_n[:g].to(torch.int64) if multi else out_n[:g].view(torch.bool)), out_a[:g]


def _merge_gathered_torch(parts, kw, multi, real_words=(), max_words=(), word_ops=None, desc=False):
    """merge_agg_partials of the gathered rows (kw key words | NULL mask | accumulator words, one tensor per part) with
    torch ops, on any device: the reference the native merge is tested against."""
    from . import ffi
    ops = list(word_ops) if word_ops is not None else []
    max_words = set(max_words) | {w for w, o in enumerate(ops) if o == ffi.MERGE_MAX}
    bit_words = {w: o for w, o in enumerate(ops) if o in (ffi.MERGE_OR, ffi.MERGE_XOR)}
    first_words = [w for w, o in enumerate(ops) if o == ffi.MERGE_FIRST_KEY]
    special = set(real_words) | max_words | set(bit_words) | {w for w, o in enumerate(ops) if o in (ffi.MERGE_FIRST_KEY, ffi.MERGE_FIRST_VALUE)}
    part_of = torch.cat([torch.full((p.shape[0],), i, dtype=torch.int64, device=p.device) for i, p in enumerate(parts)])
    allp = torch.cat(parts, dim=0)
    if allp.shape[0] == 0:
        return (allp[:, :kw], allp[:, kw], allp[:, kw + 1:]) if multi else (allp[:, 0], allp[:, 1].bool(), allp[:, 2:])
    k, nul, a = allp[:, :kw], allp[:, kw], allp[:, kw + 1:]
    if not multi:
        k = torch.where(nul.bool().view(-1, 1), torch.zeros_like(k), k)
    ident = torch.cat([nul.view(-1, 1), k], dim=1)
    uniq, inv = torch.unique(ident, dim=0, return_inverse=True)
    out = torch.zeros((uniq.shape[0], a.shape[1]), dtype=torch.int64, device=a.device)
    ng = uniq.shape[0]
    for w, o in bit_words.items():  # per bit plane: OR = any row has it, XOR = an odd number of rows have it
        for b0 in range(0, 64, 8):  # 8 one-byte planes at a time: 8 transient bytes per gathered row
            shifts = torch.arange(b0, b0 + 8, device=a.device)
            planes = ((a[:, w].view(-1, 1) >> shifts) & 1).to(torch.uint8)
            red = torch.zeros((ng, 8), dtype=torch.uint8, device=a.device)
            if o == ffi.MERGE_OR:
                red.scatter_reduce_(0, inv.view(-1, 1).expand(-1, 8), planes, reduce="amax")
            else:
                red.index_add_(0, inv, planes)  # (a uint8 sum wraps mod 256 and keeps its parity)
            out[:, w] |= ((red & 1).to(torch.int64) << shifts).sum(dim=1)  # (distinct bits: their sum is their OR)
    for w in first_words:
        has = a[:, w] != 0
        pref = part_of if desc else len(parts) - 1 - part_of  # larger = preferred part
        pref = torch.where(has, pref, torch.full_like(pref, -1))
        best = torch.full((ng,), -1, dtype=torch.int64, device=a.device).scatter_reduce_(0, inv, pref, reduce="amax")
        cand = has & (pref == best[inv])
        flipped = torch.where(cand, a[:, w] ^ SIGN, torch.full_like(a[:, w], SIGN))  # unsigned order as signed
        top = torch.full((ng,), SIGN, dtype=torch.int64, device=a.device).scatter_reduce_(0, inv, flipped, reduce="amax")
        win = cand & (flipped == top[inv])
        out[inv[win], w] = a[win, w]
        out[inv[win], w + 1] = a[win, w + 1]
    int_words = [w for w in range(a.shape[1]) if w not in special]
    if int_words:
        out[:, int_words] = torch.zeros((uniq.shape[0], len(int_words)), dtype=torch.int64, device=a.device).index_add_(0, inv, a[:, int_words])
    for w in real_words:
        s = torch.zeros(uniq.shape[0], dtype=torch.float64, device=a.device).index_add_(0, inv, a[:, w].contiguous().view(torch.float64))
        out[:, w] = s.view(torch.int64)
    for w in max_words:  # unsigned 64-bit maximum = signed maximum after flipping the top bit
        flipped = a[:, w] ^ (-(1 << 63))
        m = torch.full((uniq.shape[0],), -(1 << 63), dtype=torch.int64, device=a.device).scatter_reduce_(0, inv, flipped, reduce="amax")
        out[:, w] = m ^ (-(1 << 63))
    if multi:
        return uniq[:, 1:].contiguous(), uniq[:, 0].contiguous(), out
    return uniq[:, 1].contiguous(), uniq[:, 0].bool(), out


def limbs_to_int(lo, hi, unsigned=False):
    """Exact value of an integer SUM from its two 32-bit limb sums (python ints): hi * 2^32 + lo."""
    lo &= (1 << 64) - 1
    if unsigned:
        hi &= (1 << 64) - 1
    elif hi >= (1 << 63):
        hi -= 1 << 64
    return hi * (1 << 32) + lo


# ---- TopN ---------------------------------------------------------------------------------------------------------
def _order_word(col, null, desc, kind):
    """Order-preserving int64 ranks for one order-by column: NULL first (last when DESC), unsigned / f64 aware."""
    if kind == "f64":
        f = col.view(torch.float64)
        f = torch.where(f == 0, torch.zeros_like(f), f)
        b = f.view(torch.int64)
        w = torch.where(b < 0, ~b, b | SIGN) ^ SIGN  # total order as signed int64
    elif kind == "u64":
        w = col ^ SIGN
    else:
        w = col
    return w, null


def merge_topn(columns, nulls, order, limit):
    """columns: list of int64[n] (bits), nulls: list of bool[n]; order: [(column index, desc, kind)] with kind in
    {'i64','u64','f64'}.  Gathers every rank's rows and keeps the best `limit`, sorted."""
    rows = torch.stack(columns + [n.to(torch.int64) for n in nulls], dim=1) if columns else torch.zeros((0, 0), dtype=torch.int64)
    allr = torch.cat(_all_gather_var(rows), dim=0)
    nc = len(columns)
    idx = torch.arange(allr.shape[0], device=allr.device)
    # lexicographic sort = stable sorts from the least significant key to the most significant one
    for ci, desc, kind in reversed(order):
        w, nul = _order_word(allr[:, ci], allr[:, nc + ci].bool(), desc, kind)
        w = torch.where(nul, torch.zeros_like(w), w)  # a NULL cell may hold any bits: it must not disturb the less significant keys
        w, nul = w[idx], nul[idx]
        # asc: NULLs first, then ascending value; desc: reverse of that
        perm = torch.argsort(w, stable=True, descending=bool(desc))
        idx, nul = idx[perm], nul[perm]
        perm2 = torch.argsort(nul.to(torch.int8), stable=True, descending=not desc)
        idx = idx[perm2]
    idx = idx[:limit]
    sel = allr[idx]
    return [sel[:, i].contiguous() for i in range(nc)], [sel[:, nc + i].bool() for i in range(nc)]


# ---- checksum -------------------------------------------------------------------------------------------------------
def merge_checksum(checksum, total_kvs, total_bytes, device="cpu"):
    """XOR of the per-rank CRC folds (all_gather + local XOR), sums of the counters (all_reduce)."""
    if _world() == 1:
        return checksum, total_kvs, total_bytes
    c = torch.tensor([checksum - (1 << 64) if checksum >= (1 << 63) else checksum], dtype=torch.int64, device=device)
    parts = [torch.zeros_like(c) for _ in range(_world())]
    dist.all_gather(parts, c)
    x = 0
    for p in parts:
        x ^= int(p.item()) & ((1 << 64) - 1)
    cnt = torch.tensor([total_kvs, total_bytes], dtype=torch.int64, device=device)
    dist.all_reduce(cnt, op=dist.ReduceOp.SUM)
    return x, int(cnt[0].item()), int(cnt[1].item())


# ---- device partial tables -> torch tensors ---------------------------------------------------------------------------
class _CudaArray:
    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = {"shape": shape, "typestr": typestr, "data": (ptr, False), "version": 2}


def agg_partials_as_tensors(executor, device):
    """Wrap the executor's device-resident partial aggregation table (b2_exec_agg_partials) as torch tensors (no copy)."""
    import ctypes as C
    from . import ffi
    p = ffi.AggPartials()
    rc = ffi.lib().b2_exec_agg_partials(executor._h, C.byref(p))
    if rc != 0:
        raise RuntimeError(ffi.lib().b2_last_error_message().decode())
    n, w = p.n_groups, p.acc_words
    dev = torch.device("cuda", device)
    if n == 0:
        z = torch.zeros(0, dtype=torch.int64, device=dev)
        return z, z.bool(), torch.zeros((0, w), dtype=torch.int64, device=dev)
    acc = torch.as_tensor(_CudaArray(p.acc, (n, w), "<i8"), device=dev).clone()
    if p.has_group and p.key_words > 1:
        keys = torch.as_tensor(_CudaArray(p.keys, (n, p.key_words), "<i8"), device=dev).clone()
        nul = torch.as_tensor(_CudaArray(p.key_null, (n,), "|u1"), device=dev).to(torch.int64)
    elif p.has_group:
        keys = torch.as_tensor(_CudaArray(p.keys, (n,), "<i8"), device=dev).clone()
        nul = torch.as_tensor(_CudaArray(p.key_null, (n,), "|u1"), device=dev).bool()
    else:
        keys = torch.zeros(n, dtype=torch.int64, device=dev)
        nul = torch.zeros(n, dtype=torch.bool, device=dev)
    return keys, nul, acc


def agg_word_ops(executor):
    """How each accumulator word of the executor's partial table merges (b2_exec_agg_word_ops): a list of ffi.MERGE_*."""
    import ctypes as C
    from . import ffi
    p = ffi.AggPartials()
    rc = ffi.lib().b2_exec_agg_partials(executor._h, C.byref(p))
    if rc == 0:
        n = C.c_uint32(p.acc_words)
        ops = (C.c_uint8 * max(1, p.acc_words))()
        rc = ffi.lib().b2_exec_agg_word_ops(executor._h, ops, C.byref(n))
    if rc != 0:
        raise RuntimeError(ffi.lib().b2_last_error_message().decode())
    return list(ops[: n.value])
