"""`-m gpu`: the native final merge of gathered partial tables (b2_agg_merge) against the torch merge of dist.py on CPU
copies of the same rows: the same groups in the same order, the same dtypes, every word bit for bit.  Rows are generated
from fixed seeds: 1-4 key words, NULL masks (single-key NULL rows carry garbage key bits), keys at the int64 edges,
every merge op, FIRST in both scan directions across several parts (empty parts, parts without a key, ties inside one
part), duplicates within and across parts, wrapping sums, and 0 / 1 / 1024 / ~1e6 rows."""
import numpy as np
import pytest
import torch

from tikv_b200 import dist as bd
from tikv_b200 import ffi

pytestmark = pytest.mark.gpu

EDGES = [-(1 << 63), -1, 0, (1 << 63) - 1]
ALL_OPS = [ffi.MERGE_ADD, ffi.MERGE_MAX, ffi.MERGE_OR, ffi.MERGE_XOR, ffi.MERGE_FIRST_KEY, ffi.MERGE_FIRST_VALUE, ffi.MERGE_ADD]


def _u64(rng, n):
    return rng.integers(-(1 << 63), (1 << 63) - 1, size=n, dtype=np.int64, endpoint=True)


def gen_parts(seed, kw, sizes, ops, n_keys=40, null_frac=0.1, first_ties=True):
    """One int64[size, kw + 1 + len(ops)] tensor per part: key words drawn from a pool of n_keys values per word (edges
    included), so groups repeat within and across parts; NULL masks below 2^kw; state words by op.  FIRST keys are 0 in
    30 % of the rows and come from five values when `first_ties` (which row wins a tie is the torch reference's
    last write: serial only for small inputs)."""
    rng = np.random.default_rng(seed)
    pools = [np.concatenate([np.array(EDGES, dtype=np.int64), _u64(rng, max(0, n_keys - len(EDGES)))]) for _ in range(kw)]
    parts = []
    for n in sizes:
        rows = np.zeros((n, kw + 1 + len(ops)), dtype=np.int64)
        for k in range(kw):
            rows[:, k] = rng.choice(pools[k], size=n)
        nul = rng.random(n) < null_frac
        if kw == 1:
            rows[:, 1] = nul
            rows[nul, 0] = _u64(rng, int(nul.sum()))  # garbage bits under a NULL key: they must not split the group
        else:
            rows[:, kw] = np.where(nul, rng.integers(1, 1 << kw, size=n), 0)
        for w, o in enumerate(ops):
            c = kw + 1 + w
            if o == ffi.MERGE_FIRST_KEY:
                keys = rng.choice(np.array([1, 2, 3, -1, -(1 << 63)], dtype=np.int64), size=n) if first_ties else _u64(rng, n)
                rows[:, c] = np.where(rng.random(n) < 0.3, 0, keys)
            else:
                rows[:, c] = _u64(rng, n)  # full-width words: ADD wraps modulo 2^64
        parts.append(torch.from_numpy(rows))
    return parts


def check(parts, kw, multi, ops=None, desc=False, max_words=()):
    exp = bd._merge_gathered_torch(parts, kw, multi, max_words=max_words, word_ops=ops, desc=desc)
    allp = torch.cat(parts, dim=0).cuda()  # the gathered form: strided views of packed rows, int64 NULL masks
    got = bd._merge_native(allp[:, :kw], allp[:, kw], allp[:, kw + 1:], [p.shape[0] for p in parts], multi, max_words=max_words, word_ops=ops, desc=desc)
    for name, e, g in zip(("keys", "key_null", "acc"), exp, got):
        assert g.is_cuda and g.dtype == e.dtype and tuple(g.shape) == tuple(e.shape), (name, g.dtype, e.dtype, g.shape, e.shape)
        g = g.cpu()
        assert torch.equal(g, e), (name, (g != e).nonzero()[:5].tolist())
    return exp


@pytest.mark.parametrize("desc", [False, True], ids=["fwd", "bwd"])
@pytest.mark.parametrize("kw", [1, 2, 3, 4])
def test_every_op_across_parts(kw, desc):
    parts = gen_parts(100 + kw, kw, [0, 37, 300, 0, 64, 1], ALL_OPS, n_keys={1: 40, 2: 10, 3: 5, 4: 4}[kw])
    exp = check(parts, kw, kw > 1, ALL_OPS, desc)
    assert 10 < exp[0].shape[0] < sum(p.shape[0] for p in parts)


@pytest.mark.parametrize("kw", [1, 3])
def test_max_words_and_default_add(kw):
    parts = gen_parts(7 + kw, kw, [120, 80], [ffi.MERGE_ADD] * 4, n_keys=8)
    check(parts, kw, kw > 1)
    check(parts, kw, kw > 1, max_words=(1, 3))


def test_edge_keys_order_and_null_garbage():
    """Every key at an int64 edge, in every order, NULL rows with arbitrary key bits: the keys in signed order, then one
    NULL group (mask 1 sorts after mask 0)."""
    keys = torch.tensor(EDGES * 3 + [5, -5], dtype=torch.int64)
    nul = torch.zeros(len(keys), dtype=torch.int64)
    nul[[0, 5, 13]] = 1
    acc = torch.arange(len(keys), dtype=torch.int64).view(-1, 1)
    parts = [torch.cat([keys.view(-1, 1), nul.view(-1, 1), acc], 1)[torch.randperm(len(keys), generator=torch.Generator().manual_seed(3))]]
    k, n, a = check(parts, 1, False)
    assert n.tolist() == [False] * 5 + [True] and k.tolist() == [-(1 << 63), -1, 0, 5, (1 << 63) - 1, 0]


@pytest.mark.parametrize("desc", [False, True], ids=["fwd", "bwd"])
def test_first_rules(desc):
    """FIRST by hand: group 1 has no key in part 0 (empty), key 0 in part 1, ties of the largest key in part 2 and a
    larger key in part 3; group 2 has no nonzero key anywhere."""
    ops = [ffi.MERGE_FIRST_KEY, ffi.MERGE_FIRST_VALUE]

    def part(rows):
        return torch.tensor(rows, dtype=torch.int64).view(-1, 4)
    parts = [part([]), part([[1, 0, 0, 11], [2, 0, 0, 12]]), part([[1, 0, 5, 21], [1, 0, 9, 22], [1, 0, 9, 23], [2, 0, 0, 24]]),
             part([[1, 0, -3, 31], [1, 0, 2, 32]])]
    k, n, a = check(parts, 1, False, ops, desc)
    assert a.tolist() == ([[-3, 31], [0, 0]] if desc else [[9, 23], [0, 0]])


@pytest.mark.parametrize("n", [0, 1, 1024])
def test_small_sizes(n):
    for kw in (1, 2):
        check(gen_parts(n + kw, kw, [n], [ffi.MERGE_ADD] * 3, n_keys=2 * n + 4), kw, kw > 1)
    check([torch.zeros((0, 4), dtype=torch.int64)] * 3, 1, False, [ffi.MERGE_FIRST_KEY, ffi.MERGE_FIRST_VALUE])


def test_bench_shaped_table():
    """1024 distinct keys, one part, [count, low limb sum, high limb sum]: the shape of bench.py's C3 merge."""
    keys = torch.randperm(1024, generator=torch.Generator().manual_seed(11)).to(torch.int64)
    acc = torch.randint(0, 1 << 40, (1024, 3), generator=torch.Generator().manual_seed(12), dtype=torch.int64)
    k, n, a = bd.merge_agg_partials(keys.cuda(), torch.zeros(1024, dtype=torch.bool, device="cuda"), acc.cuda())
    assert k.dtype == torch.int64 and n.dtype == torch.bool and torch.equal(k.cpu(), torch.arange(1024))
    assert torch.equal(a.cpu(), acc[torch.argsort(keys)])
    check([torch.cat([keys.view(-1, 1), torch.zeros((1024, 1), dtype=torch.int64), acc], 1)], 1, False)


@pytest.mark.parametrize("kw", [1, 2])
def test_million_rows(kw):
    parts = gen_parts(900 + kw, kw, [250_000, 0, 500_000, 250_000], ALL_OPS, n_keys=300, first_ties=False)
    exp = check(parts, kw, kw > 1, ALL_OPS, desc=kw == 2)
    assert exp[0].shape[0] > 250


def test_rejects_bad_arguments():
    rows = torch.zeros((4, 8), dtype=torch.int64, device="cuda")
    with pytest.raises(RuntimeError, match="FIRST"):
        bd._merge_native(rows[:, :1], rows[:, 1], rows[:, 2:], [4], False, word_ops=[ffi.MERGE_ADD] * 5 + [ffi.MERGE_FIRST_KEY])
    with pytest.raises(RuntimeError, match="key words"):
        bd._merge_native(rows[:, :5], rows[:, 5], rows[:, 6:], [4], True)
