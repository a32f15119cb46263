"""Host-side plan builder: the flat POD equivalent of tipb::DagRequest that crosses the C ABI.

Mirrors the reference's test builder `DagSelect` (components/test_coprocessor/src/dag.rs) in spirit:
    DagSelect.from(table).where(...).aggr_sum(col).group_by([col]).build()
Expressions are written as trees and lowered to RPN post-order exactly like
tidb_query_expr/src/types/expr_builder.rs:251-330 does for tipb::Expr trees.
"""
import ctypes as C

from . import ffi

_INT_TPS = {ffi.TP_TINY, ffi.TP_SHORT, ffi.TP_INT24, ffi.TP_LONG, ffi.TP_LONGLONG, ffi.TP_YEAR, ffi.TP_BIT}
_REAL_TPS = {ffi.TP_FLOAT, ffi.TP_DOUBLE}


def eval_kind(tp):
    if tp in _INT_TPS:
        return "int"
    if tp in _REAL_TPS:
        return "real"
    if tp == ffi.TP_NEWDECIMAL:
        return "decimal"
    if tp in (ffi.TP_DATE, ffi.TP_DATETIME):
        return "time"
    if tp == ffi.TP_DURATION:
        return "duration"
    if tp in (ffi.TP_VARCHAR, ffi.TP_VARSTRING, ffi.TP_STRING, ffi.TP_BLOB, 0xf9, 0xfa, 0xfb, 0xff):
        return "bytes"
    return "other"


class Expr:
    """Expression tree node; `.tp/.flag` is the node's return FieldType."""

    def __init__(self, kind, tp, flag=0, sig=0, args=(), i64=0, f64=0.0, collation=0, data=None):
        self.kind, self.tp, self.flag, self.sig, self.args, self.i64, self.f64 = kind, tp, flag, sig, tuple(args), i64, f64
        self.collation, self.data = collation, data

    def rpn(self, out=None, keep=None):
        """Post-order nodes; `keep` collects the buffers bytes constants point into (the Plan owns them)."""
        out = [] if out is None else out
        for a in self.args:
            a.rpn(out, keep)
        n = ffi.RpnNode()
        n.kind, n.sig, n.n_args, n.field_tp, n.field_flag = self.kind, self.sig, len(self.args), self.tp, self.flag
        n.i64, n.f64, n.collation = self.i64, self.f64, self.collation
        if self.kind in (ffi.RPN_CONST_BYTES, ffi.RPN_CONST_DECIMAL):
            buf = C.create_string_buffer(bytes(self.data), max(1, len(self.data)))
            if keep is not None:
                keep.append(buf)
            else:
                self._buf = buf
            n.i64, n.n_args = C.addressof(buf), len(self.data)
        out.append(n)
        return out

    @property
    def ekind(self):
        return eval_kind(self.tp)


COLLATION_BINARY, COLLATION_UTF8MB4_BIN = 63, -46  # tipb FieldType.collate as TiDB sends it (field_type.rs:130-146)


def col(offset, tp=ffi.TP_LONGLONG, unsigned=False, collation=0):
    return Expr(ffi.RPN_COLUMN_REF, tp, ffi.FLAG_UNSIGNED if unsigned else 0, i64=offset, collation=collation)


def const_bytes(b, collation=COLLATION_BINARY, tp=ffi.TP_VARCHAR):
    """Bytes / String constant (tipb ExprType::Bytes / String)."""
    return Expr(ffi.RPN_CONST_BYTES, tp, 0, collation=collation, data=bytes(b))


def const_decimal(payload):
    """DECIMAL constant (tipb ExprType::MysqlDecimal); `payload` = precision byte, fraction byte, MySQL binary decimal."""
    return Expr(ffi.RPN_CONST_DECIMAL, ffi.TP_NEWDECIMAL, 0, data=bytes(payload))


def like(target, pattern, escape=92, collation=COLLATION_BINARY):
    """target LIKE pattern ESCAPE chr(escape) (impl_like.rs); `collation` is the LikeSig node's own."""
    e = fn("LIKE", target, pattern, const_int(escape))
    e.collation = collation
    return e


def const_int(v):
    return Expr(ffi.RPN_CONST_INT, ffi.TP_LONGLONG, 0, i64=int(v))


def const_uint(v):
    v = int(v)
    return Expr(ffi.RPN_CONST_UINT, ffi.TP_LONGLONG, ffi.FLAG_UNSIGNED, i64=v - (1 << 64) if v >= (1 << 63) else v)


def const_real(v):
    return Expr(ffi.RPN_CONST_REAL, ffi.TP_DOUBLE, 0, f64=float(v))


def const_time(packed, tp=ffi.TP_DATETIME):
    """DATE / DATETIME constant; `packed` = Time::to_packed_u64, what TiDB sends in ExprType::MysqlTime."""
    return Expr(ffi.RPN_CONST_TIME, tp, 0, i64=int(packed))


def const_duration(nanos):
    return Expr(ffi.RPN_CONST_DURATION, ffi.TP_DURATION, 0, i64=int(nanos))


def null(tp=ffi.TP_LONGLONG):
    return Expr(ffi.RPN_CONST_NULL, tp, 0)


def fn(sig_name, *args, ret_tp=ffi.TP_LONGLONG, unsigned=False):
    return Expr(ffi.RPN_FN, ret_tp, ffi.FLAG_UNSIGNED if unsigned else 0, sig=ffi.SIG[sig_name], args=args)


_SUFFIX = {"real": "REAL", "time": "TIME", "duration": "DURATION", "decimal": "DECIMAL"}


def _cmp(name, a, b):
    return fn(f"{name}_{_SUFFIX.get(a.ekind, 'INT')}", a, b)


def lt(a, b): return _cmp("LT", a, b)
def le(a, b): return _cmp("LE", a, b)
def gt(a, b): return _cmp("GT", a, b)
def ge(a, b): return _cmp("GE", a, b)
def eq(a, b): return _cmp("EQ", a, b)
def ne(a, b): return _cmp("NE", a, b)
def nulleq(a, b): return _cmp("NULLEQ", a, b)
def and_(a, b): return fn("LOGICAL_AND", a, b)
def or_(a, b): return fn("LOGICAL_OR", a, b)
def xor_(a, b): return fn("LOGICAL_XOR", a, b)
def not_(a): return fn("UNARY_NOT_REAL" if a.ekind == "real" else "UNARY_NOT_INT", a)
def in_(a, *values): return fn(f"IN_{_SUFFIX.get(a.ekind, 'INT')}", a, *values)
def is_null(a): return fn(f"{_SUFFIX.get(a.ekind, 'INT')}_IS_NULL", a)
def bit_and(a, b): return fn("BIT_AND", a, b, unsigned=True)   # MySQL bit operators return BIGINT UNSIGNED
def bit_or(a, b): return fn("BIT_OR", a, b, unsigned=True)
def bit_xor(a, b): return fn("BIT_XOR", a, b, unsigned=True)
def bit_neg(a): return fn("BIT_NEG", a, unsigned=True)
def cast_int_as_int(a, unsigned=False): return fn("CAST_INT_AS_INT", a, unsigned=unsigned)
def cast_int_as_real(a, unsigned=False): return fn("CAST_INT_AS_REAL", a, ret_tp=ffi.TP_DOUBLE, unsigned=unsigned)
def cast_real_as_real(a): return fn("CAST_REAL_AS_REAL", a, ret_tp=ffi.TP_DOUBLE)


def _arith(name, a, b):
    if a.ekind == "real":
        return fn(f"{name}_REAL", a, b, ret_tp=ffi.TP_DOUBLE)
    uns = bool((a.flag | b.flag) & ffi.FLAG_UNSIGNED)
    return fn(f"{name}_INT", a, b, ret_tp=ffi.TP_LONGLONG, unsigned=uns)


def plus(a, b): return _arith("PLUS", a, b)
def minus(a, b): return _arith("MINUS", a, b)
def multiply(a, b): return _arith("MULTIPLY", a, b)


def _uns(*xs):
    return any(x.flag & ffi.FLAG_UNSIGNED for x in xs)


def _typed(name, first, *args, unsigned=None):
    real = first.ekind == "real"
    return fn(f"{name}_REAL" if real else f"{name}_INT", *args, ret_tp=ffi.TP_DOUBLE if real else ffi.TP_LONGLONG,
              unsigned=(not real and _uns(first)) if unsigned is None else unsigned)


def divide(a, b): return fn("DIVIDE_REAL", a, b, ret_tp=ffi.TP_DOUBLE)                 # a / b over Real: x / 0 is NULL + warning 1365
def int_divide(a, b): return fn("INT_DIVIDE_INT", a, b, unsigned=_uns(a, b))      # a DIV b
def mod(a, b): return fn("MOD_REAL", a, b, ret_tp=ffi.TP_DOUBLE) if a.ekind == "real" else fn("MOD_INT", a, b, unsigned=_uns(a))
def neg(a): return _typed("UNARY_MINUS", a, a, unsigned=False)
def abs_(a): return fn("ABS_REAL", a, ret_tp=ffi.TP_DOUBLE) if a.ekind == "real" else fn("ABS_UINT" if _uns(a) else "ABS_INT", a, unsigned=_uns(a))
def if_null(a, b): return _typed("IF_NULL", a, a, b, unsigned=_uns(a, b) if a.ekind != "real" else False)
def if_(cond, a, b): return _typed("IF", a, cond, a, b, unsigned=_uns(a, b) if a.ekind != "real" else False)
def coalesce(*xs): return _typed("COALESCE", xs[0], *xs, unsigned=_uns(*xs) if xs[0].ekind != "real" else False)


def case_when(*xs):
    """case_when(cond1, value1, cond2, value2, ..., [else_value])"""
    return _typed("CASE_WHEN", xs[1] if len(xs) > 1 else xs[0], *xs, unsigned=False)


class ColumnDef:
    def __init__(self, col_id, tp=ffi.TP_LONGLONG, unsigned=False, not_null=False, pk_handle=False, default=None, decimal=0):
        self.col_id, self.tp, self.pk_handle, self.default, self.decimal = col_id, tp, pk_handle, default, decimal
        self.flag = (ffi.FLAG_UNSIGNED if unsigned else 0) | (ffi.FLAG_NOT_NULL if not_null else 0)


class Plan:
    """Owns every ctypes object referenced by `self.c` (a b2_dag_plan)."""

    def __init__(self):
        self._keep = []
        self._execs = []
        self.c = None
        self.columns = []

    def _expr(self, e):
        nodes = e.rpn(keep=self._keep)
        arr = (ffi.RpnNode * len(nodes))(*nodes)
        self._keep.append(arr)
        x = ffi.RpnExpr()
        x.nodes, x.n_nodes = arr, len(nodes)
        return x

    def table_scan(self, table_id, columns, desc=False):
        self.columns = list(columns)
        arr = (ffi.ColumnInfo * len(columns))()
        for i, cd in enumerate(columns):
            arr[i].col_id, arr[i].tp, arr[i].flag, arr[i].pk_handle = cd.col_id, cd.tp, cd.flag, int(cd.pk_handle)
            arr[i].decimal = cd.decimal
            if cd.default is not None:
                buf = C.create_string_buffer(bytes(cd.default), len(cd.default))
                self._keep.append(buf)
                arr[i].default_val = C.cast(buf, C.c_char_p)
                arr[i].default_len = len(cd.default)
        self._keep.append(arr)
        e = ffi.ExecutorDesc()
        e.tp, e.desc, e.table_id, e.columns, e.n_columns = ffi.EXEC_TABLE_SCAN, int(desc), table_id, arr, len(columns)
        self._execs.append(e)
        return self

    def index_scan(self, table_id, columns, desc=False):
        """BatchIndexScanExecutor: `columns` are the index columns in index order, then optionally the PK handle
        (pk_handle=True), then optionally the physical table id column (col_id -3).  Oracle only so far: the device path
        answers B2_ERR_UNSUPPORTED."""
        self.table_scan(table_id, columns, desc)
        self._execs[-1].tp = ffi.EXEC_INDEX_SCAN
        return self

    def selection(self, *conds):
        arr = (ffi.RpnExpr * len(conds))(*[self._expr(c) for c in conds])
        self._keep.append(arr)
        e = ffi.ExecutorDesc()
        e.tp, e.conditions, e.n_conditions = ffi.EXEC_SELECTION, arr, len(conds)
        self._execs.append(e)
        return self

    def projection(self, *exprs):
        """BatchProjectionExecutor: the output columns become the values of `exprs` (carried in `conditions`)."""
        arr = (ffi.RpnExpr * len(exprs))(*[self._expr(c) for c in exprs])
        self._keep.append(arr)
        e = ffi.ExecutorDesc()
        e.tp, e.conditions, e.n_conditions = ffi.EXEC_PROJECTION, arr, len(exprs)
        self._execs.append(e)
        return self

    def aggregation(self, aggs, group_by=()):
        """aggs: list of (kind, Expr) with kind in {'count','sum','avg','min','max','first','bit_and','bit_or','bit_xor'}."""
        kinds = {"count": ffi.AGG_COUNT, "sum": ffi.AGG_SUM, "avg": ffi.AGG_AVG, "min": ffi.AGG_MIN, "max": ffi.AGG_MAX,
                 "first": ffi.AGG_FIRST, "bit_and": ffi.AGG_BIT_AND, "bit_or": ffi.AGG_BIT_OR, "bit_xor": ffi.AGG_BIT_XOR}
        a = (ffi.AggrDesc * len(aggs))()
        for i, (k, ex) in enumerate(aggs):
            a[i].kind = kinds[k]
            a[i].arg = self._expr(ex)
        g = (ffi.RpnExpr * max(1, len(group_by)))(*[self._expr(x) for x in group_by])
        self._keep += [a, g]
        e = ffi.ExecutorDesc()
        e.tp, e.aggrs, e.n_aggrs, e.group_by, e.n_group_by = ffi.EXEC_AGGREGATION, a, len(aggs), g, len(group_by)
        self._execs.append(e)
        return self

    def limit(self, n):
        e = ffi.ExecutorDesc()
        e.tp, e.limit = ffi.EXEC_LIMIT, int(n)
        self._execs.append(e)
        return self

    def topn(self, order_by, limit):
        """order_by: list of (Expr, desc)."""
        o = (ffi.OrderBy * len(order_by))()
        for i, (ex, desc) in enumerate(order_by):
            o[i].expr = self._expr(ex)
            o[i].desc = int(desc)
        self._keep.append(o)
        e = ffi.ExecutorDesc()
        e.tp, e.order_by, e.n_order_by, e.limit = ffi.EXEC_TOPN, o, len(order_by), limit
        self._execs.append(e)
        return self

    def build(self, output_offsets=None):
        arr = (ffi.ExecutorDesc * len(self._execs))(*self._execs)
        self._keep.append(arr)
        p = ffi.DagPlan()
        p.executors, p.n_executors = arr, len(self._execs)
        if output_offsets is not None:
            oo = (C.c_uint32 * len(output_offsets))(*output_offsets)
            self._keep.append(oo)
            p.output_offsets, p.n_output_offsets = oo, len(output_offsets)
        self.c = p
        return self


def key_ranges(ranges):
    """ranges: list of (start_bytes, end_bytes) raw keys -> (ctypes array, keepalive)."""
    arr = (ffi.KeyRange * len(ranges))()
    keep = []
    for i, (s, e) in enumerate(ranges):
        s, e = bytes(s), bytes(e)
        keep += [s, e]
        arr[i].start, arr[i].start_len, arr[i].end, arr[i].end_len = s, len(s), e, len(e)
    return arr, keep
