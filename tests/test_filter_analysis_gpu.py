"""Differential tests of the Filter's Make()-time analyses (DESIGN.md §3.3, §3.6, §3.7): random conditions
compared bit for bit with the CPU oracle, chosen so that a wrong analysis drops or adds rows.

1. Truth-context null analysis (BodyGen::TruthStrict): Kleene trees over nullable fixed-width columns with
   their own null rates, some without a validity buffer.  A column the analysis lists has its validity
   ANDed into the keep-mask after the row loop, so listing one too many drops rows.  Every tree runs on
   the default kernel and on the row-driven kernel.
2. Dictionary-first decision (DictionaryFirstColumn): random conditions over one dictionary column,
   rooted at a strict predicate so both decisions occur, against the oracle over the decoded column and
   against the general row kernel.
3. Gated loads (PlanGate / EmitGatedGroup): random AND spines over every fixed-width type, led by a range
   over a clustered column so that whole groups die, whole groups survive and boundary groups are mixed;
   gated == ungated == oracle.
4. The random trees of test_random_trees.py over dictionary and string_view / binary_view columns.

Seeds are fixed and every failure message names its seed.  Runs on the H100 (`-m gpu`) and, through
tests/test_emu.py, under the functional simulator."""
import decimal

import numpy as np
import pyarrow as pa
import pytest

import devmem
from helpers import assert_arrays_match
from test_dictionary_gpu import decoded, dict_column
from test_random_trees import SCHEMA as TREE_SCHEMA, TYPES as TREE_TYPES, TreeGen, _batch as tree_batch
from test_string_view_gpu import views

pytestmark = pytest.mark.gpu

B, S, BIN = pa.bool_(), pa.string(), pa.binary()
I8, I16, I32, I64 = pa.int8(), pa.int16(), pa.int32(), pa.int64()
U8, U16, U32, U64 = pa.uint8(), pa.uint16(), pa.uint32(), pa.uint64()
F32, F64 = pa.float32(), pa.float64()
D32, D64, TS, T32 = pa.date32(), pa.date64(), pa.timestamp("ms"), pa.time32("ms")
DEC12, DEC38 = pa.decimal128(12, 2), pa.decimal128(38, 10)
RELOPS = ["equal", "not_equal", "less_than", "less_than_or_equal_to", "greater_than", "greater_than_or_equal_to"]
BIG = 30_001 if devmem.EMU else 70_001


def _indices(f, batch, dtype="int32"):
    return f.evaluate(batch, None, dtype).to_array().to_numpy().astype(np.uint64)


def _expect(got, want, what):
    if not np.array_equal(got, want):
        extra = np.setdiff1d(got, want)[:5]
        missing = np.setdiff1d(want, got)[:5]
        raise AssertionError("%s: %d rows selected, oracle %d; extra %s, missing %s" % (
            what, len(got), len(want), extra, missing))


def _always_true(b, s):
    return b.make_or([b.make_function("isnull", [s], B), b.make_function("isnotnull", [s], B)])


def _strip_validity(col):
    """The column with its validity buffer removed: every slot reads as valid, whatever it holds."""
    return pa.Array.from_buffers(col.type, len(col), [None] + col.buffers()[1:], offset=col.offset)


# ---- 1. truth-context null analysis ---------------------------------------------------------------
NULL_RATES = [0.0, 0.05, 0.5, 1.0]
KLEENE_COLS = [("a", I32), ("b", I64), ("c", F64), ("e", D32), ("g", I16), ("h", F32)]
KLEENE_SCHEMA = pa.schema(KLEENE_COLS + [("s", S)])


def _kleene_column(t, n, rng, rate):
    if t in (F32, F64):
        vals = np.round(rng.standard_normal(n) * 12, 1).astype(t.to_pandas_dtype())
        arr = pa.array(vals, type=t, mask=rng.random(n) < rate if rate else None)
    else:
        vals = rng.integers(-20, 21, n)
        it = pa.int32() if t == D32 else t
        arr = pa.array(vals.astype(it.to_pandas_dtype()), type=it, mask=rng.random(n) < rate if rate else None)
        arr = arr.cast(t) if t == D32 else arr
    return arr


def kleene_batch(n, seed, rates, stripped, offset):
    """Columns of KLEENE_SCHEMA with per-column null rates; the columns in `stripped` carry no validity
    buffer (so their null slots read as valid values)."""
    rng = np.random.default_rng(seed)
    cols = []
    for (name, t), rate in zip(KLEENE_COLS, rates):
        col = _kleene_column(t, n + offset, rng, rate)
        if name in stripped:
            col = _strip_validity(col)
        cols.append(col.slice(offset))
    words = np.array(["x", "yy", "", "zzz"], dtype=object)[rng.integers(0, 4, n + offset)]
    cols.append(pa.array(list(words), S, mask=rng.random(n + offset) < 0.1).slice(offset))
    return pa.RecordBatch.from_arrays(cols, schema=KLEENE_SCHEMA)


class KleeneGen:
    """Boolean trees in truth position over the columns `cols` (names of KLEENE_COLS)."""

    def __init__(self, b, rng, cols):
        self.b, self.rng, self.cols = b, rng, cols
        self.types = dict(KLEENE_COLS)

    def lit(self, t):
        v = int(self.rng.integers(-15, 16))
        if self.rng.random() < 0.04:
            return self.b.make_literal(None, t)
        return self.b.make_literal(float(v) + (0.5 if t in (F32, F64) else 0), t) if t in (F32, F64) else \
            self.b.make_literal(v, t)

    def col(self, name=None):
        name = name or self.cols[int(self.rng.integers(len(self.cols)))]
        t = self.types[name]
        return self.b.make_field(pa.field(name, t)), t

    def leaf(self, name=None):
        b, rng = self.b, self.rng
        x, t = self.col(name)
        r = rng.random()
        op = RELOPS[int(rng.integers(len(RELOPS)))]
        if r < 0.55:
            return b.make_function(op, [x, self.lit(t)], B)
        if r < 0.65 and t in (I32, I64, F64):
            return b.make_function(op, [b.make_function("add", [x, self.lit(t)], t), self.lit(t)], B)
        if r < 0.72 and t in (I32, I64):
            return b.make_in_expression(x, [int(v) for v in rng.integers(-15, 16, 3)], t)
        if r < 0.80:   # nvl in value position: a null x is replaced, so x is not strict here
            return b.make_function(op, [b.make_function("nvl", [x, self.lit(t)], t), self.lit(t)], B)
        if r < 0.87:
            return b.make_function("is_distinct_from" if rng.random() < 0.5 else "is_not_distinct_from", [x, self.lit(t)], B)
        if r < 0.94:
            return b.make_function("isnull" if rng.random() < 0.5 else "isnotnull", [x], B)
        y, u = self.col()
        if u != t:
            return b.make_function(op, [x, self.lit(t)], B)
        return b.make_function(op, [x, y], B)

    def tree(self, depth):
        b, rng = self.b, self.rng
        r = rng.random()
        if depth <= 0 or r < 0.25:
            return self.leaf()
        if r < 0.55:
            kids = [self.tree(depth - 1) for _ in range(int(rng.integers(2, 6)))]
            return b.make_and(kids) if rng.random() < 0.5 else b.make_or(kids)
        if r < 0.63:
            return b.make_function("not", [self.tree(depth - 1)], B)
        if r < 0.71:
            return b.make_if(self.tree(depth - 1), self.tree(depth - 1), self.tree(depth - 1), B)
        if r < 0.82:
            fn = ["istrue", "isfalse", "isnottrue", "isnotfalse"][int(rng.integers(4))]
            return b.make_function(fn, [self.tree(depth - 1)], B)
        if r < 0.90:
            return b.make_function("nvl", [self.tree(depth - 1), b.make_literal(bool(rng.random() < 0.5), B)], B)
        return self.leaf()

    def wide_or(self, depth):
        """An OR of three to five children over different columns: the shape whose strict set is the
        intersection of its children's."""
        names = list(self.rng.permutation(self.cols))[: int(self.rng.integers(3, 6))]
        kids = [self.leaf(n) if self.rng.random() < 0.7 else self.tree(depth - 1) for n in names]
        return self.b.make_or(kids)

    def root(self):
        r = self.rng.random()
        depth = int(self.rng.integers(1, 4))
        if r < 0.4:
            return self.wide_or(depth)
        if r < 0.7:
            kids = [self.tree(depth), self.wide_or(depth)]
            return self.b.make_and(kids if self.rng.random() < 0.5 else kids[::-1])
        return self.tree(depth + 1)


def _kleene_sizes(seed):
    return (1 if seed % 2 else 33, 4099) + ((BIG,) if seed % 3 == 0 else ())


@pytest.mark.parametrize("seed", range(60))
def test_truth_context_null_analysis(seed, gandiva, oracle):
    rng = np.random.default_rng(71_000 + seed)
    ncols = int(rng.integers(3, 7))
    cols = [n for n, _ in KLEENE_COLS[:ncols]]
    b = gandiva.TreeExprBuilder()
    cond = KleeneGen(b, rng, cols).root()
    s = b.make_field(pa.field("s", S))
    row_cond = b.make_and([cond, _always_true(b, s)])   # a string conjunct: the row-driven kernel
    default = gandiva.make_filter(KLEENE_SCHEMA, b.make_condition(cond))
    row = gandiva.make_filter(KLEENE_SCHEMA, b.make_condition(row_cond), gandiva.Configuration(string_scan=4))
    rates = [NULL_RATES[int(rng.integers(4))] for _ in KLEENE_COLS]
    stripped = {n for n in cols if rng.random() < 0.2} if seed % 4 == 1 else set()
    for n in _kleene_sizes(seed):
        offset = int(rng.integers(0, 40))
        batch = kleene_batch(n, seed * 7 + n, rates, stripped, offset)
        want = oracle.filter_indices(cond, batch, threads=2)
        what = "seed %d n=%d offset=%d rates=%s stripped=%s: %s" % (seed, n, offset, rates, sorted(stripped), cond)
        _expect(_indices(default, batch), want, "default kernel, " + what)
        _expect(_indices(row, batch), want, "row-driven kernel, " + what)


@pytest.mark.parametrize("n", [33, 4099])
def test_wide_or_is_not_strict_in_a_column_one_child_reads(n, gandiva, oracle):
    """or(a < 1, b < 2, c < 3) keeps a row whose b is null when a < 1 holds: b's validity must not be
    ANDed into the keep-mask (an OR is strict only in the columns every child is strict in)."""
    schema = pa.schema([("a", I32), ("b", I32), ("c", I32), ("s", S)])
    rng = np.random.default_rng(n)
    a = rng.integers(-3, 4, n).astype(np.int32)
    bnull = rng.random(n) < 0.5
    bnull[0] = True
    a[0] = -2   # row 0: a < 1 is true, b is null
    batch = pa.RecordBatch.from_arrays(
        [pa.array(a), pa.array(rng.integers(-3, 4, n).astype(np.int32), mask=bnull),
         pa.array(rng.integers(-3, 6, n).astype(np.int32)), pa.array(["x"] * n, S)], schema=schema)
    b = gandiva.TreeExprBuilder()
    f = lambda name: b.make_field(schema.field(name))
    cond = b.make_or([b.make_function("less_than", [f(name), b.make_literal(v, I32)], B)
                      for name, v in (("a", 1), ("b", 2), ("c", 3))])
    want = oracle.filter_indices(cond, batch)
    assert 0 in want
    assert np.count_nonzero(bnull[want.astype(np.int64)]) > 0
    default = gandiva.make_filter(schema, b.make_condition(cond))
    row = gandiva.make_filter(schema, b.make_condition(b.make_and([cond, _always_true(b, f("s"))])),
                              gandiva.Configuration(string_scan=4))
    _expect(_indices(default, batch), want, "default kernel, n=%d" % n)
    _expect(_indices(row, batch), want, "row-driven kernel, n=%d" % n)


# ---- 2. dictionary-first decision -----------------------------------------------------------------
LIKE_PATTERNS = ["%AI%", "M%", "%L", "_A%", "%", "", "SHIP", "%ö%", "REG%AIR", "%BRASS"]
WORD_LITS = ["MAIL", "SHIP", "AIR", "", "FOB", "héllo wörld", "RAIL", "ZZZ"]


class DictGen:
    """Conditions over the one column `d` (utf8 or binary values)."""

    def __init__(self, b, rng, d, vt):
        self.b, self.rng, self.d, self.vt = b, rng, d, vt

    def word(self):
        w = str(self.rng.choice(WORD_LITS))
        return w if self.vt == S else w.encode()

    def strict(self):
        """A predicate that is null whenever d is."""
        b, rng, d, vt = self.b, self.rng, self.d, self.vt
        kinds = ["equal", "in", "relop"] + (["like", "starts_with", "in_upper", "substr"] if vt == S else [])
        k = kinds[int(rng.integers(len(kinds)))]
        if k == "equal":
            return b.make_function("equal" if rng.random() < 0.6 else "not_equal", [d, b.make_literal(self.word(), vt)], B)
        if k == "in":
            return b.make_in_expression(d, [self.word() for _ in range(int(rng.integers(1, 4)))], vt)
        if k == "relop":
            return b.make_function(RELOPS[int(rng.integers(2, 6))], [d, b.make_literal(self.word(), vt)], B)
        if k == "like":
            return b.make_function("like", [d, b.make_literal(str(rng.choice(LIKE_PATTERNS)), S)], B)
        if k == "starts_with":
            return b.make_function("starts_with", [d, b.make_literal(self.word()[:2], S)], B)
        if k == "in_upper":
            return b.make_in_expression(b.make_function("upper", [d], S), [self.word().upper() for _ in range(2)], S)
        sub = b.make_function("substr", [d, b.make_literal(1, I64), b.make_literal(3, I64)], S)
        return b.make_function("equal", [sub, b.make_literal(self.word()[:3], S)], B)

    def tree(self, depth):
        b, rng, d, vt = self.b, self.rng, self.d, self.vt
        r = rng.random()
        if depth <= 0 or r < 0.3:
            r2 = rng.random()
            if r2 < 0.6:
                return self.strict()
            if r2 < 0.75:
                return b.make_function("isnull" if rng.random() < 0.5 else "isnotnull", [d], B)
            if r2 < 0.88 and vt == S:   # null d reads as the replacement
                w = self.word()
                return b.make_function("equal", [b.make_function("nvl", [d, b.make_literal(w, S)], S), b.make_literal(w, S)], B)
            if vt == S:
                ln = b.make_function("char_length", [d], I32)
                return b.make_function("is_distinct_from", [ln, b.make_literal(int(rng.integers(0, 5)), I32)], B)
            return self.strict()
        if r < 0.6:
            kids = [self.tree(depth - 1) for _ in range(int(rng.integers(2, 4)))]
            return b.make_and(kids) if rng.random() < 0.5 else b.make_or(kids)
        if r < 0.7:
            return b.make_function("not", [self.tree(depth - 1)], B)
        if r < 0.8:
            return b.make_if(self.tree(depth - 1), self.tree(depth - 1), self.tree(depth - 1), B)
        if r < 0.9:
            fn = ["istrue", "isfalse", "isnottrue", "isnotfalse"][int(rng.integers(4))]
            return b.make_function(fn, [self.tree(depth - 1)], B)
        return b.make_function("nvl", [self.tree(depth - 1), b.make_literal(bool(rng.random() < 0.5), B)], B)

    def root(self):
        rng = self.rng
        depth = int(rng.integers(1, 4))
        if rng.random() < 0.65:
            kids = [self.strict(), self.tree(depth)]
            kids = kids if rng.random() < 0.5 else kids[::-1]
            return self.b.make_and(kids) if rng.random() < 0.5 else self.b.make_or(kids)
        return self.tree(depth)


INDEX_TYPES = [I8, I16, I32, I64]


def _dictionary_seed(gandiva, oracle, seed, col):
    """Makes both Filters of one random condition over `col` (all Make()s of a test come before its first
    evaluation, so a cache of compiled kernels covers them); returns the check, which evaluates both
    paths and returns the dictionary_first value."""
    batch = pa.RecordBatch.from_arrays([col, pa.array(["s%d" % (i % 7) for i in range(len(col))], S)], names=["d", "s"])
    plain = decoded(batch)
    vt = col.type.value_type
    conds = []
    for bt in (batch, plain):   # the same tree twice: over the dictionary field and over the decoded one
        b = gandiva.TreeExprBuilder()
        conds.append((b, DictGen(b, np.random.default_rng(81_000 + seed), b.make_field(bt.schema.field("d")), vt).root()))
    (b, cond), (_, want_cond) = conds
    want = oracle.filter_indices(want_cond, plain, threads=2)
    first = gandiva.make_filter(batch.schema, b.make_condition(cond))
    general = gandiva.make_filter(batch.schema, b.make_condition(
        b.make_and([cond, _always_true(b, b.make_field(batch.schema.field("s")))])))
    what = "seed %d n=%d %s: %s" % (seed, len(col), col.type, want_cond)

    def check():
        _expect(_indices(first, batch), want, "dictionary_first=%d, %s" % (first.kernel_info["dictionary_first"], what))
        _expect(_indices(general, batch), want, "general path, " + what)
        assert general.kernel_info["dictionary_first"] == 0, what
        return first.kernel_info["dictionary_first"]
    return check


@pytest.mark.parametrize("chunk", range(4))
def test_dictionary_first_decision(chunk, gandiva, oracle):
    """Eight seeds per chunk over every index width and both value types; each chunk must take both
    decisions in at least a quarter of its seeds, so neither path goes untested."""
    checks = []
    for seed in range(8 * chunk, 8 * chunk + 8):
        rng = np.random.default_rng(seed)
        vt = BIN if seed % 4 == 3 else S
        col = dict_column(int(rng.choice([777, 4099])), INDEX_TYPES[seed % 4], seed=seed, card=int(rng.integers(3, 13)),
                          idx_offset=int(rng.integers(0, 9)), dict_offset=int(rng.integers(0, 3)), value_type=vt)
        checks.append(_dictionary_seed(gandiva, oracle, seed, col))
    paths = [check() for check in checks]
    assert 2 <= sum(paths) <= 6, paths


@pytest.mark.parametrize("edge", ["empty_dictionary", "all_null_indices", "one_row"])
def test_dictionary_first_decision_edges(edge, gandiva, oracle):
    checks = []
    for seed in range(100, 106):
        col = {"empty_dictionary": lambda: dict_column(777, INDEX_TYPES[seed % 4], seed=seed, card=0),
               "all_null_indices": lambda: dict_column(1000, INDEX_TYPES[seed % 4], seed=seed, null_idx=1.0),
               "one_row": lambda: dict_column(1, INDEX_TYPES[seed % 4], seed=seed, null_idx=0.0)}[edge]()
        checks.append(_dictionary_seed(gandiva, oracle, seed, col))
    for check in checks:
        check()


# ---- 3. gated loads: random AND spines ------------------------------------------------------------
GATE_TYPES = [I8, I16, I32, I64, U8, U16, U32, U64, F32, F64, D32, D64, TS, T32, DEC12, DEC38]
GATE_CONFIGS = [{}, {"stages": 4}, {"rows_per_thread": 2, "block_threads": 128}, {"rows_per_thread": 8, "block_threads": 256}]
TREEGEN_TYPES = {I32, I64, F32, F64, D32, D64, TS, T32}


def _float_column(t, n, rng):
    ft = np.dtype(t.to_pandas_dtype())
    fi = np.finfo(ft)
    vals = (rng.standard_normal(n) * 50).astype(ft)
    special = np.array([np.nan, -np.nan, np.inf, -np.inf, 0.0, -0.0, fi.smallest_subnormal, -fi.smallest_subnormal,
                        fi.tiny, fi.max, -fi.max, 1.0], dtype=ft)
    pick = rng.random(n) < 0.06
    vals[pick] = special[rng.integers(0, len(special), int(pick.sum()))]
    return vals


def _int_column(npt, n, rng):
    info = np.iinfo(npt)
    lo, hi = max(int(info.min), -100), min(int(info.max), 100)
    vals = rng.integers(lo, hi + 1, n).astype(npt)
    edge = np.array([info.min, info.max, info.min + 1, info.max - 1, 0], dtype=npt)
    pick = rng.random(n) < 0.03
    vals[pick] = edge[rng.integers(0, len(edge), int(pick.sum()))]
    return vals


def _decimal_column(t, n, rng, mask):
    """decimal128 from its 16-byte two's-complement words: small values, the largest and smallest of
    the precision, and a few with a high word."""
    unscaled = [int(v) for v in rng.integers(-20000, 20001, n)]
    limit = 10 ** t.precision - 1
    for i in np.nonzero(rng.random(n) < 0.03)[0]:
        unscaled[i] = [limit, -limit, 10 ** (t.precision - 1), -(10 ** (t.precision - 1)), 0][int(rng.integers(5))]
    raw = b"".join((u & ((1 << 128) - 1)).to_bytes(16, "little") for u in unscaled)
    validity = pa.py_buffer(np.packbits(~mask, bitorder="little").tobytes()) if mask.any() else None
    return pa.Array.from_buffers(t, n, [validity, pa.py_buffer(raw)], null_count=int(mask.sum()))


def gate_column(t, n, rng, null_rate):
    mask = rng.random(n) < null_rate
    if pa.types.is_decimal128(t):
        return _decimal_column(t, n, rng, mask)
    if t in (F32, F64):
        return pa.array(_float_column(t, n, rng), type=t, mask=mask if null_rate else None)
    if t in (D32, T32):
        vals = rng.integers(0, 200, n).astype(np.int32) if t == D32 else rng.integers(0, 86_400_000, n).astype(np.int32)
        return pa.array(vals, pa.int32(), mask=mask if null_rate else None).cast(t)
    if t in (D64, TS):
        vals = rng.integers(0, 200, n).astype(np.int64) * 86_400_000
        if t == TS:
            vals += rng.integers(0, 86_400_000, n)
        return pa.array(vals, pa.int64(), mask=mask if null_rate else None).cast(t)
    return pa.array(_int_column(t.to_pandas_dtype(), n, rng), type=t, mask=mask if null_rate else None)


def gate_batch(schema, n, seed, null_rates):
    """`k` = row // 500 (int16, no nulls) followed by the random columns of `schema`."""
    rng = np.random.default_rng(seed)
    cols = [pa.array((np.arange(n) // 500).astype(np.int16), I16)]
    for f, rate in zip(list(schema)[1:], null_rates):
        cols.append(gate_column(f.type, n, rng, rate))
    return pa.RecordBatch.from_arrays(cols, schema=schema)


class GateGen:
    def __init__(self, gandiva, b, rng, schema, sample):
        self.b, self.rng, self.schema, self.sample = b, rng, schema, sample
        self.tree = TreeGen(gandiva, b, rng)
        # hash functions observe a NaN's bits, which differ between x86 and sm_90a (test_random_trees.py)
        self.tree.sigs = {t: [s for s in sigs if not s[0].startswith("hash")] for t, sigs in self.tree.sigs.items()}
        self.tree.fields = {}
        for f in list(schema)[1:]:
            if f.type in TREEGEN_TYPES:
                self.tree.fields.setdefault(f.type, []).append(f)

    def literal(self, f):
        """A value of the column (so comparisons select some rows), or an edge of its type."""
        vals = self.sample[f.name]
        t = f.type
        if len(vals) and self.rng.random() < 0.8:
            v = vals[int(self.rng.integers(len(vals)))]
        elif pa.types.is_decimal128(t):
            v = decimal.Decimal(0)
        elif t in (F32, F64):
            v = float(self.rng.choice([np.nan, np.inf, -np.inf, -0.0, 0.0]))
        else:
            v = 0
        if pa.types.is_decimal128(t):
            return self.b.make_literal(decimal.Decimal(v), t)
        if t in (F32, F64):
            return self.b.make_literal(float(v), t)
        return self.b.make_literal(int(v), t)

    def simple(self, f):
        """A predicate over column f (every type, decimal and unsigned included)."""
        b, rng, t = self.b, self.rng, f.type
        x = b.make_field(f)
        r = rng.random()
        same = [g for g in list(self.schema)[1:] if g.type == t and g.name != f.name]
        if r < (0.35 if same else 0.55):
            return b.make_function(RELOPS[int(rng.integers(len(RELOPS)))], [x, self.literal(f)], B)
        if r < 0.7:
            if same:   # a two-column conjunct
                y = b.make_field(same[int(rng.integers(len(same)))])
                return b.make_function(RELOPS[int(rng.integers(len(RELOPS)))], [x, y], B)
            return b.make_function(RELOPS[int(rng.integers(len(RELOPS)))], [self.literal(f), x], B)
        if r < 0.8:
            return b.make_and([b.make_function("greater_than_or_equal_to", [x, self.literal(f)], B),
                               b.make_function("less_than_or_equal_to", [x, self.literal(f)], B)])
        if r < 0.9 and not pa.types.is_decimal128(t):
            return b.make_function("is_distinct_from", [x, self.literal(f)], B)
        return b.make_function("isnotnull", [x], B)

    def conjunct(self, fields):
        f = fields[int(self.rng.integers(len(fields)))]
        if f.type in TREEGEN_TYPES and self.rng.random() < 0.4:
            return self.tree.gen(B, int(self.rng.integers(1, 3)))
        return self.simple(f)


def _gate_setup(gandiva, seed):
    rng = np.random.default_rng(91_000 + seed)
    types = [GATE_TYPES[int(i)] for i in rng.choice(len(GATE_TYPES), int(rng.integers(2, 6)), replace=False)]
    if rng.random() < 0.6:   # two columns of one type: conjuncts that compare them span two stages
        types.insert(int(rng.integers(1, len(types) + 1)), types[int(rng.integers(len(types)))])
    schema = pa.schema([("k", I16)] + [("c%d" % i, t) for i, t in enumerate(types)])
    null_rates = [float(rng.choice([0.0, 0.0, 0.02, 0.3])) for _ in types]
    n = BIG + int(rng.integers(0, 64))
    batch = gate_batch(schema, n, seed, null_rates)
    sample = {f.name: [v for v in batch.column(i).to_pylist()[:400] if v is not None] for i, f in enumerate(schema)}
    for f in schema:
        if pa.types.is_temporal(f.type):
            it = pa.int32() if f.type.bit_width == 32 else pa.int64()
            sample[f.name] = [v for v in batch.column(f.name).view(it).to_pylist()[:400] if v is not None]
    b = gandiva.TreeExprBuilder()
    gen = GateGen(gandiva, b, rng, schema, sample)
    k = b.make_field(schema.field("k"))
    groups = n // 500 + 1
    lo = int(rng.integers(0, groups))
    hi = lo + int(rng.integers(1, max(2, groups // 2)))
    conj = [b.make_and([b.make_function("greater_than_or_equal_to", [k, b.make_literal(lo, I16)], B),
                        b.make_function("less_than", [k, b.make_literal(hi, I16)], B)])]
    fields = list(schema)[1:]
    used = []
    for _ in range(int(rng.integers(1, 5))):
        pool = used if used and rng.random() < 0.3 else fields   # some conjuncts repeat an earlier column
        f = pool[int(rng.integers(len(pool)))]
        used.append(f)
        conj.append(gen.conjunct([f]))
    cond = b.make_and(conj)
    cfg = GATE_CONFIGS[seed % len(GATE_CONFIGS)]
    return b, schema, batch, cond, cfg


def _gate_seed(gandiva, oracle, seed):
    """Makes the gated / ungated pair of one seed; returns the check, which evaluates both on the whole
    batch, on a slice at an offset that is not a multiple of 32 and on a short tail, and returns the
    number of gated stages."""
    b, schema, batch, cond, cfg = _gate_setup(gandiva, seed)
    on = gandiva.make_filter(schema, b.make_condition(cond), gandiva.Configuration(filter_gating=0, **cfg))
    off = gandiva.make_filter(schema, b.make_condition(cond), gandiva.Configuration(filter_gating=1, **cfg))
    stages = on.kernel_info["gated_stages"]
    assert off.kernel_info["gated_stages"] == 0
    if stages == 0:
        assert on.llvm_ir == off.llvm_ir, "seed %d: a filter that does not gate must keep its kernel" % seed

    def check():
        n = batch.num_rows
        off_ = 1 + (seed * 13) % 31   # never a multiple of 32
        for part, dtypes in ((batch, ("int32",)), (batch.slice(off_, min(n - off_, 30_000)), ("int16", "int64")),
                             (batch.slice(7, 1 + seed % 97), ("int32",))):
            want = oracle.filter_indices(cond, part, threads=2)
            what = "seed %d cfg=%s stages=%d n=%d offset=%d: %s" % (seed, cfg, stages, part.num_rows,
                                                                  part.column(0).offset, cond)
            for dtype in dtypes:
                _expect(_indices(on, part, dtype), want, "gated %s, %s" % (dtype, what))
                _expect(_indices(off, part, dtype), want, "ungated %s, %s" % (dtype, what))
        return stages
    return check


@pytest.mark.parametrize("chunk", range(6))
def test_gated_loads_random_spines(chunk, gandiva, oracle):
    """Ten seeds per chunk: gated == ungated == oracle.  Most seeds must gate (the range over `k` reads
    2 bytes of the row) and some with three stages or more, so the dense load of all-alive groups runs."""
    checks = [_gate_seed(gandiva, oracle, seed) for seed in range(10 * chunk, 10 * chunk + 10)]
    stages = [check() for check in checks]
    assert sum(s > 0 for s in stages) >= 6, stages
    assert max(stages) >= 3, stages


# ---- 4. the random trees over encoded string columns ----------------------------------------------
def _encode_dictionary(col, rng):
    """`col` as a dictionary: a random index width, unused entries, a null entry that some null rows
    point at (the others have a null index), a sliced dictionary and sliced indices."""
    vals = col.to_pylist()
    binary = pa.types.is_binary(col.type)
    mk = (lambda s: s.encode()) if binary else (lambda s: s)
    uniq = sorted({v for v in vals if v is not None})
    entries = uniq + [mk("unused %d" % i) for i in range(int(rng.integers(0, 4)))] + [None]
    entries = [entries[int(i)] for i in rng.permutation(len(entries))]
    junk = int(rng.integers(0, 3))
    dictionary = pa.array([mk("junk")] * junk + entries, type=col.type).slice(junk)
    pos = {v: i for i, v in enumerate(entries) if v is not None}
    null_entry = entries.index(None)
    idx = np.array([pos[v] if v is not None else null_entry for v in vals], dtype=np.int64)
    null_idx = np.array([v is None and rng.random() < 0.5 for v in vals], dtype=bool)
    widths = [I16, I32, I64] + ([I8] if len(entries) < 128 else [])
    it = widths[int(rng.integers(len(widths)))]
    lead = int(rng.integers(0, 5))
    indices = pa.array(np.concatenate([np.zeros(lead, np.int64), idx]).astype(it.to_pandas_dtype()), type=it,
                       mask=np.concatenate([np.zeros(lead, bool), null_idx]))
    return pa.DictionaryArray.from_arrays(indices, dictionary).slice(lead)


def _encoded(batch, seed):
    """The batch with s, u and z each a dictionary or a string_view / binary_view column."""
    rng = np.random.default_rng(seed)
    cols, fields = [], []
    for f, col in zip(batch.schema, batch.columns):
        if f.name in ("s", "u", "z"):
            if rng.random() < 0.5:
                col = _encode_dictionary(col, rng)
            else:
                col, twin = views(col.to_pylist(), nbuf=int(rng.integers(1, 4)), seed=seed, binary=f.name == "z")
                assert twin.equals(batch.column(f.name))
        cols.append(col)
        fields.append(pa.field(f.name, col.type))
    return pa.RecordBatch.from_arrays(cols, schema=pa.schema(fields))


def _encoded_gen(gandiva, b, seed, schema):
    g = TreeGen(gandiva, b, np.random.default_rng(seed))
    g.fields = {}
    for f in TREE_SCHEMA:
        g.fields.setdefault(f.type, []).append(schema.field(f.name))   # keyed by the plain type
    return g


def _encodings(batch):
    return [(f.name, str(f.type)) for f in batch.schema if f.name in ("s", "u", "z")]


@pytest.mark.parametrize("seed", range(12))
def test_random_projector_trees_over_encoded_strings(seed, gandiva, oracle):
    b = gandiva.TreeExprBuilder()
    rng = np.random.default_rng(2000 + seed)
    out_types = [TREE_TYPES[int(rng.integers(len(TREE_TYPES)))] for _ in range(int(rng.integers(1, 4)))]
    depth = int(rng.integers(2, 5))
    g = _encoded_gen(gandiva, b, 3000 + seed, TREE_SCHEMA)
    roots = [g.gen(t, depth) for t in out_types]
    runs = []
    for n in (1, 1000 + seed, 4099):   # each size encodes the columns differently: one Projector each
        plain = tree_batch(n, seed + n)
        enc = _encoded(plain, 17 * seed + n)
        g = _encoded_gen(gandiva, b, 3000 + seed, enc.schema)
        enc_roots = [g.gen(t, depth) for t in out_types]
        runs.append((n, plain, enc, gandiva.make_projector(enc.schema, [b.make_expression(r, pa.field("o%d" % i, t))
                                                                        for i, (r, t) in enumerate(zip(enc_roots, out_types))], None)))
    for n, plain, enc, p in runs:
        got = p.evaluate(enc)
        want = oracle.project(roots, out_types, plain, threads=2)
        for i, (gv, wv) in enumerate(zip(got, want)):
            assert_arrays_match(gv, wv, "seed %d n=%d %s out %d: %s" % (seed, n, _encodings(enc), i, roots[i]))


@pytest.mark.parametrize("seed", range(12))
def test_random_filter_trees_over_encoded_strings(seed, gandiva, oracle):
    b = gandiva.TreeExprBuilder()
    depth = int(np.random.default_rng(6000 + seed).integers(2, 5))
    scans = (0, 8) if seed % 3 == 0 else (0,)   # every third seed: the view shortcut off too
    cond = _encoded_gen(gandiva, b, 7000 + seed, TREE_SCHEMA).gen(B, depth)
    runs = []
    for n in (1, 2000 + seed, 9001):
        plain = tree_batch(n, seed + n)
        enc = _encoded(plain, 19 * seed + n)
        enc_cond = _encoded_gen(gandiva, b, 7000 + seed, enc.schema).gen(B, depth)
        for scan in scans:
            runs.append((n, scan, plain, enc, gandiva.make_filter(enc.schema, b.make_condition(enc_cond),
                                                                  gandiva.Configuration(string_scan=scan))))
    for n, scan, plain, enc, f in runs:
        want = oracle.filter_indices(cond, plain, threads=2)
        _expect(_indices(f, enc), want, "seed %d n=%d string_scan=%d %s: %s" % (seed, n, scan, _encodings(enc), cond))
