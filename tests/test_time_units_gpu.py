"""timestamp[s|us|ns], time32[s] and time64[us|ns] columns on the GPU (DESIGN.md §2, §3.2).

- Unit twins: the same Projector and Filter trees run over seeded data in one unit and over the same
  instants in a finer one; boolean / integer / date results are equal, timestamp results scale by the
  factor, SelectionVectors are identical.  The millisecond kernels are oracle-checked elsewhere.
- Arbitrary and extreme ticks: extraction, truncation, castDATE, castVARCHAR, unit casts, parsing and
  to_timestamp against numpy datetime64, pyarrow.compute and Python integers.
- pyarrow's `test_in_expr_todo` timestamp and time cases at pyarrow's default units.
- A Q6-shaped range Filter over nullable timestamp[us] / [ns] columns: host, device-resident and
  Arrow C Device batches."""
import ctypes as C
import datetime

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import devmem

pytestmark = pytest.mark.gpu

TPS = {"s": 1, "ms": 1000, "us": 10 ** 6, "ns": 10 ** 9}
TT = {"s": pa.time32("s"), "ms": pa.time32("ms"), "us": pa.time64("us"), "ns": pa.time64("ns")}
N = 3_001 if devmem.EMU else 50_021
I64, I32, B = pa.int64(), pa.int32(), pa.bool_()
INT64_MIN, INT64_MAX = -2 ** 63, 2 ** 63 - 1


def _wrap(x):
    x &= (1 << 64) - 1
    return x - (1 << 64) if x >= 1 << 63 else x


def _twin_batch(unit, seed=0, n=N):
    """Columns t, u (instants within +-70 years of 1970 in `unit`, 10 % nulls) and n (small counts)."""
    rng = np.random.default_rng(seed)
    span = 70 * 365 * 86400 * TPS[unit]
    t = rng.integers(-span, span, n)
    u = np.where(rng.random(n) < 0.2, t + rng.integers(-40 * 86400, 40 * 86400, n) * TPS[unit], rng.integers(-span, span, n))
    cnt = rng.integers(-1000, 1000, n).astype(np.int32)
    mt, mu = rng.random(n) < 0.1, rng.random(n) < 0.1
    return t, u, cnt, mt, mu


def _batch(unit, t, u, cnt, mt, mu):
    ts = pa.timestamp(unit)
    return pa.RecordBatch.from_arrays([pa.array(t, ts, mask=mt), pa.array(u, ts, mask=mu), pa.array(cnt, I32)],
                                      names=["t", "u", "n"])


def _exprs(b, schema, unit):
    """(name, node, result type) of every tree the twin test runs at `unit`."""
    ts, tt = pa.timestamp(unit), TT[unit]
    t, u, n = (b.make_field(schema.field(x)) for x in ("t", "u", "n"))
    out = []
    for f in ("extractYear", "extractMonth", "extractDay", "extractHour", "extractMinute", "extractSecond",
              "extractDoy", "extractDow", "extractQuarter", "extractWeek", "extractDecade", "extractCentury",
              "extractMillennium", "extractEpoch"):
        out.append((f, b.make_function(f, [t], I64), I64))
    for f in ("Second", "Minute", "Hour", "Day", "Week", "Month", "Quarter", "Year", "Decade", "Century"):
        out.append(("date_trunc_" + f, b.make_function("date_trunc_" + f, [t], ts), ts))
    for f in ("Second", "Minute", "Hour", "Day", "Week", "Month", "Quarter", "Year"):
        out.append(("timestampadd" + f, b.make_function("timestampadd" + f, [n, t], ts), ts))
        out.append(("timestampdiff" + f, b.make_function("timestampdiff" + f, [t, u], I32), I32))
    out += [("add_months", b.make_function("add_months", [t, n], ts), ts),
            ("date_add", b.make_function("date_add", [t, n], ts), ts),
            ("date_sub", b.make_function("date_sub", [t, n], ts), ts),
            ("months_between", b.make_function("months_between", [t, u], pa.float64()), pa.float64()),
            ("datediff", b.make_function("datediff", [t, u], I32), I32),
            ("castDATE", b.make_function("castDATE", [t], pa.date64()), pa.date64()),
            ("last_day", b.make_function("last_day", [t], pa.date64()), pa.date64()),
            ("castTIME", b.make_function("castTIME", [t], tt), tt),
            ("hour(castTIME)", b.make_function("extractHour", [b.make_function("castTIME", [t], tt)], I64), I64),
            ("second(castTIME)", b.make_function("extractSecond", [b.make_function("castTIME", [t], tt)], I64), I64),
            ("less_than", b.make_function("less_than", [t, u], B), B),
            ("equal", b.make_function("equal", [t, u], B), B),
            ("is_distinct_from", b.make_function("is_distinct_from", [t, u], B), B),
            ("isnull", b.make_function("isnull", [t], B), B),
            ("nvl", b.make_function("nvl", [t, u], ts), ts),
            ("if", b.make_if(b.make_function("less_than", [t, u], B), t, u, ts), ts)]
    return out


def _ints(a):
    """(values as Python-comparable int64 / float64 numpy, validity) of an engine result."""
    valid = np.asarray(a.is_valid().to_numpy(zero_copy_only=False), dtype=bool)
    if pa.types.is_boolean(a.type) or pa.types.is_floating(a.type):
        vals = a.fill_null(False if pa.types.is_boolean(a.type) else 0.0).to_numpy(zero_copy_only=False)
    else:
        vals = a.view(I64 if a.type.bit_width == 64 else I32).fill_null(0).to_numpy(zero_copy_only=False).astype(np.int64)
    return vals, valid


@pytest.mark.parametrize("coarse,fine", [("ms", "us"), ("ms", "ns"), ("s", "ms")])
def test_unit_twins(gandiva, coarse, fine):
    factor = TPS[fine] // TPS[coarse]
    t, u, cnt, mt, mu = _twin_batch(coarse, seed=factor)
    bc = _batch(coarse, t, u, cnt, mt, mu)
    bf = _batch(fine, t * factor, u * factor, cnt, mt, mu)
    b = gandiva.TreeExprBuilder()
    ec, ef = _exprs(b, bc.schema, coarse), _exprs(b, bf.schema, fine)
    pc_ = gandiva.make_projector(bc.schema, [b.make_expression(x, pa.field("o%d" % i, rt)) for i, (_, x, rt) in enumerate(ec)], None)
    pf = gandiva.make_projector(bf.schema, [b.make_expression(x, pa.field("o%d" % i, rt)) for i, (_, x, rt) in enumerate(ef)], None)
    rc, rf = pc_.evaluate(bc), pf.evaluate(bf)
    for (name, _, rt), gc, gf in zip(ec, rc, rf):
        assert gf.type == ef[[e[0] for e in ef].index(name)][2]
        vc, okc = _ints(gc)
        vf, okf = _ints(gf)
        assert np.array_equal(okc, okf), name
        scale = factor if (pa.types.is_timestamp(rt) or pa.types.is_time(rt)) else 1
        if pa.types.is_floating(rt):
            assert np.array_equal(vc[okc].view(np.int64), vf[okf].view(np.int64)), name
        else:
            assert np.array_equal(vc[okc] * scale, vf[okf]), name
    # Filters: comparisons, IN and a Kleene OR give the same rows
    sels = []
    for unit, batch, f in ((coarse, bc, 1), (fine, bf, factor)):
        ts = pa.timestamp(unit)
        tf, uf = b.make_field(batch.schema.field("t")), b.make_field(batch.schema.field("u"))
        lo, hi = int(t[5]) * f, int(t[7]) * f
        cond = b.make_or([
            b.make_and([b.make_function("greater_than_or_equal_to", [tf, b.make_literal(min(lo, hi), ts)], B),
                        b.make_function("less_than", [tf, b.make_literal(max(lo, hi), ts)], B)]),
            b.make_in_expression(uf, [int(x) * f for x in u[:50:3]], ts),
            b.make_function("equal", [b.make_function("extractDow", [tf], I64), b.make_literal(3, I64)], B)])
        sels.append(gandiva.make_filter(batch.schema, b.make_condition(cond)).evaluate(batch).to_array().to_numpy())
    assert len(sels[0]) > 0 and np.array_equal(sels[0], sels[1])


def _extreme_ticks(seed, n=4_000):
    rng = np.random.default_rng(seed)
    v = rng.integers(INT64_MIN + 1, INT64_MAX, n, dtype=np.int64, endpoint=True)
    small = rng.integers(-10 ** 15, 10 ** 15, n // 4)
    return np.concatenate([np.array([INT64_MIN + 1, INT64_MAX, 0, -1, 1], np.int64), v, small.astype(np.int64)])


def _project1(gandiva, arr, name, rt, extra=()):
    b = gandiva.TreeExprBuilder()
    batch = pa.RecordBatch.from_arrays([arr], names=["t"])
    node = b.make_function(name, [b.make_field(batch.schema.field("t"))] + list(extra), rt)
    return gandiva.make_projector(batch.schema, [b.make_expression(node, pa.field("o", rt))], None).evaluate(batch)[0]


@pytest.mark.parametrize("unit", ["s", "ms", "us", "ns"])
def test_calendar_at_extreme_ticks(gandiva, unit):
    ticks = _extreme_ticks(TPS[unit])
    arr = pa.array(ticks, pa.timestamp(unit))
    tpd = 86400 * TPS[unit]
    days = np.array([int(x) // tpd for x in ticks], dtype=np.int64)   # Python floor division
    tod = np.array([int(x) - (int(x) // tpd) * tpd for x in ticks], dtype=np.int64)
    d = days.astype("M8[D]")
    month = d.astype("M8[M]")
    want = {"extractYear": d.astype("M8[Y]").astype(np.int64) + 1970,
            "extractMonth": month.astype(np.int64) % 12 + 1,
            "extractDay": (d - month.astype("M8[D]")).astype(np.int64) + 1,
            "extractHour": tod // (3600 * TPS[unit]),
            "extractMinute": tod // (60 * TPS[unit]) % 60,
            "extractSecond": tod // TPS[unit] % 60}
    for name, w in want.items():
        got = _project1(gandiva, arr, name, I64).to_numpy()
        assert np.array_equal(got, w), name
    got = _project1(gandiva, arr, "date_trunc_Day", pa.timestamp(unit)).cast(I64).to_numpy()
    assert got.tolist() == [_wrap(int(x) * tpd) for x in days]
    got = _project1(gandiva, arr, "castDATE", pa.date64()).cast(I64).to_numpy()
    assert got.tolist() == [_wrap(int(x) * 86400000) for x in days]
    got = _project1(gandiva, arr, "castTIME", TT[unit])
    got = got.view(pa.int32() if got.type.bit_width == 32 else I64).to_numpy().astype(np.int64)
    assert np.array_equal(got, tod)
    # within pyarrow's range (years 1..9999): castVARCHAR spells what pc.cast spells
    lo, hi = -62135596800 * TPS[unit], 253402300799 * TPS[unit]
    inr = ticks[(ticks >= lo) & (ticks <= hi)]
    a = pa.array(inr, pa.timestamp(unit))
    got = _project1(gandiva, a, "castVARCHAR", pa.string(), [gandiva.TreeExprBuilder().make_literal(40, I64)])
    assert got.to_pylist() == pc.cast(a, pa.string()).to_pylist()


@pytest.mark.parametrize("src", ["s", "ms", "us", "ns"])
def test_unit_casts(gandiva, src):
    ticks = _extreme_ticks(7 + TPS[src])
    arr = pa.array(ticks, pa.timestamp(src))
    for dst in ("s", "ms", "us", "ns"):
        if dst == src:
            continue
        got = _project1(gandiva, arr, "castTIMESTAMP", pa.timestamp(dst)).cast(I64).to_numpy()
        if TPS[dst] > TPS[src]:
            want = [_wrap(int(x) * (TPS[dst] // TPS[src])) for x in ticks]
        else:
            want = [int(x) // (TPS[src] // TPS[dst]) for x in ticks]   # floor, as numpy's astype
            small = np.abs(ticks) < 10 ** 15
            assert np.array_equal(ticks[small].astype("M8[%s]" % src).astype("M8[%s]" % dst).astype(np.int64),
                                  np.array(want)[small])
        assert got.tolist() == want, dst
    # int64 and date64 sources
    got = _project1(gandiva, pa.array(ticks, I64), "castTIMESTAMP", pa.timestamp(src)).cast(I64).to_numpy()
    assert np.array_equal(got, ticks)
    ms = ticks // 1000
    got = _project1(gandiva, pa.array(ms, pa.date64()), "castTIMESTAMP", pa.timestamp(src)).cast(I64).to_numpy()
    want = [_wrap(int(x) * TPS[src] // 1000) if TPS[src] >= 1000 else int(x) // 1000 for x in ms]
    assert got.tolist() == want


@pytest.mark.parametrize("unit", ["s", "ms", "us", "ns"])
def test_parse_and_to_timestamp(gandiva, unit):
    rng = np.random.default_rng(TPS[unit] % 97)
    texts, want = [], []
    for i in range(600):
        secs = int(rng.integers(-2 * 10 ** 9, 4 * 10 ** 9))
        nd = i % 10
        frac = "".join(str(int(x)) for x in rng.integers(0, 10, nd))
        dt = datetime.datetime(1970, 1, 1) + datetime.timedelta(seconds=secs)
        texts.append(dt.strftime("%Y-%m-%d %H:%M:%S") + ("." + frac if nd else ""))
        sub = int((frac + "0" * 9)[:9]) if nd else 0
        want.append(secs * TPS[unit] + sub * TPS[unit] // 10 ** 9)
    got = _project1(gandiva, pa.array(texts), "castTIMESTAMP", pa.timestamp(unit)).cast(I64).to_pylist()
    assert got == want
    secs = rng.integers(-2 * 10 ** 9, 4 * 10 ** 9, 500)
    got = _project1(gandiva, pa.array(secs, I64), "to_timestamp", pa.timestamp(unit)).cast(I64).to_numpy()
    assert got.tolist() == [int(s) * TPS[unit] for s in secs]
    fs = secs / 7.0
    got = _project1(gandiva, pa.array(fs, pa.float64()), "to_timestamp", pa.timestamp(unit)).cast(I64).to_numpy()
    assert got.tolist() == [int(np.trunc(x * TPS[unit])) for x in fs]
    got = _project1(gandiva, pa.array(secs, I64), "to_time", TT[unit])
    got = got.view(pa.int32() if got.type.bit_width == 32 else I64).to_numpy().astype(np.int64)
    assert got.tolist() == [(int(s) * TPS[unit]) % (86400 * TPS[unit]) for s in secs]


def test_in_expr_todo_at_pyarrow_default_units(gandiva):
    """The timestamp and time cases of pyarrow's test_in_expr_todo (skipped there upstream)."""
    utc = datetime.timezone.utc
    d1 = datetime.datetime.fromtimestamp(1542238951.621877, utc).replace(tzinfo=None)
    d2 = datetime.datetime.fromtimestamp(1542238911.621877, utc).replace(tzinfo=None)
    d3 = datetime.datetime.fromtimestamp(1542238051.621877, utc).replace(tzinfo=None)
    for values, t in (([d1, d2, d3], pa.timestamp("us")), ([d1.time(), d2.time(), d3.time()], pa.time64("us"))):
        arr = pa.array(values)
        assert arr.type == t
        table = pa.Table.from_arrays([arr], ["a"])
        b = gandiva.TreeExprBuilder()
        node_a = b.make_field(table.schema.field("a"))
        cond = b.make_in_expression(node_a, [values[1]], t)
        f = gandiva.make_filter(table.schema, b.make_condition(cond))
        result = f.evaluate(table.to_batches()[0], pa.default_memory_pool())
        assert result.to_array().to_pylist() == [1]


def _q6_batch(unit, n, seed=11):
    rng = np.random.default_rng(seed)
    ms = rng.integers(694224000000, 915148800000, n)   # 1992 .. 1998 in ms
    x = rng.integers(0, 50, n).astype(np.int32)
    mask = rng.random(n) < 0.01
    f = TPS[unit] // 1000
    return pa.RecordBatch.from_arrays([pa.array(ms * f, pa.timestamp(unit), mask=mask), pa.array(x, I32)],
                                      names=["ts", "x"])


def _q6_filter(gandiva, schema, unit):
    b = gandiva.TreeExprBuilder()
    ts, x = b.make_field(schema.field("ts")), b.make_field(schema.field("x"))
    f = TPS[unit] // 1000
    lo, hi = 757382400000 * f, 788918400000 * f   # [1994-01-01, 1995-01-01)
    cond = b.make_and([b.make_function("greater_than_or_equal_to", [ts, b.make_literal(lo, pa.timestamp(unit))], B),
                       b.make_function("less_than", [ts, b.make_literal(hi, pa.timestamp(unit))], B),
                       b.make_function("less_than", [x, b.make_literal(24, I32)], B)])
    return gandiva.make_filter(schema, b.make_condition(cond))


def _to_device(keep, buf):
    d = devmem.DevBuf(max(buf.size, 1) + 64, np.uint8, fill=0)
    devmem.synchronize()
    import gandiva_b200
    gandiva_b200.memcpy_htod(0, d.ptr, np.frombuffer(buf, dtype=np.uint8).copy())
    keep.append(d)
    return d.ptr


def test_range_filter(gandiva):
    n = 20_011 if devmem.EMU else 4_000_037
    base = _q6_batch("ms", n)
    fms = _q6_filter(gandiva, base.schema, "ms")
    want = fms.evaluate(base).to_array().to_numpy()
    assert 0 < len(want) < n
    for unit in ("us", "ns"):
        batch = _q6_batch(unit, n)
        f = _q6_filter(gandiva, batch.schema, unit)
        got = f.evaluate(batch).to_array().to_numpy()
        assert np.array_equal(got, want), unit
        assert f.kernel_info["gated_stages"] == fms.kernel_info["gated_stages"]
        # device-resident batch
        keep = []
        cols = []
        for c in batch.columns:
            bb = c.buffers()
            cols.append((_to_device(keep, bb[0]) if bb[0] is not None and c.null_count else 0, _to_device(keep, bb[1]), 0, c.offset))
        sel = devmem.DevBuf(n + 8, np.uint32, fill=0)
        devmem.synchronize()
        cnt = f.evaluate_device(n, cols, sel.ptr, n, "UINT32", devmem.stream(), sync=True)
        assert np.array_equal(sel.numpy()[:cnt], want), unit
        # Arrow C Device path: a filter, and a projector whose timestamp result is exported in the unit
        imported = gandiva.ArrowDeviceBatch.from_record_batch(batch)
        res = f.evaluate_arrow(imported, "UINT32")
        st = gandiva.ArrowSchemaC()
        pa.uint32()._export_to_c(C.addressof(st))
        got = pa.Array._import_from_c_device(res.address, C.addressof(st))
        assert np.array_equal(got.to_numpy().astype(np.int64), want)
        b = gandiva.TreeExprBuilder()
        node = b.make_function("date_trunc_Day", [b.make_field(batch.schema.field("ts"))], pa.timestamp(unit))
        p = gandiva.make_projector(batch.schema, [b.make_expression(node, pa.field("d", pa.timestamp(unit)))], None)
        out = p.evaluate_arrow(imported)
        assert out.schema.children[0].contents.format == (b"tsn:" if unit == "ns" else b"tsu:")
        rb = out.to_record_batch()
        assert rb.schema.field("d").type == pa.timestamp(unit)
        assert rb.column(0).equals(p.evaluate(batch)[0])
        imported.release()
