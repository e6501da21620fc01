"""DRAM traffic of the gated fixed-width Filter, counted on the CPU from the synthetic lineitem columns
(the oracle's generator: the same rows bench.py generates on the device for a seed).

    python tools/filter_sectors.py [--workload q6] [--rows 16777216] [--seed 42]

For a condition's stage plan (the columns each stage loads and the conjuncts it ANDs in, as the kernel
plans them: columns by first appearance on the AND spine, each conjunct in the stage of its last column)
it prints the rows every stage keeps and, for each gated column and DRAM fetch granularity of 32 / 64 /
128 B, the fraction of the column's segments that hold at least one row alive when it is loaded.  The
bytes per row follow: the first stage's columns in full, every gated column times its touched fraction,
plus 4 B per selected row (the UINT32 SelectionVector).  Dividing a measured kernel time by the ungated
kernel's bytes/s (tools/gated_filter_bench.py) gives the effective bytes per row the GPU moved; the table
shows which fetch granularity that corresponds to.

The stage plans below restate, in numpy, what the kernel's planner (PlanGate) makes of each workload's
condition (the conditions of tools/gated_filter_bench.py); the tool checks the stage count against the
compiled kernel's `gated_stages` and says so where the engine does not gate the condition at all."""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import oracle  # noqa: E402

# (column kind of oracle.generate_lineitem, name, dtype)
COLS = {"ship": (0, "l_shipdate", np.int32), "disc": (1, "l_discount", np.float64), "qty": (2, "l_quantity", np.float64)}


def plans():
    """Per workload: stages as (columns loaded, predicate over the loaded columns)."""
    ship_q6 = lambda c: (c["ship"] >= 8766) & (c["ship"] < 9131)  # noqa: E731
    disc = lambda c: (c["disc"] >= 0.05) & (c["disc"] <= 0.07)    # noqa: E731
    qty = lambda c: c["qty"] < 24.0                                 # noqa: E731
    return {
        "q6": [(["ship"], ship_q6), (["disc"], disc), (["qty"], qty)],
        "dense_first": [(["ship"], lambda c: (c["ship"] >= 8035) & (c["ship"] < 10562)), (["disc"], disc), (["qty"], qty)],
        "reversed": [(["qty"], qty), (["disc"], disc), (["ship"], ship_q6)],
        "two_column": [(["disc", "qty"], lambda c: c["disc"] * 100.0 < c["qty"]), (["ship"], ship_q6)],
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="q6", choices=sorted(plans()))
    ap.add_argument("--rows", type=int, default=16 << 20)
    ap.add_argument("--seed", type=int, default=42)
    a = ap.parse_args()
    n = a.rows
    cols = {}
    for key, (kind, _, dt) in COLS.items():
        vals, _ = oracle.generate_lineitem(kind, a.seed, 0, n, 0, threads=os.cpu_count() or 1)
        cols[key] = np.frombuffer(vals, dt, count=n)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import cases
    import gandiva_b200 as gandiva
    from gated_filter_bench import condition
    tb = gandiva.TreeExprBuilder()
    engine = gandiva.make_filter(cases.Q6_SCHEMA, tb.make_condition(condition(tb, a.workload))).kernel_info["gated_stages"]
    if engine == 0:
        print("the engine does not gate this condition (kernel attribute gated_stages = 0); the table shows what gating would move")
    else:
        assert engine == len(plans()[a.workload]), (engine, len(plans()[a.workload]))
    grains = (32, 64, 128)
    alive = np.ones(n, dtype=bool)
    dense = 0.0
    gated = {g: 0.0 for g in grains}
    print("workload %s, %d rows, seed %d" % (a.workload, n, a.seed))
    print("| stage | columns | rows alive when loaded | %s | rows kept after the stage |" %
          " | ".join("%d B segments touched" % g for g in grains))
    print("|---|---|---|%s---|" % ("---|" * len(grains)))
    for s, (names, pred) in enumerate(plans()[a.workload]):
        touched = []
        for g in grains:
            if s == 0:
                touched.append(1.0)
                continue
            frac = 0.0
            for name in names:
                w = np.dtype(COLS[name][2]).itemsize
                seg = np.zeros((n * w + g - 1) // g, dtype=bool)
                seg[(np.flatnonzero(alive) * w) // g] = True
                frac += seg.mean() * w
                gated[g] += seg.mean() * w
            touched.append(frac / sum(np.dtype(COLS[x][2]).itemsize for x in names))
        if s == 0:
            dense = float(sum(np.dtype(COLS[x][2]).itemsize for x in names))
        was = alive.mean()
        alive = alive & pred(cols)
        print("| %d | %s | %.2f %% | %s | %.3f %% |" % (s, ", ".join(COLS[x][1] for x in names), 100 * was,
                                                     " | ".join("%.1f %%" % (100 * t) for t in touched), 100 * alive.mean()))
    sel = alive.mean()
    ungated = sum(np.dtype(c[2]).itemsize for c in COLS.values()) + 4 * sel
    print()
    print("| DRAM fetch granularity | bytes/row | vs ungated %.2f |" % ungated)
    print("|---|---|---|")
    for g in grains:
        bpr = dense + gated[g] + 4 * sel
        print("| %d B | %.2f | %.2fx |" % (g, bpr, ungated / bpr))


if __name__ == "__main__":
    main()
