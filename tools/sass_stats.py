"""Static SASS facts of the kernels the bench configs use (no GPU needed: NVRTC + cuobjdump):
registers, stack, SASS instruction count and the mnemonics that show how data moves (UBLKCP = TMA
bulk copy, SYNCS = mbarrier, LDGSTS = cp.async, LDG.E.128 / .64, VOTE / SHFL / BAR).
  python tools/sass_stats.py > sass_stats.md"""
import collections
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    dump = tempfile.mkdtemp(prefix="gdv_sass_")
    os.environ["GDV_DUMP_DIR"] = dump
    os.environ["GDV_EAGER_NONULL"] = "1"
    import pyarrow as pa
    import cases
    import gandiva_b200 as g
    b = g.TreeExprBuilder()
    made = []

    def note(label, obj):
        made.append((label, obj.kernel_info["name"]))
    note("config 2: Q6 filter, 256 threads x 4 chunks per warp (what batches >= 32 M rows get)", g.make_filter(
        cases.Q6_SCHEMA, b.make_condition(cases.q6_condition(b)), g.Configuration(block_threads=256, stages=4)))
    note("config 2: Q6 filter, 256 threads x 1 chunk (small batches)", g.make_filter(
        cases.Q6_SCHEMA, b.make_condition(cases.q6_condition(b)), g.Configuration(block_threads=256, stages=1)))
    exprs = [b.make_expression(r, pa.field("o%d" % i, t)) for i, (r, t) in enumerate(cases.q1_outputs(b))]
    note("config 3: Q1 projector, TMA loader", g.make_projector(cases.Q1_SCHEMA, exprs, None, "NONE", g.Configuration(loader=2)))
    note("config 4: string filter, key-driven (256 threads)", g.make_filter(
        cases.COMMENT_SCHEMA, b.make_condition(cases.comment_condition(b))))
    note("config 4: string filter, row-driven cooperative scan (512 threads)", g.make_filter(
        cases.COMMENT_SCHEMA, b.make_condition(cases.comment_condition(b)), g.Configuration(block_threads=512, string_scan=4)))
    schema, outs, _ = cases.case_arith("add", pa.int32())(b)
    note("config 1: add(int32, int32) projector", g.make_projector(schema, [b.make_expression(outs[0][0], pa.field("c", pa.int32()))], None))
    labels = dict((name, label) for label, name in made)
    print("| kernel (nullable / no-null variant) | regs | stack | SASS instr | data movement mnemonics |")
    print("|---|---|---|---|---|")
    for f in sorted(os.listdir(dump)):
        if not f.endswith(".cubin"):
            continue
        name = f[:-6]
        src = open(os.path.join(dump, name + ".cu")).readline()
        variant = "no-null" if "no input has nulls" in src else "nullable"
        res = subprocess.run(["cuobjdump", "-res-usage", os.path.join(dump, f)], capture_output=True, text=True).stdout
        regs = re.search(r"REG:(\d+)", res).group(1)
        stack = re.search(r"STACK:(\d+)", res).group(1)
        sass = subprocess.run(["cuobjdump", "-sass", os.path.join(dump, f)], capture_output=True, text=True).stdout
        ops = collections.Counter()
        n = 0
        for line in sass.splitlines():
            m = re.match(r"\s+/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\d\s+)?([A-Z0-9_.]+)", line)
            if not m:
                continue
            n += 1
            op = m.group(1)
            for key in ("UBLKCP", "SYNCS", "LDGSTS", "LDG.E.EF.128", "LDG.E.128", "LDG.E.EF.64", "LDG.E.EF", "LDS", "STG", "VOTE", "SHFL", "BAR"):
                if op.startswith(key):
                    ops[key] += 1
                    break
        label = labels.get(name, "(lazily built variant)")
        # the eager no-null variant has another name: label by kernel kind
        if name not in labels:
            label = "variant of: " + ("filter" if "filter" in name else "projector")
        print("| %s, %s `%s` | %s | %s | %d | %s |" % (label, variant, name[-8:], regs, stack, n,
                                                     ", ".join("%s x%d" % kv for kv in sorted(ops.items()))))


if __name__ == "__main__":
    main()
