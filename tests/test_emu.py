"""CPU-side execution of the GPU parity suite under the functional SIMT simulator (tests/emu).

The unmodified product stack (ctypes mirror -> C-ABI -> runtime -> CUDA driver calls -> the
kernels the fuser generates) runs in a SUBPROCESS whose LD_LIBRARY_PATH puts tests/emu/lib's
stand-in libcuda.so.1 / libnvrtc.so.12 in front of the real ones; the generated CUDA source is
compiled for the host against tests/emu/gdv_emu.h and every CUDA thread is a fiber.  The simulator
is test infrastructure only: it checks kernel *logic* (tails, validity windows, ballots, scans,
look-back, staging protocols, function semantics) against the oracle without a GPU; the `-m gpu`
run of the very same test functions on the H100 stays the parity gate.

Every `gpu`-marked test runs (about a minute on 8 cores, compiled kernels are cached under
/tmp/gdv_emu_cache_<uid>, outside the tree); GDV_EMU_SELECT=<pytest -k expression> narrows it while developing."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

def _run(select, timeout):
    import emu
    env = emu.env()
    cmd = [sys.executable, "-m", "pytest", os.path.join(ROOT, "tests"), "-m", "gpu", "-q", "-x",
           "-p", "no:cacheprovider", "-n", str(min(8, os.cpu_count() or 1))]
    if select:
        cmd += ["-k", select]
    return subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=timeout)


def test_gpu_suite_under_simulator():
    res = _run(os.environ.get("GDV_EMU_SELECT"), 3000)
    tail = res.stdout[-4000:] + res.stderr[-2000:]
    assert res.returncode == 0, tail
    assert " passed" in res.stdout, tail


def test_simulator_is_not_reachable_from_the_product():
    """Nothing under gandiva_b200/ or include/ names the simulator (the only seam is the
    GDV_HOST_EMU guard around the inline-PTX primitives of the device sources)."""
    hits = []
    for base in ("gandiva_b200", "include"):
        for dirpath, _, files in os.walk(os.path.join(ROOT, base)):
            for f in files:
                if f.endswith((".so", ".pyc", ".o")):
                    continue
                text = open(os.path.join(dirpath, f), errors="replace").read()
                if "tests/emu" in text and "gdv_emu.h" not in text:
                    hits.append(os.path.join(dirpath, f))
                if "gdv_emu_" in text or "GDV_EMU_" in text:
                    hits.append(os.path.join(dirpath, f))
    assert hits == [], hits
