"""Fill gandiva_b200/_cubin_cache with sm_90a cubins of kernels the `-m gpu` suite makes, on a box
WITHOUT a GPU.  NVRTC needs no device: the suite is simply run here with GDV_CUBIN_CACHE_DIR set and
GDV_EAGER_NONULL=1 (the no-null variants are built at Make() too); every Make() compiles with the
real NVRTC and lands in the cache, every test then fails at its first Evaluate (no driver), which is
expected and ignored.  The GPU box finds the cubins through GDV_CUBIN_CACHE_DIR (tests/conftest.py)
and skips those compilations; kernels that are only built at Evaluate (other index widths, the
large-batch variants) are still compiled there.  Entries are keyed by the full generated source, the device library text
and options, so a stale entry can never be picked up.

`--pack` stores the result as gandiva_b200/_cubin_cache.tar.xz (about 27 MB instead of 170 MB; git-ignored
like every built artefact, shipped with the snapshot) and removes the directory; tests/conftest.py
unpacks the archive on the box when the directory is missing."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    cache = os.path.join(ROOT, "gandiva_b200", "_cubin_cache")
    os.makedirs(cache, exist_ok=True)
    env = dict(os.environ, GDV_CUBIN_CACHE_DIR=cache, GDV_EAGER_NONULL="1")
    env.pop("GDV_EMU", None)
    before = len([f for f in os.listdir(cache) if f.endswith(".cubin")])
    subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests"), "-m", "gpu", "-q", "-p", "no:cacheprovider",
                    "-n", str(min(8, os.cpu_count() or 1))], env=env, cwd=ROOT,
                   stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    after = [f for f in os.listdir(cache) if f.endswith(".cubin")]
    size = sum(os.path.getsize(os.path.join(cache, f)) for f in after)
    print("cubin cache: %d -> %d entries, %.1f MB" % (before, len(after), size / 1e6))
    if "--pack" in sys.argv[1:]:
        import shutil
        import tarfile
        archive = cache + ".tar.xz"
        with tarfile.open(archive, "w:xz", preset=3) as tar:
            tar.add(cache, arcname="_cubin_cache")
        shutil.rmtree(cache)
        print("packed into %s (%.1f MB)" % (archive, os.path.getsize(archive) / 1e6))


if __name__ == "__main__":
    main()
