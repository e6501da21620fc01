import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


# Kernels compiled before (here, without a GPU: NVRTC needs none) are loaded instead of recompiled:
# tools/populate_cubin_cache.py fills this in-tree directory, which travels to the GPU box with
# the snapshot like the built .so files (*.cubin is git-ignored).
_CUBIN_CACHE = os.path.join(ROOT, "gandiva_b200", "_cubin_cache")
if (not os.path.isdir(_CUBIN_CACHE) and os.path.exists(_CUBIN_CACHE + ".tar.xz") and os.environ.get("GDV_EMU") != "1"
        and os.environ.get("PYTEST_XDIST_WORKER") is None and os.path.exists("/dev/nvidiactl")):   # only where a GPU is
    import tarfile
    try:   # the packed form tools/populate_cubin_cache.py --pack leaves (a few seconds to unpack)
        with tarfile.open(_CUBIN_CACHE + ".tar.xz") as _tar:
            _tar.extractall(os.path.dirname(_CUBIN_CACHE), filter="data")
    except Exception as _e:   # a broken archive only costs the compilations
        print("cubin cache archive not usable: %s" % _e)
if os.path.isdir(_CUBIN_CACHE) and os.environ.get("GDV_EMU") != "1":
    os.environ.setdefault("GDV_CUBIN_CACHE_DIR", _CUBIN_CACHE)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")
    # build the native libraries once per session if they are missing (in-tree .so files
    # normally travel with the snapshot)
    import importlib.util
    spec = importlib.util.spec_from_file_location(
        "gdv_build", os.path.join(ROOT, "gandiva_b200", "build.py"))
    _build = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(_build)
    if not (os.path.exists(_build.LIB) and os.path.exists(_build.ORACLE_LIB)):
        _build.build_all()


@pytest.fixture(scope="session")
def gandiva():
    import gandiva_b200
    return gandiva_b200


@pytest.fixture(scope="session")
def oracle():
    import oracle as _oracle
    return _oracle


def pytest_collection_modifyitems(config, items):
    """A kernel that never finishes must fail its test, not hang the GPU box until the runner's own
    limit: every gpu-marked test gets a generous pytest-timeout (thread method: the process exits,
    the driver tears the context down)."""
    if not config.pluginmanager.hasplugin("timeout"):
        return
    for item in items:
        if item.get_closest_marker("gpu") is not None and item.get_closest_marker("timeout") is None:
            item.add_marker(pytest.mark.timeout(900, method="thread"))
