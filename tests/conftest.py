import os
import sys
from pathlib import Path

import numpy as np
import pytest

REPO = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(REPO))
sys.path.insert(0, str(REPO / "oracle"))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def _cuda_devices() -> int:
    try:
        import ctypes
        rt = ctypes.CDLL("libcudart.so")
        n = ctypes.c_int(0)
        return n.value if rt.cudaGetDeviceCount(ctypes.byref(n)) == 0 else 0
    except OSError:
        try:
            import torch
            return torch.cuda.device_count()
        except Exception:
            return 0


def pytest_collection_modifyitems(config, items):
    """Plain `pytest tests` on a CPU-only machine: the gpu-marked tests are SKIPPED (there is no CPU fallback to run them
    on), so the suite is green without `-m "not gpu"`.  On a GPU box nothing is skipped."""
    if any(item.get_closest_marker("gpu") for item in items) and _cuda_devices() == 0:
        skip = pytest.mark.skip(reason="no CUDA device: flowgger_b200 has no CPU fallback")
        for item in items:
            if item.get_closest_marker("gpu"):
                item.add_marker(skip)


@pytest.fixture(scope="session")
def oracle():
    import pyoracle
    pyoracle.build()
    return pyoracle


@pytest.fixture(scope="session")
def native():
    import flowgger_b200
    from flowgger_b200 import build as fb_build
    fb_build.build_all()
    return flowgger_b200


def first_diff(gpu_buf, gpu_offs, ora_buf, ora_offs, data, offsets, limit=5):
    """Indices + text of the first lines whose canonical dumps differ."""
    n = len(gpu_offs) - 1
    glen = np.diff(gpu_offs)
    olen = np.diff(ora_offs)
    out = []
    # cheap path: find the first position where cumulative offsets or bytes diverge
    for i in range(n):
        g = gpu_buf[gpu_offs[i]:gpu_offs[i + 1]]
        o = ora_buf[ora_offs[i]:ora_offs[i + 1]]
        if g != o:
            line = bytes(data[offsets[i]:offsets[i + 1]])
            out.append((i, line, g, o))
            if len(out) >= limit:
                break
    return out


def assert_parity(dec, oracle_mod, fmt, data, offsets, cfg=None, resident=False):
    """GPU (through the C ABI) vs oracle on the same lines: canonical dumps must be byte-identical."""
    if resident:
        dec.upload(data, offsets)
        dec.parse_resident()
        res = dec.download()
    else:
        res = dec.decode(data, offsets)
    gbuf, goffs = dec.dump(res, data, offsets, nthreads=os.cpu_count() or 4)
    obuf, ooffs = oracle_mod.decode_dump(fmt, data, offsets, cfg, nthreads=os.cpu_count() or 4)
    if gbuf == obuf and np.array_equal(goffs, ooffs):
        return res
    diffs = first_diff(gbuf, goffs, obuf, ooffs, data, offsets)
    msg = "\n".join(f"line {i}: {line!r}\n   gpu: {g!r}\n   ref: {o!r}" for i, line, g, o in diffs)
    raise AssertionError(f"{len(diffs)}+ lines differ from the oracle:\n{msg}")
