import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100)")


def pytest_collection_modifyitems(config, items):
    """`pytest tests` on a host without a CUDA device skips the gpu-marked tests instead of failing them."""
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:       # noqa: BLE001
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device visible (gpu-marked tests need an H100)")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def lib_built():
    from sonata_b200 import _native, build
    if not os.path.exists(_native.LIB_PATH):
        build.build()
    return _native.lib()


@pytest.fixture(scope="session")
def voice_paths(lib_built):
    from sonata_b200 import voicegen
    d = voicegen.default_voice_dir()
    return {q: voicegen.write_voice(d, q) for q in ("medium", "high")}


@pytest.fixture(scope="session")
def oracle_weights():
    from oracle import vits_oracle as vo
    from sonata_b200 import voicegen
    cache = {}

    def get(q):
        if q not in cache:
            cache[q] = vo.to_torch(voicegen.make_tensors(q))
        return cache[q]
    return get
