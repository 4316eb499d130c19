import pathlib
import sys

import pytest

ROOT = pathlib.Path(__file__).resolve().parent.parent
for p in (str(ROOT), str(ROOT / "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on the H100 with -m gpu)")
    config.addinivalue_line("markers", "ref: needs oracle/_ref (the compiled reference; built where the reference sources exist)")


def pytest_collection_modifyitems(config, items):
    import oracle_lib
    oracle_lib.build()
    if not oracle_lib.have_ref():
        skip = pytest.mark.skip(reason="oracle/_ref/libsela_ref.so not built (no reference sources here)")
        for it in items:
            if "ref" in it.keywords:
                it.add_marker(skip)
