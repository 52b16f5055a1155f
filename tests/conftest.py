import gzip
import os
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100: run with -m gpu)")


@pytest.fixture(scope="session", autouse=True)
def _built():
    """CPU-side artefacts (oracle, host-sim, product .so) are built once per session; idempotent."""
    import __graft_entry__ as g
    g.build()
    yield


XML_GOLDEN = ROOT / "tests" / "golden" / "xml"


@pytest.fixture(scope="session")
def reference_resources(tmp_path_factory):
    """The reference's test resources (zstd-jni src/test/resources) the tests decode, rebuilt from the reduced copy in
    tests/golden/xml (tests/golden/make_golden_xml.py): the plaintext unpacked, the concatenated streams made as the
    reference's regenerate.sh makes them."""
    d = tmp_path_factory.mktemp("resources")
    (d / "xml").write_bytes(gzip.decompress((XML_GOLDEN / "xml.gz").read_bytes()))
    for f in XML_GOLDEN.iterdir():
        if f.name != "xml.gz":
            (d / f.name).write_bytes(f.read_bytes())
    for name in ("xml-1", "xml-1-sized"):
        (d / f"{name}x2.zst").write_bytes((d / f"{name}.zst").read_bytes() * 2)
    return d
