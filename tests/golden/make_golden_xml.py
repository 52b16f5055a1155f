"""Generates tests/golden/xml/: a reduced copy of the reference's own test resources (zstd-jni src/test/resources), which
tests/conftest.py turns back into the resource directory the tests read (fixture `reference_resources`).

The resources are a 5.3 MB text file `xml` and streams made from it by their regenerate.sh.  Stored here, following that
script on the first XML_BYTES of `xml` (two 128 KB blocks) with the compiled reference (oracle/_ref/libzstd-oracle.so):
  xml.gz                   the plaintext (gzip: an encoder independent of the one under test)
  xml-{1,3,6,9}.zst        streaming, unknown content size, no checksum (`cat xml | zstd --no-check -N`)
  xml-1-sized.zst          one-shot with the content size (`zstd --no-check -1 xml`)
  xml-advanced.zst         explicit parameters wlog=23,slog=4,tlen=32,mml=7,strat=7,hlog=16,clog=15
  xmlsmall, xmlsmall-sized.zst   the reference's own files, verbatim (102 / 103 bytes)
The concatenations (xml-1x2.zst, xml-1-sizedx2.zst) are made by the fixture.

usage: python tests/golden/make_golden_xml.py <zstd-jni checkout>/src/test/resources
"""
import gzip
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent.parent))

from tests.oracle_util import ref, ref_compress_params, ref_stream_compress  # noqa: E402

XML_BYTES = 160000
ADVANCED = {"windowLog": 23, "searchLog": 4, "targetLength": 32, "minMatch": 7, "strategy": 7, "hashLog": 16, "chainLog": 15}


def main(resources: Path) -> None:
    assert ref() is not None, "oracle/_ref/libzstd-oracle.so missing: run `make -C oracle ref`"
    out = HERE / "xml"
    out.mkdir(exist_ok=True)
    xml = (resources / "xml").read_bytes()[:XML_BYTES]
    (out / "xml.gz").write_bytes(gzip.compress(xml, 9, mtime=0))
    for level in (1, 3, 6, 9):
        (out / f"xml-{level}.zst").write_bytes(ref_stream_compress(xml, level))
    (out / "xml-1-sized.zst").write_bytes(ref_compress_params(xml, 1, {}))
    (out / "xml-advanced.zst").write_bytes(ref_compress_params(xml, 3, ADVANCED))
    for name in ("xmlsmall", "xmlsmall-sized.zst"):
        (out / name).write_bytes((resources / name).read_bytes())


if __name__ == "__main__":
    main(Path(sys.argv[1]))
