"""Generates tests/golden/* from the reference compiled in place (oracle/_ref/libzstd-oracle.so).

Run in the dev container (needs /root/reference to have built oracle/_ref):
    python -m tests.golden.make_golden
The fixtures are small on purpose; inputs are regenerated from the deterministic corpus generator or a seeded
generator (regenerate_input), only their SHA-256 is stored.  Nothing here runs on the GPU box except regenerate_input().
"""
from __future__ import annotations

import hashlib
import json
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent.parent))


def regenerate_input(spec: dict) -> bytes:
    from zstd_jni_b200 import corpus
    from tests import cases
    if spec["kind"] == "corpus":
        return corpus.chunk(spec["index"])[: spec["size"]].tobytes()
    if spec["kind"] == "special":
        return dict(cases.special_cases())[spec["name"]]
    if spec["kind"] == "multi":
        return b"".join(corpus.chunk(i).tobytes() for i in spec["indices"])[: spec["size"]]
    import numpy as np
    if spec["kind"] == "tokens":           # random tokens of `width` bytes drawn from a vocabulary of `vocab` random tokens
        rng = np.random.default_rng(spec["seed"])
        voc = rng.integers(0, 256, (spec["vocab"], spec["width"]), dtype=np.uint8)
        return voc[rng.integers(0, spec["vocab"], -(-spec["size"] // spec["width"]))].reshape(-1)[: spec["size"]].tobytes()
    if spec["kind"] == "alphabet":         # independent bytes from the first `alpha` letters
        rng = np.random.default_rng(spec["seed"])
        return (rng.integers(0, spec["alpha"], spec["size"], dtype=np.uint8) + 33).tobytes()
    if spec["kind"] == "planted":          # `copies` x (fresh bytes from an alphabet, then a copy of an earlier stretch)
        rng = np.random.default_rng(spec["seed"])
        out = bytearray(rng.integers(0, spec["alpha"], spec["fresh"], dtype=np.uint8).tobytes())
        for _ in range(spec["copies"]):
            n = int(rng.integers(8, 25)); at = int(rng.integers(0, max(1, len(out) - n)))
            out += bytes(out[at:at + n])
            out += rng.integers(0, spec["alpha"], int(rng.integers(1, spec["fresh"] + 1)), dtype=np.uint8).tobytes()
        return bytes(out)
    if spec["kind"] == "samecodes":        # `count` x (64 ... 80 fresh bytes, then 10 bytes from 61 ... 124 back): one LL / OF / ML code each
        rng = np.random.default_rng(spec["seed"])
        out = bytearray(rng.integers(0, 256, 40, dtype=np.uint8).tobytes())
        for k in range(spec["count"]):
            out += rng.integers(0, 256, int(rng.integers(64, 81)), dtype=np.uint8).tobytes()
            d = 61 + (29 * k) % 64         # never one of the last three offsets: no repcodes
            out += bytes(out[len(out) - d:len(out) - d + 10])
        return bytes(out) + rng.integers(0, 256, 16, dtype=np.uint8).tobytes()      # (no match is looked for in the last bytes)
    if spec["kind"] == "repeat":
        return bytes([spec["byte"]]) * spec["size"]
    raise KeyError(spec["kind"])


# ---- decode-only frames from the reference's other encoders (optimal parsers, explicit parameters), one block each
EXPERIMENTAL_IDS = {"literalCompressionMode": 1002, "splitAfterSequences": 1010, "blockSplitterLevel": 1017}
NO_SPLIT = {"blockSplitterLevel": 1, "splitAfterSequences": 2}      # the optimal levels split 128 KB inputs into several blocks by default


def ref_compress_ids(data: bytes, level: int, params: dict) -> bytes:
    """The compiled reference with explicit and experimental parameters (names of CPARAM_IDS / EXPERIMENTAL_IDS)."""
    import ctypes as C
    from tests.oracle_util import CPARAM_IDS, ERR_MAX, ref
    R = ref()
    cctx = R.ZSTD_createCCtx()
    try:
        R.ZSTD_CCtx_setParameter(cctx, 100, level)
        for k, v in params.items():
            assert R.ZSTD_CCtx_setParameter(cctx, {**CPARAM_IDS, **EXPERIMENTAL_IDS}[k], v) <= ERR_MAX, k
        cap = len(data) + (len(data) >> 8) + 1024
        out = C.create_string_buffer(cap)
        n = R.ZSTD_compress2(cctx, out, cap, data, len(data))
        assert n <= ERR_MAX
        return out.raw[:n]
    finally:
        R.ZSTD_freeCCtx(cctx)


def foreign_frames():
    """(name, input spec, level, params, frame, note) for every foreign fixture.  Seeds are searched where a feature needs an exact
    value; every frame is one the staged decoder takes itself (tests/golden/frame_info.py FrameInfo.staged)."""
    from tests.golden.frame_info import EDGE_NBSEQ, parse_frame
    out = []

    def add(name, spec, level, params, frame=None, note=None):
        data = regenerate_input(spec)
        z = frame if frame is not None else ref_compress_ids(data, level, {**NO_SPLIT, **params})
        assert parse_frame(z).staged, name
        out.append((name, spec, level, params, z, note))
        return z

    def search(name, level, params, specs, want):
        for spec in specs:
            z = ref_compress_ids(regenerate_input(spec), level, {**NO_SPLIT, **params})
            if want(parse_frame(z)):
                return add(name, spec, level, params, z)
        raise AssertionError(f"no seed reaches {name}")

    # the most sequences a 128 KB block gets: random 3-byte tokens, minMatch 3 (three-byte sequence count)
    best = None
    for vocab in (150, 200, 256, 300):
        spec = {"kind": "tokens", "seed": 0, "vocab": vocab, "width": 3, "size": 131070}
        z = ref_compress_ids(regenerate_input(spec), 19, {**NO_SPLIT, "minMatch": 3})
        if best is None or parse_frame(z).nb_seq > parse_frame(best[1]).nb_seq:
            best = (spec, z)
    add("L19_mm3_maxseq", best[0], 19, {"minMatch": 3}, best[1])
    add("L22_tokens4", {"kind": "tokens", "seed": 1, "vocab": 3000, "width": 4, "size": 131072}, 22, {})
    add("L16_tokens5", {"kind": "tokens", "seed": 2, "vocab": 2000, "width": 5, "size": 100000}, 16, {})
    add("L13_alpha8", {"kind": "alphabet", "seed": 3, "alpha": 8, "size": 60000}, 13, {})
    # sequence counts on the walk -> value link depth and the k_order bucket edge; raw literals (incompressible fresh bytes)
    levels = (19, 13, 16, 22)
    for k, n in enumerate(EDGE_NBSEQ):
        search(f"L{levels[k % 4]}_nbseq{n}", levels[k % 4], {},
               ({"kind": "planted", "seed": s, "alpha": 256, "fresh": 40, "copies": n} for s in range(300)), lambda i, n=n: i.nb_seq == n)
    # Huffman literals of 8 ... 63 bytes next to 1 ... 31 sequences (btultra2 compresses literal sections from 8 bytes on)
    for k, (n, fresh) in enumerate(((2, 8), (5, 8), (11, 6), (24, 3))):
        search(f"L19_huf_small_{k}", 19, {},
               ({"kind": "planted", "seed": s, "alpha": 4, "fresh": fresh, "copies": n} for s in range(300)),
               lambda i: i.lit_mode == 2 and 8 <= i.lit_size <= 63 and 1 <= i.nb_seq <= 31)
    # one length / offset code throughout: RLE mode in all three positions
    search("L19_rle_tables", 19, {}, ({"kind": "samecodes", "seed": s, "count": 24} for s in range(300)),
           lambda i: i.modes == ("rle", "rle", "rle"))
    # literal-only compressed blocks: Huffman 255 bytes (one stream) and 256 bytes (four streams)
    for size in (255, 256):
        search(f"L19_huf_lit{size}", 19, {}, ({"kind": "alphabet", "seed": s, "alpha": 40, "size": size} for s in range(300)),
               lambda i: i.lit_mode == 2 and i.nb_seq == 0)
    search("L22_huf_lit_only", 22, {}, ({"kind": "alphabet", "seed": s, "alpha": 24, "size": 90} for s in range(300)),
           lambda i: i.lit_mode == 2 and i.nb_seq == 0)
    # explicit parameters: minMatch 3, a small window, literal compression disabled
    add("L19_mm3_w12_rawlit", {"kind": "alphabet", "seed": 4, "alpha": 8, "size": 4000}, 19,
        {"minMatch": 3, "windowLog": 12, "literalCompressionMode": 2})
    add("L19_mm3_w10_rawlit", {"kind": "tokens", "seed": 5, "vocab": 60, "width": 3, "size": 1000}, 19,
        {"minMatch": 3, "windowLog": 10, "literalCompressionMode": 2})
    add("L13_mm3_rawlit_big", {"kind": "tokens", "seed": 6, "vocab": 500, "width": 3, "size": 120000}, 13,
        {"minMatch": 3, "literalCompressionMode": 2})
    # RLE literals next to sequences: the reference writes them only when all (>= 8) literals are one byte, which a block of one
    # repeated byte never has (one literal, then a match); so the raw one-byte literals section of that frame is re-typed as RLE
    spec = {"kind": "repeat", "byte": 97, "size": 1000}
    z = bytearray(ref_compress_ids(regenerate_input(spec), 19, NO_SPLIT))
    i = parse_frame(bytes(z)); at = i.header_size + 3
    assert i.lit_mode == 0 and i.lit_size == 1 and z[at] == 0x08 and i.nb_seq == 1
    z[at] = 0x09                           # literals section header: RLE, one byte
    add("L19_rle_lit", spec, 19, {}, bytes(z), "raw literals section of the reference frame re-typed as RLE")
    return out


def main():
    from tests.oracle_util import ref, ref_compress, ref_decompress, ref_stream_compress
    assert ref() is not None, "oracle/_ref/libzstd-oracle.so missing: run `make -C oracle ref`"
    man = {"generator": "tests/golden/make_golden.py", "reference": "libzstd " + ref().ZSTD_versionString().decode() + " (luben/zstd-jni 1.5.7-16 src/main/native)",
           "oneshot": [], "decode_only": [], "errors": []}
    for f in HERE.glob("*.zst"):
        f.unlink()
    specs = []
    for cls, idx in ((0, 0), (1, 1), (2, 2), (4, 4), (5, 5), (7, 7), (7, 15), (7, 23)):
        for size in (0, 1, 6, 7, 64, 255, 256, 1000, 1024, 5000, 16384, 16385):
            if cls in (7,) and size not in (0, 7, 1000, 16385):
                continue
            specs.append({"kind": "corpus", "index": idx, "size": size})
    for idx in (1, 5, 7, 15, 23, 31):
        specs.append({"kind": "corpus", "index": idx, "size": 131072})
    for name in ("zeros-128k", "period-3", "long-match", "four-symbols-50k"):
        specs.append({"kind": "special", "name": name})
    n = 0
    for spec in specs:
        data = regenerate_input(spec)
        for level in ((3, 1) if len(data) <= 5000 or spec["kind"] == "special" else (3,)):
            frame = ref_compress(data, level)
            assert not isinstance(frame, int)
            if len(frame) > 20000:
                continue
            fn = f"oneshot_{n:03d}_L{level}.zst"; n += 1
            (HERE / fn).write_bytes(frame)
            man["oneshot"].append({"file": fn, "level": level, "input": spec, "input_sha256": hashlib.sha256(data).hexdigest(), "frame_size": len(frame)})
    # lazy levels (row match finder, cost-based table selection): the 128 KB inputs and the specials again
    for spec in specs:
        data = regenerate_input(spec)
        if len(data) <= 16384:
            continue
        for level in (9, 6, 5, 12):
            frame = ref_compress(data, level)
            assert not isinstance(frame, int)
            if len(frame) > 20000:
                continue
            fn = f"oneshot_{n:03d}_L{level}.zst"; n += 1
            (HERE / fn).write_bytes(frame)
            man["oneshot"].append({"file": fn, "level": level, "input": spec, "input_sha256": hashlib.sha256(data).hexdigest(), "frame_size": len(frame)})
    # hash-chain finder (levels 4, 6) and binary tree (level 9) on small inputs
    for spec in specs:
        data = regenerate_input(spec)
        if spec["kind"] != "corpus" or spec["size"] not in (1000, 5000, 16384):
            continue
        for level in (4, 6, 9):
            frame = ref_compress(data, level)
            assert not isinstance(frame, int)
            fn = f"oneshot_{n:03d}_L{level}.zst"; n += 1
            (HERE / fn).write_bytes(frame)
            man["oneshot"].append({"file": fn, "level": level, "input": spec, "input_sha256": hashlib.sha256(data).hexdigest(), "frame_size": len(frame)})
    # decode-only: the reference's streaming path (multi-block, unknown content size, repeat modes)
    multi = {"kind": "multi", "indices": [1, 9, 5, 17], "size": 450000}
    data = regenerate_input(multi)
    for level, checksum in ((1, False), (3, False), (3, True), (9, False)):
        z = ref_stream_compress(data, level, checksum=checksum)
        fn = f"stream_L{level}{'_xxh' if checksum else ''}.zst"
        (HERE / fn).write_bytes(z)
        man["decode_only"].append({"file": fn, "size": len(data), "sha256": hashlib.sha256(data).hexdigest(), "input": multi})
    z3 = ref_stream_compress(data[:150000], 3)
    skippable = b"\x50\x2a\x4d\x18" + (7).to_bytes(4, "little") + b"skipped"
    (HERE / "concat_skippable.zst").write_bytes(skippable + z3 + skippable + z3)
    man["decode_only"].append({"file": "concat_skippable.zst", "size": 300000, "sha256": hashlib.sha256(data[:150000] * 2).hexdigest(), "input": None})
    from tests.golden.frame_info import REQUIRED_FEATURES, features
    seen = set()
    for name, spec, level, params, z, note in foreign_frames():
        data = regenerate_input(spec)
        fn = f"foreign_{name}.zst"
        (HERE / fn).write_bytes(z)
        e = {"file": fn, "size": len(data), "sha256": hashlib.sha256(data).hexdigest(), "input": spec, "level": level, "params": params,
             "features": features(z)}
        if note:
            e["note"] = note
        man["decode_only"].append(e)
        seen |= set(e["features"])
    assert REQUIRED_FEATURES <= seen, sorted(REQUIRED_FEATURES - seen)
    # error behaviour pinned by the reference
    base = ref_compress(regenerate_input({"kind": "corpus", "index": 1, "size": 20000}), 3)
    probes = {"err_truncated_end.zst": base[:-1], "err_truncated_mid.zst": base[: len(base) // 2], "err_bad_magic.zst": b"\x00" + base[1:],
              "err_reserved_bit.zst": base[:4] + bytes([base[4] | 0x08]) + base[5:], "err_trailing_garbage.zst": base + b"\x01\x02\x03\x04\x05\x06\x07\x08\x09"}
    for fn, blob in probes.items():
        r = ref_decompress(blob, 20000)
        assert isinstance(r, int), fn
        (HERE / fn).write_bytes(blob)
        man["errors"].append({"file": fn, "cap": 20000, "code": -r})
    r = ref_decompress(base, 19999)
    (HERE / "err_dst_too_small.zst").write_bytes(base)
    man["errors"].append({"file": "err_dst_too_small.zst", "cap": 19999, "code": -r})
    (HERE / "manifest.json").write_text(json.dumps(man, indent=1))
    total = sum(f.stat().st_size for f in HERE.glob("*.zst"))
    print(len(man["oneshot"]), "one-shot,", len(man["decode_only"]), "decode-only,", len(man["errors"]), "error fixtures;", total, "bytes")


if __name__ == "__main__":
    main()
