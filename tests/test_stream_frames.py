"""A frame of many blocks streamed segment by segment (zstdb200_fstream_*, ZSTD_decompressStream).

CPU: the host instantiation (tests/hostsim/libzb_hostsim_stream.so): segments decoded from their own copy of the input with the history
in a ring, cut at every block boundary; the fused decoder's resume entry from every block boundary, on valid frames (bytes) and on
frames damaged after the resume point (error codes of the whole-frame fused decode).
GPU: the public frame-stream handle and ZSTD_decompressStream on reference-made frames, in pieces of several sizes.
"""
from __future__ import annotations

import ctypes as C
import random
from pathlib import Path

import pytest

from tests.oracle_util import ERR_MAX, hostsim_decompress, oracle_decompress, ref, ref_stream_compress

ROOT = Path(__file__).resolve().parent.parent
GOLDEN = ROOT / "tests" / "golden"
MB = sorted(p for p in GOLDEN.glob("mb_*.zst"))


def _lib():
    L = C.CDLL(str(ROOT / "tests" / "hostsim" / "libzb_hostsim_stream.so"))
    L.zbst_decode.restype = C.c_size_t
    L.zbst_decode.argtypes = [C.c_void_p, C.c_size_t, C.c_char_p, C.c_size_t, C.c_uint, C.c_uint, C.c_uint, C.c_int, C.POINTER(C.c_int)]
    return L


def stream_decode(frame: bytes, cap: int, seg_blocks: int, resume_from: int = 1 << 30, ring_log: int = 0, stream: bool = False):
    """(status, bytes or negative error code): status 0 decoded, 1 error, 2 the segment decoder could not vouch for a segment.
    stream: the resume entry as the frame stream runs it, with the last window copied out of the ring as its history."""
    out = C.create_string_buffer(max(cap, 1))
    st = C.c_int(-1)
    n = _lib().zbst_decode(out, cap, frame, len(frame), seg_blocks, resume_from, ring_log, 1 if stream else 0, C.byref(st))
    if st.value == 1:
        assert n > ERR_MAX
        return 1, -((1 << 64) - n)
    return st.value, out.raw[:n]


def _blocks(frame: bytes) -> int:
    fhd = frame[4]
    did, single, fcs = fhd & 3, (fhd >> 5) & 1, fhd >> 6
    pos = 5 + (not single) + (4 if did == 3 else did) + ((1 << fcs) if fcs else 0) + (1 if single and not fcs else 0)
    n = 0
    while pos + 3 <= len(frame):
        bh = int.from_bytes(frame[pos:pos + 3], "little")
        pos += 3 + (1 if (bh >> 1) & 3 == 1 else bh >> 3)
        n += 1
        if bh & 1:
            return n
    return 0


def _valid():
    out = []
    for p in MB:
        f = p.read_bytes()
        want = oracle_decompress(f, 1 << 24)
        if isinstance(want, bytes) and _blocks(f) >= 2 and stream_decode(f, len(want), 0)[0] == 0:      # exactly one frame
            out.append((p.name, f, want))
    return out


def _window_log(frame: bytes) -> int:
    return (frame[5] >> 3) + 10 if not (frame[4] >> 5) & 1 else 0


@pytest.mark.parametrize("name,frame,want", _valid(), ids=[v[0] for v in _valid()])
def test_ring_segments_every_cut(name, frame, want):
    """Segments of every length, from their own staged input, the history read from the smallest ring that holds the window and one
    segment (so copies straddle its wrap and reach exactly the window back)."""
    n = _blocks(frame)
    for seg in range(1, n + 1):
        st, got = stream_decode(frame, len(want), seg)
        assert st == 0 and got == want, (name, seg, st)


@pytest.mark.parametrize("name,frame,want", _valid(), ids=[v[0] for v in _valid()])
def test_resume_every_block_boundary(name, frame, want):
    n = _blocks(frame)
    for k in range(n):
        for seg in (1, 3, n):
            for stream in (False, True):
                st, got = stream_decode(frame, len(want), seg, resume_from=k, stream=stream)
                assert st == 0 and got == want, (name, k, seg, stream)


@pytest.mark.parametrize("name", ["mb_L1.zst", "mb_L19.zst", "mb_L3_w10_raw_rle.zst", "mb_L3_xxh.zst", "mb_L9.zst"])
def test_resume_corruptions_match_whole_frame_fused(name):
    """Single-bit flips after the resume point: the resumed decode gives the whole-frame fused decode's bytes or error code."""
    frame = (GOLDEN / name).read_bytes()
    want = oracle_decompress(frame, 1 << 24)
    cap = len(want)
    n = _blocks(frame)
    rnd = random.Random(name)
    # block offsets, to put each flip after the resume point
    fhd = frame[4]
    pos = 5 + (not (fhd >> 5) & 1) + (4 if fhd & 3 == 3 else fhd & 3) + ((1 << (fhd >> 6)) if fhd >> 6 else 0) + (1 if (fhd >> 5) & 1 and not fhd >> 6 else 0)
    starts = []
    for _ in range(n):
        starts.append(pos)
        bh = int.from_bytes(frame[pos:pos + 3], "little")
        pos += 3 + (1 if (bh >> 1) & 3 == 1 else bh >> 3)
    checked = 0
    for _ in range(120):
        k = rnd.randrange(1, n)
        b = bytearray(frame)
        i = rnd.randrange(starts[k] + 3, len(b))
        b[i] ^= 1 << rnd.randrange(8)
        b = bytes(b)
        if _blocks(b) != n:
            continue            # a block header of the damaged frame moved: the stream would stage other blocks
        whole = hostsim_decompress(b, cap)
        st, got = stream_decode(b, cap, 2, resume_from=k)
        if st == 2:
            continue            # the segment path before the resume point met the damage
        assert got == whole, (name, k, i)
        checked += 1
    assert checked >= 40


def test_stream_damage_matches_the_reference_stream():
    """The frame stream as the host instantiation runs it (4-block segments, the last window as the resume entry's history) on bit flips
    in the second half of reference frames, against the compiled reference's ZSTD_decompressStream: the same error code, or a class
    DESIGN.md section 5 documents."""
    if ref() is None:
        pytest.skip("oracle/_ref not built")
    from collections import Counter

    from tests.golden.frame_info import reference_difference
    from tests.oracle_util import ref_compress_flags
    R = _ref_stream_lib()
    data = _text(3 << 20, 77)
    rnd = random.Random(11)
    classes = Counter()
    for frame in (ref_stream_compress(data, 3, 1 << 20, True), ref_compress_flags(data, 3, checksum=False)):
        for _ in range(60):
            b = bytearray(frame)
            i = rnd.randrange(len(b) // 2, len(b) - 4)
            b[i] ^= 1 << rnd.randrange(8)
            b = bytes(b)
            want, _, _ = _dstream(b, 131075, 131072, lib=R)
            st, got = stream_decode(b, 1 << 24, 4, resume_from=0, stream=True)
            got = got if st == 1 else 0
            if got == want:
                classes["equal"] += 1
                continue
            cls = reference_difference(frame, b, 1 << 24, want, got)
            assert cls, (i, got, want)
            classes[cls] += 1
    assert classes["equal"] >= 100, classes


# ---------------------------------------------------------------- GPU
def _text(n: int, seed: int) -> bytes:
    import numpy as np
    rnd = np.random.default_rng(seed)
    words = rnd.integers(97, 123, size=(4000, 8), dtype=np.uint8)
    words[:, 7] = 32
    return words[rnd.zipf(1.4, size=n // 8 + 1) % 4000].tobytes()[:n]


class _Stream:
    """The public frame-stream handle on its own batch context."""

    def __init__(self, seg_blocks: int, pipeline: int = 1):
        from zstd_jni_b200 import _native
        self.L = _native.lib()
        self.ctx = self.L.zstdb200_create(0)
        assert self.ctx
        assert self.L.zstdb200_set_option(self.ctx, b"dec_segment_blocks", seg_blocks) == 0
        assert self.L.zstdb200_set_option(self.ctx, b"dec_pipeline", pipeline) == 0

    def close(self):
        self.L.zstdb200_free(self.ctx)

    def decode(self, frame: bytes, pieces, outs, early=None):
        """Feeds `frame` in pieces of the sizes `pieces` yields into output buffers of the sizes `outs` yields.  Returns (bytes or
        error code, stats, most bytes held, bytes out when `early` compressed bytes had been fed)."""
        L = self.L
        fs = C.c_void_p()
        h = L.zstdb200_fstream_open(self.ctx, frame, len(frame), 0, 1 << 31, C.byref(fs))
        assert h <= ERR_MAX, h
        out = bytearray()
        held, at_early = 0, None
        pos = h
        try:
            r = 1
            while r == 1:
                k = min(next(pieces), len(frame) - pos)
                piece = frame[pos:pos + k]
                sp = C.c_size_t(0)
                while True:
                    cap = next(outs)
                    buf = C.create_string_buffer(cap)
                    dp = C.c_size_t(0)
                    r = L.zstdb200_fstream_decode(self.ctx, fs, piece, len(piece), C.byref(sp), buf, cap, C.byref(dp))
                    out += buf.raw[:dp.value]
                    held = max(held, L.zstdb200_fstream_stats(fs, 2))
                    if r != 1 or (sp.value == len(piece) and dp.value < cap):
                        break
                pos += sp.value
                if early is not None and at_early is None and pos >= early:
                    at_early = len(out)
                if r == 1 and pos >= len(frame):
                    break
            stats = (L.zstdb200_fstream_stats(fs, 0), L.zstdb200_fstream_stats(fs, 1))
        finally:
            L.zstdb200_fstream_free(fs)
        res = bytes(out) if r == 0 else (-((1 << 64) - r) if r > ERR_MAX else "incomplete")
        return res, stats, held, at_early, bytes(out)


def _sizes(kind, seed):
    rnd = random.Random(seed)
    while True:
        yield kind if isinstance(kind, int) else rnd.randint(1, kind[1])


@pytest.mark.gpu
@pytest.mark.parametrize("level", [1, 3, 19])
def test_gpu_handle_pieces(level):
    if ref() is None:
        pytest.skip("oracle/_ref not built")
    data = _text((6 if level == 19 else 24) << 20, level)
    s = _Stream(8)
    try:
        for checksum in (False, True):
            frame = ref_stream_compress(data, level, 1 << 20, checksum)
            for pieces, outs in ((131075, 131072), (("r", 300000), ("r", 400000)), (7, 1 << 20), (1 << 22, 1)):
                if pieces == 7 or outs == 1:
                    short = ref_stream_compress(data[: 2 << 20], level, 1 << 20, checksum)      # a few segments, byte-sized feeds
                    f, want = short, data[: 2 << 20]
                else:
                    f, want = frame, data
                got, (dec, res), held, _, _ = s.decode(f, _sizes(pieces, 1), _sizes(outs, 2))
                assert got == want, (level, checksum, pieces, outs)
                assert dec >= 2 and res == 0
                assert held <= 8 * (131072 + 3) + 8 * (131072 + 32)
    finally:
        s.close()


@pytest.mark.gpu
def test_gpu_handle_resume_entry_only():
    """dec_pipeline 0: every segment on the fused decoder's resume entry."""
    if ref() is None:
        pytest.skip("oracle/_ref not built")
    data = _text(12 << 20, 4)
    s = _Stream(8, pipeline=0)
    try:
        for level, checksum in ((1, True), (3, False), (19, True)):
            frame = ref_stream_compress(data, level, 1 << 20, checksum)
            got, (dec, res), _, _, _ = s.decode(frame, _sizes(("r", 1 << 20), level), _sizes(("r", 1 << 20), level + 1))
            assert got == data and dec == 0 and res >= 12
    finally:
        s.close()


@pytest.mark.gpu
def test_gpu_handle_window_logs():
    if ref() is None:
        pytest.skip("oracle/_ref not built")
    from tests.oracle_util import ref_compress_params
    s = _Stream(16)
    try:
        for wl in (17, 20, 24, 27):
            data = _text(6 << 20, wl)
            data = data[: 3 << 20] + data[: 3 << 20]
            frame = ref_compress_params(data, 3, {"windowLog": wl}, checksum=wl % 2 == 0)
            got, (dec, res), _, _, _ = s.decode(frame, _sizes(("r", 1 << 20), wl), _sizes(("r", 1 << 20), wl))
            assert got == data and dec >= 2 and res == 0, wl
    finally:
        s.close()


@pytest.mark.gpu
def test_gpu_handle_damage_late():
    """Damage late in a frame of many segments: the bytes handed out are a prefix of the content and the call ends in an error."""
    if ref() is None:
        pytest.skip("oracle/_ref not built")
    data = _text(16 << 20, 9)
    frame = ref_stream_compress(data, 3, 1 << 20, True)
    rnd = random.Random(3)
    s = _Stream(8)
    try:
        cases = [frame[:-1] + bytes([frame[-1] ^ 1])]                 # wrong checksum
        for _ in range(6):
            b = bytearray(frame)
            i = rnd.randrange(len(b) * 3 // 4, len(b) - 4)
            b[i] ^= 1 << rnd.randrange(8)
            cases.append(bytes(b))
        for b in cases:
            # the damage is in the last quarter of the input: the segments before it are handed out intact; the damaged segment's bytes
            # may differ, as the reference's do when a damaged block still decodes, and the call ends in an error
            got, _, _, _, out = s.decode(b, _sizes(131075, 0), _sizes(1 << 20, 0))
            assert isinstance(got, int) and got < 0
            assert out[: len(data) // 2] == data[: min(len(out), len(data) // 2)]
        got, _, _, _, out = s.decode(cases[0], _sizes(131075, 0), _sizes(1 << 20, 0))
        assert got == -22 and out == data                            # checksum_wrong after the last byte
    finally:
        s.close()


def _dstream(frame: bytes, piece: int, out_size: int, long_max: int = 0, early: int | None = None, lib=None, digest: bool = False):
    """ZSTD_decompressStream of this library (or of `lib`, the compiled reference) over `frame` in pieces of `piece` bytes into a buffer of
    `out_size`.  Returns (0 or the error code, the bytes out -- or their sha256 and length with `digest` --, the bytes out once `early`
    input bytes had been fed)."""
    import hashlib

    from zstd_jni_b200 import _native
    L = lib or _native.lib()
    z = L.ZSTD_createDCtx()
    if long_max:
        assert L.ZSTD_DCtx_setParameter(z, 100, long_max) == 0
    out = bytearray()
    h, total = hashlib.sha256(), 0
    dst = C.create_string_buffer(out_size)
    at_early = None
    code = 0
    try:
        pos = 0
        while pos < len(frame) and not code:
            src = frame[pos:pos + piece]
            ib = _native.InBuffer(C.cast(C.c_char_p(src), C.c_void_p), len(src), 0)
            while True:
                ob = _native.OutBuffer(C.cast(dst, C.c_void_p), out_size, 0)
                r = L.ZSTD_decompressStream(z, C.byref(ob), C.byref(ib))
                got = dst.raw[:ob.pos]
                if digest:
                    h.update(got); total += len(got)
                else:
                    out += got
                if r > ERR_MAX:
                    code = -((1 << 64) - r)
                    break
                if ib.pos == ib.size and ob.pos < out_size:
                    break
            pos += len(src)
            if early is not None and at_early is None and pos >= early:
                at_early = bytes(out)
        return code, ((h.hexdigest(), total) if digest else bytes(out)), at_early
    finally:
        L.ZSTD_freeDCtx(z)


def _ref_stream_lib():
    R = ref()
    R.ZSTD_decompressStream.restype = C.c_size_t
    R.ZSTD_decompressStream.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    return R


@pytest.mark.gpu
def test_gpu_decompress_stream_past_one_segment():
    """A 96 MB frame (768 blocks, past the default segment of 512): output starts after the first segment's input, bytes exact."""
    if ref() is None:
        pytest.skip("oracle/_ref not built")
    data = _text(96 << 20, 21)
    frame = ref_stream_compress(data, 1, 4 << 20, True)
    code, got, early = _dstream(frame, 131075, 131072, early=len(frame) * 4 // 5)
    assert code == 0 and got == data
    assert early and data.startswith(early)
    code, got, _ = _dstream(frame, 7 << 20, 1 << 20)
    assert code == 0 and got == data


@pytest.mark.gpu
def test_gpu_decompress_stream_window_log_28():
    """windowLog 28 under setLongMax(28): a random 144 MB run repeated, so long-distance matches reach back more than 2^27 bytes."""
    if ref() is None:
        pytest.skip("oracle/_ref not built")
    import hashlib

    import numpy as np
    a = np.random.default_rng(28).integers(0, 256, size=144 << 20, dtype=np.uint8).tobytes()
    data = a + a[: 48 << 20]
    R = ref()
    cctx = R.ZSTD_createCCtx()
    try:
        for k, v in ((100, 1), (101, 28), (160, 1), (201, 1)):        # level, windowLog, long-distance matching, checksum
            assert R.ZSTD_CCtx_setParameter(cctx, k, v) <= ERR_MAX
        cap = len(data) + (len(data) >> 7) + (1 << 20)
        out = C.create_string_buffer(cap)
        n = R.ZSTD_compress2(cctx, out, cap, data, len(data))
        assert n <= ERR_MAX
        frame = C.string_at(out, n)
    finally:
        R.ZSTD_freeCCtx(cctx)
    del out
    assert len(frame) < len(a) + (8 << 20)            # the repeat was found: it reaches back 144 MB > 2^27
    from zstd_jni_b200 import _native
    fh = _native.FrameHeader()
    assert _native.lib().ZSTD_getFrameHeader(C.byref(fh), frame, 32) == 0
    assert (1 << 27) < fh.windowSize <= (1 << 28)      # more than the default limit admits
    code, (digest, total), _ = _dstream(frame, 1 << 22, 1 << 22, long_max=28, digest=True)
    assert code == 0 and total == len(data) and digest == hashlib.sha256(data).hexdigest()


@pytest.mark.gpu
def test_gpu_decompress_stream_compressed_past_2gib():
    """An incompressible 2.06 GiB input: the reference writes raw blocks, the frame's compressed size passes 2^31."""
    if ref() is None:
        pytest.skip("oracle/_ref not built")
    import hashlib

    import numpy as np
    data = np.random.default_rng(31).integers(0, 256, size=(2 << 30) + (64 << 20), dtype=np.uint8).tobytes()
    R = ref()
    cap = len(data) + (len(data) >> 7) + (1 << 20)
    out = C.create_string_buffer(cap)
    n = R.ZSTD_compress(out, cap, data, len(data), 1)
    assert n <= ERR_MAX and n > (1 << 31)
    frame = memoryview(out).cast("B")[:n].tobytes()
    del out
    want = hashlib.sha256(data).hexdigest()
    del data
    code, (digest, total), _ = _dstream(frame, 1 << 24, 1 << 24, digest=True)
    assert code == 0 and total == (2 << 30) + (64 << 20) and digest == want


def _damage_report() -> list:
    """Run in a process with ZSTDB200_DEC_SEGMENT_BLOCKS=4: damaged frames of many 4-block segments through ZSTD_decompressStream of
    this library and of the compiled reference.  One row per case: name, frame, damaged frame, our code, the reference's code, whether
    our bytes out are a prefix of the reference's."""
    from tests.oracle_util import ref_compress_flags
    R = _ref_stream_lib()
    rows = []
    data = _text(3 << 20, 77)
    streamed = ref_stream_compress(data, 3, 1 << 20, True)          # no content size, checksum
    sized = ref_compress_flags(data, 3, checksum=False)                # content size, no checksum
    assert _blocks(streamed) > 16 and _blocks(sized) > 16

    def case(name, frame, damaged, piece=131075):
        c1, o1, _ = _dstream(damaged, piece, 131072)
        c2, o2, _ = _dstream(damaged, piece, 131072, lib=R)
        k = min(len(o1), len(o2))       # the reference does not count the bytes of the call that fails, this library does
        rows.append({"name": name, "frame": frame.hex(), "damaged": damaged.hex(), "ours": c1, "ref": c2, "prefix": o1[:k] == o2[:k],
                     "ours_len": len(o1), "ref_len": len(o2)})

    c1, o1, _ = _dstream(streamed, 7, 131072)
    rows.append({"name": "valid, 7-byte pieces", "ours": c1, "ref": 0, "prefix": o1 == data})
    case("wrong checksum", streamed, streamed[:-1] + bytes([streamed[-1] ^ 0x40]))
    fhd = sized[4]
    fcs_at = 5 + (not (fhd >> 5) & 1) + (4 if fhd & 3 == 3 else fhd & 3)
    fcs_len = (1 << (fhd >> 6)) if fhd >> 6 else 0
    assert fcs_len >= 4
    size = int.from_bytes(sized[fcs_at:fcs_at + fcs_len], "little")
    for d in (1, -1):
        case("content size %+d" % d, sized, sized[:fcs_at] + (size + d).to_bytes(fcs_len, "little") + sized[fcs_at + fcs_len:])
    for cut in (len(streamed) // 2, len(streamed) - 5, len(streamed) - 1):
        case("truncated to %d" % cut, streamed, streamed[:cut])
    rnd = random.Random(11)
    for frame in (streamed, sized):
        for _ in range(40):
            b = bytearray(frame)
            i = rnd.randrange(len(b) // 2, len(b) - 4)
            b[i] ^= 1 << rnd.randrange(8)
            case("bit flip at %d" % i, frame, bytes(b))
    return rows


@pytest.mark.gpu
def test_gpu_damage_matches_the_reference_stream():
    """Damage late in a frame of many segments, through ZSTD_decompressStream against the compiled reference's: a wrong checksum, the
    content size off by one either way, truncations and bit flips.  The error codes are equal, or a bit flip falls in a class DESIGN.md
    section 5 documents (frame_info.reference_difference); the bytes both hand out agree."""
    if ref() is None:
        pytest.skip("oracle/_ref not built")
    import json
    import os
    import subprocess
    import sys
    from collections import Counter

    from tests.golden.frame_info import reference_difference
    env = dict(os.environ, ZSTDB200_DEC_SEGMENT_BLOCKS="4")
    code = "import json; from tests.test_stream_frames import _damage_report; print('ROWS' + json.dumps(_damage_report()))"
    p = subprocess.run([sys.executable, "-c", code], cwd=str(ROOT), env=env, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stderr[-3000:]
    rows = json.loads(p.stdout[p.stdout.index("ROWS") + 4:])
    classes = Counter()
    for r in rows:
        assert r["prefix"], r["name"]
        if r["ours"] == r["ref"]:
            classes["equal"] += 1
            continue
        assert r["name"].startswith("bit flip"), (r["name"], r["ours"], r["ref"])
        cls = reference_difference(bytes.fromhex(r["frame"]), bytes.fromhex(r["damaged"]), 1 << 24, r["ref"], r["ours"])
        assert cls, (r["name"], r["ours"], r["ref"])
        classes[cls] += 1
    print("damage classes:", dict(classes))
    assert classes["equal"] >= len(rows) * 3 // 4, classes
