"""Items of several frames decoded frame by frame, and checksummed single-block frames on the staged decoder.

CPU: the host instantiation of the decoder's source (tests/hostsim/zb_hostsim_items.cpp, compiled by this module):
  - item_walk lists the frames of concatenations of golden fixtures, reference frames with and without content size and checksum,
    skippable and empty frames, cut at every byte and followed by garbage -- frame by frame the reference's walk
    (ZSTD_findFrameCompressedSize, ZSTD_getFrameContentSize), and the item is split exactly where the rule allows;
  - xxh64_warp on the emulated warp equals the serial xxh64 at every length 0..600, in a sweep up to 128 KB and at offsets 0..15;
  - the staged decoder takes checksummed one-block frames and gives the fused decoder's bytes and error codes on checksum and block
    damage.
GPU: zstdb200_decompress_batch (decompressBatch, Zstd.decompress, ZstdDecompressCtx) on valid and damaged multi-frame items and on
checksummed batches, against a dec_pipeline 0 context (the fused kernel on whole items) and the reference.
"""
from __future__ import annotations

import ctypes as C
import random
import subprocess
from pathlib import Path

import numpy as np
import pytest

from tests.oracle_util import (ERR_MAX, hostsim_compress_flags, hostsim_decompress, ref, ref_compress_flags, ref_decompress,
                               ref_stream_compress, staged_decompress)

ROOT = Path(__file__).resolve().parent.parent
GOLDEN = ROOT / "tests" / "golden"
UNKNOWN = (1 << 64) - 1


@pytest.fixture(scope="module")
def items_lib(tmp_path_factory):
    src = ROOT / "tests" / "hostsim" / "zb_hostsim_items.cpp"
    so = tmp_path_factory.mktemp("hostsim_items") / "libzb_hostsim_items.so"
    subprocess.run(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-Wall", "-Wno-unused-function", "-x", "c++", str(src), "-o", str(so)],
                   check=True)
    L = C.CDLL(str(so))
    L.zbi_item_walk.restype = C.c_uint
    L.zbi_item_walk.argtypes = [C.c_char_p, C.c_size_t, C.c_ulonglong, C.POINTER(C.c_ulonglong), C.c_uint, C.POINTER(C.c_int)]
    L.zbi_xxh64.restype = C.c_ulonglong
    L.zbi_xxh64.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.c_int, C.POINTER(C.c_int)]
    L.zbi_staged_mode.restype = C.c_uint
    L.zbi_staged_mode.argtypes = [C.c_char_p, C.c_size_t, C.c_size_t]
    L.zbi_decode_list.restype = C.c_size_t
    L.zbi_decode_list.argtypes = [C.c_char_p, C.POINTER(C.c_ulonglong), C.POINTER(C.c_ulonglong), C.c_size_t, C.c_int, C.POINTER(C.c_ubyte),
                                  C.POINTER(C.c_ulonglong), C.POINTER(C.c_ulonglong), C.c_size_t, C.POINTER(C.c_int), C.POINTER(C.c_size_t)]
    return L


def item_walk(L, item: bytes, cap: int):
    """(frames [(srcOff, srcSize, contentSize or None, skippable)], split)."""
    k = 4096
    out = (C.c_ulonglong * (7 * k))()
    split = C.c_int(0)
    n = L.zbi_item_walk(item, len(item), cap, out, k, C.byref(split))
    frames = []
    for j in range(min(n, k)):
        o = out[7 * j: 7 * j + 7]
        frames.append((o[0], o[1], None if o[6] else (o[2] if o[5] else None), bool(o[6])))
    return frames, bool(split.value)


def _ref_walk(item: bytes):
    """The reference's frames of the item: [(srcOff, srcSize, contentSize or None, skippable)], and whether the walk reached the end."""
    R = ref()
    R.ZSTD_findFrameCompressedSize.restype = C.c_size_t
    R.ZSTD_findFrameCompressedSize.argtypes = [C.c_char_p, C.c_size_t]
    R.ZSTD_getFrameContentSize.restype = C.c_ulonglong
    R.ZSTD_getFrameContentSize.argtypes = [C.c_char_p, C.c_size_t]
    out, pos = [], 0
    while pos < len(item):
        rest = item[pos:]
        n = R.ZSTD_findFrameCompressedSize(rest, len(rest))
        if n > ERR_MAX or n == 0:
            return out, False
        skippable = len(rest) >= 4 and (int.from_bytes(rest[:4], "little") & 0xFFFFFFF0) == 0x184D2A50
        cs = R.ZSTD_getFrameContentSize(rest, len(rest))
        out.append((pos, n, None if skippable or cs >= UNKNOWN - 1 else cs, skippable))
        pos += n
    return out, True


def _expected_split(frames, complete, cap):
    if not complete or len(frames) < 2:
        return False
    zs = [f for f in frames if not f[3]]
    if any(f[2] is None for f in zs[:-1]):
        return False
    return sum(f[2] or 0 for f in zs) <= cap


def _skippable(n: int, magic_low: int = 0) -> bytes:
    return (0x184D2A50 + magic_low).to_bytes(4, "little") + n.to_bytes(4, "little") + bytes((i * 7) & 0xFF for i in range(n))


def _data(seed: int, n: int) -> bytes:
    rnd = random.Random(seed)
    words = [bytes(rnd.choice(b"abcdefghij") for _ in range(rnd.randrange(2, 9))) for _ in range(200)]
    out = bytearray()
    while len(out) < n:
        out += rnd.choice(words) + b" "
    return bytes(out[:n])


def _ref_frames():
    """Reference frames: with and without content size and checksum, empty, multi-block one-shot."""
    out = []
    for k, (cs, ck) in enumerate([(True, False), (True, True), (False, False), (False, True)]):
        out.append(ref_compress_flags(_data(k, 5000 + 999 * k), 3, checksum=ck, content_size=cs))
    out.append(ref_compress_flags(b"", 3))
    out.append(ref_compress_flags(b"", 3, checksum=True))
    out.append(ref_compress_flags(_data(9, 300_000), 1))      # three blocks
    assert all(isinstance(f, bytes) for f in out)
    return out


def _walk_inputs():
    gold = [GOLDEN / "mb_L1.zst", GOLDEN / "mb_L3_xxh.zst", GOLDEN / "oneshot_000_L3.zst", GOLDEN / "oneshot_001_L1.zst",
            GOLDEN / "mb_two_frames_skippable.zst", GOLDEN / "concat_skippable.zst"] + sorted(GOLDEN.glob("stream_L*.zst"))[:3]
    g = [p.read_bytes() for p in gold if p.exists()]
    r = _ref_frames()
    sk = [_skippable(n, n % 16) for n in (0, 1, 7, 64, 300)]
    items = {}
    items["gold-concat"] = b"".join(g)
    for k, f in enumerate(g):
        items[f"gold-{k}-alone"] = f
        items[f"gold-{k}-twice"] = f + f
    items["ref-all"] = b"".join(r)
    items["ref-sized-only"] = r[0] + r[1] + r[4] + r[6]
    items["ref-middle-unsized"] = r[0] + r[2] + r[1]
    items["ref-last-unsized"] = r[0] + r[1] + r[3]
    for k, s in enumerate(sk):
        items[f"skip-{k}-between"] = r[0] + s + r[1]
        items[f"skip-{k}-first-last"] = s + r[1] + r[0] + s
        items[f"skip-{k}-alone-twice"] = s + s
    items["empty-frames"] = r[4] + r[5] + r[4]
    items["garbage"] = r[0] + r[1] + b"\x01\x02\x03"
    items["garbage-magic"] = r[0] + r[1] + r[0][:4]
    return items


def test_item_walk_matches_reference(items_lib):
    checked = 0
    for name, item in _walk_inputs().items():
        want, complete = _ref_walk(item)
        total = sum(f[2] or 0 for f in want if not f[3])
        for cap in sorted({total - 1, total, total + 1, total + 100_000} - {-1}):
            got, split = item_walk(items_lib, item, cap)
            assert got == want[:len(got)], name
            if complete:
                assert len(got) == len(want), name
            assert split == _expected_split(want, complete, cap), (name, cap)
            if split and all(f[2] is not None for f in want if not f[3]):
                # the reference decodes it whole into exactly the declared sizes
                dec = ref_decompress(item, cap)
                assert isinstance(dec, bytes) and len(dec) == total, (name, dec if isinstance(dec, int) else len(dec))
            checked += 1
    assert checked > 100


def test_item_walk_every_cut(items_lib):
    r = _ref_frames()
    item = r[1] + _skippable(5) + r[0] + r[6]
    whole, _ = _ref_walk(item)
    bounds = {f[0] for f in whole} | {len(item)}
    for cut in range(len(item) + 1):
        part = item[:cut]
        want, complete = _ref_walk(part)
        got, split = item_walk(items_lib, part, 1 << 22)
        assert got == want[:len(got)], cut
        assert split == _expected_split(want, complete, 1 << 22), cut
        if split:
            assert cut in bounds
    # and followed by garbage at every length up to 12 bytes
    for g in range(1, 13):
        got, split = item_walk(items_lib, item + bytes(range(1, g + 1)), 1 << 22)
        assert not split and len(got) == len(whole)


def test_xxh64_warp_equals_serial(items_lib):
    rnd = random.Random(5)
    buf = bytes(rnd.getrandbits(8) for _ in range(131072 + 16))
    u = C.c_int(0)

    def h(data, off, lanes):
        v = items_lib.zbi_xxh64(data, len(data), off, lanes, C.byref(u))
        assert u.value == 1, (len(data), off, lanes)
        return v

    for n in range(0, 601):
        d = buf[n:2 * n]
        assert h(d, 0, 32) == h(d, 0, 1), n
    for n in list(range(601, 131073, 4099)) + [131071, 131072]:
        d = buf[:n]
        assert h(d, 0, 32) == h(d, 0, 1), n
    for off in range(16):
        for n in (0, 31, 32, 33, 255, 256, 257, 1000, 4099):
            d = buf[off:off + n]
            want = h(d, 0, 1)
            for lanes in (4, 8, 16, 32):
                assert h(d, off, lanes) == want, (off, n, lanes)
    # the published XXH64 of seed 0: the empty input
    assert h(b"", 0, 32) == 0xEF46DB3751D8E999


def decode_list(L, items, caps, reserve_ok: bool):
    """(entries, split flags, entry input offsets, entry output offsets, reservations asked, entries asked for)."""
    n = len(items)
    so = [0]
    for it in items:
        so.append(so[-1] + len(it))
    do = [0]
    for c in caps:
        do.append(do[-1] + c)
    emax = 1 << 16
    e_src, e_dst = (C.c_ulonglong * (emax + 1))(), (C.c_ulonglong * (emax + 1))()
    split = (C.c_ubyte * n)()
    asked, asked_for = C.c_int(0), C.c_size_t(0)
    m = L.zbi_decode_list(b"".join(items), (C.c_ulonglong * (n + 1))(*so), (C.c_ulonglong * (n + 1))(*do), n, 1 if reserve_ok else 0, split,
                          e_src, e_dst, emax, C.byref(asked), C.byref(asked_for))
    return m, list(split), list(e_src[:m + 1]), list(e_dst[:m + 1]), asked.value, asked_for.value, so, do


def test_decode_list_keeps_items_whole_without_workspace(items_lib):
    """The decode list cuts an item only when the workspaces of every entry can be had, and only when its frames are large enough to
    pay for an entry each; otherwise every item stays whole -- the same list of items a dec_pipeline 0 call decodes."""
    r = _ref_frames()
    big = [ref_compress_flags(_data(400 + k, 100_000), 3) for k in range(3)]
    splittable = big[0] + _skippable(7) + big[1] + big[2]
    empties = r[4] * 16384                                     # 16 384 empty frames: legal, nothing to gain from a split
    small = b"".join(ref_compress_flags(_data(500 + k, 1000), 3) for k in range(8))
    items = [big[0], splittable, empties, small, splittable]
    caps = [100_000, 300_000, 0, 8000, 300_001]
    m, split, e_src, e_dst, asked, asked_for, so, do = decode_list(items_lib, items, caps, True)
    assert split == [0, 1, 0, 0, 1] and m == 5 + 3 + 3 and asked == 1 and asked_for == m
    # the split item's entries: each frame's input, outputs at the declared sizes (the skippable frame: nothing)
    frames, _ = _ref_walk(splittable)
    assert e_src[1:5] == [so[1] + f[0] for f in frames]
    assert e_dst[1:5] == [do[1], do[1] + 100_000, do[1] + 100_000, do[1] + 200_000]
    assert e_src[-1] == so[-1] and e_dst[-1] == do[-1]
    # the workspaces cannot be had: every item whole
    m, split, e_src, e_dst, asked, asked_for, so, do = decode_list(items_lib, items, caps, False)
    assert (m, split, e_src, e_dst, asked) == (5, [0] * 5, so, do, 1)
    # nothing to split: the reservation is not even asked for
    m, split, e_src, e_dst, asked, _, so, do = decode_list(items_lib, [big[0], empties, small], [100_000, 0, 8000], True)
    assert (m, split, e_src, e_dst, asked) == (3, [0] * 3, so, do, 0)


def _checksummed_frames():
    out = []
    for level in (1, 3, 9, 19):
        # (level 19 beyond 64 KB writes blocks the staged decoder refuses with or without a checksum)
        for k, n in enumerate((37, 4000, 65536, 120_000 if level < 19 else 30_000)):
            data = _data(level * 10 + k, n)
            out.append((f"ref-L{level}-{n}", ref_compress_flags(data, level, checksum=True), data))
    for level in (1, 3):
        for k, n in enumerate((100, 50_000, 131072)):
            data = _data(100 + level * 10 + k, n)
            out.append((f"own-L{level}-{n}", hostsim_compress_flags(data, level, checksum=True), data))
    out.append(("raw", ref_compress_flags(bytes(random.Random(3).getrandbits(8) for _ in range(3000)), 3, checksum=True), None))
    out.append(("rle", ref_compress_flags(b"\x07" * 5000, 3, checksum=True), b"\x07" * 5000))
    return out


@pytest.mark.parametrize("emu", [False, True])
def test_staged_decoder_takes_checksummed_frames(items_lib, emu):
    frames = _checksummed_frames()
    if emu:      # (the emulator is slow: the smaller frames, and fewer flips)
        frames = [f for f in frames if len(f[1]) < 20_000]
    for name, frame, data in frames:
        assert isinstance(frame, bytes), name
        if data is None:
            data = hostsim_decompress(frame, 1 << 17)
        assert items_lib.zbi_staged_mode(frame, len(frame), len(data)) != 0, name
        assert staged_decompress(frame, len(data), emu=emu) == data, name
        assert staged_decompress(frame, len(data), emu=emu, misalign=5) == data, name
        cap = len(data)
        # every single-bit flip of the stored checksum
        for bit in range(32 if not emu else 8):
            b = bytearray(frame)
            b[len(b) - 4 + bit // 8] ^= 1 << (bit % 8)
            b = bytes(b)
            got = staged_decompress(b, cap, emu=emu)
            assert got == hostsim_decompress(b, cap) == -22, (name, bit)
        # seeded flips in the block
        rnd = random.Random(name)
        flips = 200 if not emu else 10
        for _ in range(flips):
            b = bytearray(frame)
            i = rnd.randrange(6, len(b) - 4)
            b[i] ^= 1 << rnd.randrange(8)
            b = bytes(b)
            assert staged_decompress(b, cap, emu=emu) == hostsim_decompress(b, cap), (name, i)


# ------------------------------------------------------------------------------------------------------------------------ GPU
def _ctx(pipeline: int):
    from zstd_jni_b200.zstd import ZstdBatchContext
    ctx = ZstdBatchContext(0)
    ctx.setOption("dec_pipeline", pipeline)
    return ctx


def _counters(ctx):
    from zstd_jni_b200 import _native
    L = _native.lib()
    return (L.zstdb200_split_items(ctx._live(), 0), L.zstdb200_split_items(ctx._live(), 1),
            L.zstdb200_segment_frames(ctx._live(), 0), L.zstdb200_segment_frames(ctx._live(), 1))


def _multi_block_frames(item: bytes) -> int:
    """Frames of more than one block in an item (by the reference's walk and a block count of each frame)."""
    frames, _ = _ref_walk(item)
    n = 0
    for off, size, _cs, skippable in frames:
        if skippable:
            continue
        f = item[off:off + size]
        fhd = f[4]
        did, single, fcs = fhd & 3, (fhd >> 5) & 1, fhd >> 6
        pos = 5 + (not single) + (4 if did == 3 else did) + ((1 << fcs) if fcs else 0) + (1 if single and not fcs else 0)
        blocks = 0
        while True:
            bh = int.from_bytes(f[pos:pos + 3], "little")
            pos += 3 + (1 if (bh >> 1) & 3 == 1 else bh >> 3)
            blocks += 1
            if bh & 1:
                break
        n += blocks >= 2
    return n


def _valid_items():
    """(name, item, content) of valid multi-frame items: compressChunks streams, ZstdCompressCtx's multi-frame output, ZstdOutputStream,
    concatenated reference frames (multi-block ones included), skippable and empty frames, a last frame without a content size."""
    from zstd_jni_b200.zstd import ZstdBatchContext, ZstdCompressCtx, ZstdOutputStream
    import io
    items = []
    ctx = ZstdBatchContext(0)
    for level in (1, 3, 19):
        for ck in (0, 1):
            data = _data(level + 50 * ck, 700_000 if level != 19 else 300_000)
            ctx.setOption("checksum", ck)
            chunk = 131072 if level < 19 else 65536          # (the optimal-parser levels take at most 64 KB)
            stream, _sizes = ctx.compressChunks(np.frombuffer(data, dtype=np.uint8), chunk, level)
            items.append((f"chunks-L{level}-ck{ck}", stream.tobytes(), data))
    ctx.setOption("checksum", 0)
    ctx.close()
    data = _data(77, 600_000)
    with ZstdCompressCtx() as cc:
        cc.setLevel(3)
        cc.setMultiFrame(True)
        items.append(("cctx-multiframe", cc.compress(data), data))
    sink = io.BytesIO()
    os_ = ZstdOutputStream(sink, 3)
    for k in range(0, len(data), 100_000):
        os_.write(data[k:k + 100_000])
        os_.flush()
    os_.close()
    items.append(("output-stream", sink.getvalue(), data))
    r = [(_data(200 + k, n), ck) for k, (n, ck) in enumerate([(40_000, 0), (131072, 1), (500_000, 0), (300_000, 1), (9, 0)])]
    frames = [ref_compress_flags(d, 3, checksum=bool(ck)) for d, ck in r]
    content = b"".join(d for d, _ in r)
    items.append(("ref-concat-with-multiblock", b"".join(frames), content))
    items.append(("ref-skippable-between", frames[0] + _skippable(10) + frames[1] + _skippable(0, 3) + frames[2] + _skippable(300),
                  r[0][0] + r[1][0] + r[2][0]))
    empty = ref_compress_flags(b"", 3)
    items.append(("ref-empty-frames", empty + frames[0] + empty + frames[1] + empty, r[0][0] + r[1][0]))
    last_unsized = ref_compress_flags(r[1][0], 3, content_size=False)
    items.append(("ref-last-unsized", frames[0] + frames[3] + last_unsized, r[0][0] + r[3][0] + r[1][0]))
    items.append(("ref-stream-multiblock-last", frames[0] + ref_stream_compress(r[2][0], 3), r[0][0] + r[2][0]))
    return items


@pytest.mark.gpu
def test_gpu_valid_multiframe_items():
    from zstd_jni_b200.zstd import Zstd, ZstdDecompressCtx
    items = _valid_items()
    single = [(ref_compress_flags(_data(900 + k, 60_000), 3), _data(900 + k, 60_000)) for k in range(3)]
    ctx = _ctx(1)
    for name, item, content in items:
        before = _counters(ctx)
        got = ctx.decompressBatch([single[0][0], item, single[1][0], item, single[2][0]],
                                  [len(single[0][1]), len(content), len(single[1][1]), len(content), len(single[2][1])])
        assert got[1] == content and got[3] == content, name
        assert [got[0], got[2], got[4]] == [s[1] for s in single], name
        after = _counters(ctx)
        assert after[0] == before[0] + 2 and after[1] == before[1], (name, before, after)
        mb = _multi_block_frames(item)
        assert after[2] == before[2] + 2 * mb and after[3] == before[3], (name, mb, before, after)
        assert Zstd.decompress(item, len(content)) == content, name
        with ZstdDecompressCtx() as dc:
            assert dc.decompress(item, len(content)) == content, name
            dst = bytearray(len(content) + 20)
            src = b"\xAA" * 7 + item + b"\xBB" * 3
            n = dc.decompressByteArray(dst, 11, len(content) + 9, src, 7, len(item))
            assert n == len(content) and bytes(dst[11:11 + n]) == content, name
    ctx.close()


def _damaged(item: bytes, content_len: int, rnd: random.Random):
    """(what, item, capacity) variants of a valid multi-frame item."""
    frames, _ = _ref_walk(item)
    out = []
    for k, (off, size, _cs, skippable) in enumerate(frames):
        for _ in range(3):
            b = bytearray(item)
            i = rnd.randrange(off, off + size)
            b[i] ^= 1 << rnd.randrange(8)
            out.append((f"flip-frame{k}-{i}", bytes(b), content_len))
        out.append((f"cut-{k}-", item[:off + size - 1], content_len))
        out.append((f"cut-{k}", item[:off + size], content_len))
        out.append((f"cut-{k}+", item[:off + size + 1], content_len))
    zs = [f for f in frames if not f[3]]
    mid = zs[len(zs) // 2]
    b = bytearray(item)
    b[mid[0] + mid[1] - 1] ^= 0x10            # the middle frame's stored checksum or its last block's last byte
    out.append(("middle-tail", bytes(b), content_len))
    fhd = item[mid[0] + 4]
    if fhd >> 6:                              # the middle frame's content size field +-1
        did, single = fhd & 3, (fhd >> 5) & 1
        p = mid[0] + 5 + (not single) + (4 if did == 3 else did)
        w = 1 << (fhd >> 6)
        v = int.from_bytes(item[p:p + w], "little")
        for d in (-1, 1):
            b = bytearray(item)
            b[p:p + w] = ((v + d) % (1 << (8 * w))).to_bytes(w, "little")
            out.append((f"middle-size{d:+d}", bytes(b), content_len))
    out.append(("trailing-garbage", item + b"\x00\x01\x02", content_len))
    for dc in (-1, 0, 1):
        out.append((f"capacity{dc:+d}", item, content_len + dc))
    return out


@pytest.mark.gpu
def test_gpu_damaged_items_equal_fused():
    items = _valid_items()
    picks = [it for it in items if it[0] in ("chunks-L3-ck1", "chunks-L1-ck0", "ref-concat-with-multiblock", "ref-skippable-between",
                                              "ref-last-unsized", "cctx-multiframe")]
    rnd = random.Random(11)
    new, old = _ctx(1), _ctx(0)
    compared = 0
    for name, item, content in picks:
        cases = _damaged(item, len(content), rnd)
        got = new.decompressBatch([c[1] for c in cases], [c[2] for c in cases], raise_on_error=False)
        want = old.decompressBatch([c[1] for c in cases], [c[2] for c in cases], raise_on_error=False)
        for (what, b, cap), g, w in zip(cases, got, want):
            assert g == w, (name, what)
            r = ref_decompress(b, cap)
            if isinstance(r, bytes) or isinstance(w, bytes):
                assert r == w, (name, what)
            else:
                # the documented exception: a damaged Huffman literal stream is corruption_detected here
                assert w == r or w == -20, (name, what, w, r)
            compared += 1
    assert compared > 100
    new.close(); old.close()


@pytest.mark.gpu
def test_gpu_items_too_small_to_split_stay_whole():
    """Items whose frames regenerate too little to pay for an entry each (16 384 empty frames, a run of 1 KB frames) are not split and
    give the dec_pipeline 0 result."""
    empty = ref_compress_flags(b"", 3)
    small = [_data(600 + k, 1000) for k in range(40)]
    items = [empty * 16384, b"".join(ref_compress_flags(d, 3) for d in small), empty * 3 + b"\x00"]
    caps = [0, 40_000, 0]
    new, old = _ctx(1), _ctx(0)
    before = _counters(new)
    got = new.decompressBatch(items, caps, raise_on_error=False)
    assert got == old.decompressBatch(items, caps, raise_on_error=False)
    assert got[0] == b"" and got[1] == b"".join(small)
    assert _counters(new)[:2] == before[:2]
    new.close(); old.close()


@pytest.mark.gpu
def test_gpu_checksummed_batches_equal_fused():
    from zstd_jni_b200.zstd import ZstdBatchContext
    n = 8192
    rng = np.random.default_rng(3)
    words = rng.integers(97, 123, size=(4096, 8), dtype=np.uint8)
    data = words[rng.integers(0, 4096, size=n * 131072 // 8)].reshape(-1)[: n * 131072].tobytes()
    ctx = ZstdBatchContext(0)
    ctx.setOption("checksum", 1)
    stream, sizes = ctx.compressChunks(np.frombuffer(data, dtype=np.uint8), 131072, 3)
    ctx.close()
    stream = stream.tobytes()
    offs = np.concatenate([[0], np.cumsum(sizes.astype(np.int64))])
    frames = [stream[offs[i]:offs[i + 1]] for i in range(n)]
    assert all((f[4] >> 2) & 1 for f in frames[:8])
    caps = [131072] * n
    ref_frames = [ref_compress_flags(_data(300 + k, 20_000 + 997 * k), level, checksum=True) for k, level in enumerate((1, 3, 9, 19))]
    rnd = random.Random(4)
    extra, extra_caps = [], []
    for f in ref_frames + frames[:16]:
        cap = 131072
        extra += [f]; extra_caps += [cap]
        b = bytearray(f); b[-1 - rnd.randrange(4)] ^= 1 << rnd.randrange(8); extra += [bytes(b)]; extra_caps += [cap]
        b = bytearray(f); i = rnd.randrange(8, len(f) - 4); b[i] ^= 1 << rnd.randrange(8); extra += [bytes(b)]; extra_caps += [cap]
    new, old = _ctx(1), _ctx(0)
    # the staged pipeline takes the checksummed frames: the fused kernel, which skips them, is left with almost nothing to do
    new.setOption("timing", 1)
    new.kernelTimes()
    assert b"".join(new.decompressBatch(frames, caps)) == data
    times = new.kernelTimes()
    new.setOption("timing", 0)
    assert times["k_decompress"][0] < 0.05 * times["k_dec_exec"][0], times
    got = new.decompressBatch(frames + extra, caps + extra_caps, raise_on_error=False)
    want = old.decompressBatch(frames + extra, caps + extra_caps, raise_on_error=False)
    assert b"".join(got[:n]) == data
    for k, (g, w) in enumerate(zip(got, want)):
        assert g == w, k
    assert sum(1 for g in got[n:] if g == -22) >= len(ref_frames) + 16 - 2
    new.close(); old.close()
