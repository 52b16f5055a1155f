"""The decode list (items of several frames cut into their frames), the segment decoder and the staged decoder behind every host-memory
decompression call, in both frame formats.

CPU: the host instantiation of the decoder's source (tests/hostsim/zb_hostsim_format.cpp, compiled by this module):
  - the magicless frame_walk / item_walk / seg_walk of frames with their magic number stripped list the same frames, and the same block
    refs 4 bytes earlier, as the walks of the original frames (golden multi-block fixtures, cross-frame items, magicless.json frames);
  - a magicless frame whose first four bytes read like a skippable magic number (0x184D2A5x) is walked and decoded as a frame;
  - the staged decoder on magicless single-block frames, valid and damaged, gives the fused decoder's bytes and error codes.
GPU: zstdb200_decompress_batch (dec_pipeline 1 and 0), zstdb200_decompress_frames (one and two slices) and
zstdb200_decompress_frames_begin/_end (two operations in flight) on the same valid, damaged and magicless items: identical bytes and
results, equal to the reference; the counters grow by what a host walk of the items predicts.
"""
from __future__ import annotations

import ctypes as C
import hashlib
import json
import random
import subprocess
from pathlib import Path

import numpy as np
import pytest

from tests.golden.make_golden import cross_frame_items, regenerate_input
from tests.oracle_util import (ERR_MAX, hostsim_compress_flags, hostsim_decompress_magicless, ref, ref_compress_flags, ref_decompress,
                               ref_decompress_magicless)

ROOT = Path(__file__).resolve().parent.parent
GOLDEN = ROOT / "tests" / "golden"
MAGICLESS = json.loads((GOLDEN / "magicless.json").read_text())
SPLIT_MIN_BYTES = 32768          # zb_decode_list.cuh: bytes regenerated per entry, on average, by an item that is split


@pytest.fixture(scope="module")
def flib(tmp_path_factory):
    src = ROOT / "tests" / "hostsim" / "zb_hostsim_format.cpp"
    so = tmp_path_factory.mktemp("hostsim_format") / "libzb_hostsim_format.so"
    subprocess.run(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-Wall", "-Wno-unused-function", "-x", "c++", str(src), "-o", str(so)],
                   check=True)
    L = C.CDLL(str(so))
    L.zbf_item_walk.restype = C.c_uint
    L.zbf_item_walk.argtypes = [C.c_char_p, C.c_size_t, C.c_ulonglong, C.c_uint, C.POINTER(C.c_ulonglong), C.c_uint, C.POINTER(C.c_int)]
    L.zbf_frame_walk.restype = C.c_uint
    L.zbf_frame_walk.argtypes = [C.c_char_p, C.c_size_t, C.c_uint, C.c_int, C.POINTER(C.c_ulonglong), C.c_uint, C.POINTER(C.c_uint)]
    L.zbf_staged.restype = C.c_size_t
    L.zbf_staged.argtypes = [C.c_void_p, C.c_size_t, C.c_char_p, C.c_size_t, C.c_uint, C.POINTER(C.c_uint)]
    return L


def item_walk(L, item: bytes, cap: int, magicless: bool):
    """([(srcOff, srcSize, contentSize, nBlocks, checksum, hasContentSize, skippable)], split)."""
    k = 4096
    out = (C.c_ulonglong * (7 * k))()
    split = C.c_int(0)
    n = L.zbf_item_walk(item, len(item), cap, 1 if magicless else 0, out, k, C.byref(split))
    return [tuple(out[7 * j: 7 * j + 7]) for j in range(min(n, k))], bool(split.value)


def frame_walk(L, item: bytes, magicless: bool, seg: bool = False):
    """(block count, [(header offset, header)], stored checksum)."""
    k = 1 << 16
    refs = (C.c_ulonglong * k)()
    xxh = C.c_uint(0)
    n = L.zbf_frame_walk(item, len(item), 1 if magicless else 0, 1 if seg else 0, refs, k, C.byref(xxh))
    return n, [(r & 0xFFFFFFFF, r >> 32) for r in refs[:n]], xxh.value


def staged(L, frame: bytes, cap: int, magicless: bool):
    out = C.create_string_buffer(max(cap, 1))
    mode = C.c_uint(0)
    n = L.zbf_staged(out, cap, frame, len(frame), 1 if magicless else 0, C.byref(mode))
    return (out.raw[:n] if n <= ERR_MAX else -((1 << 64) - n)), mode.value


def _data(seed: int, n: int) -> bytes:
    rnd = random.Random(seed)
    words = [bytes(rnd.choice(b"abcdefghij") for _ in range(rnd.randrange(2, 9))) for _ in range(200)]
    out = bytearray()
    while len(out) < n:
        out += rnd.choice(words) + b" "
    return bytes(out[:n])


def _frames_of(L, item: bytes):
    """The frames of an item of zstd frames (no skippable ones), by the magic-format walk."""
    frames, _ = item_walk(L, item, 1 << 40, False)
    assert sum(f[1] for f in frames) == len(item) and not any(f[6] for f in frames)
    return [item[f[0]:f[0] + f[1]] for f in frames]


def _magic_items(L):
    """(name, [frames with their magic number]) of zstd frames only: the golden multi-block fixtures, the cross-frame items, the frames
    of magicless.json (with the magic number put back)."""
    out = []
    for p in sorted(GOLDEN.glob("mb_*.zst")):
        z = p.read_bytes()
        frames, _ = item_walk(L, z, 1 << 40, False)
        if any(f[6] for f in frames):
            continue                  # (a skippable frame has no magicless form)
        out.append((p.name, [z[f[0]:f[0] + f[1]] for f in frames]))
    for name, item, _cap, _code in cross_frame_items():
        out.append((name, _frames_of(L, item)))
    for e in MAGICLESS["frames"]:
        z = hostsim_compress_flags(regenerate_input(e["input"]), e["level"], e["checksum"], e["content_size"], magicless=True)
        assert hashlib.sha256(z).hexdigest() == e["sha256"]
        out.append((f"magicless-L{e['level']}-{e['checksum']}-{e['content_size']}", [bytes.fromhex("28b52ffd") + z]))
    return out


def test_magicless_walks_match_magic_walks(flib):
    items = _magic_items(flib)
    assert len(items) >= 12 and any(len(f) >= 2 for _, f in items)
    for name, frames in items:
        assert all(f[:4] == bytes.fromhex("28b52ffd") for f in frames), name
        item, bare = b"".join(frames), b"".join(f[4:] for f in frames)
        for cap in (1 << 40, 0):
            want, wsplit = item_walk(flib, item, cap, False)
            got, gsplit = item_walk(flib, bare, cap, True)
            assert len(got) == len(want) == len(frames) and gsplit == wsplit, (name, cap)
            for k, (g, w) in enumerate(zip(got, want)):
                assert g == (w[0] - 4 * k, w[1] - 4) + w[2:], (name, k)
        # the magicless walk does not take the frames with their magic number (it reads 0x28 as a descriptor with the reserved bit set)
        assert item_walk(flib, item, 1 << 40, True)[0] == []
        for f in frames:
            for seg in (False, True):
                n, refs, xxh = frame_walk(flib, f, False, seg)
                m, mrefs, mxxh = frame_walk(flib, f[4:], True, seg)
                assert (m, mxxh) == (n, xxh) and mrefs == [(o - 4, h) for o, h in refs], (name, seg)
                assert frame_walk(flib, f[4:], False, seg)[0] == 0
                assert n >= 1 or seg, name


def _lookalike(data: bytes) -> bytes:
    """A magicless frame of `data` (6477 bytes) whose first four bytes read 0x184D2A50, a skippable magic number: descriptor 0x50 (2-byte
    content size, window byte), window byte 0x2A (40 KB), content size 0x184D + 256 = 6477, then the blocks of a frame of the same
    content."""
    assert len(data) == 6477
    z = hostsim_compress_flags(data, 3)
    fhd = z[4]
    assert fhd == 0x60 and (fhd >> 5) & 1          # one-shot: single segment, 2-byte content size
    return bytes([0x50, 0x2A, 0x4D, 0x18]) + z[7:]


def test_skippable_lookalike_is_a_frame(flib):
    data = _data(31, 6477)
    f = _lookalike(data)
    assert int.from_bytes(f[:4], "little") == 0x184D2A50
    frames, split = item_walk(flib, f, len(data), True)
    assert frames == [(0, len(f), 6477, 1, 0, 1, 0)] and not split
    two, split = item_walk(flib, f + f, 2 * len(data), True)
    assert [x[0] for x in two] == [0, len(f)] and split
    # the magic-format walk reads a skippable frame (of a length the item does not hold)
    assert item_walk(flib, f, len(data), False)[0] == []
    n, refs, _ = frame_walk(flib, f, True)
    assert n == 1 and refs[0][0] == 4
    got, mode = staged(flib, f, len(data), True)
    assert mode != 0 and got == data == hostsim_decompress_magicless(f, len(data))
    assert hostsim_decompress_magicless(f + f, 2 * len(data)) == data + data
    if ref() is not None:
        assert ref_decompress_magicless(f, len(data)) == data
        assert ref_decompress_magicless(f + f, 2 * len(data)) == data + data


def _magicless_single_block():
    out = []
    for e in MAGICLESS["frames"]:
        data = regenerate_input(e["input"])
        out.append((f"golden-L{e['level']}", hostsim_compress_flags(data, e["level"], e["checksum"], e["content_size"], magicless=True), data))
    for k, (n, level, ck) in enumerate([(37, 1, False), (4000, 3, True), (65536, 3, False), (131072, 1, True), (100_000, 9, False)]):
        data = _data(40 + k, n)
        out.append((f"own-L{level}-{n}", hostsim_compress_flags(data, level, checksum=ck, magicless=True), data))
    out.append(("lookalike", _lookalike(_data(31, 6477)), _data(31, 6477)))
    return out


def test_staged_magicless_equals_fused(flib):
    rnd = random.Random(7)
    taken = 0
    for name, f, data in _magicless_single_block():
        cap = len(data)
        got, mode = staged(flib, f, cap, True)
        assert got == data == hostsim_decompress_magicless(f, cap), name
        taken += mode != 0
        # the same frame in the other format is not the staged decoder's
        assert staged(flib, f, cap, False)[1] == 0
        for _ in range(60):
            b = bytearray(f)
            i = rnd.randrange(len(b))
            b[i] ^= 1 << rnd.randrange(8)
            b = bytes(b)
            assert staged(flib, b, cap, True)[0] == hostsim_decompress_magicless(b, cap), (name, i)
        for cut in (len(f) - 1, len(f) // 2):
            assert staged(flib, f[:cut], cap, True)[0] == hostsim_decompress_magicless(f[:cut], cap), (name, cut)
        assert staged(flib, f, cap - 1, True)[0] == hostsim_decompress_magicless(f, cap - 1), name
    # every frame with a content size is the staged decoder's
    assert taken >= len(_magicless_single_block()) - sum(1 for e in MAGICLESS["frames"] if not e["content_size"])


# ------------------------------------------------------------------------------------------------------------------------ GPU
def _lib():
    from zstd_jni_b200 import _native
    return _native.lib()


def _ctx(pipeline: int = 1, magicless: int = 0):
    from zstd_jni_b200.zstd import ZstdBatchContext
    ctx = ZstdBatchContext(0)
    ctx.setOption("dec_pipeline", pipeline)
    ctx.setOption("magicless", magicless)
    return ctx


def _counters(ctx):
    L = _lib()
    return (L.zstdb200_split_items(ctx._live(), 0), L.zstdb200_split_items(ctx._live(), 1),
            L.zstdb200_segment_frames(ctx._live(), 0), L.zstdb200_segment_frames(ctx._live(), 1))


def _results(out: np.ndarray, offs, res):
    """Per item: its bytes, or the negative error code."""
    return [out[offs[i]:offs[i] + r].tobytes() if r <= ERR_MAX else -((1 << 64) - r) for i, r in enumerate(res)]


def call_batch(ctx, items, caps):
    return ctx.decompressBatch(items, caps, raise_on_error=False)


def call_frames(ctx, items, caps, slices):
    ctx.setOption("host_slices_dec", slices)
    stream = np.frombuffer(b"".join(items), dtype=np.uint8)
    out = np.zeros(max(sum(caps), 1), dtype=np.uint8)
    n = len(items)
    fs = (C.c_size_t * n)(*[len(x) for x in items])
    ds = (C.c_size_t * n)(*caps)
    _lib().zstdb200_decompress_frames(ctx._live(), C.c_void_p(stream.ctypes.data), fs, n, C.c_void_p(out.ctypes.data), sum(caps), ds)
    ctx.setOption("host_slices_dec", 2)
    return _results(out, np.concatenate([[0], np.cumsum(caps)]).astype(np.int64), list(ds))


def call_begin_end(ctx, items, caps, slots=(1, 3)):
    """Two operations in flight: the first half of the items on one slot, the second half on another, both begun before either ends."""
    L = _lib()
    h = len(items) // 2
    parts = [(items[:h], caps[:h]), (items[h:], caps[h:])]
    keep = []
    for slot, (its, cs) in zip(slots, parts):
        stream = np.frombuffer(b"".join(its) or b"\x00", dtype=np.uint8)
        out = np.zeros(max(sum(cs), 1), dtype=np.uint8)
        fs = (C.c_size_t * len(its))(*[len(x) for x in its])
        ds = (C.c_size_t * len(its))(*cs)
        r = L.zstdb200_decompress_frames_begin(ctx._live(), slot, C.c_void_p(stream.ctypes.data), fs, len(its), C.c_void_p(out.ctypes.data),
                                               sum(cs), ds)
        assert r <= ERR_MAX, r
        keep.append((stream, out, fs, ds, cs))
    got = []
    for slot, (stream, out, fs, ds, cs) in zip(slots, keep):
        res = (C.c_size_t * len(cs))()
        L.zstdb200_decompress_frames_end(ctx._live(), slot, res)
        got += _results(out, np.concatenate([[0], np.cumsum(cs)]).astype(np.int64), list(res))
    return got


def call_device(ctx, items, caps):
    import torch
    L = _lib()
    dev = torch.device("cuda:0")
    so = np.concatenate([[0], np.cumsum([len(x) for x in items])]).astype(np.int64)
    do = np.concatenate([[0], np.cumsum(caps)]).astype(np.int64)
    d_src = torch.from_numpy(np.frombuffer(b"".join(items), dtype=np.uint8).copy()).to(dev)
    d_so, d_do = torch.from_numpy(so).to(dev), torch.from_numpy(do).to(dev)
    d_dst = torch.zeros(max(int(do[-1]), 1), dtype=torch.uint8, device=dev)
    d_res = torch.zeros(len(items), dtype=torch.int64, device=dev)
    s = torch.cuda.Stream()
    assert L.zstdb200_decompress_device(ctx.handle, len(items), d_src.data_ptr(), d_so.data_ptr(), d_dst.data_ptr(), d_do.data_ptr(),
                                        d_res.data_ptr(), s.cuda_stream) == 0
    s.synchronize()
    res = [int(x) & ((1 << 64) - 1) for x in d_res.cpu().numpy()]
    return _results(d_dst.cpu().numpy(), do, res)


CALLS = [("batch", lambda c, i, k: call_batch(c, i, k)), ("frames-1", lambda c, i, k: call_frames(c, i, k, 1)),
         ("frames-2", lambda c, i, k: call_frames(c, i, k, 2)), ("begin-end", lambda c, i, k: call_begin_end(c, i, k))]


def _predict(L, item: bytes, cap: int, magicless: bool = False):
    """(items split, frames on the segment decoder) that a host walk of the item predicts: the decode list's rule (zb_decode_list.cuh),
    and seg_walk of each entry."""
    frames, split = item_walk(L, item, cap, magicless)
    if split:
        zs = [f for f in frames if not f[6]]
        regen = sum(f[2] for f in zs) if all(f[5] for f in zs) else cap
        split = regen // len(frames) >= SPLIT_MIN_BYTES
    if split:
        return 1, sum(1 for f in frames if frame_walk(L, item[f[0]:f[0] + f[1]], magicless, seg=True)[0])
    return 0, 1 if frame_walk(L, item, magicless, seg=True)[0] else 0


def _gpu_items():
    """(name, item, content) of valid items: reference multi-block fixtures (checksummed ones among them), compressChunks streams,
    ZstdCompressCtx's multi-frame output, ZstdOutputStream, skippable frames, a last frame without a content size, the cross-frame item
    that decodes, and 128 KB frames."""
    from tests.test_multiframe_items import _valid_items
    items = []
    for p in sorted(GOLDEN.glob("mb_*.zst")):
        z = p.read_bytes()
        d = ref_decompress(z, 1 << 24)
        assert isinstance(d, bytes), p.name
        items.append((p.name, z, d))
    for name, item, cap, code in cross_frame_items():
        if code is None:
            d = ref_decompress(item, cap)
            assert isinstance(d, bytes)
            items.append((name, item, d))
    items += _valid_items()
    return items


def _ordinary(n: int):
    from zstd_jni_b200 import corpus
    from zstd_jni_b200.zstd import ZstdBatchContext
    data = corpus.corpus(n, size=131072).reshape(-1)
    with ZstdBatchContext(0) as c:
        stream, sizes = c.compressChunks(data, 131072, 3)
    offs = np.concatenate([[0], np.cumsum(sizes.astype(np.int64))])
    s = stream.tobytes()
    return [(f"chunk-{i}", s[offs[i]:offs[i + 1]], data[i * 131072:(i + 1) * 131072].tobytes()) for i in range(n)]


def _compare_calls(items, caps, magicless: int = 0, expect=None):
    """Every call on the items; each call's results, the dec_pipeline 0 batch's first.  Returns them by call name."""
    old, new = _ctx(0, magicless), _ctx(1, magicless)
    want = call_batch(old, items, caps)
    got = {"batch-fused": want}
    for name, call in CALLS:
        got[name] = call(new, items, caps)
    old.close(); new.close()
    for name, g in got.items():
        for k, (a, b) in enumerate(zip(g, want)):
            assert a == b, (name, k, a if isinstance(a, int) else len(a), b if isinstance(b, int) else len(b))
    return got


@pytest.mark.gpu
def test_gpu_calls_agree_and_count(flib):
    mix = _gpu_items()
    plain = _ordinary(512)
    items = [m[1] for m in mix] + [p[1] for p in plain]
    caps = [len(m[2]) for m in mix] + [len(p[2]) for p in plain]
    want = [m[2] for m in mix] + [p[2] for p in plain]
    assert len(items) >= 512 + 20
    got = _compare_calls(items, caps)
    for k, w in enumerate(want):
        assert got["batch"][k] == w, (k, items[k][:8])
    # the counters: each call splits the items the host walk predicts and decodes their frames of many blocks on segments, none deferred
    split, seg = 0, 0
    for item, cap in zip(items, caps):
        a, b = _predict(flib, item, cap)
        split += a; seg += b
    assert split >= 10 and seg >= 5
    ctx = _ctx(1)
    for name, call in CALLS:
        before = _counters(ctx)
        assert call(ctx, items, caps) == want, name
        after = _counters(ctx)
        assert (after[0] - before[0], after[1] - before[1], after[2] - before[2], after[3] - before[3]) == (split, 0, seg, 0), (name, before, after)
    ctx.close()


def _wrong_checksum(z: bytes) -> bytes:
    b = bytearray(z)
    b[-2] ^= 0x40
    return bytes(b)


@pytest.mark.gpu
def test_gpu_damaged_items_equal_fused_in_every_call():
    from tests.test_multiframe_items import _damaged, _valid_items
    rnd = random.Random(23)
    picks = [it for it in _valid_items() if it[0] in ("chunks-L3-ck1", "ref-concat-with-multiblock", "ref-skippable-between",
                                                       "ref-last-unsized", "output-stream")]
    cases = []
    for name, item, content in picks:
        cases += [(f"{name}:{what}", b, cap) for what, b, cap in _damaged(item, len(content), rnd)]
    # a wrong stored checksum on a frame of many blocks: alone, and inside a split item
    xxh = (GOLDEN / "mb_L3_xxh.zst").read_bytes()
    xd = ref_decompress(xxh, 1 << 24)
    cases.append(("mb_L3_xxh:checksum", _wrong_checksum(xxh), len(xd)))
    big = ref_compress_flags(_data(5, 300_000), 3, checksum=True)
    lead = ref_compress_flags(_data(6, 100_000), 3)
    cases.append(("split:checksum", lead + _wrong_checksum(big), 400_000))
    cases.append(("split:checksum-valid", lead + big, 400_000))
    cross = cross_frame_items()
    cases += [(name, item, cap) for name, item, cap, _code in cross]
    items, caps = [c[1] for c in cases], [c[2] for c in cases]
    got = _compare_calls(items, caps)
    for (name, item, cap), g in zip(cases, got["batch"]):
        r = ref_decompress(item, cap)
        # (the documented exception: a damaged Huffman literal stream is corruption_detected here)
        assert g == r or g == -20, (name, g if isinstance(g, int) else len(g), r if isinstance(r, int) else len(r))
    k = len(cases) - len(cross)
    assert got["batch"][k - 1] == _data(6, 100_000) + _data(5, 300_000) and got["batch"][k - 2] == -22 and got["batch"][k - 3] == -22


def _magicless_items():
    """(name, item, content) in the magicless format: compressChunks frames and streams, reference frames of one and of many blocks,
    their concatenation, the skippable lookalike."""
    from zstd_jni_b200.zstd import ZstdBatchContext
    out = []
    data = _data(61, 900_000)
    with ZstdBatchContext(0) as c:
        c.setOption("magicless", 1)
        for ck in (0, 1):
            c.setOption("checksum", ck)
            stream, sizes = c.compressChunks(np.frombuffer(data, dtype=np.uint8), 131072, 3)
            s = stream.tobytes()
            offs = np.concatenate([[0], np.cumsum(sizes.astype(np.int64))])
            out.append((f"chunks-ck{ck}", s, data))
            out += [(f"chunk-ck{ck}-{i}", s[offs[i]:offs[i + 1]], data[i * 131072:(i + 1) * 131072]) for i in range(len(sizes))]
    for k, (n, ck) in enumerate([(5000, False), (131072, True), (400_000, False), (700_000, True)]):
        d = _data(70 + k, n)
        z = ref_compress_flags(d, 3, checksum=ck, magicless=True)
        assert isinstance(z, bytes) and ref_decompress_magicless(z, n) == d
        out.append((f"ref-{n}-ck{int(ck)}", z, d))
    out.append(("ref-concat", out[-1][1] + out[-3][1] + out[-4][1], out[-1][2] + out[-3][2] + out[-4][2]))
    la = _data(31, 6477)
    out.append(("lookalike", _lookalike(la), la))
    out.append(("lookalike-twice-and-ref", _lookalike(la) + _lookalike(la) + out[-3][1], la + la + out[-3][2]))
    return out


@pytest.mark.gpu
def test_gpu_magicless_items_on_the_parallel_decoders(flib):
    mix = _magicless_items()
    items, caps, want = [m[1] for m in mix], [len(m[2]) for m in mix], [m[2] for m in mix]
    for (name, item, content) in mix:
        assert ref_decompress_magicless(item, len(content)) == content, name
    got = _compare_calls(items, caps, magicless=1)
    assert got["batch"] == want
    # damaged: bit flips and cuts, the same results as the fused kernel in every call
    rnd = random.Random(5)
    bad, bcaps = [], []
    for (name, item, content) in mix:
        for _ in range(3):
            b = bytearray(item); b[rnd.randrange(len(b))] ^= 1 << rnd.randrange(8); bad.append(bytes(b)); bcaps.append(len(content))
        bad.append(item[:-1]); bcaps.append(len(content))
    _compare_calls(bad, bcaps, magicless=1)
    # the frames of many blocks go to the segment decoder, in every call; the device call takes the single-block frames on the staged
    # decoder
    seg = sum(_predict(flib, it, cap, True)[1] for it, cap in zip(items, caps))
    assert seg >= 4
    ctx, old = _ctx(1, 1), _ctx(0, 1)
    for name, call in CALLS:
        before = _counters(ctx)
        assert call(ctx, items, caps) == want, name
        assert _counters(ctx)[2] - before[2] == seg and _counters(ctx)[3] == before[3], name
    singles = [k for k, (name, _i, _c) in enumerate(mix) if name.startswith("chunk-") or name in ("ref-5000-ck0", "ref-131072-ck1", "lookalike")]
    si, sc = [items[k] for k in singles], [caps[k] for k in singles]
    assert call_device(ctx, si, sc) == [want[k] for k in singles] == call_device(old, si, sc)
    sb, sbc = bad[:len(bad) // 2], bcaps[:len(bcaps) // 2]
    assert call_device(ctx, sb, sbc) == call_device(old, sb, sbc)
    ctx.close(); old.close()


@pytest.mark.gpu
def test_gpu_magicless_single_block_batch_is_staged():
    """8192 magicless single-block frames: the staged decoder takes them, the fused kernel is left with almost nothing to do."""
    from zstd_jni_b200.zstd import ZstdBatchContext
    n = 8192
    rng = np.random.default_rng(3)
    words = rng.integers(97, 123, size=(4096, 8), dtype=np.uint8)
    data = words[rng.integers(0, 4096, size=n * 131072 // 8)].reshape(-1)[: n * 131072].tobytes()
    with ZstdBatchContext(0) as c:
        c.setOption("magicless", 1)
        stream, sizes = c.compressChunks(np.frombuffer(data, dtype=np.uint8), 131072, 3)
    stream = stream.tobytes()
    offs = np.concatenate([[0], np.cumsum(sizes.astype(np.int64))])
    frames = [stream[offs[i]:offs[i + 1]] for i in range(n)]
    assert frames[0][:4] != bytes.fromhex("28b52ffd")
    caps = [131072] * n
    new = _ctx(1, 1)
    new.setOption("timing", 1)
    new.kernelTimes()
    assert b"".join(new.decompressBatch(frames, caps)) == data
    times = new.kernelTimes()
    new.setOption("timing", 0)
    assert times["k_decompress"][0] < 0.05 * times["k_dec_exec"][0], times
    new.close()
