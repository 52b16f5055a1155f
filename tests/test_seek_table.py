"""Seek tables (the seekable format): written by zstdb200_compress_items_device with option seek_table, and read by
zstdb200_decompress_ranges_device to locate the frames that hold a range without walking the frames before it.

The module holds a plain-Python writer and reader of the table, built from the format: an item's frames, then a skippable frame of
magic 0x184D2A5E whose content is one entry per frame -- Compressed_Size, Decompressed_Size, and the low 32 bits of the frame's XXH64
when the descriptor's bit 7 is set -- then Number_Of_Frames, the descriptor and 0x8F92EAB1.  Frames and decoding come from the compiled
reference (oracle/_ref).

CPU: the host instantiation of both sides (tests/hostsim/zb_hostsim_seek.cpp): the compress plan over stand-in frames against the
model's layout, with and without checksums and for items of 0, 1, 2 and many chunks; the capacity sum and the 0x8000000-entry limit at
the planning functions; the table's structural checks, one failure each; and the ranges call located through tables -- on one lane and
on the emulated 32-lane warp -- at every entry boundary and one byte either side, in parts of 3 entries, against the model.
GPU: compress_items_device with tables at levels 1, 3 and 19 against the option-off streams and the model's tables, decoded whole by
the reference and by decompress_items_device; the ranges call with tables against the same call without them; foreign seekable items
whose frames declare no content size; damaged tables; dec_pipeline 0; and the magicless refusals.
"""
from __future__ import annotations

import ctypes as C
import random
import struct
import subprocess
from pathlib import Path

import numpy as np
import pytest

from tests import frame_writer as fw
from tests.oracle_util import ERR_MAX, ref, ref_compress_flags, ref_decompress, ref_stream_compress
from tests.test_device_ranges import UNKNOWN, _data, model, ref_frame

ROOT = Path(__file__).resolve().parent.parent
U64 = C.c_ulonglong
M64 = (1 << 64) - 1
BLOCK = 128 << 10
SKIPPABLE_MAGIC, SEEKABLE_MAGIC, FRAMES_MAX = 0x184D2A5E, 0x8F92EAB1, 0x8000000
E_CORRUPTION, E_CHECKSUM, E_PARAMETER_UNSUPPORTED, E_DST_SIZE_TOO_SMALL, E_FRAME_INDEX_TOO_LARGE = 20, 22, 40, 70, 100


def err(code):
    return (1 << 64) - code


def _code(r):
    return (1 << 64) - r if r > ERR_MAX else 0


# ---------------------------------------------------------------------------------------------------------------------------- the model
def write_table(entries, checksum: bool) -> bytes:
    """The table of entries (compressed size, decompressed size, checksum)."""
    body = b"".join(struct.pack("<II", c, d) + (struct.pack("<I", x) if checksum else b"") for c, d, x in entries)
    return struct.pack("<II", SKIPPABLE_MAGIC, len(body) + 9) + body + struct.pack("<IBI", len(entries), 0x80 if checksum else 0, SEEKABLE_MAGIC)


def read_table(item: bytes):
    """(entries, checksum) of the item's table when it is valid by every rule, the entries' sum included; else None."""
    if len(item) < 17 or struct.unpack_from("<I", item, len(item) - 4)[0] != SEEKABLE_MAGIC:
        return None
    k, desc = struct.unpack_from("<IB", item, len(item) - 9)
    if desc & 0x7C or k > FRAMES_MAX:
        return None
    E = 12 if desc & 0x80 else 8
    T = 8 + E * k + 9
    if T > len(item):
        return None
    magic, fsize = struct.unpack_from("<II", item, len(item) - T)
    if magic != SKIPPABLE_MAGIC or fsize != E * k + 9:
        return None
    entries = [struct.unpack_from("<II", item, len(item) - T + 8 + E * j) + ((struct.unpack_from("<I", item, len(item) - T + 16 + E * j)[0],)
               if E == 12 else (0,)) for j in range(k)]
    if sum(e[0] for e in entries) != len(item) - T:
        return None
    return entries, E == 12


def xxh32_low(data: bytes) -> int:
    """The low 32 bits of XXH64 (seed 0): the content checksum the reference writes for data."""
    return struct.unpack("<I", ref_compress_flags(data, 1, checksum=True)[-4:])[0]


def seekable(frames_and_contents, checksum: bool) -> bytes:
    """Frames followed by the table that lists them; each given as (frame, its content or None for a skippable frame)."""
    entries = [(len(f), len(c or b""), xxh32_low(c or b"") if checksum else 0) for f, c in frames_and_contents]
    return b"".join(f for f, _ in frames_and_contents) + write_table(entries, checksum)


def model_seek(items, reqs):
    """Per request: the bytes or negative code the call returns with seek tables -- through the table when the item has a valid one,
    else walked (test_device_ranges.model)."""
    out = []
    for i, b, ln in reqs:
        t = read_table(items[i]) if i < len(items) and ln else None
        if t is None:
            out.append(model(items, [(i, b, ln)])[0])
            continue
        entries, checksum = t
        x, e, pos, at, got, fail = items[i], b + ln, 0, 0, [], None
        for cs, ds, xx in entries:
            if at >= e:
                break
            if ds == 0 or at + ds <= b:
                pos, at = pos + cs, at + ds
                continue
            if (at < b or at + ds > e) and ds > BLOCK:
                fail = -E_PARAMETER_UNSUPPORTED
                break
            f = ref_frame(x[pos:], False)
            if isinstance(f, int):
                fail = f
                break
            size, fcs, skippable = f
            if skippable or size != cs or (fcs != UNKNOWN and fcs != ds):
                fail = -E_CORRUPTION
                break
            d = ref_decompress(x[pos:pos + cs], ds)
            if isinstance(d, int) or len(d) != ds:
                fail = d if isinstance(d, int) else -E_CORRUPTION
                break
            if checksum and xxh32_low(d) != xx:
                fail = -E_CHECKSUM
                break
            got.append(d[max(b - at, 0):min(e, at + ds) - at])
            pos, at = pos + cs, at + ds
        out.append(fail if fail is not None else b"".join(got))
    return out


def entry_ranges(i, item, reach=2):
    """Requests at every entry boundary of the item's table and one byte either side: empty, one byte, to the next `reach` boundaries
    +-1, to the end and past it."""
    t = read_table(item)
    marks = [0]
    for _, ds, _ in t[0]:
        marks.append(marks[-1] + ds)
    end = marks[-1]
    points = sorted({p for m in marks for p in (m - 1, m, m + 1) if p >= 0} | {end + 3})
    reqs = set()
    for p in points:
        ends = {p, p + 1, end, end + 7} | {q + d for q in [m for m in marks if m > p][:reach] for d in (-1, 0, 1)}
        reqs |= {(i, p, q - p) for q in ends if q >= p}
    return sorted(reqs)


def _needs_ref():
    if ref() is None:
        pytest.skip("the compiled reference (oracle/_ref) is not built")


def compress_bound(n):
    return n + (n >> 8) + ((BLOCK - n) >> 11 if n < BLOCK else 0)


def chunks_of(size, cs):
    return [min(cs, size - a) for a in range(0, size, cs)] or [0]


def seek_capacity(sizes, cs, checksum):
    E = 12 if checksum else 8
    return sum(sum(compress_bound(c) for c in chunks_of(s, cs)) + 17 + E * len(chunks_of(s, cs)) for s in sizes)


# ---------------------------------------------------------------------------------------------------------------------------- CPU
@pytest.fixture(scope="module")
def seek_lib(tmp_path_factory):
    src = ROOT / "tests" / "hostsim" / "zb_hostsim_seek.cpp"
    so = tmp_path_factory.mktemp("zb_hostsim_seek") / "libzb_hostsim_seek.so"
    subprocess.run(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-Wall", "-Wno-unused-function", "-x", "c++", str(src), "-o", str(so)],
                   check=True)
    L = C.CDLL(str(so))
    P64 = C.POINTER(U64)
    L.zbs_citem_item.restype = None
    L.zbs_citem_item.argtypes = [U64, U64, C.c_uint, P64]
    L.zbs_citems.restype = None
    L.zbs_citems.argtypes = [P64, C.c_size_t, U64, U64, C.c_uint, C.c_uint, P64, C.POINTER(C.c_uint), C.c_char_p, P64, P64]
    L.zbs_table_read.restype = C.c_int
    L.zbs_table_read.argtypes = [C.c_char_p, C.c_size_t, P64]
    L.zbs_ranges.restype = None
    L.zbs_ranges.argtypes = [C.c_char_p, P64, C.c_size_t, C.c_size_t, P64, P64, P64, C.c_uint, C.c_uint, C.c_int, C.c_char_p, P64, P64]
    return L


def _arr(v):
    return (U64 * max(len(v), 1))(*v)


def host_citems(L, sizes, cs, frames, xxh, E, capacity=None, P=3):
    """The host plan: (output bytes up to the end offset, offsets, results)."""
    if capacity is None:
        capacity = seek_capacity(sizes, cs, E == 12) if E else sum(sum(compress_bound(c) for c in chunks_of(s, cs)) for s in sizes)
    out = C.create_string_buffer(b"\xee" * capacity, max(capacity, 1))
    do, res = _arr([0] * (len(sizes) + 1)), _arr([0] * len(sizes))
    L.zbs_citems(_arr(sizes), len(sizes), cs, capacity, P, E, _arr(frames), (C.c_uint * max(len(xxh), 1))(*xxh), out, do, res)
    return out.raw[:do[len(sizes)]], list(do), list(res)


def model_citems(sizes, cs, frames, xxh, checksum):
    """The stream the plan writes for stand-in frames: per item its frames (chunk j's: its byte j & 0xFF, the last four its xxh with
    checksums), then its table."""
    out, j = [], 0
    for s in sizes:
        entries, body = [], b""
        for c in chunks_of(s, cs):
            f = bytes([j & 0xFF]) * frames[j]
            if checksum:
                f = f[:-4] + struct.pack("<I", xxh[j])
            body += f
            entries.append((frames[j], c, xxh[j] if checksum else 0))
            j += 1
        out.append(body + write_table(entries, checksum))
    return out


@pytest.mark.parametrize("checksum", [False, True])
def test_citem_tables_layout(seek_lib, checksum):
    cs = 100
    sizes = [0, 1, 100, 101, 200, 999, 0, 5000, 37]       # 0, 1, 2 and many chunks, exact multiples, empty items between
    rnd = random.Random(7)
    frames = [rnd.randrange(9, compress_bound(c) + 1) for s in sizes for c in chunks_of(s, cs)]
    xxh = [rnd.randrange(1 << 32) for _ in frames]
    E = 12 if checksum else 8
    for P in (3, 4, 64):
        out, do, res = host_citems(seek_lib, sizes, cs, frames, xxh, E, P=P)
        want = model_citems(sizes, cs, frames, xxh, checksum)
        assert out == b"".join(want), P
        assert res == [len(w) for w in want] and do == list(np.cumsum([0] + [len(w) for w in want]))
        for w in want:
            t = read_table(w)
            assert t is not None and t[1] == checksum
    if not checksum:      # without tables the same plan packs the frames alone
        out0, _, res0 = host_citems(seek_lib, sizes, cs, frames, xxh, 0)
        assert out0 == b"".join(w[:-(17 + 8 * len(chunks_of(s, cs)))] for w, s in zip(want, sizes))
        assert res0 == [len(w) - 17 - 8 * len(chunks_of(s, cs)) for w, s in zip(want, sizes)]


def test_citem_failures_and_capacity(seek_lib):
    cs, sizes = 100, [250, 50, 0, 300]
    m = sum(len(chunks_of(s, cs)) for s in sizes)
    frames, xxh = [40 + j for j in range(m)], [j * 77 for j in range(m)]
    cap = seek_capacity(sizes, cs, False)
    bad = list(frames)
    bad[1] = err(E_PARAMETER_UNSUPPORTED)      # item 0's second frame fails; the others keep their tables
    out, do, res = host_citems(seek_lib, sizes, cs, bad, xxh, 8)
    want = model_citems(sizes, cs, frames, xxh, False)
    assert res[0] == err(E_PARAMETER_UNSUPPORTED) and res[1:] == [len(w) for w in want[1:]]
    for i in (1, 2, 3):
        assert out[do[i]:do[i + 1]] == want[i]
    _, do, res = host_citems(seek_lib, sizes, cs, frames, xxh, 8, capacity=cap)
    assert res == [len(w) for w in want]
    _, do, res = host_citems(seek_lib, sizes, cs, frames, xxh, 8, capacity=cap - 1)
    assert res == [err(E_DST_SIZE_TOO_SMALL)] * 4 and do == [0] * 5


def test_capacity_sum_and_frame_limit(seek_lib):
    out = _arr([0] * 4)
    for size, cs in ((0, 100), (1, 100), (100, 100), (101, 100), (5 * BLOCK + 3, BLOCK), (10_000, 1000)):
        for E in (8, 12):
            seek_lib.zbs_citem_item(size, cs, E, out)
            k = len(chunks_of(size, cs))
            assert list(out) == [k, sum(compress_bound(c) for c in chunks_of(size, cs)) + 17 + E * k, 17 + E * k, M64], (size, cs, E)
        seek_lib.zbs_citem_item(size, cs, 0, out)
        assert out[2] == 0 and out[3] == M64 and out[1] == sum(compress_bound(c) for c in chunks_of(size, cs))
    seek_lib.zbs_citem_item(FRAMES_MAX, 1, 8, out)                 # the most entries a table holds
    assert out[0] == FRAMES_MAX and out[2] == 17 + 8 * FRAMES_MAX and out[3] == M64
    seek_lib.zbs_citem_item(FRAMES_MAX + 1, 1, 12, out)            # one more: the item fails, no table
    assert out[0] == FRAMES_MAX + 1 and out[2] == 0 and out[3] == E_FRAME_INDEX_TOO_LARGE
    seek_lib.zbs_citem_item(FRAMES_MAX + 1, 1, 0, out)
    assert out[3] == M64


def test_table_validity(seek_lib):
    frames = [b"x" * 10, b"y" * 20]
    good = b"".join(frames) + write_table([(10, 5, 0), (20, 7, 0)], False)
    t = _arr([0] * 3)
    assert seek_lib.zbs_table_read(good, len(good), t) == 1 and list(t) == [30 + 8, 2, 8]
    goodx = b"".join(frames) + write_table([(10, 5, 1), (20, 7, 2)], True)
    assert seek_lib.zbs_table_read(goodx, len(goodx), t) == 1 and list(t) == [38, 2, 12]
    empty = write_table([], False)
    assert seek_lib.zbs_table_read(empty, 17, t) == 1 and list(t) == [8, 0, 8]
    desc = len(good) - 5

    def edit(at, val):
        x = bytearray(good)
        x[at:at + len(val)] = val
        return bytes(x)

    failures = [
        empty[:16],                                              # shorter than 17 bytes
        edit(len(good) - 1, b"\x8e"),                            # the seekable magic number
        edit(desc, b"\x04"), edit(desc, b"\x40"),                # reserved bits
        good[:-9] + struct.pack("<IBI", FRAMES_MAX + 1, 0, SEEKABLE_MAGIC),      # k over the limit
        good[:-9] + struct.pack("<IBI", 5, 0, SEEKABLE_MAGIC),   # a table larger than the item
        edit(30, b"\x5f"),                                       # the skippable magic number
        edit(34, struct.pack("<I", 2 * 8 + 10)),                 # Frame_Size
        edit(desc, b"\x80"),                                     # the checksum flag changes E, so the header no longer matches
    ]
    for k, x in enumerate(failures):
        assert seek_lib.zbs_table_read(x, len(x), t) == 0, k
        assert read_table(x) is None, k
    assert seek_lib.zbs_table_read(edit(desc, b"\x03"), len(good), t) == 1      # bits 1-0 are ignored
    # the entries' sum is checked where they are read: an item whose sum is off is walked (below)
    assert read_table(edit(38, struct.pack("<I", 11))) is None


def host_seek_ranges(L, items, reqs, P=3, S=1, emu=False):
    so, do = [0], [0]
    for x in items:
        so.append(so[-1] + len(x))
    for _, _, ln in reqs:
        do.append(do[-1] + ln)
    dst = C.create_string_buffer(b"\xa5" * do[-1], max(do[-1], 1))
    res, stats = _arr([0] * len(reqs)), _arr([0] * 6)
    L.zbs_ranges(b"".join(items), _arr(so), len(items), len(reqs), _arr([r[0] for r in reqs]), _arr([r[1] for r in reqs]), _arr(do), P, S,
                 int(emu), dst, res, stats)
    out, got = dst.raw[:do[-1]], []
    for k in range(len(reqs)):
        r = res[k]
        if r > ERR_MAX:
            got.append(-_code(r))
            continue
        got.append(out[do[k]:do[k] + r])
        assert out[do[k] + r:do[k + 1]] == b"\xa5" * (do[k + 1] - do[k] - r), k
    return got, list(stats)


def _seekable_items(checksum):
    pieces = [(_data(k, 700 + 613 * k)) for k in range(6)]
    frames = [(ref_compress_flags(c, 1 + k % 3, checksum=k % 2 == 0), c) for k, c in enumerate(pieces)]
    empty = (ref_compress_flags(b"", 3), b"")
    stream = _data(50, 3000)
    return [
        seekable(frames[:4], checksum),
        seekable([empty, frames[0], empty, (fw.skippable(9), None), frames[1], empty], checksum),
        seekable([(ref_stream_compress(stream, 3, 1000), stream), frames[2], (ref_stream_compress(pieces[3], 1, 500), pieces[3])], checksum),
        seekable([(ref_compress_flags(_data(60, 200_000), 3), _data(60, 200_000)), frames[5]], checksum),      # larger than a partial slot
        seekable([], checksum),
    ]


@pytest.mark.parametrize("checksum", [False, True])
def test_ranges_located_through_tables(seek_lib, checksum):
    _needs_ref()
    items = _seekable_items(checksum)
    reqs = [r for i, x in enumerate(items) for r in entry_ranges(i, x, reach=3)]
    want = model_seek(items, reqs)
    assert any(w == -E_PARAMETER_UNSUPPORTED for w in want) and b"" in want
    for emu, P, S in ((False, 3, 1), (True, 3, 1), (False, 5, 2)):
        got, stats = host_seek_ranges(seek_lib, items, reqs, P, S, emu)
        for k, (g, w) in enumerate(zip(got, want)):
            assert g == w, (emu, k, reqs[k], g if isinstance(g, int) else len(g), w if isinstance(w, int) else len(w))
        assert stats[5] == sum(1 for r in reqs if r[2]) and stats[4] == 0 and stats[1] <= P and stats[2] <= S


def test_ranges_fall_back_to_the_walk(seek_lib):
    """Items whose table fails a check, the entries' sum included, and items without one, are walked exactly as without tables."""
    _needs_ref()
    good = _seekable_items(False)[0]
    plain = b"".join(ref_compress_flags(_data(70 + k, 900), 1) for k in range(3))
    T = 8 + 8 * 4 + 9
    off = bytearray(good)
    off[len(good) - T + 8:len(good) - T + 12] = struct.pack("<I", struct.unpack_from("<I", good, len(good) - T + 8)[0] + 1)
    reserved = bytearray(good)
    reserved[-5] = 0x10
    items = [bytes(off), bytes(reserved), plain, plain + struct.pack("<I", SEEKABLE_MAGIC)]
    reqs = [r for i, x in enumerate(items[:3]) for r in [(i, 0, 50), (i, 690, 30), (i, 0, 10_000)]] + [(3, 0, 100)]
    want = model(items, reqs)
    for emu in (False, True):
        got, stats = host_seek_ranges(seek_lib, items, reqs, 3, 1, emu)
        assert got == want and stats[5] == 0


def test_damaged_tables_on_the_host(seek_lib):
    _needs_ref()
    contents = [_data(80 + k, 3000 + 100 * k) for k in range(4)]
    frames = [ref_compress_flags(c, 1) for c in contents]
    entries = [(len(f), len(c), xxh32_low(c)) for f, c in zip(frames, contents)]
    body = b"".join(frames)
    swapped = [entries[0], (entries[1][0], entries[2][1], entries[1][2]), (entries[2][0], entries[1][1], entries[2][2]), entries[3]]
    moved = [(entries[0][0] + 5, entries[0][1], entries[0][2]), (entries[1][0] - 5,) + entries[1][1:]] + entries[2:]
    wrong = entries[:2] + [(entries[2][0], entries[2][1], entries[2][2] ^ 1), entries[3]]
    items = [body + write_table(swapped, False), body + write_table(moved, False), body + write_table(wrong, True)]
    total = sum(len(c) for c in contents)
    reqs = [(i, b, ln) for i in range(3) for b, ln in ((0, 100), (3000, 200), (6500, 100), (0, total), (9500, 50))]
    want = model_seek(items, reqs)
    assert want[0] == contents[0][:100] and want[1] == -E_CORRUPTION                     # swapped Decompressed_Size
    assert want[5] == -E_CORRUPTION and isinstance(want[6], int) and want[7] == contents[2][400:500]      # a moved Compressed_Size
    assert want[10] == contents[0][:100] and want[12] == -E_CHECKSUM                     # a wrong Checksum
    got, _ = host_seek_ranges(seek_lib, items, reqs)
    assert got == want


# ---------------------------------------------------------------------------------------------------------------------------- GPU
def _lib():
    from zstd_jni_b200 import _native
    return _native.lib()


def _ctx(pipeline=1, **options):
    from zstd_jni_b200.zstd import ZstdBatchContext
    ctx = ZstdBatchContext(0)
    ctx.setOption("dec_pipeline", pipeline)
    for k, v in options.items():
        ctx.setOption(k, v)
    return ctx


def _gpu_ranges(items, reqs, pipeline=1, **options):
    from tests.test_device_ranges import _dev, _dev64, _host_offsets, call_ranges
    d_src, d_so = _dev(b"".join(items)), _dev64(_host_offsets(items))
    with _ctx(pipeline, **options) as ctx:
        return call_ranges(ctx, d_src, d_so, len(items), reqs)


def compress_items(contents, level, cs, capacity=None, **options):
    """compress_items_device's streams (or per-item codes) and the call's return, copied back."""
    import torch
    from tests.test_device_ranges import _dev, _dev64, _host_offsets, _u64
    n = len(contents)
    d_src, d_so = _dev(b"".join(contents)), _dev64(_host_offsets(contents))
    if capacity is None:
        capacity = seek_capacity([len(c) for c in contents], cs, bool(options.get("checksum")))
    d_c = torch.zeros(max(capacity, 1), dtype=torch.uint8, device="cuda:0")
    d_co = torch.zeros(n + 1, dtype=torch.int64, device="cuda:0")
    d_cres = torch.zeros(n, dtype=torch.int64, device="cuda:0")
    with _ctx(1, **options) as ctx:
        r = _lib().zstdb200_compress_items_device(ctx.handle, level, cs, n, d_src.data_ptr(), d_so.data_ptr(), d_c.data_ptr(), capacity,
                                                  d_co.data_ptr(), d_cres.data_ptr(), None)
        assert _lib().zstdb200_sync(ctx.handle, None) == 0
    co, res, c = _u64(d_co), _u64(d_cres), d_c.cpu().numpy().tobytes()
    return r, [c[co[i]:co[i + 1]] if res[i] <= ERR_MAX else -_code(res[i]) for i in range(n)], co, res, c


def _read_skippable(frame: bytes):
    R = ref()
    f = R.ZSTD_readSkippableFrame
    f.restype, f.argtypes = C.c_size_t, [C.c_char_p, C.c_size_t, C.POINTER(C.c_uint), C.c_char_p, C.c_size_t]
    out, variant = C.create_string_buffer(len(frame)), C.c_uint(99)
    r = f(out, len(frame), C.byref(variant), frame, len(frame))
    assert r <= ERR_MAX, _code(r)
    return out.raw[:r], variant.value


@pytest.mark.gpu
@pytest.mark.parametrize("level,cs", [(1, BLOCK), (3, BLOCK), (3, 4096), (1, 1000), (19, 4096), (19, 1000)])
@pytest.mark.parametrize("checksum", [0, 1])
def test_compress_items_with_tables(level, cs, checksum):
    _needs_ref()
    import torch
    from tests.test_device_ranges import _dev, _dev64, _host_offsets, _u64
    sizes = (0, 1, 777, cs - 1, cs, cs + 1, 2 * cs, 3 * cs + cs // 2, 0)
    contents = [_data(level * 10 + k + checksum, n) for k, n in enumerate(sizes)]
    r, off, _, _, _ = compress_items(contents, level, cs, capacity=seek_capacity(sizes, cs, False) * 2, checksum=checksum)
    assert r == 0 and all(isinstance(x, bytes) for x in off)
    r, on, co, _, _ = compress_items(contents, level, cs, checksum=checksum, seek_table=1)      # capacity exact
    assert r == 0
    for x, y, c in zip(off, on, contents):
        frames, pos = [], 0
        while pos < len(x):
            size = ref_frame(x[pos:], False)[0]
            frames.append(x[pos:pos + size])
            pos += size
        entries = [(len(f), p, struct.unpack("<I", f[-4:])[0] if checksum else 0) for f, p in zip(frames, chunks_of(len(c), cs))]
        assert y == x + write_table(entries, bool(checksum))
        assert ref_decompress(y, len(c)) == c
        body, variant = _read_skippable(y[len(x):])
        assert variant == 14 and body == y[len(x) + 8:]
        if checksum:
            assert [e[2] for e in entries] == [xxh32_low(c[a:a + cs]) for a in range(0, max(len(c), 1), cs)]
    # decompress_items_device regenerates the packed output, packed exactly
    packed = b"".join(on)
    d_src, d_so = _dev(packed), _dev64(co)
    total = sum(sizes)
    d_dst = torch.zeros(total + 1, dtype=torch.uint8, device="cuda:0")
    d_do = torch.zeros(len(on) + 1, dtype=torch.int64, device="cuda:0")
    d_res = torch.zeros(len(on), dtype=torch.int64, device="cuda:0")
    with _ctx(1) as ctx:
        assert _lib().zstdb200_decompress_items_device(ctx.handle, len(on), d_src.data_ptr(), d_so.data_ptr(), d_dst.data_ptr(), total + 1,
                                                       d_do.data_ptr(), d_res.data_ptr(), None) == 0
        assert _lib().zstdb200_sync(ctx.handle, None) == 0
    assert _u64(d_res) == list(sizes) and _u64(d_do)[-1] == total
    assert d_dst.cpu().numpy().tobytes()[:total] == b"".join(contents)
    # one byte short: every item dstSize_tooSmall
    r, short, co, res, _ = compress_items(contents, level, cs, capacity=seek_capacity(sizes, cs, bool(checksum)) - 1, checksum=checksum,
                                          seek_table=1)
    assert r == 0 and short == [-E_DST_SIZE_TOO_SMALL] * len(sizes) and co == [0] * (len(sizes) + 1)


@pytest.mark.gpu
def test_magicless_with_tables_is_refused():
    import torch
    d = torch.zeros(64, dtype=torch.int64, device="cuda:0")
    with _ctx(1, magicless=1, seek_table=1) as ctx:
        assert _lib().zstdb200_compress_items_device(ctx.handle, 3, BLOCK, 1, d.data_ptr(), d.data_ptr(), d.data_ptr(), 512, d.data_ptr(),
                                                     d.data_ptr(), None) == err(E_PARAMETER_UNSUPPORTED)
        assert _lib().zstdb200_decompress_ranges_device(ctx.handle, 1, d.data_ptr(), d.data_ptr(), 1, d.data_ptr(), d.data_ptr(), d.data_ptr(),
                                                        d.data_ptr(), d.data_ptr(), None) == err(E_PARAMETER_UNSUPPORTED)
        assert _lib().zstdb200_sync(ctx.handle, None) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("level,cs,checksum", [(3, BLOCK, 0), (1, 4096, 1), (3, 1000, 0)])
def test_ranges_with_tables_match_the_walk(level, cs, checksum):
    from tests.test_device_ranges import _random_ranges
    sizes = (0, 1, 777, cs, cs + 1, 3 * cs + cs // 2, 20_000, 5 * BLOCK + 3)
    contents = [_data(500 + level * 10 + k, n) for k, n in enumerate(sizes)]
    _, items, _, _, _ = compress_items(contents, level, cs, checksum=checksum, seek_table=1)
    rnd = random.Random(level * 1000 + cs)
    reqs = [r for i, x in enumerate(items) for r in entry_ranges(i, x, reach=1)][::3]
    reqs += _random_ranges(rnd, list(sizes), 300, 3 * cs)
    rnd.shuffle(reqs)
    reqs += reqs[:50] + [(i, 0, len(c)) for i, c in enumerate(contents)]      # repeated, overlapping, unordered, whole
    off = _gpu_ranges(items, reqs)
    assert off == [contents[i][b:b + ln] for i, b, ln in reqs]
    assert _gpu_ranges(items, reqs, seek_table=1) == off
    assert _gpu_ranges(items, reqs, pipeline=0, seek_table=1) == off


@pytest.mark.gpu
def test_more_entries_than_a_part_and_partial_entries_than_its_scratch():
    content = _data(300, 600 * 1000)
    _, items, _, _, _ = compress_items([content], 3, 1000, seek_table=1)
    reqs = [(0, 0, len(content)), (0, 1, len(content) - 2)] + [(0, k * 1000 + 17, 100) for k in range(600)]
    got = _gpu_ranges(items, reqs, seek_table=1)
    assert got == [content[b:b + ln] for _, b, ln in reqs]
    assert got == _gpu_ranges(items, reqs)


@pytest.mark.gpu
@pytest.mark.parametrize("checksum", [False, True])
def test_foreign_seekable_items(checksum):
    """Frames of the reference's streaming compressor declare no content size: with a table they are read, without it they are not."""
    _needs_ref()
    contents = [_data(700 + k, 30_000 + 5_000 * k) for k in range(5)]
    frames = [(ref_stream_compress(c, 3, 7_000, checksum=k % 2 == 1), c) for k, c in enumerate(contents)]
    items = [seekable(frames, checksum), seekable([frames[1], (fw.skippable(3), None), frames[2]], checksum)]
    reqs = [r for i, x in enumerate(items) for r in entry_ranges(i, x)]
    want = model_seek(items, reqs)
    assert all(isinstance(w, bytes) for w in want)
    assert _gpu_ranges(items, reqs, seek_table=1) == want
    assert _gpu_ranges(items, reqs, pipeline=0, seek_table=1) == want
    assert all(g == -E_PARAMETER_UNSUPPORTED for g, r in zip(_gpu_ranges(items, reqs), reqs) if r[2])


@pytest.mark.gpu
def test_damaged_tables():
    _needs_ref()
    contents = [_data(800 + k, 40_000) for k in range(4)] + [_data(900, 200_000)]
    frames = [ref_compress_flags(c, 3) for c in contents]
    entries = [(len(f), len(c), xxh32_low(c)) for f, c in zip(frames, contents)]
    body = b"".join(frames)
    good = body + write_table(entries, True)
    structural = bytearray(good)
    structural[-5] = 0x84                                                # a reserved bit: walked as without tables
    swapped = entries[:1] + [(entries[1][0], entries[2][1] + 1, entries[1][2])] + entries[2:]
    moved = [(entries[0][0] + 9,) + entries[0][1:], (entries[1][0] - 9,) + entries[1][1:]] + entries[2:]
    wrong = entries[:2] + [(entries[2][0], entries[2][1], entries[2][2] ^ 0x100)] + entries[3:]
    damaged = bytearray(body)
    damaged[len(frames[0]) + len(frames[1]) // 2] ^= 0x5A                # frame 1, outside the ranges below
    items = [bytes(structural), body + write_table(swapped, True), body + write_table(moved, True), body + write_table(wrong, True),
             bytes(damaged) + write_table(entries, True), good]
    reqs = [(i, b, ln) for i in range(len(items)) for b, ln in ((100, 1000), (40_000, 300), (85_000, 500), (125_000, 100), (160_000, 200_000))]
    want = model_seek(items, reqs)
    got = _gpu_ranges(items, reqs, seek_table=1)
    assert got == want
    assert got[0:5] == _gpu_ranges(items[:1], reqs[0:5]) == model(items[:1], reqs[0:5])      # a structural failure: walked
    assert got[6] == -E_CORRUPTION and got[5] == contents[0][100:1100]                 # swapped Decompressed_Size
    assert got[10] == -E_CORRUPTION and isinstance(got[11], int) and got[12] == contents[2][5_000:5_500]   # a moved Compressed_Size
    assert got[17] == -E_CHECKSUM and got[16] == contents[1][:300]                     # a wrong Checksum
    assert got[20] == contents[0][100:1100] and got[22] == contents[2][5_000:5_500] and isinstance(got[21], int)   # a damaged frame
    assert got[29] == contents[4] and got[28] == contents[3][5_000:5_100]
    # a partial entry over 131072 bytes
    assert _gpu_ranges([good], [(0, 170_000, 10), (0, 160_000, 200_000)], seek_table=1) == [-E_PARAMETER_UNSUPPORTED, contents[4]]
