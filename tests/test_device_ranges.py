"""zstdb200_decompress_ranges_device: byte ranges of items in device memory regenerated from the frames that hold them, located on the GPU.

CPU: the host instantiation of the call (tests/hostsim/zb_hostsim_ranges.cpp, compiled by this module), run in parts of 3 entries of
which 1 or 2 may be covered in part, so that requests span parts, against a plain-Python model built on the compiled reference: its
ZSTD_findFrameCompressedSize and ZSTD_getFrameHeader_advanced for the walk, its ZSTD_decompress of each covered frame alone.  Items: the
golden multi-block, multi-frame, skippable, streamed (no content size) and err_* items, golden one-shot frames without their magic
number on a magicless call, and reference-made items with empty and skippable frames.  Ranges: at every frame boundary and one byte
either side, empty, past the end and whole items, and requests for items that do not exist.
GPU: the call against the same model, with a canary around every request's output: compress_items_device output at levels 1, 3 and 19,
128 KB, 4 KB and 1000-byte chunks, with a checksum, magicless and without content sizes; reference frames with skippable frames between
them; the multi-block mb_*.zst frames covered wholly and in part; ranges that overlap, repeat and come in any item order; one request of
more entries than a part holds and more partial entries than a part's scratch; a damaged frame outside the range, one inside it and a
wrong checksum; m == 0, dec_pipeline 0, the call-level errors, and the call returning before its work is done.
"""
from __future__ import annotations

import ctypes as C
import random
import subprocess
from pathlib import Path

import numpy as np
import pytest

from tests import frame_writer as fw
from tests.oracle_util import ERR_MAX, ref, ref_compress_flags, ref_decompress, ref_decompress_magicless, ref_stream_compress

ROOT = Path(__file__).resolve().parent.parent
GOLDEN = ROOT / "tests" / "golden"
U64 = C.c_ulonglong
M64 = (1 << 64) - 1
UNKNOWN = M64
BLOCK = 128 << 10
E_PARAMETER_UNSUPPORTED, E_OUT_OF_BOUND, E_CORRUPTION, E_CHECKSUM, E_SRC_SIZE_WRONG = 40, 42, 20, 22, 72


def err(code):
    return (1 << 64) - code


# ---------------------------------------------------------------------------------------------------------------------------- the model
class _FrameHeader(C.Structure):
    _fields_ = [("frameContentSize", C.c_ulonglong), ("windowSize", C.c_ulonglong), ("blockSizeMax", C.c_uint), ("frameType", C.c_int),
                ("headerSize", C.c_uint), ("dictID", C.c_uint), ("checksumFlag", C.c_uint), ("_r1", C.c_uint), ("_r2", C.c_uint)]


def _code(r):
    return (1 << 64) - r if r > ERR_MAX else 0


def ref_frame(rest: bytes, magicless: bool):
    """The frame that starts rest, as the reference walks it: (compressed size, content size or UNKNOWN, skippable), or the negative
    error code ZSTD_findFrameCompressedSize gives (in the magicless format the same walk around ZSTD_getFrameHeader_advanced)."""
    R = ref()
    gh = R.ZSTD_getFrameHeader_advanced
    gh.restype, gh.argtypes = C.c_size_t, [C.POINTER(_FrameHeader), C.c_char_p, C.c_size_t, C.c_int]
    if not magicless:
        fc = R.ZSTD_findFrameCompressedSize
        fc.restype, fc.argtypes = C.c_size_t, [C.c_char_p, C.c_size_t]
        size = fc(rest, len(rest))
        if _code(size):
            return -_code(size)
        zfh = _FrameHeader()
        assert gh(C.byref(zfh), rest, len(rest), 0) == 0
        return size, zfh.frameContentSize, zfh.frameType == 1
    zfh = _FrameHeader()
    r = gh(C.byref(zfh), rest, len(rest), 1)
    if r:
        return -(_code(r) or E_SRC_SIZE_WRONG)
    p = zfh.headerSize
    while True:
        if len(rest) - p < 3:
            return -E_SRC_SIZE_WRONG
        bh = int.from_bytes(rest[p:p + 3], "little")
        kind = (bh >> 1) & 3
        if kind == 3:
            return -E_CORRUPTION
        size = 1 if kind == 1 else bh >> 3
        if 3 + size > len(rest) - p:
            return -E_SRC_SIZE_WRONG
        p += 3 + size
        if bh & 1:
            break
    if zfh.checksumFlag:
        if len(rest) - p < 4:
            return -E_SRC_SIZE_WRONG
        p += 4
    return p, zfh.frameContentSize, False


def model(items, reqs, magicless=False):
    """Per request (item, begin, length): the bytes the call returns, or the negative error code -- the first failure in item order."""
    dec = ref_decompress_magicless if magicless else ref_decompress
    out = []
    for i, b, ln in reqs:
        if i >= len(items):
            out.append(-E_OUT_OF_BOUND)
            continue
        x, e, pos, at, got, fail = items[i], b + ln, 0, 0, [], None
        while ln and pos < len(x) and at < e:
            f = ref_frame(x[pos:], magicless)
            if isinstance(f, int):
                fail = f
                break
            size, cs, skippable = f
            if not skippable:
                if cs == UNKNOWN:
                    fail = -E_PARAMETER_UNSUPPORTED
                    break
                if cs and at + cs > b:
                    if (at < b or at + cs > e) and cs > BLOCK:
                        fail = -E_PARAMETER_UNSUPPORTED
                        break
                    d = dec(x[pos:pos + size], cs)
                    if isinstance(d, int):
                        fail = d
                        break
                    if len(d) != cs:
                        fail = -E_CORRUPTION
                        break
                    got.append(d[max(b - at, 0):min(e, at + cs) - at])
                at += cs
            pos += size
        out.append(fail if fail is not None else b"".join(got))
    return out


def boundaries(x: bytes, magicless=False):
    """The content offsets at which the item's frames start, and its content size (as far as the walk goes)."""
    pos, at, marks = 0, 0, [0]
    while pos < len(x):
        f = ref_frame(x[pos:], magicless)
        if isinstance(f, int):
            break
        size, cs, skippable = f
        if not skippable and cs != UNKNOWN:
            at += cs
            marks.append(at)
        pos += size
    return marks


def boundary_ranges(i, x, magicless=False, reach=2):
    """Requests at every boundary and one byte either side: empty, one byte, to the next `reach` boundaries +-1, to the end and past it."""
    marks = boundaries(x, magicless)
    end = marks[-1]
    points = sorted({p for m in marks for p in (m - 1, m, m + 1) if p >= 0} | {end + 3})
    reqs = set()
    for p in points:
        ends = {p, p + 1, end, end + 7}
        later = [m for m in marks if m > p][:reach]
        ends |= {q + d for q in later for d in (-1, 0, 1)}
        reqs |= {(i, p, q - p) for q in ends if q >= p}
    return sorted(reqs)


# ---------------------------------------------------------------------------------------------------------------------------- CPU
@pytest.fixture(scope="module")
def ranges_lib(tmp_path_factory):
    src = ROOT / "tests" / "hostsim" / "zb_hostsim_ranges.cpp"
    so = tmp_path_factory.mktemp("zb_hostsim_ranges") / "libzb_hostsim_ranges.so"
    subprocess.run(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-Wall", "-Wno-unused-function", "-x", "c++", str(src), "-o", str(so)],
                   check=True)
    L = C.CDLL(str(so))
    P64 = C.POINTER(U64)
    L.zbr_ranges.restype = None
    L.zbr_ranges.argtypes = [C.c_char_p, P64, C.c_size_t, C.c_size_t, P64, P64, P64, C.c_uint, C.c_uint, C.c_int, C.c_char_p, P64, P64]
    return L


def _arr(v):
    return (U64 * max(len(v), 1))(*v)


def host_ranges(L, items, reqs, P=3, S=1, magicless=False):
    """The host instantiation of the call: per request its bytes or negative code, and the part statistics.  Every request's output
    starts as a canary; what the call does not return stays one."""
    so = [0]
    for x in items:
        so.append(so[-1] + len(x))
    do = [0]
    for _, _, ln in reqs:
        do.append(do[-1] + ln)
    dst = C.create_string_buffer(b"\xa5" * do[-1], max(do[-1], 1))
    res, stats = _arr([0] * len(reqs)), _arr([0] * 5)
    L.zbr_ranges(b"".join(items), _arr(so), len(items), len(reqs), _arr([r[0] for r in reqs]), _arr([r[1] for r in reqs]), _arr(do), P, S,
                 int(magicless), dst, res, stats)
    out = dst.raw[:do[-1]]
    got = []
    for k in range(len(reqs)):
        r = res[k]
        if r > ERR_MAX:
            got.append(-_code(r))
            continue
        got.append(out[do[k]:do[k] + r])
        assert out[do[k] + r:do[k + 1]] == b"\xa5" * (do[k + 1] - do[k] - r), k      # nothing past a short read
    return got, list(stats)


def _check_host(L, items, magicless=False, reach=2, P=3, S=1):
    reqs = [r for i, x in enumerate(items) for r in boundary_ranges(i, x, magicless, reach)]
    reqs += [(len(items), 0, 5), (len(items) + 7, 3, 0)]
    want = model(items, reqs, magicless)
    got, stats = host_ranges(L, items, reqs, P, S, magicless)
    for k, (g, w) in enumerate(zip(got, want)):
        assert g == w, (k, reqs[k], g if isinstance(g, int) else len(g), w if isinstance(w, int) else len(w))
    assert stats[4] == 0 and stats[1] <= P and stats[2] <= S
    return got, stats


def _data(seed: int, n: int) -> bytes:
    rnd = np.random.default_rng(seed)
    words = rnd.integers(97, 123, size=(500, 8), dtype=np.uint8)
    words[:, 7] = 32
    return words[rnd.zipf(1.4, size=n // 8 + 1) % 500].tobytes()[:n]


def _needs_ref():
    if ref() is None:
        pytest.skip("the compiled reference (oracle/_ref) is not built")


def test_golden_items(ranges_lib):
    _needs_ref()
    names = sorted(p.name for p in GOLDEN.glob("*.zst") if p.name.startswith(("mb_", "concat_", "stream_", "err_", "oneshot_00")))
    items = [(GOLDEN / n).read_bytes() for n in names]
    got, stats = _check_host(ranges_lib, items)
    assert stats[0] > 10
    assert -E_PARAMETER_UNSUPPORTED in got and any(isinstance(g, bytes) and len(g) > BLOCK for g in got)      # partial and whole mb_ frames
    assert {g for g in got if isinstance(g, int)} - {-E_PARAMETER_UNSUPPORTED, -E_OUT_OF_BOUND}      # the err_ items' own codes


def test_golden_frames_magicless(ranges_lib):
    _needs_ref()
    frames = [(GOLDEN / f"oneshot_{k:03d}_L{1 + 2 * (k % 2 == 0)}.zst").read_bytes()[4:] for k in range(8)]
    items = [frames[0] + frames[1] + frames[2], frames[3], frames[4] + frames[5][:-3], frames[6] + frames[7] + frames[0]]
    _check_host(ranges_lib, items, magicless=True, P=3, S=2)


def test_reference_items_with_empty_and_skippable_frames(ranges_lib):
    _needs_ref()
    pieces = [ref_compress_flags(_data(k, 700 + 613 * k), 1 + k % 3, checksum=k % 3 == 0) for k in range(8)]
    empty = ref_compress_flags(b"", 3)
    items = [
        b"".join(pieces[:5]),
        empty + pieces[0] + empty + fw.skippable(9) + pieces[1] + empty,
        fw.skippable(0) + empty + empty,
        pieces[2] + ref_stream_compress(_data(50, 3000), 3, 1000) + pieces[3],      # a frame without a content size, after one with
        pieces[4] + pieces[5][:-1],
        pieces[6] + b"\x00\x01\x02" + pieces[7],
        b"",
        ref_compress_flags(_data(60, 200_000), 3) + pieces[1],                      # a multi-block frame larger than a partial slot
    ]
    got, stats = _check_host(ranges_lib, items, reach=3)
    assert stats[0] > 20 and stats[2] == 1
    assert b"" in got and -E_PARAMETER_UNSUPPORTED in got
    _check_host(ranges_lib, items[:2], reach=3, P=5, S=2)


def test_part_planning_spans_requests(ranges_lib):
    """Requests of many entries in parts of 3 and 4, and many partial entries, against the model; every part is full unless it
    reaches a partial entry beyond its scratch or the end."""
    _needs_ref()
    pieces = [ref_compress_flags(_data(100 + k, 500 + 50 * k), 1) for k in range(12)]
    item = b"".join(pieces)
    total = sum(500 + 50 * k for k in range(12))
    rnd = random.Random(3)
    reqs = [(0, 0, total), (0, 10, total - 20)] + [(0, rnd.randrange(total), rnd.randrange(1, 1500)) for _ in range(40)]
    want = model([item], reqs)
    for P, S in ((3, 1), (4, 2), (5, 5), (64, 3)):
        got, stats = host_ranges(ranges_lib, [item], reqs, P, S)
        assert got == want and stats[1] <= P and stats[2] <= S and stats[4] == 0


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


def _dev(b: bytes):
    import torch
    return torch.from_numpy(np.frombuffer(b or b"\0", dtype=np.uint8).copy()).to("cuda:0")


def _dev64(v):
    import torch
    return torch.tensor([int(x) for x in v] or [0], dtype=torch.int64, device="cuda:0")


def _u64(t):
    return [int(x) & M64 for x in t.cpu().numpy()]


GUARD = 16      # bytes of a guard request between two requests: an item that does not exist, so nothing is written there


def call_ranges(ctx, d_src, src_offsets, n, reqs, stream=None):
    """The call with a guard request before and after every request.  Returns per request its bytes or negative code, after checking
    that every guard and every byte past a short read still holds the canary."""
    import torch
    full = [(n + 1, 0, GUARD)]
    for r in reqs:
        full += [r, (n + 1, 0, GUARD)]
    do = [0]
    for _, _, ln in full:
        do.append(do[-1] + ln)
    d_items, d_begins, d_do = _dev64([r[0] for r in full]), _dev64([r[1] for r in full]), _dev64(do)
    d_dst = torch.full((max(do[-1], 1),), 0xA5, dtype=torch.uint8, device="cuda:0")
    d_res = torch.zeros(len(full), dtype=torch.int64, device="cuda:0")
    s = stream or torch.cuda.Stream()
    assert _lib().zstdb200_decompress_ranges_device(ctx.handle, n, d_src.data_ptr(), src_offsets.data_ptr(), len(full), d_items.data_ptr(),
                                                    d_begins.data_ptr(), d_dst.data_ptr(), d_do.data_ptr(), d_res.data_ptr(), s.cuda_stream) == 0
    s.synchronize()
    res, out = _u64(d_res), d_dst.cpu().numpy().tobytes()
    got = []
    for k, r in enumerate(res):
        if k % 2 == 0:
            assert r == err(E_OUT_OF_BOUND) and out[do[k]:do[k + 1]] == b"\xa5" * GUARD, k
            continue
        if r > ERR_MAX:
            got.append(-_code(r))
            continue
        assert out[do[k] + r:do[k + 1]] == b"\xa5" * (do[k + 1] - do[k] - r), k
        got.append(out[do[k]:do[k] + r])
    return got


def _host_offsets(items):
    return np.concatenate([[0], np.cumsum([len(x) for x in items])]).astype(np.int64)


def check_items(items, reqs, magicless=False, pipelines=(1,)):
    """The call on items held in device memory, against the model; the same results on every dec_pipeline asked for."""
    d_src, d_so = _dev(b"".join(items)), _dev64(_host_offsets(items))
    want = model(items, reqs, magicless)
    for pipeline in pipelines:
        with _ctx(pipeline, magicless=int(magicless)) as ctx:
            got = call_ranges(ctx, d_src, d_so, len(items), reqs)
        for k, (g, w) in enumerate(zip(got, want)):
            assert g == w, (pipeline, k, reqs[k], g if isinstance(g, int) else len(g), w if isinstance(w, int) else len(w))
    return want


def _random_ranges(rnd, items_content, count, most):
    reqs = []
    for _ in range(count):
        i = rnd.randrange(len(items_content))
        size = items_content[i]
        b = rnd.randrange(size + 2) if size else rnd.randrange(3)
        reqs.append((i, b, rnd.randrange(0, most)))
    return reqs


def _compress_on_gpu(ctx, items, level, cs):
    """compress_items_device's streams of items, copied back."""
    import torch
    n = len(items)
    d_src, d_so = _dev(b"".join(items)), _dev64(_host_offsets(items))
    ccap = sum(len(x) + (len(x) >> 7) + 1024 * (len(x) // cs + 1) for x in items)
    d_c = torch.zeros(ccap, dtype=torch.uint8, device="cuda:0")
    d_co = torch.zeros(n + 1, dtype=torch.int64, device="cuda:0")
    d_cres = torch.zeros(n, dtype=torch.int64, device="cuda:0")
    assert _lib().zstdb200_compress_items_device(ctx.handle, level, cs, n, d_src.data_ptr(), d_so.data_ptr(), d_c.data_ptr(), ccap,
                                                 d_co.data_ptr(), d_cres.data_ptr(), None) == 0
    assert _lib().zstdb200_sync(ctx.handle, None) == 0
    assert all(r <= ERR_MAX for r in _u64(d_cres))
    co, c = _u64(d_co), d_c.cpu().numpy().tobytes()
    return [c[co[i]:co[i + 1]] for i in range(n)]


@pytest.mark.gpu
@pytest.mark.parametrize("level,cs,options", [(1, BLOCK, {}), (3, BLOCK, {}), (3, 4096, {}), (3, 1000, {}), (19, 65536, {}),
                                              (3, BLOCK, {"checksum": 1}), (3, BLOCK, {"magicless": 1}), (3, BLOCK, {"content_size": 0})])
def test_items_from_compress_items_device(level, cs, options):
    sizes = (0, 1, 777, cs - 1, cs, cs + 1, 3 * cs + cs // 2, 20_000, 5 * BLOCK + 3)
    contents = [_data(level * 10 + k, n) for k, n in enumerate(sizes)]
    with _ctx(1, **options) as ctx:
        items = _compress_on_gpu(ctx, contents, level, cs)
    magicless = bool(options.get("magicless"))
    rnd = random.Random(level * 1000 + cs)
    reqs = [r for i, x in enumerate(items) for r in boundary_ranges(i, x, magicless, reach=1)][::3]
    reqs += _random_ranges(rnd, [len(x) for x in contents], 300, 3 * cs)
    reqs += [(i, 0, len(x)) for i, x in enumerate(contents)]
    want = check_items(items, reqs, magicless)
    if options.get("content_size", 1) == 0:
        assert all(w == -E_PARAMETER_UNSUPPORTED for w, r in zip(want, reqs) if r[2] and contents[r[0]])
    else:
        assert all(w == contents[i][b:b + ln] for w, (i, b, ln) in zip(want, reqs))


@pytest.mark.gpu
def test_reference_frames_with_skippable_frames_between_them():
    pieces = [ref_compress_flags(_data(200 + k, 30_000 + 7_000 * k), 1 + 2 * (k % 3), checksum=k % 2 == 1) for k in range(10)]
    items = [b"".join(p + fw.skippable(k % 5, k % 16) for k, p in enumerate(pieces)), fw.skippable(3) + pieces[3] + pieces[4],
             pieces[5] + ref_compress_flags(b"", 1) + pieces[6]]
    rnd = random.Random(5)
    reqs = [r for i, x in enumerate(items) for r in boundary_ranges(i, x)]
    reqs += _random_ranges(rnd, [sum(30_000 + 7_000 * k for k in range(10)), 30_000 + 7_000 * 7, 30_000 + 7_000 * 11], 200, 90_000)
    rnd.shuffle(reqs)
    reqs += reqs[:50]      # repeated, overlapping, in any item order
    check_items(items, reqs, pipelines=(1, 0))


@pytest.mark.gpu
def test_multi_block_frames_wholly_and_in_part():
    names = sorted(p.name for p in GOLDEN.glob("mb_*.zst"))
    items = [(GOLDEN / n).read_bytes() for n in names]
    reqs = [r for i, x in enumerate(items) for r in boundary_ranges(i, x)]
    want = check_items(items, reqs)
    assert -E_PARAMETER_UNSUPPORTED in want and any(isinstance(w, bytes) and len(w) > BLOCK for w in want)


@pytest.mark.gpu
def test_more_entries_than_a_part_and_more_partial_entries_than_its_scratch():
    content = _data(300, 600 * 1000)
    with _ctx(1, timing=1) as ctx:
        item = _compress_on_gpu(ctx, [content], 3, 1000)[0]
    # one request of 600 entries (parts hold 512 here), and 600 requests of one partial entry each (a part's scratch holds half its slots)
    reqs = [(0, 0, len(content)), (0, 1, len(content) - 2)]
    reqs += [(0, k * 1000 + 17, 100) for k in range(600)]
    want = check_items([item], reqs)
    assert want == [content[b:b + ln] for _, b, ln in reqs]
    d_src, d_so = _dev(item), _dev64([0, len(item)])
    with _ctx(1) as ctx:
        ctx.setOption("timing", 1)
        assert call_ranges(ctx, d_src, d_so, 1, reqs) == want
        times = ctx.kernelTimes()
    assert "k_range_locate" in times and "k_range_parts" in times and "k_range_finish" in times, times


@pytest.mark.gpu
def test_damaged_frames_inside_and_outside_the_range():
    contents = [_data(400 + k, 50_000) for k in range(6)]
    pieces = [ref_compress_flags(c, 3, checksum=True) for c in contents]
    bad = bytearray(pieces[2])
    bad[len(bad) // 2] ^= 0x5A                          # inside the frame's blocks
    ck = bytearray(pieces[4])
    ck[-1] ^= 0x01                                      # the stored checksum
    cut = pieces[5][:-7]                                # truncated: the walk cannot pass it
    item = pieces[0] + pieces[1] + bytes(bad) + pieces[3] + bytes(ck) + cut
    reqs = [(0, 0, 100_000), (0, 150_000, 50_000), (0, 60_000, 100), (0, 110_000, 100), (0, 210_000, 100), (0, 0, 300_000),
            (0, 120_000, 100_000), (0, 260_000, 10), (0, 0, 250_000)]
    want = check_items([item], reqs, pipelines=(1, 0))
    assert want[0] == contents[0] + contents[1] and want[1] == contents[3] and want[2] == contents[1][10_000:10_100]
    assert isinstance(want[3], int) and want[4] == -E_CHECKSUM and want[5] == want[3]
    assert want[6] == want[3] and want[7] == -E_SRC_SIZE_WRONG and want[8] == want[3]
    assert want[3] == ref_decompress(bytes(bad), 50_000)


@pytest.mark.gpu
def test_call_level_cases_and_dec_pipeline_0():
    import torch
    pieces = [ref_compress_flags(_data(500 + k, 40_000), 1) for k in range(4)]
    items = [b"".join(pieces), pieces[0]]
    reqs = [(1, 5, 10), (0, 39_990, 20), (5, 0, 4), (0, 0, 0), (0, 160_000, 10), (0, 159_995, 10)]
    want = check_items(items, reqs, pipelines=(1, 0))
    assert want == [pieces and _data(500, 40_000)[5:15], _data(500, 40_000)[39_990:] + _data(501, 40_000)[:10], -E_OUT_OF_BOUND, b"", b"",
                    _data(503, 40_000)[-5:]]
    L = _lib()
    d_res = torch.full((1,), -1, dtype=torch.int64, device="cuda:0")
    with _ctx(1) as ctx:
        assert L.zstdb200_decompress_ranges_device(ctx.handle, 1, 0, 0, 0, 0, 0, 0, 0, d_res.data_ptr(), None) == 0      # m == 0
        assert L.zstdb200_sync(ctx.handle, None) == 0 and d_res.cpu().tolist() == [-1]
        assert L.zstdb200_decompress_ranges_device(ctx.handle, 1, 0, 0, 1 << 31, 0, 0, 0, 0, 0, None) == err(E_SRC_SIZE_WRONG)
        assert L.zstdb200_decompress_ranges_device(ctx.handle, 1 << 31, 0, 0, 1, 0, 0, 0, 0, 0, None) == err(E_SRC_SIZE_WRONG)
        assert L.zstdb200_last_error() is not None


@pytest.mark.gpu
def test_call_returns_before_its_work_is_done():
    import torch
    content = _data(600, 64 << 20)
    with _ctx(1) as ctx:
        item = _compress_on_gpu(ctx, [content], 3, BLOCK)[0]
        d_src, d_so = _dev(item), _dev64([0, len(item)])
        m = 64
        do = [k << 20 for k in range(m + 1)]
        d_items, d_begins, d_do = _dev64([0] * m), _dev64([k << 20 for k in range(m)]), _dev64(do)
        d_dst = torch.zeros(m << 20, dtype=torch.uint8, device="cuda:0")
        d_res = torch.zeros(m, dtype=torch.int64, device="cuda:0")
        s = torch.cuda.Stream()
        L = _lib()
        args = (ctx.handle, 1, d_src.data_ptr(), d_so.data_ptr(), m, d_items.data_ptr(), d_begins.data_ptr(), d_dst.data_ptr(), d_do.data_ptr(),
                d_res.data_ptr(), s.cuda_stream)
        assert L.zstdb200_decompress_ranges_device(*args) == 0      # the first call builds the graph
        s.synchronize()
        d_dst.zero_()
        torch.cuda.synchronize()
        assert L.zstdb200_decompress_ranges_device(*args) == 0
        assert not s.query()
        s.synchronize()
        assert d_res.cpu().tolist() == [1 << 20] * m
        assert bytes(d_dst.cpu().numpy()) == content
