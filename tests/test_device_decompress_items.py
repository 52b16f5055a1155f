"""zstdb200_decompress_bound_device / zstdb200_decompress_items_device: every item's room found from its frames on the GPU, and the items
decoded into those rooms, with nothing from the host.

CPU: the host instantiation of the call's plan (tests/hostsim/zb_hostsim_ditems.cpp, compiled by this module).  The device bound of an
item equals the compiled reference's ZSTD_decompressBound and this library's host ZSTD_decompressBound on the golden multi-block,
multi-frame, skippable and streamed (no content size) frames, library-made multi-frame items, streams of ZSTD_compressStream2, every
truncation of several items, trailing garbage, empty items, a reserved bit and a window beyond the limit; magicless items equal the
reference's frame walk over ZSTD_getFrameHeader_advanced with ZSTD_f_zstd1_magicless.  The scan of the rooms and the fit check equal a
plain computation, at a capacity equal to the total, one byte short, and with a saturated sum.
GPU: compress_items_device then decompress_items_device on one stream gives the items back and their offsets, at levels 1, 3 and 19, with
a checksum, magicless and without content sizes; reference-made items decode to the reference's bytes in rooms of the reference's bound,
and corrupt or truncated items get zstdb200_decompress_device's results without touching their neighbours; 8192 x 128 KB, 64 x 16 MB,
20 000 items of 0-300 KB, one 1 GiB frame and more split entries than one part holds; a short capacity writes nothing and leaves the
plan; n == 0, dec_pipeline 0, the bound call alone, and the call returns before its work is done.
"""
from __future__ import annotations

import ctypes as C
import random
import subprocess
from pathlib import Path

import numpy as np
import pytest

from tests.oracle_util import (ERR_MAX, hostsim_compress_flags, ref, ref_compress_flags, ref_decompress, ref_decompress_magicless,
                               ref_stream_compress)

ROOT = Path(__file__).resolve().parent.parent
GOLDEN = ROOT / "tests" / "golden"
U64 = C.c_ulonglong
M64 = (1 << 64) - 1
UNKNOWN, ERROR = M64, M64 - 1
E_SRC_SIZE_WRONG, E_DST_SIZE_TOO_SMALL = 72, 70
BLOCK = 128 << 10


def err(code):
    return (1 << 64) - code


# ---------------------------------------------------------------------------------------------------------------------------- CPU
@pytest.fixture(scope="module")
def plan_lib(tmp_path_factory):
    src = ROOT / "tests" / "hostsim" / "zb_hostsim_ditems.cpp"
    so = tmp_path_factory.mktemp("zb_hostsim_ditems") / "libzb_hostsim_ditems.so"
    subprocess.run(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-Wall", "-Wno-unused-function", "-x", "c++", str(src), "-o", str(so)],
                   check=True)
    L = C.CDLL(str(so))
    P64 = C.POINTER(U64)
    L.zbd_bound.restype = U64
    L.zbd_bound.argtypes = [C.c_char_p, C.c_size_t, C.c_uint]
    L.zbd_plan.restype = C.c_int
    L.zbd_plan.argtypes = [P64, C.c_size_t, U64, P64, P64, P64, P64, P64, P64]
    return L


def _host_bound_fn():
    from zstd_jni_b200 import _native
    f = _native.lib().ZSTD_decompressBound
    f.restype, f.argtypes = C.c_ulonglong, [C.c_char_p, C.c_size_t]
    return f


class _FrameHeader(C.Structure):
    _fields_ = [("frameContentSize", C.c_ulonglong), ("windowSize", C.c_ulonglong), ("blockSizeMax", C.c_uint), ("frameType", C.c_int),
                ("headerSize", C.c_uint), ("dictID", C.c_uint), ("checksumFlag", C.c_uint), ("_r1", C.c_uint), ("_r2", C.c_uint)]


def ref_walk_bound(item: bytes, magicless: bool) -> int:
    """ZSTD_findFrameSizeInfo's walk summed as ZSTD_decompressBound sums it, around the reference's own header parser
    (ZSTD_getFrameHeader_advanced, in either format): the reference exports no bound for ZSTD_f_zstd1_magicless."""
    R = ref()
    f = R.ZSTD_getFrameHeader_advanced
    f.restype, f.argtypes = C.c_size_t, [C.POINTER(_FrameHeader), C.c_char_p, C.c_size_t, C.c_int]
    pos, bound = 0, 0
    while pos < len(item):
        rest = item[pos:]
        if not magicless and len(rest) >= 8 and int.from_bytes(rest[:4], "little") & 0xFFFFFFF0 == 0x184D2A50:
            size = int.from_bytes(rest[4:8], "little")
            if size + 8 > 0xFFFFFFFF or size + 8 > len(rest):
                return ERROR
            pos += size + 8
            continue
        zfh = _FrameHeader()
        if f(C.byref(zfh), rest, len(rest), 1 if magicless else 0) != 0:
            return ERROR
        p, blocks = zfh.headerSize, 0
        while True:
            if len(rest) - p < 3:
                return ERROR
            bh = int.from_bytes(rest[p:p + 3], "little")
            kind, size = (bh >> 1) & 3, (1 if (bh >> 1) & 3 == 1 else bh >> 3)
            if kind == 3 or 3 + size > len(rest) - p:
                return ERROR
            p += 3 + size
            blocks += 1
            if bh & 1:
                break
        if zfh.checksumFlag:
            if len(rest) - p < 4:
                return ERROR
            p += 4
        fcs = zfh.frameContentSize
        if fcs == ERROR:
            return ERROR
        bound = (bound + (fcs if fcs != UNKNOWN else blocks * zfh.blockSizeMax)) & M64
        pos += p
    return bound


def _golden_items():
    names = sorted(p.name for p in GOLDEN.glob("*.zst") if p.name.startswith(("mb_", "concat_", "stream_", "err_", "oneshot_00")))
    return [(GOLDEN / n).read_bytes() for n in names]


def _data(seed: int, n: int) -> bytes:
    rnd = np.random.default_rng(seed)
    return np.resize(rnd.integers(97, 109, size=max(1, min(n, 5000)), dtype=np.uint8), n).tobytes()


def _multi_frame(seed, size, cs, **kw):
    """The stream compress_items_device writes for an item: one hostsim frame per chunk of cs bytes."""
    x = _data(seed, size)
    return b"".join(hostsim_compress_flags(x[k:k + cs], 3, **kw) for k in range(0, max(size, 1), cs))


def _frame(fcs: int, blocks, wl_byte=None, reserved=False):
    """A frame of raw blocks declaring content size fcs (None: none; 8-byte field), its window descriptor wl_byte (None: single segment)."""
    single = wl_byte is None
    fhd = (0 if fcs is None else 3 << 6) | (0x20 if single else 0) | (0x08 if reserved else 0)
    if fcs is None and single:
        fhd = 0x20
    out = b"\x28\xb5\x2f\xfd" + bytes([fhd]) + (b"" if single else bytes([wl_byte]))
    out += (fcs or 0).to_bytes(8, "little") if fcs is not None else (b"\0" if single else b"")
    for k, b in enumerate(blocks):
        out += ((len(b) << 3) | (k == len(blocks) - 1)).to_bytes(3, "little") + b
    return out


def _corpus():
    items = _golden_items()
    items += [_multi_frame(s, n, cs) for s, (n, cs) in enumerate([(300_000, BLOCK), (10_000, 4096), (0, BLOCK), (BLOCK, BLOCK)])]
    items += [_multi_frame(9, 200_000, 65536, checksum=True), _multi_frame(10, 200_000, BLOCK, content_size=False)]
    if ref() is not None:
        items += [ref_stream_compress(_data(20, 400_000), 3), ref_stream_compress(_data(21, 300_000), 1, 50_000, checksum=True)]
        items += [ref_compress_flags(_data(22, 1000), 19) + ref_compress_flags(b"", 3) + ref_compress_flags(_data(23, 300_000), 1)]
    skip = (0x184D2A53).to_bytes(4, "little") + (5).to_bytes(4, "little") + b"abcde"
    good = items[-1]
    items += [b"", skip, skip + good + skip, good + b"\0", good + b"\x28\xb5\x2f", good[:-1], b"\x28\xb5\x2f\xfd",
              _frame(1000, [b"x" * 1000], reserved=True), _frame(None, [b"y" * 10, b"z" * 7], wl_byte=(31 - 10) << 3),
              _frame(None, [b"y" * 10, b"z" * 7], wl_byte=(32 - 10) << 3), _frame(5, [b"abcde"]), _frame(UNKNOWN, [b"ab", b"c"]),
              _frame(ERROR, [b"ab"]), _frame(M64 - 200, [b"ab"]) + _frame(M64 - 300, [b"cd"]),
              (0x184D2A50).to_bytes(4, "little") + (0xFFFFFFF8).to_bytes(4, "little"), bytes([0x3F, 0, 0, 0, 0, 0, 0, 0, 0])]
    return items


def test_device_bound_matches_the_reference_and_the_host_bound(plan_lib):
    if ref() is None:
        pytest.skip("the compiled reference (oracle/_ref) is not built")
    R = ref()
    R.ZSTD_decompressBound.restype, R.ZSTD_decompressBound.argtypes = C.c_ulonglong, [C.c_char_p, C.c_size_t]
    host = _host_bound_fn()
    for x in _corpus():
        want = R.ZSTD_decompressBound(x, len(x))
        assert plan_lib.zbd_bound(x, len(x), 0) == want
        assert ref_walk_bound(x, False) == want                 # the helper the magicless items are held to
        if b"\xff" * 8 not in x:      # (the host bound takes a declared size of 2^64-1 as a size; the reference, as none)
            assert host(x, len(x)) == want


def test_device_bound_on_every_truncation(plan_lib):
    if ref() is None:
        pytest.skip("the compiled reference (oracle/_ref) is not built")
    R = ref()
    R.ZSTD_decompressBound.restype, R.ZSTD_decompressBound.argtypes = C.c_ulonglong, [C.c_char_p, C.c_size_t]
    skip = (0x184D2A5F).to_bytes(4, "little") + (3).to_bytes(4, "little") + b"xyz"
    items = [_multi_frame(1, 9000, 4096), _multi_frame(2, 2000, 4096, checksum=True) + skip + _multi_frame(3, 50, 4096),
             (GOLDEN / "mb_two_frames_skippable.zst").read_bytes()[:3000], ref_stream_compress(_data(4, 5000), 3, 1000, checksum=True)]
    for x in items:
        for k in range(len(x) + 1):
            want = R.ZSTD_decompressBound(x[:k], k)
            assert plan_lib.zbd_bound(x[:k], k, 0) == want, k


def test_device_bound_of_magicless_items(plan_lib):
    if ref() is None:
        pytest.skip("the compiled reference (oracle/_ref) is not built")
    items = [_multi_frame(s, n, cs, magicless=True) for s, (n, cs) in enumerate([(300_000, BLOCK), (10_000, 4096), (0, BLOCK)])]
    items += [_multi_frame(5, 100_000, 30_000, magicless=True, content_size=False, checksum=True)]
    items += [ref_compress_flags(_data(6, 200_000), 3, magicless=True) + ref_compress_flags(_data(7, 777), 1, magicless=True, checksum=True)]
    skip = (0x184D2A50).to_bytes(4, "little") + (2).to_bytes(4, "little") + b"ab"     # a frame header in this format, not a skippable frame
    items += [b"", skip, items[0] + skip, items[1][:-1], items[1] + b"\0", bytes([0x08, 0, 0, 0])]
    for x in items:
        want = ref_walk_bound(x, True)
        assert plan_lib.zbd_bound(x, len(x), 1) == want
    x = items[1]
    for k in range(len(x) + 1):
        assert plan_lib.zbd_bound(x[:k], k, 1) == ref_walk_bound(x[:k], True), k


def device_plan(L, bounds, cap, src_off=None, decoded=None):
    n = len(bounds)
    a = lambda k: (U64 * max(k, 1))()
    src_off = src_off or list(range(n + 1))
    decoded = decoded or [7] * n
    dst_off, run_src, run_dst, results = a(n + 1), a(n + 1), a(n + 1), a(n)
    fits = L.zbd_plan((U64 * max(n, 1))(*bounds), n, cap, (U64 * (n + 1))(*src_off), (U64 * max(n, 1))(*decoded), dst_off, run_src, run_dst,
                      results)
    return bool(fits), list(dst_off[:n + 1]), list(run_src[:n + 1]), list(run_dst[:n + 1]), list(results[:n])


def host_plan(bounds, cap, src_off, decoded):
    off, s = [], 0
    for b in bounds:
        off.append(s)
        s = min(M64, s + (0 if b == ERROR else b))
    off.append(s)
    fits = s <= cap
    zeros = [0] * len(off)
    return fits, off, (src_off if fits else zeros), (off if fits else zeros), (decoded if fits else [err(E_DST_SIZE_TOO_SMALL)] * len(bounds))


@pytest.mark.parametrize("n", [1, 5, 1023, 1024, 1025, 3000, 40_000])
def test_plan_scan_and_fit(plan_lib, n):
    rnd = random.Random(n)
    bounds = [rnd.choice([0, ERROR, rnd.randrange(1, 1 << 20), 1 << 30]) if rnd.random() < 0.3 else rnd.randrange(0, 300_000) for _ in range(n)]
    src_off = sorted(rnd.randrange(0, 1 << 40) for _ in range(n + 1))
    decoded = [rnd.choice([rnd.randrange(0, 1 << 20), err(20), err(E_SRC_SIZE_WRONG)]) for _ in range(n)]
    total = host_plan(bounds, M64, src_off, decoded)[1][-1]
    for cap in (total, total - 1, total + 1, 0, M64):
        if cap < 0:
            continue
        got = device_plan(plan_lib, bounds, cap, src_off, decoded)
        assert got == host_plan(bounds, cap, src_off, decoded), cap
        assert got[0] == (cap >= total)


@pytest.mark.parametrize("n", [3, 1500, 70_000])
def test_plan_saturates(plan_lib, n):
    rnd = random.Random(7 + n)
    bounds = [rnd.randrange(0, 1 << 20) for _ in range(n)]
    at = rnd.sample(range(n), 3)
    for k, i in enumerate(at):      # the sum passes 2^64 at one item, then stays there; an ERROR item takes no room
        bounds[i] = [M64 - 1000, 1 << 63, ERROR][k]
    src_off = list(range(n + 1))
    want = host_plan(bounds, M64 - 1, src_off, [1] * n)
    assert want[1][-1] == M64 and not want[0]
    assert device_plan(plan_lib, bounds, M64 - 1, src_off, [1] * n) == want
    assert device_plan(plan_lib, bounds, M64, src_off, [1] * n) == host_plan(bounds, M64, src_off, [1] * n)


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


def _u64(t):
    return [int(x) & M64 for x in t.cpu().numpy()]


def _dev(data: bytes):
    import torch
    return torch.from_numpy(np.frombuffer(data or b"\0", dtype=np.uint8).copy()).to("cuda:0")


def _offsets(sizes):
    import torch
    return torch.from_numpy(np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)).to("cuda:0")


def call_items(ctx, items, cap=None, sentinel=0):
    """decompress_items_device: (per item its bytes or the negative error code, the output offsets, d_dst as it was left).
    cap: the output's capacity (default: the rooms' total, from zstdb200_decompress_bound_device)."""
    import torch
    n = len(items)
    d_src, d_so = _dev(b"".join(items)), _offsets([len(x) for x in items])
    if cap is None:
        cap = call_bound(ctx, items)[1][-1]
    d_dst = torch.full((max(cap, 1),), sentinel, dtype=torch.uint8, device="cuda:0")
    d_do = torch.full((n + 1,), -1, dtype=torch.int64, device="cuda:0")
    d_res = torch.zeros(max(n, 1), dtype=torch.int64, device="cuda:0")
    s = torch.cuda.Stream()
    r = _lib().zstdb200_decompress_items_device(ctx.handle, n, d_src.data_ptr(), d_so.data_ptr(), d_dst.data_ptr(), cap, d_do.data_ptr(),
                                                d_res.data_ptr(), s.cuda_stream)
    assert r == 0, r
    s.synchronize()
    do, res, out = _u64(d_do), _u64(d_res)[:n], d_dst.cpu().numpy()
    got = [out[do[i]:do[i] + r].tobytes() if r <= ERR_MAX else -((1 << 64) - r) for i, r in enumerate(res)]
    return got, do, out


def call_bound(ctx, items, with_bounds=True):
    """decompress_bound_device: (the bounds, the output offsets)."""
    import torch
    n = len(items)
    d_src, d_so = _dev(b"".join(items)), _offsets([len(x) for x in items])
    d_do = torch.full((n + 1,), -1, dtype=torch.int64, device="cuda:0")
    d_b = torch.full((max(n, 1),), -1, dtype=torch.int64, device="cuda:0")
    s = torch.cuda.Stream()
    assert _lib().zstdb200_decompress_bound_device(ctx.handle, n, d_src.data_ptr(), d_so.data_ptr(), d_do.data_ptr(),
                                                   d_b.data_ptr() if with_bounds else None, s.cuda_stream) == 0
    s.synchronize()
    return _u64(d_b)[:n], _u64(d_do)


def _rooms(offsets):
    return [offsets[i + 1] - offsets[i] for i in range(len(offsets) - 1)]


def _round_trip(items, level, cs, **options):
    """compress_items_device, then decompress_items_device on its output, on one stream with no host copy between."""
    import torch
    n = len(items)
    with _ctx(1, **options) as ctx:
        d_src, d_so = _dev(b"".join(items)), _offsets([len(x) for x in items])
        ccap = sum(len(x) + (len(x) >> 7) + 1024 * (len(x) // cs + 1) for x in items)
        d_c = torch.zeros(ccap, dtype=torch.uint8, device="cuda:0")
        d_co = torch.zeros(n + 1, dtype=torch.int64, device="cuda:0")
        d_cres = torch.zeros(n, dtype=torch.int64, device="cuda:0")
        total = sum(len(x) for x in items)
        cap = total if options.get("content_size", 1) else sum(max(1, -(-len(x) // cs)) * BLOCK for x in items)
        d_out = torch.zeros(max(cap, 1), dtype=torch.uint8, device="cuda:0")
        d_oo = torch.zeros(n + 1, dtype=torch.int64, device="cuda:0")
        d_res = torch.zeros(n, dtype=torch.int64, device="cuda:0")
        s = torch.cuda.Stream()
        L = _lib()
        assert L.zstdb200_compress_items_device(ctx.handle, level, cs, n, d_src.data_ptr(), d_so.data_ptr(), d_c.data_ptr(), ccap,
                                                d_co.data_ptr(), d_cres.data_ptr(), s.cuda_stream) == 0
        assert L.zstdb200_decompress_items_device(ctx.handle, n, d_c.data_ptr(), d_co.data_ptr(), d_out.data_ptr(), cap, d_oo.data_ptr(),
                                                  d_res.data_ptr(), s.cuda_stream) == 0
        s.synchronize()
        assert all(r <= ERR_MAX for r in _u64(d_cres))
        oo, res, out = _u64(d_oo), _u64(d_res), d_out.cpu().numpy()
        assert res == [len(x) for x in items]
        assert [out[oo[i]:oo[i] + len(x)].tobytes() for i, x in enumerate(items)] == items
        return oo


def _text(seed, n):
    rnd = np.random.default_rng(seed)
    words = rnd.integers(97, 123, size=(2000, 8), dtype=np.uint8)
    words[:, 7] = 32
    return words[rnd.zipf(1.4, size=n // 8 + 1) % 2000].tobytes()[:n]


def _varied(seed, cs):
    return [_text(seed + k, n) for k, n in enumerate((0, 1, 777, cs - 1, cs, cs + 1, 3 * cs + cs // 2, 0, 20_000, 5 * BLOCK + 3))]


@pytest.mark.gpu
@pytest.mark.parametrize("level,cs,options", [(1, BLOCK, {}), (3, BLOCK, {}), (19, 65536, {}), (3, 4096, {}), (3, BLOCK, {"checksum": 1}),
                                              (3, BLOCK, {"magicless": 1}), (3, BLOCK, {"content_size": 0}),
                                              (3, 65536, {"checksum": 1, "content_size": 0, "magicless": 1})])
def test_round_trip_after_compress_items_device(level, cs, options):
    items = _varied(level * 10, cs)
    oo = _round_trip(items, level, cs, **options)
    if options.get("content_size", 1):
        assert oo == list(np.cumsum([0] + [len(x) for x in items]))       # packed: the original item offsets


def _compare_with_device_call(items, magicless=0, pipeline=1):
    """decompress_items_device against decompress_device on the same rooms, and the reference's bytes where the reference decodes."""
    from tests.test_device_split import call_device
    with _ctx(pipeline, magicless=magicless) as ctx:
        bounds, offs = call_bound(ctx, items)
        got, do, _ = call_items(ctx, items)
        assert do == offs
        assert got == call_device(ctx, items, _rooms(offs))
    if ref() is not None:
        dec = ref_decompress_magicless if magicless else ref_decompress
        for x, g, room, b in zip(items, got, _rooms(offs), bounds):
            if not magicless:
                R = ref()
                R.ZSTD_decompressBound.restype, R.ZSTD_decompressBound.argtypes = C.c_ulonglong, [C.c_char_p, C.c_size_t]
                assert b == R.ZSTD_decompressBound(x, len(x))
            else:
                assert b == ref_walk_bound(x, True)
            w = dec(x, room)
            if isinstance(w, bytes):
                assert g == w
    return got


@pytest.mark.gpu
def test_reference_items_with_corruptions_among_them():
    good = [ref_compress_flags(_text(1, 300_000), 3), ref_compress_flags(_text(2, 100_000), 19, checksum=True),
            ref_stream_compress(_text(3, 700_000), 1), ref_stream_compress(_text(4, 200_000), 3, 50_000, checksum=True),
            b"".join(ref_compress_flags(_text(10 + k, BLOCK), 3) for k in range(6)),
            b"".join(ref_compress_flags(_text(20 + k, 40_000), 1) for k in range(4)) + ref_stream_compress(_text(30, 50_000), 3),
            ref_compress_flags(b"", 3), b"", (GOLDEN / "concat_skippable.zst").read_bytes(), (GOLDEN / "mb_L3_xxh.zst").read_bytes()]
    bad = []
    for k, x in enumerate(good[:6]):
        flipped = bytearray(x)
        flipped[len(x) // 2] ^= 0x40
        bad += [bytes(flipped), x[:len(x) // 3], x + b"\x01\x02", x[:-1]]
    items = [y for pair in zip(bad, (good * 3)[:len(bad)]) for y in pair]
    got = _compare_with_device_call(items)
    for x, g in zip(items[1::2], got[1::2]):      # every good item between the bad ones regenerates whole
        if x:
            assert g == ref_decompress(x, 1 << 21)


@pytest.mark.gpu
def test_magicless_and_dec_pipeline_0():
    items = [b"".join(ref_compress_flags(_text(40 + k, BLOCK), 3, magicless=True) for k in range(4)),
             ref_compress_flags(_text(50, 600_000), 1, magicless=True), b""]
    items.append(items[0][:-2])
    assert _compare_with_device_call(items, magicless=1) == _compare_with_device_call(items, magicless=1, pipeline=0)
    plain = [ref_compress_flags(_text(60, 300_000), 3), ref_stream_compress(_text(61, 300_000), 3), b"junk"]
    assert _compare_with_device_call(plain, pipeline=0) == _compare_with_device_call(plain, pipeline=1)


@pytest.mark.gpu
def test_shapes_8192_items_of_128k_and_64_of_16m():
    for n, size in ((8192, BLOCK), (64, 16 << 20)):
        data = _text(n, n * size)
        items = [data[i * size:(i + 1) * size] for i in range(n)]
        _round_trip(items, 1, BLOCK)


@pytest.mark.gpu
def test_shapes_20000_mixed_items():
    rng = np.random.default_rng(2)
    sizes = [int(x) for x in rng.integers(0, 300 << 10, size=20_000)]
    sizes[::997] = [0] * len(sizes[::997])
    data = _text(5, sum(sizes))
    offs = np.concatenate([[0], np.cumsum(sizes)])
    _round_trip([data[offs[i]:offs[i + 1]] for i in range(len(sizes))], 1, BLOCK)


@pytest.mark.gpu
def test_shapes_one_1gib_frame_and_more_split_entries_than_a_part():
    data = _text(6, 1 << 30)
    frame = ref_compress_flags(data, 1)
    with _ctx(1, timing=1) as ctx:
        got, do, _ = call_items(ctx, [frame])
        assert do == [0, 1 << 30] and got == [data]
        times = ctx.kernelTimes()
        assert "k_ditem_plan" in times and "k_seg_loop" in times, times
        # 4 items of 200 one-block frames: 800 entries, more than the 512 of one part
        items = [b"".join(ref_compress_flags(data[(k * 200 + j) * 40_000:(k * 200 + j + 1) * 40_000], 3) for j in range(200)) for k in range(4)]
        got, do, _ = call_items(ctx, items)
        assert got == [data[k * 8_000_000:(k + 1) * 8_000_000] for k in range(4)]


@pytest.mark.gpu
def test_short_capacity_writes_nothing_and_leaves_the_plan():
    import torch
    items = [ref_compress_flags(_text(70 + k, 100_000 + 999 * k), 3) for k in range(20)] + [b"bad", ref_stream_compress(_text(90, 400_000), 1)]
    with _ctx() as ctx:
        bounds, plan = call_bound(ctx, items)
        total = plan[-1]
        for cap in (total - 1, 0):
            got, do, out = call_items(ctx, items, cap=cap, sentinel=0xA5)
            assert got == [-E_DST_SIZE_TOO_SMALL] * len(items) and do == plan
            assert (out[:max(cap, 1)] == 0xA5).all()
        # again with d_dstOffsets[n] bytes
        got, do, _ = call_items(ctx, items, cap=total)
        assert do == plan and got[:20] == [_text(70 + k, 100_000 + 999 * k) for k in range(20)] and got[-1] == _text(90, 400_000)
        # n == 0
        d_do = torch.full((1,), -1, dtype=torch.int64, device="cuda:0")
        L = _lib()
        assert L.zstdb200_decompress_items_device(ctx.handle, 0, 0, 0, 0, 0, d_do.data_ptr(), 0, None) == 0
        assert L.zstdb200_sync(ctx.handle, None) == 0 and d_do.cpu().tolist() == [0]
        d_do.fill_(-1)
        assert L.zstdb200_decompress_bound_device(ctx.handle, 0, 0, 0, d_do.data_ptr(), 0, None) == 0
        assert L.zstdb200_sync(ctx.handle, None) == 0 and d_do.cpu().tolist() == [0]
        assert L.zstdb200_decompress_items_device(ctx.handle, 1 << 31, 0, 0, 0, 0, 0, 0, None) == err(E_SRC_SIZE_WRONG)
        assert L.zstdb200_decompress_bound_device(ctx.handle, 1 << 31, 0, 0, 0, 0, None) == err(E_SRC_SIZE_WRONG)


@pytest.mark.gpu
def test_bound_call_alone():
    items = _corpus()
    R = ref()
    R.ZSTD_decompressBound.restype, R.ZSTD_decompressBound.argtypes = C.c_ulonglong, [C.c_char_p, C.c_size_t]
    with _ctx() as ctx:
        bounds, offs = call_bound(ctx, items)
        assert bounds == [R.ZSTD_decompressBound(x, len(x)) for x in items]
        assert ERROR in bounds
        want, s = [0], 0
        for b in bounds:
            s = min(M64, s + (0 if b == ERROR else b))
            want.append(s)
        assert offs == want
        assert call_bound(ctx, items, with_bounds=False)[1] == offs


@pytest.mark.gpu
def test_device_call_returns_before_the_decompression_is_done():
    import torch
    data = _text(8, 256 << 20)
    items = [ref_compress_flags(data[k << 20:(k + 1) << 20], 3) for k in range(256)]
    n = len(items)
    d_src, d_so = _dev(b"".join(items)), _offsets([len(x) for x in items])
    d_dst = torch.zeros(len(data), dtype=torch.uint8, device="cuda:0")
    d_do = torch.zeros(n + 1, dtype=torch.int64, device="cuda:0")
    d_res = torch.zeros(n, dtype=torch.int64, device="cuda:0")
    L = _lib()
    with _ctx() as ctx:
        s = torch.cuda.Stream()
        args = (ctx.handle, n, d_src.data_ptr(), d_so.data_ptr(), d_dst.data_ptr(), len(data), d_do.data_ptr(), d_res.data_ptr(), s.cuda_stream)
        assert L.zstdb200_decompress_items_device(*args) == 0      # the first call builds the graphs
        s.synchronize()
        d_dst.zero_()
        torch.cuda.synchronize()
        assert L.zstdb200_decompress_items_device(*args) == 0
        assert not s.query()
        s.synchronize()
        assert d_res.cpu().tolist() == [1 << 20] * n and d_do.cpu().tolist() == [k << 20 for k in range(n + 1)]
        assert bytes(d_dst.cpu().numpy()) == data
