"""Multi-block, multi-frame and magicless items of zstdb200_decompress_device on the segment loop the GPU drives itself.

CPU: the host instantiation of the loop (tests/hostsim/zb_hostsim_loop.cpp, compiled by this module): items routed by the device walk,
their blocks cut into segments of 1, 2, 3 and 7 blocks that start and end inside frames and cross frames and items.  Every item the loop
keeps regenerates the reference's bytes; an item it marks goes to the fused decoder.  Cuts at every byte, trailing garbage, bit flips and
truncations never give bytes the fused decoder would not.
GPU: zstdb200_decompress_device against a dec_pipeline 0 context (the fused kernel) and the reference: reference-made multi-block frames,
concatenations with skippable and one-block frames, mixed calls, more than 16384 items, a magicless context, dec_segment_blocks 4,
corruptions; the call returns before its work is done, and the loop shows in the kernel times.
"""
from __future__ import annotations

import ctypes as C
import random
import subprocess
from pathlib import Path

import numpy as np
import pytest

from tests.oracle_util import (ERR_MAX, hostsim_decompress, hostsim_decompress_magicless, ref_compress_flags, ref_compress_params,
                               ref_decompress, ref_decompress_magicless, ref_stream_compress)

ROOT = Path(__file__).resolve().parent.parent
GOLDEN = ROOT / "tests" / "golden"
U64 = C.c_ulonglong


@pytest.fixture(scope="module")
def loop_lib(tmp_path_factory):
    src = ROOT / "tests" / "hostsim" / "zb_hostsim_loop.cpp"
    so = tmp_path_factory.mktemp("hostsim_loop") / "libzb_hostsim_loop.so"
    subprocess.run(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-Wall", "-Wno-unused-function", "-x", "c++", str(src), "-o", str(so)],
                   check=True)
    L = C.CDLL(str(so))
    L.zbl_item_blocks.restype = U64
    L.zbl_item_blocks.argtypes = [C.c_char_p, C.c_size_t, C.c_int]
    L.zbl_min_blocks.restype = U64
    L.zbl_min_blocks.argtypes = [C.POINTER(U64), C.c_size_t, U64]
    L.zbl_loop.restype = C.c_uint
    L.zbl_loop.argtypes = [C.c_char_p, C.POINTER(U64), C.c_size_t, C.c_char_p, C.POINTER(U64), C.POINTER(U64), C.POINTER(C.c_int),
                           C.c_uint, C.c_int, C.c_uint, C.c_int]
    return L


def run_loop(L, items, caps, B, magicless=False, seed=1, emu=0):
    """[(status, bytes)] per item: 0 decoded by the loop, 1 marked for the fused decoder, 2 not routed to the loop."""
    n = len(items)
    so = (U64 * (n + 1))(*np.concatenate([[0], np.cumsum([len(x) for x in items])]).astype(np.uint64).tolist())
    do = (U64 * (n + 1))(*np.concatenate([[0], np.cumsum(caps)]).astype(np.uint64).tolist())
    dst = C.create_string_buffer(max(int(do[n]), 1) + 64)
    res, st = (U64 * max(n, 1))(), (C.c_int * max(n, 1))()
    L.zbl_loop(b"".join(items), so, n, dst, do, res, st, B, 1 if magicless else 0, seed, emu)
    return [(st[i], dst.raw[do[i]:do[i] + res[i]] if st[i] == 0 else None) for i in range(n)]


def _data(seed: int, n: int) -> bytes:
    rnd = random.Random(seed)
    words = [bytes(rnd.choice(b"abcdefghijklmnop") for _ in range(rnd.randrange(2, 10))) for _ in range(300)]
    out = bytearray()
    while len(out) < n:
        out += rnd.choice(words) + (b" " if rnd.random() < 0.9 else bytes([rnd.randrange(256)]))
    return bytes(out[:n])


def _skippable(n: int, low: int = 0) -> bytes:
    return (0x184D2A50 + low).to_bytes(4, "little") + n.to_bytes(4, "little") + bytes((i * 13) & 0xFF for i in range(n))


def _mb_fixtures():
    return [p.read_bytes() for p in sorted(GOLDEN.glob("mb_*.zst"))] + [(GOLDEN / "concat_skippable.zst").read_bytes()]


def _valid_items():
    """Items the loop takes: the multi-block fixtures, and concatenations with skippable frames, frames without a content size, checksummed
    and one-block frames."""
    mb = _mb_fixtures()
    one = [ref_compress_flags(_data(k, 3000 + 700 * k), 3, checksum=k % 2 == 1, content_size=k % 3 != 2) for k in range(6)]
    unsized = ref_stream_compress(_data(40, 300_000), 3, checksum=True)
    items = mb + [
        mb[0] + _skippable(17, 3) + mb[1],
        one[0] + one[1] + one[2],
        b"".join(one) + _skippable(0),
        _skippable(5) + unsized + one[3],
        unsized + unsized,
        mb[2] + one[4] + mb[3] + _skippable(40, 15) + one[5],
        b"".join(one * 11),
    ]
    return items


def _check_against_fused(items, caps, got, magicless=False):
    fused = hostsim_decompress_magicless if magicless else hostsim_decompress
    for k, (item, cap, (st, b)) in enumerate(zip(items, caps, got)):
        if st == 0:
            assert fused(item, cap) == b, k


@pytest.mark.parametrize("B,emu", [(1, 0), (2, 0), (3, 1), (7, 0), (64, 0)])
def test_loop_regenerates_reference_bytes(loop_lib, B, emu):
    items = _valid_items()
    want = [ref_decompress(x, 1 << 22) for x in items]
    assert all(isinstance(w, bytes) for w in want)
    caps = [len(w) for w in want]
    got = run_loop(loop_lib, items, caps, B, seed=B, emu=emu)
    for k, ((st, b), w) in enumerate(zip(got, want)):
        assert st == 0, k
        assert b == w, k
    assert loop_lib.zbl_item_blocks(items[0], len(items[0]), 0) >= 2


def test_loop_routing_leaves_other_items(loop_lib):
    one = ref_compress_flags(_data(3, 5000), 3)
    items = [one, b"", _skippable(9), _skippable(9) + _skippable(3), one + b"\x00", one[:-1], b"\x28\xb5\x2f\xfd"]
    assert [loop_lib.zbl_item_blocks(x, len(x), 0) for x in items] == [0] * len(items)
    assert [s for s, _ in run_loop(loop_lib, items, [6000] * len(items), 3)] == [2] * len(items)
    assert loop_lib.zbl_item_blocks(one + _skippable(1), len(one) + 9, 0) == 1      # two frames, one block


def test_loop_capacity_and_magicless(loop_lib):
    items = _valid_items()[:4]
    want = [ref_decompress(x, 1 << 22) for x in items]
    short = [len(w) - 1 for w in want]
    got = run_loop(loop_lib, items, short, 3)
    assert [s for s, _ in got] == [1] * len(items)
    m = [ref_compress_flags(_data(50 + k, 150_000 + 9000 * k), 1 + 2 * k, checksum=k == 1, magicless=True) for k in range(3)]
    m1 = ref_compress_flags(_data(60, 4000), 3, magicless=True)
    mitems = m + [m[0] + m1 + m[1], m1 + m1]
    mwant = [ref_decompress_magicless(x, 1 << 21) for x in mitems]
    assert all(isinstance(w, bytes) for w in mwant)
    for B in (2, 7):
        got = run_loop(loop_lib, mitems, [len(w) for w in mwant], B, magicless=True)
        assert got == [(0, w) for w in mwant]
    # a skippable frame's magic starts a (bad) frame in the magicless format: not taken
    assert loop_lib.zbl_item_blocks(m[0] + _skippable(4), len(m[0]) + 12, 1) == 0


def test_loop_takes_few_long_items_and_leaves_many_short_ones(loop_lib):
    """seg_loop_min_blocks: the loop for long items and for few items, the fused kernel's warps for many short ones."""
    def least(blocks, warps=2112):
        return loop_lib.zbl_min_blocks((U64 * len(blocks))(*blocks), len(blocks), warps)
    assert least([8192]) == 1                                  # one 1 GiB frame
    assert least([64] * 128) == 1                              # 128 items of 64 one-block frames
    assert least([2]) == 1 and least([2] * 100) == 1           # few items
    assert least([2] * 8192) > 2                               # thousands of files just over 128 KB
    assert least([3] * 4096) > 3                               # thousands of items of a few frames
    t = least([2] * 8191 + [8192])                             # ... with one long item among them: only that one
    assert 2 < t <= 8192
    assert least([]) == 1 and least([2] * 8192, warps=1) == 1


def test_loop_cuts_and_garbage(loop_lib):
    mb = _mb_fixtures()
    base = [mb[5], ref_compress_flags(_data(7, 2000), 3) + _skippable(6) + ref_compress_flags(_data(8, 1500), 1, checksum=True)]
    items, caps = [], []
    for x in base:
        cap = len(ref_decompress(x, 1 << 22))
        for cut in range(len(x) + 1):
            items.append(x[:cut]); caps.append(cap)
        for g in (b"\x00", b"\x01\x02\x03", x[:4], _skippable(3)[:6]):
            items.append(x + g); caps.append(cap)
    for B in (2, 7):
        got = run_loop(loop_lib, items, caps, B, seed=B)
        _check_against_fused(items, caps, got)
        assert sum(1 for s, _ in got if s == 0) >= 2


def test_loop_corruptions(loop_lib):
    rnd = random.Random(5)
    items, caps = [], []
    for x in _mb_fixtures():
        cap = len(ref_decompress(x, 1 << 22))
        for _ in range(30):
            z = bytearray(x)
            for _ in range(rnd.choice((1, 1, 2, 5))):
                p = rnd.randrange(len(z))
                z[p] ^= 1 << rnd.randrange(8)
            items.append(bytes(z)); caps.append(cap)
        for _ in range(10):
            items.append(x[:rnd.randrange(len(x))] + x[rnd.randrange(len(x)):]); caps.append(cap)
    for B in (3, 7):
        got = run_loop(loop_lib, items, caps, B, seed=B)
        _check_against_fused(items, caps, got)


# ---------------------------------------------------------------------------------------------------------------------------- GPU
def _lib():
    from zstd_jni_b200 import _native
    return _native.lib()


def _ctx(pipeline=1, magicless=0, seg_blocks=None):
    from zstd_jni_b200.zstd import ZstdBatchContext
    ctx = ZstdBatchContext(0)
    ctx.setOption("dec_pipeline", pipeline)
    if magicless:
        ctx.setOption("magicless", 1)
    if seg_blocks:
        assert _lib().zstdb200_set_option(ctx.handle, b"dec_segment_blocks", seg_blocks) == 0
    return ctx


def call_device(ctx, items, caps):
    """Per item: its bytes, or the negative error code."""
    import torch
    dev = torch.device("cuda:0")
    so = np.concatenate([[0], np.cumsum([len(x) for x in items])]).astype(np.int64)
    do = np.concatenate([[0], np.cumsum(caps)]).astype(np.int64)
    d_src = torch.from_numpy(np.frombuffer(b"".join(items) or b"\0", dtype=np.uint8).copy()).to(dev)
    d_so, d_do = torch.from_numpy(so).to(dev), torch.from_numpy(do).to(dev)
    d_dst = torch.zeros(max(int(do[-1]), 1), dtype=torch.uint8, device=dev)
    d_res = torch.zeros(len(items), dtype=torch.int64, device=dev)
    s = torch.cuda.Stream()
    assert _lib().zstdb200_decompress_device(ctx.handle, len(items), d_src.data_ptr(), d_so.data_ptr(), d_dst.data_ptr(), d_do.data_ptr(),
                                             d_res.data_ptr(), s.cuda_stream) == 0
    s.synchronize()
    res = [int(x) & ((1 << 64) - 1) for x in d_res.cpu().numpy()]
    out = d_dst.cpu().numpy()
    return [out[do[i]:do[i] + r].tobytes() if r <= ERR_MAX else -((1 << 64) - r) for i, r in enumerate(res)]


def _both(items, caps, magicless=0, seg_blocks=None):
    with _ctx(1, magicless, seg_blocks) as new, _ctx(0, magicless) as old:
        got = call_device(new, items, caps)
        assert got == call_device(old, items, caps)
        segs = (_lib().zstdb200_segment_frames(new.handle, 0), _lib().zstdb200_segment_frames(new.handle, 1))
        assert segs == (0, 0)      # the counters count host-memory calls only
    return got


def _gpu_valid_items():
    items = _valid_items()
    for level in (1, 3, 19):
        for ck, cs in ((False, True), (True, True), (False, False), (True, False)):
            items.append(ref_compress_flags(_data(100 + level, 400_000), level, checksum=ck, content_size=cs))
    for wl in (17, 20, 23, 27):
        f = ref_compress_params(_data(200 + wl, 700_000), 3, {"windowLog": wl}, checksum=wl % 2 == 1)
        assert isinstance(f, bytes)
        items.append(f)
    items.append(ref_stream_compress(_data(300, 1_000_000), 19))
    return items


@pytest.mark.gpu
def test_device_call_on_multi_block_and_multi_frame_items():
    items = _gpu_valid_items()
    want = [ref_decompress(x, 1 << 22) for x in items]
    singles = [ref_compress_flags(_data(400 + k, 20_000 + 500 * k), 3) for k in range(40)]
    swant = [ref_decompress(x, 1 << 20) for x in singles]
    mixed = [x for pair in zip(singles, items) for x in pair] + singles[len(items):]
    mwant = [x for pair in zip(swant, want) for x in pair] + swant[len(items):]
    assert _both(mixed, [len(w) for w in mwant]) == mwant
    assert _both(items, [len(w) for w in want], seg_blocks=4) == want


@pytest.mark.gpu
def test_device_call_more_than_16384_items():
    rnd = random.Random(9)
    one = [ref_compress_flags(_data(500 + k, 1500 + 97 * k), 1 + k % 3, checksum=k % 4 == 0) for k in range(24)]
    items = []
    for i in range(16500):
        k = rnd.randrange(len(one))
        items.append(one[k] if i % 3 == 0 else one[k] + one[(k + 1) % len(one)] + (_skippable(i % 7) if i % 5 == 0 else b""))
    items[16400] = _mb_fixtures()[0]
    want = [ref_decompress(x, 1 << 20) for x in items]
    assert _both(items, [len(w) for w in want]) == want


@pytest.mark.gpu
def test_device_call_magicless():
    m = [ref_compress_flags(_data(600 + k, 300_000 + 9000 * k), 1 + 2 * k, checksum=k == 1, magicless=True) for k in range(3)]
    m1 = ref_compress_flags(_data(610, 4000), 3, magicless=True)
    items = m + [m[0] + m1 + m[1], m1 + m1, m1]
    want = [ref_decompress_magicless(x, 1 << 21) for x in items]
    assert _both(items, [len(w) for w in want], magicless=1) == want


@pytest.mark.gpu
def test_device_call_corruptions_and_capacity():
    rnd = random.Random(11)
    base = _mb_fixtures() + [ref_compress_flags(_data(700, 400_000), 3, checksum=True)]
    items, caps = [], []
    for x in base:
        cap = len(ref_decompress(x, 1 << 22))
        for _ in range(40):
            z = bytearray(x)
            for _ in range(rnd.choice((1, 2, 4))):
                p = rnd.randrange(len(z))
                z[p] ^= 1 << rnd.randrange(8)
            items.append(bytes(z)); caps.append(cap)
        for _ in range(8):
            items.append(x[:rnd.randrange(len(x))]); caps.append(cap)
        items.append(x); caps.append(cap - 1)
        items.append(x + b"\x07"); caps.append(cap)
    for seg_blocks in (None, 4):
        got = _both(items, caps, seg_blocks=seg_blocks)
        for k, (item, cap) in enumerate(zip(items, caps)):
            r = ref_decompress(item, cap)
            if isinstance(r, bytes) and isinstance(got[k], bytes):
                assert got[k] == r, k


@pytest.mark.gpu
def test_device_call_returns_before_the_work_is_done_and_is_timed():
    import torch
    chunk = np.frombuffer(_data(800, 1 << 22), dtype=np.uint8)
    data = np.tile(chunk, 256)
    data[::4093] = np.arange(len(data[::4093]), dtype=np.uint64).astype(np.uint8)      # not one long match
    frame = ref_compress_flags(data.tobytes(), 1)
    assert isinstance(frame, bytes)
    dev = torch.device("cuda:0")
    d_src = torch.from_numpy(np.frombuffer(frame, dtype=np.uint8).copy()).to(dev)
    d_so = torch.tensor([0, len(frame)], dtype=torch.int64, device=dev)
    d_do = torch.tensor([0, len(data)], dtype=torch.int64, device=dev)
    d_dst = torch.zeros(len(data), dtype=torch.uint8, device=dev)
    d_res = torch.zeros(1, dtype=torch.int64, device=dev)
    L = _lib()
    with _ctx(1) as ctx:
        ctx.setOption("timing", 1)
        s = torch.cuda.Stream()
        args = (ctx.handle, 1, d_src.data_ptr(), d_so.data_ptr(), d_dst.data_ptr(), d_do.data_ptr(), d_res.data_ptr(), s.cuda_stream)
        assert L.zstdb200_decompress_device(*args) == 0      # the first call builds the loop
        s.synchronize()
        ctx.kernelTimes()
        assert L.zstdb200_decompress_device(*args) == 0
        assert not s.query()
        s.synchronize()
        assert int(d_res.cpu()[0]) == len(data)
        assert torch.equal(d_dst.cpu(), torch.from_numpy(data))
        times = ctx.kernelTimes()
        # the loop regenerated the frame itself: the fused kernel, one warp taking minutes on it, had nothing to decode again
        assert times["k_decompress(marked)"][0] < 0.05 * times["k_seg_loop"][0], times
