"""Items of one-block frames cut into their frames on the GPU in zstdb200_decompress_device, for the staged decoder.

CPU: the host instantiation of the device call's decode list (tests/hostsim/zb_hostsim_split.cpp, compiled by this module).  For
reference-made and library-made items -- concatenations with skippable frames, frames without a content size, magicless items, cuts at
every byte, trailing garbage, capacities one byte short and long, 32767 and 32768 bytes per frame on average -- the device lists the
entries plan_decode_list lists for every item it splits, and leaves every other item to the routing it had before.  Settling an item's
entries gives the fused decoder's result and code, also for a frame short of its declared size, a wrong checksum, bit flips and
truncations.
GPU: zstdb200_decompress_device against a dec_pipeline 0 context (the fused kernel) and the reference: items of 64 one-block frames from
ZSTD_compress2 with ZSTDB200_c_multiFrame and from concatenated reference frames, 4096 items of 2-4 frames, mixed calls with items on the
segment loop, more than 16384 items, more entries than one part holds, checksums, magicless items and corruptions; the call returns
before its work is done, and the split shows in the kernel times.
"""
from __future__ import annotations

import ctypes as C
import random
import subprocess
from pathlib import Path

import numpy as np
import pytest

from tests import frame_writer as fw
from tests.oracle_util import (ERR_MAX, hostsim_compress_flags, hostsim_decompress, hostsim_decompress_magicless, ref_compress_flags,
                               ref_decompress, ref_decompress_magicless)

ROOT = Path(__file__).resolve().parent.parent
GOLDEN = ROOT / "tests" / "golden"
U64 = C.c_ulonglong
SPLIT_MIN_BYTES = 32768


def _build(tmp_path_factory, name):
    src = ROOT / "tests" / "hostsim" / f"{name}.cpp"
    so = tmp_path_factory.mktemp(name) / f"lib{name}.so"
    subprocess.run(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-Wall", "-Wno-unused-function", "-x", "c++", str(src), "-o", str(so)],
                   check=True)
    return C.CDLL(str(so))


@pytest.fixture(scope="module")
def split_lib(tmp_path_factory):
    L = _build(tmp_path_factory, "zb_hostsim_split")
    L.zbs_device_plan.restype = U64
    L.zbs_device_plan.argtypes = [C.c_char_p, C.POINTER(U64), C.POINTER(U64), C.c_size_t, C.c_int, U64, C.POINTER(C.c_ubyte), C.POINTER(U64),
                                  C.POINTER(C.c_uint), C.c_size_t]
    L.zbs_host_plan.restype = U64
    L.zbs_host_plan.argtypes = [C.c_char_p, C.POINTER(U64), C.POINTER(U64), C.c_size_t, C.c_int, C.POINTER(C.c_ubyte), C.POINTER(U64),
                                C.POINTER(C.c_uint), C.c_size_t]
    L.zbs_route.restype = None
    L.zbs_route.argtypes = [C.c_char_p, C.c_size_t, U64, C.c_int, C.POINTER(C.c_uint), C.POINTER(U64)]
    L.zbs_decode.restype = None
    L.zbs_decode.argtypes = [C.c_char_p, C.POINTER(U64), C.POINTER(U64), C.c_size_t, C.c_int, C.c_char_p, C.POINTER(U64), C.POINTER(C.c_int)]
    return L


@pytest.fixture(scope="module")
def loop_lib(tmp_path_factory):
    """The segment loop's routing as it stood before items were split (tests/hostsim/zb_hostsim_loop.cpp)."""
    L = _build(tmp_path_factory, "zb_hostsim_loop")
    L.zbl_item_blocks.restype = U64
    L.zbl_item_blocks.argtypes = [C.c_char_p, C.c_size_t, C.c_int]
    return L


def _offsets(sizes):
    v = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint64).tolist() if len(sizes) else [0]
    return (U64 * len(v))(*v)


def _entries(e4, items, m):
    out = {}
    for j in range(m):
        out.setdefault(items[j], []).append(tuple(e4[4 * j: 4 * j + 4]))
    return out


def plans(L, items, caps, magicless=False, max_entries=1 << 20):
    """(device taken per item, device entries per item, host split per item, host entries per item)."""
    n = len(items)
    so, do = _offsets([len(x) for x in items]), _offsets(caps)
    src = b"".join(items)
    emax = 1 << 16
    taken, split = (C.c_ubyte * max(n, 1))(), (C.c_ubyte * max(n, 1))()
    de4, he4 = (U64 * (4 * emax))(), (U64 * (4 * emax))()
    dit, hit = (C.c_uint * emax)(), (C.c_uint * emax)()
    dm = L.zbs_device_plan(src, so, do, n, int(magicless), max_entries, taken, de4, dit, emax)
    hm = L.zbs_host_plan(src, so, do, n, int(magicless), split, he4, hit, emax)
    assert dm <= emax and hm <= emax
    return list(taken[:n]), _entries(de4, dit, dm), list(split[:n]), _entries(he4, hit, hm)


def route(L, item, cap, magicless=False):
    e, b = C.c_uint(), U64()
    L.zbs_route(item, len(item), cap, int(magicless), C.byref(e), C.byref(b))
    return e.value, b.value


def settle(L, items, caps, magicless=False):
    """[(status, result)] per item, result the bytes or the negative error code; status 0 whole, 1 split, 2 split and decoded again."""
    n = len(items)
    so, do = _offsets([len(x) for x in items]), _offsets(caps)
    dst = C.create_string_buffer(max(sum(caps), 1) + 64)
    res, st = (U64 * max(n, 1))(), (C.c_int * max(n, 1))()
    L.zbs_decode(b"".join(items), so, do, n, int(magicless), dst, res, st)
    return [(st[i], dst.raw[do[i]:do[i] + res[i]] if res[i] <= ERR_MAX else -((1 << 64) - res[i])) for i in range(n)]


def _data(seed: int, n: int) -> bytes:
    rnd = random.Random(seed)
    words = [bytes(rnd.choice(b"abcdefghijklmnop") for _ in range(rnd.randrange(2, 10))) for _ in range(300)]
    out = bytearray()
    while len(out) < n:
        out += rnd.choice(words) + (b" " if rnd.random() < 0.9 else bytes([rnd.randrange(256)]))
    return bytes(out[:n])


def _tiny(seed: int, n: int) -> bytes:
    """Content that compresses to a few dozen bytes: items of such frames can be cut at every byte."""
    return bytes((seed + k) & 0xFF for k in range(7)) * (n // 7) + b"x" * (n % 7)


def _frames(make=ref_compress_flags):
    """One-block frames of 33-120 KB: with and without content size and checksum, at levels 1 and 3."""
    out = []
    for k in range(6):
        f = make(_data(k, 33_000 + 17_000 * k), 1 + 2 * (k % 2), checksum=k % 3 == 1, content_size=k % 4 != 3)
        assert isinstance(f, bytes)
        out.append(f)
    return out


def _items(make=ref_compress_flags):
    f = _frames(make)
    sk = fw.skippable
    mb = [(GOLDEN / "mb_L1.zst").read_bytes(), (GOLDEN / "mb_L3_xxh.zst").read_bytes()]
    one = [(GOLDEN / f"oneshot_{k:03d}_L{1 + 2 * (k % 2 == 0)}.zst").read_bytes() for k in range(4)]
    return {
        "three": f[0] + f[1] + f[2],
        "all-sized": f[0] + f[1] + f[2] + f[4] + f[5],
        "last-unsized": f[0] + f[1] + f[3],
        "middle-unsized": f[0] + f[3] + f[1],
        "skippable-between": f[4] + sk(17, 3) + f[5] + sk(0, 15),
        "skippable-first": sk(40, 1) + f[2] + f[1],
        "two-skippable": sk(5) + sk(9, 2),
        "one-frame": f[1],
        "sixty-four": b"".join(f[k % 3] for k in range(64)),
        "with-multi-block": f[4] + mb[0] + f[5],
        "multi-block-twice": mb[1] + mb[1],
        "golden-oneshots": b"".join(one),
        "garbage": f[0] + f[1] + b"\x01\x02\x03",
        "garbage-magic": f[0] + f[1] + f[0][:4],
        "empty": b"",
    }


def _content(x, magicless=False):
    r = (ref_decompress_magicless if magicless else ref_decompress)(x, 1 << 23)
    return r if isinstance(r, bytes) else None


def _check_plans(L, items, caps, magicless=False):
    taken, dev, split, host = plans(L, items, caps, magicless)
    for i, x in enumerate(items):
        if taken[i]:
            assert split[i], i                                     # one split rule
            assert dev[i] == host[i], i                            # the same entries
            e, b = route(L, x, caps[i], magicless)
            assert e == len(host[i]) and b == 0
        else:
            assert i not in dev
    return taken, split


def test_device_plan_lists_the_host_plans_entries(split_lib):
    for make in (ref_compress_flags, hostsim_compress_flags):
        named = _items(make)
        items = list(named.values())
        want = [_content(x) for x in items]
        for delta in (0, -1, 1):                                   # capacities one byte short and one byte long
            caps = [len(w) + delta if w is not None else 1 << 20 for w in want]
            taken, split = _check_plans(split_lib, items, caps)
            k = {name: i for i, name in enumerate(named)}
            if delta >= 0:
                assert all(taken[k[n]] for n in ("three", "all-sized", "last-unsized", "skippable-between", "skippable-first", "sixty-four"))
            assert not any(taken[k[n]] for n in ("middle-unsized", "two-skippable", "one-frame", "garbage", "garbage-magic", "empty"))
            assert not taken[k["with-multi-block"]]                 # stays on the loop
            assert route(split_lib, items[k["with-multi-block"]], caps[k["with-multi-block"]])[1] == 5


def test_device_plan_at_the_split_minimum(split_lib):
    for avg in (SPLIT_MIN_BYTES - 1, SPLIT_MIN_BYTES):
        split = int(avg >= SPLIT_MIN_BYTES)
        sizes = [(4 * avg) // 3, (4 * avg) // 3, 4 * avg - 2 * ((4 * avg) // 3)]      # three frames and a skippable one: 4 entries
        frames = [ref_compress_flags(_tiny(k, n), 3) for k, n in enumerate(sizes)]
        pair = [ref_compress_flags(_tiny(5 + k, avg), 1) for k in range(2)]
        items = [frames[0] + fw.skippable(3) + frames[1] + frames[2], pair[0] + pair[1], frames[0] + frames[1] + frames[2]]
        caps = [4 * avg, 2 * avg, 4 * avg]
        taken, _ = _check_plans(split_lib, items, caps)
        assert taken == [split, split, 1]


def test_device_plan_cuts_garbage_and_magicless(split_lib):
    frames = [ref_compress_flags(_tiny(k, 40_000 + 999 * k), 1 + 2 * (k % 2), checksum=k == 1, content_size=k != 2) for k in range(3)]
    base = frames[0] + fw.skippable(6, 9) + frames[1] + frames[2]
    cap = 140_000                                                  # (the last frame has no size: it gets the rest)
    items = [base[:cut] for cut in range(len(base) + 1)] + [base + g for g in (b"\x00", b"\x28\xb5\x2f\xfd", fw.skippable(3)[:6])]
    taken, _ = _check_plans(split_lib, items, [cap] * len(items))
    assert taken[len(base)] == 1
    m = [ref_compress_flags(_data(50 + k, 40_000 + 9000 * k), 1 + 2 * k, checksum=k == 1, content_size=k != 2, magicless=True)
         for k in range(3)]
    mitems = [m[0] + m[1] + m[2], m[2] + m[0], m[0] + fw.skippable(4) + m[1], m[0] + m[1] + b"\x00"]
    mcaps = [len(_content(x, True) or b"") or 1 << 20 for x in mitems]
    taken, _ = _check_plans(split_lib, mitems, mcaps, magicless=True)
    assert taken == [1, 0, 0, 0]                                   # m[2] has no size; a skippable magic starts a (bad) frame


def test_device_plan_limit_and_routing(split_lib, loop_lib):
    f = _frames()
    items = [f[0] + f[1], f[1] + f[2] + f[4], f[2] + f[0]]
    caps = [len(_content(x)) for x in items]
    taken, dev, _, host = plans(split_lib, items, caps, max_entries=5)
    assert taken == [1, 1, 0]                                      # the third item's entries would end past the list
    assert dev == {0: host[0], 1: host[1]}
    # every item the device does not split is routed as before: the loop's candidates by their blocks, the others by the other decoders
    others = list(_items().values()) + [(GOLDEN / p).read_bytes() for p in ("mb_L9.zst", "mb_two_frames_skippable.zst", "concat_skippable.zst")]
    for x in others:
        cap = len(_content(x) or b"") or 1 << 20
        e, b = route(split_lib, x, cap)
        if not e:
            assert b == loop_lib.zbl_item_blocks(x, len(x), 0)


def _short_frame(rnd, n):
    """A frame that declares one byte more than it regenerates."""
    content = fw.text(rnd, n)
    f = bytearray(fw._write(content, fw.Frame([fw.Block(size=len(content), lit=fw.Lit("huf"))], window_log=17, fcs_bytes=4), rnd))
    at = 4 + 1 + 1
    f[at:at + 4] = (int.from_bytes(f[at:at + 4], "little") + 1).to_bytes(4, "little")
    return bytes(f), content


def _check_settle(L, items, caps, magicless=False):
    fused = hostsim_decompress_magicless if magicless else hostsim_decompress
    got = settle(L, items, caps, magicless)
    for k, (x, cap, (st, r)) in enumerate(zip(items, caps, got)):
        assert r == fused(x, cap), k
    return [st for st, _ in got]


def test_settling_gives_the_fused_decoders_result(split_lib):
    rnd = random.Random(3)
    f = _frames()
    good = [f[0] + f[1] + f[2], f[1] + fw.skippable(8) + f[4], f[0] + f[1] + f[3]]
    caps = [len(_content(x)) for x in good]
    assert _check_settle(split_lib, good, caps) == [1, 1, 1]
    short, content = _short_frame(rnd, 40_000)
    assert ref_decompress(short, 1 << 20) != content
    bad = [f[0] + short + f[1]]
    ck = bytearray(f[1]); ck[-2] ^= 0x10                          # the stored checksum of a checksummed frame
    bad.append(f[0] + bytes(ck) + f[2])
    for x in good:
        for _ in range(12):
            z = bytearray(x)
            z[rnd.randrange(len(z))] ^= 1 << rnd.randrange(8)
            bad.append(bytes(z))
        for _ in range(4):
            cut = rnd.randrange(len(x))
            bad.append(x[:cut] + x[cut + rnd.randrange(1, 40):])
    bcaps = [max(caps) + 40_001] * len(bad)
    st = _check_settle(split_lib, bad, bcaps)
    assert st[0] == 2 and st[1] == 2 and st.count(2) >= 6


# ---------------------------------------------------------------------------------------------------------------------------- GPU
def _lib():
    from zstd_jni_b200 import _native
    return _native.lib()


def _ctx(pipeline=1, magicless=0):
    from zstd_jni_b200.zstd import ZstdBatchContext
    ctx = ZstdBatchContext(0)
    ctx.setOption("dec_pipeline", pipeline)
    if magicless:
        ctx.setOption("magicless", 1)
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


def _both(items, caps, magicless=0, timing=False):
    """The device call on a dec_pipeline 1 and a dec_pipeline 0 context: the same bytes and codes; and the reference's bytes wherever the
    reference regenerates the item.  Returns the results and, with timing, the new context's kernel times."""
    ref = ref_decompress_magicless if magicless else ref_decompress
    with _ctx(1, magicless) as new, _ctx(0, magicless) as old:
        if timing:
            new.setOption("timing", 1)
        got = call_device(new, items, caps)
        times = new.kernelTimes() if timing else None
        assert got == call_device(old, items, caps)
    for k, (x, cap) in enumerate(zip(items, caps)):
        r = ref(x, cap)
        if isinstance(r, bytes):
            assert got[k] == r, k
        else:
            assert isinstance(got[k], int), k
    return got, times


def _pieces(n, size, seed, level=3, **kw):
    contents = [_data(seed + k, size) for k in range(n)]
    return [ref_compress_flags(c, level, **kw) for c in contents], contents


@pytest.mark.gpu
def test_device_call_splits_items_of_64_frames():
    from zstd_jni_b200.zstd import ZstdCompressCtx
    frames, contents = _pieces(64, 128 << 10, 1000)
    items, want = [], []
    for i in range(128):
        order = [(i * 5 + k) % 64 for k in range(64)]
        items.append(b"".join(frames[k] for k in order)); want.append(b"".join(contents[k] for k in order))
    got, times = _both(items, [len(w) for w in want], timing=True)
    assert got == want
    assert times["k_split_parts"][0] > 0 and times["k_decompress(marked)"][0] < 0.05 * times["k_split_parts"][0], times
    data = _data(1100, 64 << 17)
    with ZstdCompressCtx() as c:
        c.setLevel(3).setMultiFrame(True)
        z = c.compress(data)
    got, _ = _both([z] * 16, [len(data)] * 16)
    assert got == [data] * 16


@pytest.mark.gpu
def test_device_call_splits_many_short_items_and_mixed_calls():
    frames, contents = _pieces(64, 128 << 10, 2000, level=1)
    groups = [[(g * 7 + j) % 64 for j in range(2 + g % 3)] for g in range(64)]
    items = [b"".join(frames[j] for j in groups[i % 64]) for i in range(4096)]
    want = [b"".join(contents[j] for j in groups[i % 64]) for i in range(4096)]
    assert _both(items, [len(w) for w in want])[0] == want
    singles, scontents = _pieces(40, 20_000, 2100)
    mb = [(GOLDEN / p).read_bytes() for p in ("mb_L1.zst", "mb_L12.zst", "mb_L3_xxh.zst", "mb_two_frames_skippable.zst")]
    mixed, caps = [], []
    for k in range(120):
        x = (singles[k % 40], mb[k % 4], items[k], frames[k % 64] + mb[0] + frames[(k + 1) % 64])[k % 4]
        mixed.append(x); caps.append(len(_content(x)))
    _both(mixed, caps)


@pytest.mark.gpu
def test_device_call_more_items_than_a_part_and_more_entries():
    frames = [ref_compress_flags(_tiny(k, 33_000 + 100 * k), 1 + k % 3, checksum=k % 4 == 0) for k in range(16)]
    small = [ref_compress_flags(_data(3000 + k, 1000 + 37 * k), 3) for k in range(16)]
    items = []
    for i in range(16500):
        items.append(frames[i % 16] + frames[(i + 3) % 16] + frames[(i + 5) % 16] if i % 50 == 0 else small[i % 16])
    caps = [len(_content(x)) for x in items]
    _both(items, caps)
    few = [b"".join(frames[(i + k) % 16] for k in range(2 + i % 5)) for i in range(200)]     # 800 entries, 512 per part
    _both(few, [len(_content(x)) for x in few])


@pytest.mark.gpu
def test_device_call_checksums_magicless_and_corruptions():
    rnd = random.Random(7)
    f, c = _pieces(8, 60_000, 4000, checksum=True)
    items = [f[0] + f[1] + f[2], f[3] + fw.skippable(11) + f[4]]
    ck = bytearray(f[5]); ck[-1] ^= 0x08
    items.append(f[6] + bytes(ck) + f[7])
    short, _ = _short_frame(rnd, 40_000)
    items.append(f[0] + short + f[1])
    for x in items[:2]:
        for _ in range(20):
            z = bytearray(x)
            z[rnd.randrange(len(z))] ^= 1 << rnd.randrange(8)
            items.append(bytes(z))
        for _ in range(5):
            cut = rnd.randrange(len(x))
            items.append(x[:cut] + x[cut + rnd.randrange(1, 40):])
    caps = [200_000] * len(items)
    got, _ = _both(items, caps)
    assert got[0] == c[0] + c[1] + c[2] and isinstance(got[2], int) and isinstance(got[3], int)
    m = [ref_compress_flags(_data(5000 + k, 40_000 + 9000 * k), 1 + 2 * (k % 2), checksum=k == 1, magicless=True) for k in range(4)]
    mitems = [m[0] + m[1] + m[2], m[3] + m[0], m[1]]
    _both(mitems, [len(_content(x, True)) for x in mitems], magicless=1)


@pytest.mark.gpu
def test_device_call_returns_before_the_split_work_is_done():
    import torch
    frames, contents = _pieces(16, 128 << 10, 6000)
    items = [b"".join(frames[(i + k) % 16] for k in range(64)) for i in range(64)]
    want = b"".join(b"".join(contents[(i + k) % 16] for k in range(64)) for i in range(64))
    dev = torch.device("cuda:0")
    so = np.concatenate([[0], np.cumsum([len(x) for x in items])]).astype(np.int64)
    do = np.arange(65, dtype=np.int64) * (64 << 17)
    d_src = torch.from_numpy(np.frombuffer(b"".join(items), dtype=np.uint8).copy()).to(dev)
    d_so, d_do = torch.from_numpy(so).to(dev), torch.from_numpy(do).to(dev)
    d_dst = torch.zeros(int(do[-1]), dtype=torch.uint8, device=dev)
    d_res = torch.zeros(64, dtype=torch.int64, device=dev)
    L = _lib()
    with _ctx(1) as ctx:
        s = torch.cuda.Stream()
        args = (ctx.handle, 64, d_src.data_ptr(), d_so.data_ptr(), d_dst.data_ptr(), d_do.data_ptr(), d_res.data_ptr(), s.cuda_stream)
        assert L.zstdb200_decompress_device(*args) == 0      # the first call builds the graphs
        s.synchronize()
        assert L.zstdb200_decompress_device(*args) == 0
        assert not s.query()
        s.synchronize()
        assert d_res.cpu().tolist() == [64 << 17] * 64
        assert bytes(d_dst.cpu().numpy()) == want
