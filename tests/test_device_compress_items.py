"""zstdb200_compress_items_device: items in device memory cut into chunks, compressed and packed into multi-frame streams on the GPU.

CPU: the host instantiation of the call's plan (tests/hostsim/zb_hostsim_citems.cpp, compiled by this module), in parts of as few as 3
slots, against a plain computation with chunk_count: every chunk's input range and item, the padding slots (empty, at the end of their
part, never packed), every frame's packed offset, every item's output offsets and result -- random item sizes around the chunk size,
chunk sizes 1, 4096 and 131072, a capacity at the bound and one byte short of it, and error frames in the middle of items.
GPU: the call against the reference's one-shot frames of every chunk (or zstdb200_compress_chunks without the compiled reference) at
levels 1, 3, 9 and 19, with a checksum, without content sizes, magicless and with explicit parameters; 8192 items of 128 KB, 64 of 16 MB,
20 000 of 0-300 KB, more chunks than one part holds and empty items; the per-frame refusals and a short capacity; the streams decode
again on zstdb200_decompress_device; and the call returns before its work is done.
"""
from __future__ import annotations

import ctypes as C
import random
import subprocess
from pathlib import Path

import numpy as np
import pytest

from tests.oracle_util import ERR_MAX, ref, ref_compress_flags, ref_compress_params

ROOT = Path(__file__).resolve().parent.parent
U64 = C.c_ulonglong
BLOCK = 128 << 10
E_PARAMETER_UNSUPPORTED, E_PARAMETER_OUT_OF_BOUND, E_DST_SIZE_TOO_SMALL = 40, 42, 70


def err(code):
    return (1 << 64) - code


def compress_bound(x):
    return x + (x >> 8) + (((BLOCK - x) >> 11) if x < BLOCK else 0)


def chunks_of(size, cs):
    """The (start, end) of an item's chunks, relative to the item: one empty chunk for an empty item."""
    return [(q * cs, min((q + 1) * cs, size)) for q in range(max(1, -(-size // cs)))]


def items_bound(sizes, cs):
    return sum(compress_bound(e - s) for size in sizes for s, e in chunks_of(size, cs))


# ---------------------------------------------------------------------------------------------------------------------------- CPU
@pytest.fixture(scope="module")
def plan_lib(tmp_path_factory):
    src = ROOT / "tests" / "hostsim" / "zb_hostsim_citems.cpp"
    so = tmp_path_factory.mktemp("zb_hostsim_citems") / "libzb_hostsim_citems.so"
    subprocess.run(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-Wall", "-Wno-unused-function", "-x", "c++", str(src), "-o", str(so)],
                   check=True)
    L = C.CDLL(str(so))
    P64 = C.POINTER(U64)
    L.zbc_plan.restype = None
    L.zbc_plan.argtypes = [P64, C.c_size_t, U64, U64, C.c_uint, P64, U64, P64, P64, C.POINTER(C.c_uint), P64, C.c_size_t, P64, P64, P64]
    return L


def device_plan(L, sizes, cs, cap, P, frames, pad_frame=13):
    """The plan as the kernels run it: per chunk (start, end, item, packed offset), the output offsets, the results and the stats."""
    n = len(sizes)
    m = sum(len(chunks_of(s, cs)) for s in sizes)
    a = lambda k, t=U64: (t * max(k, 1))()
    start, end, item, packed = a(m), a(m), a(m, C.c_uint), a(m)
    dst_off, results, stats = a(n + 1), a(n), a(5)
    L.zbc_plan((U64 * max(n, 1))(*sizes), n, cs, cap, P, (U64 * max(m, 1))(*frames), pad_frame, start, end, item, packed, m, dst_off, results,
               stats)
    chunks = list(zip(start[:m], end[:m], item[:m], packed[:m]))
    return chunks, list(dst_off[:n + 1]), list(results[:n]), list(stats)


def host_plan(sizes, cs, cap, frames):
    """The same from chunk_count alone: chunks in item order, packed back to back, errors taking no room."""
    chunks, at = [], 0
    for i, size in enumerate(sizes):
        chunks += [(at + s, at + e, i) for s, e in chunks_of(size, cs)]
        at += size
    if items_bound(sizes, cs) > cap:
        return None, [0] * (len(sizes) + 1), [err(E_DST_SIZE_TOO_SMALL)] * len(sizes)
    packed, dst_off, results, first_err, pos = [], [None] * len(sizes), [0] * len(sizes), [None] * len(sizes), 0
    for (s, e, i), r in zip(chunks, frames):
        if dst_off[i] is None:
            dst_off[i] = pos
        packed.append((s, e, i, pos))
        if r > ERR_MAX:
            first_err[i] = first_err[i] or r
        else:
            results[i] += r
            pos += r
    return packed, dst_off + [pos], [e or r for e, r in zip(first_err, results)]


def _sizes(rnd, cs, n, top):
    special = [0, 1, cs - 1, cs, cs + 1, 0, 2 * cs, 3 * cs + 1]
    return [rnd.choice(special) if rnd.random() < 0.3 else rnd.randrange(0, top) for _ in range(n)]


def _frames(rnd, sizes, cs, errors=0.0):
    out = []
    for size in sizes:
        for s, e in chunks_of(size, cs):
            out.append(err(rnd.choice((E_PARAMETER_UNSUPPORTED, 72, 1))) if rnd.random() < errors else rnd.randrange(9, compress_bound(e - s) + 1))
    return out


def _check(L, sizes, cs, cap, P, frames):
    chunks, dst_off, results, stats = device_plan(L, sizes, cs, cap, P, frames)
    want_chunks, want_off, want_res = host_plan(sizes, cs, cap, frames)
    assert results == want_res and dst_off == want_off
    if want_chunks is None:
        assert stats[:2] == [0, 0]                                  # no part runs
        return stats
    m = len(want_chunks)
    assert chunks == want_chunks and stats[0] == m
    assert stats[1] == -(-m // P)                                   # parts
    assert stats[2] == stats[1] * P - m and stats[3] == 0 and stats[4] == 0      # padding: empty, at the part's end, never packed
    return stats


@pytest.mark.parametrize("cs", [1, 4096, 131072])
def test_plan_matches_chunk_count(plan_lib, cs):
    rnd = random.Random(cs)
    top = 40 if cs == 1 else 4 * cs
    for trial in range(12):
        sizes = _sizes(rnd, cs, rnd.randrange(1, 60), top)
        frames = _frames(rnd, sizes, cs)
        bound = items_bound(sizes, cs)
        for P in (3, 7, min(16384, len(sizes) + bound // cs)):
            _check(plan_lib, sizes, cs, bound, P, frames)
            _check(plan_lib, sizes, cs, bound + 1000, P, frames)


@pytest.mark.parametrize("cs", [1, 4096, 131072])
def test_plan_capacity_one_byte_short(plan_lib, cs):
    rnd = random.Random(100 + cs)
    sizes = _sizes(rnd, cs, 30, 40 if cs == 1 else 3 * cs)
    frames = _frames(rnd, sizes, cs)
    bound = items_bound(sizes, cs)
    _check(plan_lib, sizes, cs, bound, 3, frames)
    _, dst_off, results, _ = device_plan(plan_lib, sizes, cs, bound - 1, 3, frames)
    assert results == [err(E_DST_SIZE_TOO_SMALL)] * len(sizes) and dst_off == [0] * (len(sizes) + 1)


def test_plan_error_frame_in_the_middle_of_an_item(plan_lib):
    cs = 4096
    sizes = [10_000, 5 * cs + 7, 0, 3 * cs, 1]
    rnd = random.Random(5)
    frames = _frames(rnd, sizes, cs)
    good = device_plan(plan_lib, sizes, cs, items_bound(sizes, cs), 3, frames)
    # item 1's chunks are 3 .. 8: its third and fifth frames fail
    bad = list(frames)
    bad[5], bad[7] = err(E_PARAMETER_UNSUPPORTED), err(72)
    stats = _check(plan_lib, sizes, cs, items_bound(sizes, cs), 3, bad)
    _, dst_off, results, _ = device_plan(plan_lib, sizes, cs, items_bound(sizes, cs), 3, bad)
    assert results[1] == err(E_PARAMETER_UNSUPPORTED)                              # the first error among the item's frames
    assert results[:1] + results[2:] == good[2][:1] + good[2][2:]
    lost = frames[5] + frames[7]                                                   # the failed frames take no room ...
    assert dst_off[:2] == good[1][:2] and dst_off[2:] == [x - lost for x in good[1][2:]]      # ... and the items after keep their streams
    assert stats[1] == 5


def test_plan_with_random_errors_and_many_parts(plan_lib):
    rnd = random.Random(9)
    for cs in (1, 4096, 131072):
        sizes = _sizes(rnd, cs, 200, 40 if cs == 1 else 3 * cs)
        frames = _frames(rnd, sizes, cs, errors=0.1)
        _check(plan_lib, sizes, cs, items_bound(sizes, cs), 3, frames)


# ---------------------------------------------------------------------------------------------------------------------------- GPU
def _lib():
    from zstd_jni_b200 import _native
    return _native.lib()


def _data(rng, n):
    """Compressible bytes: a small alphabet, in a random block of at most 8 MB repeated."""
    block = rng.integers(97, 113, size=min(n, 8 << 20), dtype=np.uint8)
    return np.resize(block, n).tobytes() if n else b""


def call_items(ctx, items, level, cs, cap=None, stream=None):
    """(per item its stream or the negative error code, the output offsets).  cap: the output's capacity (default: the bound)."""
    import torch
    dev = torch.device("cuda:0")
    n = len(items)
    so = np.concatenate([[0], np.cumsum([len(x) for x in items])]).astype(np.int64)
    cap = items_bound([len(x) for x in items], cs) if cap is None else cap
    d_src = torch.from_numpy(np.frombuffer(b"".join(items) or b"\0", dtype=np.uint8).copy()).to(dev)
    d_so = torch.from_numpy(so).to(dev)
    d_dst = torch.zeros(max(cap, 1), dtype=torch.uint8, device=dev)
    d_do = torch.full((n + 1,), -1, dtype=torch.int64, device=dev)
    d_res = torch.zeros(max(n, 1), dtype=torch.int64, device=dev)
    s = stream or torch.cuda.Stream()
    r = _lib().zstdb200_compress_items_device(ctx.handle, level, cs, n, d_src.data_ptr(), d_so.data_ptr(), d_dst.data_ptr(), cap, d_do.data_ptr(),
                                             d_res.data_ptr(), s.cuda_stream)
    assert r == 0, r
    s.synchronize()
    do = [int(x) for x in d_do.cpu().numpy()]
    res = [int(x) & ((1 << 64) - 1) for x in d_res.cpu().numpy()[:n]]
    out = d_dst.cpu().numpy()
    got = []
    for i, r in enumerate(res):
        assert do[i] <= do[i + 1]
        got.append(out[do[i]:do[i + 1]].tobytes() if r <= ERR_MAX else -((1 << 64) - r))
        if r <= ERR_MAX:
            assert r == do[i + 1] - do[i]
    return got, do


def want_streams(ctx, items, level, cs, flags=None, params=None):
    """Per item the reference's one-shot frames of its chunks, concatenated; zstdb200_compress_chunks's stream without the reference."""
    out = []
    for x in items:
        if ref() is not None:
            pieces = [x[s:e] for s, e in chunks_of(len(x), cs)]
            frames = [ref_compress_params(p, level, params, checksum=(flags or {}).get("checksum", False)) if params else
                      ref_compress_flags(p, level, **(flags or {})) for p in pieces]
            out.append(next((f for f in frames if isinstance(f, int)), None) or b"".join(frames))
        else:
            out.append(ctx.compressChunks(x, cs, level)[0].tobytes())
    return out


def _ctx(**options):
    from zstd_jni_b200.zstd import ZstdBatchContext
    ctx = ZstdBatchContext(0)
    for k, v in options.items():
        ctx.setOption(k, v)
    return ctx


def _varied(cs, seed):
    rng = np.random.default_rng(seed)
    return [_data(rng, n) for n in (0, 1, 777, cs - 1, cs, cs + 1, 3 * cs + cs // 2, 0, 20_000)]


@pytest.mark.gpu
@pytest.mark.parametrize("level,cs", [(1, BLOCK), (3, BLOCK), (9, BLOCK), (19, 65536), (3, 4096)])
def test_streams_are_the_references_frames(level, cs):
    items = _varied(cs, level)
    with _ctx() as ctx:
        got, _ = call_items(ctx, items, level, cs)
        assert got == want_streams(ctx, items, level, cs)


@pytest.mark.gpu
@pytest.mark.parametrize("options", [{"checksum": 1}, {"content_size": 0}, {"magicless": 1}, {"checksum": 1, "content_size": 0, "magicless": 1}])
def test_streams_with_frame_options(options):
    items = _varied(BLOCK, 7)
    flags = {"checksum": bool(options.get("checksum", 0)), "content_size": bool(options.get("content_size", 1)),
             "magicless": bool(options.get("magicless", 0))}
    with _ctx(**options) as ctx:
        got, _ = call_items(ctx, items, 3, BLOCK)
        assert got == want_streams(ctx, items, 3, BLOCK, flags=flags)
        if not options.get("magicless"):
            assert all(g[:4] == b"\x28\xb5\x2f\xfd" for g in got)


@pytest.mark.gpu
def test_streams_with_explicit_parameters():
    params = {"hashLog": 14, "minMatch": 5, "strategy": 2}
    items = _varied(BLOCK, 8)
    with _ctx() as ctx:
        plain = call_items(ctx, items, 3, BLOCK)[0]
        for k, v in params.items():
            ctx.setOption("c_" + k, v)
        got, _ = call_items(ctx, items, 3, BLOCK)                # the graph is built again for the options it runs with
        assert got == want_streams(ctx, items, 3, BLOCK, params=params) and got != plain
        for k in params:
            ctx.setOption("c_" + k, 0)
        assert call_items(ctx, items, 3, BLOCK)[0] == plain


def _batch_streams(ctx, items, level, cs):
    """Every chunk through zstdb200_compress_batch (one frame each, as the reference's one-shot frame), concatenated per item."""
    pieces = [x[s:e] for x in items for s, e in chunks_of(len(x), cs)]
    frames = ctx.compressBatch(pieces, level)
    out, k = [], 0
    for x in items:
        c = len(chunks_of(len(x), cs))
        out.append(b"".join(frames[k:k + c]))
        k += c
    return out


def _round_trip(items, streams, do):
    """The packed streams, at the call's output offsets, through zstdb200_decompress_device on a context with default options."""
    from tests.test_device_split import call_device
    assert [sum(len(s) for s in streams[:i]) for i in range(len(streams) + 1)] == do
    with _ctx() as ctx:
        assert call_device(ctx, streams, [len(x) for x in items]) == items


@pytest.mark.gpu
def test_shapes_8192_items_of_128k_and_64_of_16m():
    rng = np.random.default_rng(1)
    with _ctx() as ctx:
        for n, size in ((8192, BLOCK), (64, 16 << 20)):
            data = _data(rng, n * size)
            items = [data[i * size:(i + 1) * size] for i in range(n)]
            got, do = call_items(ctx, items, 1, BLOCK)
            assert b"".join(got) == ctx.compressChunks(data, BLOCK, 1)[0].tobytes()      # the items tile the chunks of the whole
            if n == 64:
                _round_trip(items, got, do)


@pytest.mark.gpu
def test_shapes_20000_mixed_items_and_several_parts():
    rng = np.random.default_rng(2)
    sizes = [int(x) for x in rng.integers(0, 300 << 10, size=20_000)]
    sizes[::997] = [0] * len(sizes[::997])
    data = _data(rng, sum(sizes))
    offs = np.concatenate([[0], np.cumsum(sizes)])
    items = [data[offs[i]:offs[i + 1]] for i in range(len(sizes))]
    with _ctx(timing=1) as ctx:
        got, do = call_items(ctx, items, 1, BLOCK)
        times = ctx.kernelTimes()
        assert times["k_compress_parts"][1] == 1 and "k_parse+k_entropy" not in times, times
        assert got == _batch_streams(ctx, items, 1, BLOCK)
        _round_trip(items, got, do)
        # more than 16384 chunks of 4 KB: items cross the parts
        small = items[1:501]
        many = [x for x in small if x]
        assert sum(len(chunks_of(len(x), 4096)) for x in many) > 16384
        got, do = call_items(ctx, many, 3, 4096)
        assert got == _batch_streams(ctx, many, 3, 4096)
        _round_trip(many, got, do)
        empty = [b""] * 5 + [items[1]] + [b""] * 3
        got, do = call_items(ctx, empty, 3, BLOCK)
        assert got == _batch_streams(ctx, empty, 3, BLOCK)
        assert do[0] == 0 and len(got[0]) > 0                  # an empty item is one empty frame


@pytest.mark.gpu
def test_refusals_and_a_short_capacity():
    rng = np.random.default_rng(3)
    items = [_data(rng, n) for n in (0, 1000, 65536, 65537, BLOCK, 200_000, 50_000)]
    with _ctx() as ctx:
        got, do = call_items(ctx, items, 19, BLOCK)
        for x, g in zip(items, got):
            if len(x) > 65536:
                assert g == -E_PARAMETER_UNSUPPORTED
            else:
                assert g == want_streams(ctx, [x], 19, BLOCK)[0]
        bound = items_bound([len(x) for x in items], BLOCK)
        got, do = call_items(ctx, items, 3, BLOCK, cap=bound - 1)
        assert got == [-E_DST_SIZE_TOO_SMALL] * len(items) and do == [0] * (len(items) + 1)
        assert call_items(ctx, items, 3, BLOCK, cap=bound)[0] == want_streams(ctx, items, 3, BLOCK)
        L = _lib()
        for cs in (0, BLOCK + 1):                               # refused before anything is queued
            assert L.zstdb200_compress_items_device(ctx.handle, 3, cs, 1, 0, 0, 0, 0, 0, 0, 0) == err(E_PARAMETER_OUT_OF_BOUND)
        assert call_items(ctx, [], 3, BLOCK)[1] == [0]


@pytest.mark.gpu
def test_device_call_returns_before_the_compression_is_done():
    import torch
    rng = np.random.default_rng(4)
    items = [_data(rng, 1 << 20) for _ in range(256)]
    want = b"".join(items)
    dev = torch.device("cuda:0")
    so = np.arange(257, dtype=np.int64) << 20
    cap = items_bound([1 << 20] * 256, BLOCK)
    d_src = torch.from_numpy(np.frombuffer(want, dtype=np.uint8).copy()).to(dev)
    d_so = torch.from_numpy(so).to(dev)
    d_dst = torch.zeros(cap, dtype=torch.uint8, device=dev)
    d_do = torch.zeros(257, dtype=torch.int64, device=dev)
    d_res = torch.zeros(256, dtype=torch.int64, device=dev)
    L = _lib()
    with _ctx() as ctx:
        s = torch.cuda.Stream()
        args = (ctx.handle, 9, BLOCK, 256, d_src.data_ptr(), d_so.data_ptr(), d_dst.data_ptr(), cap, d_do.data_ptr(), d_res.data_ptr(), s.cuda_stream)
        assert L.zstdb200_compress_items_device(*args) == 0      # the first call builds the graph
        s.synchronize()
        assert L.zstdb200_compress_items_device(*args) == 0
        assert not s.query()
        s.synchronize()
        do = d_do.cpu().tolist()
        assert d_res.cpu().tolist() == [do[i + 1] - do[i] for i in range(256)]
        assert bytes(d_dst.cpu().numpy()[:do[-1]]) == ctx.compressChunks(want, BLOCK, 9)[0].tobytes()
