"""Host-memory decompression of multi-block, multi-frame and magicless items through each call, against dec_pipeline 0 (every item
whole on the fused kernel).

Workloads (host memory in and out, outputs compared with the input before anything is reported, best of 3 after a warm-up):
  stream   one 1 GiB level-3 frame of many blocks made by the reference's streaming compressor: decompress_frames and _begin/_end
           (dec_pipeline 0: a 64 MiB frame of the same kind, one run -- one warp walks it at about 10 MB/s)
  concat   128 items of 64 concatenated 128 KB level-3 frames: decompress_frames and _begin/_end
  magicless  8192 x 128 KB magicless level-3 frames: decompress_batch, decompress_frames, _begin/_end, decompress_device
Also: the host time of one _begin on 8192 128 KB frames (what bench.py's end-to-end leg queues), and the device memory a 1 GiB
streaming frame leaves allocated on each of the four work sets.

Run from the repository root on a machine with the GPU: python scripts/gpu_frame_list_decode.py [--out FILE]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from zstd_jni_b200 import _native, corpus  # noqa: E402
from zstd_jni_b200.zstd import ZstdBatchContext  # noqa: E402
from tests.oracle_util import ref_stream_compress  # noqa: E402

L = _native.lib()
GiB = 1 << 30


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def pinned(nbytes):
    import torch
    return torch.empty(max(nbytes, 1), dtype=torch.uint8).pin_memory().numpy()


def ctx(pipeline, magicless=0):
    c = ZstdBatchContext(0)
    c.setOption("dec_pipeline", pipeline)
    c.setOption("magicless", magicless)
    return c


def frames_call(c, src, sizes, dst, caps):
    n = len(sizes)
    fs, ds = (C.c_size_t * n)(*sizes), (C.c_size_t * n)(*caps)
    r = L.zstdb200_decompress_frames(c._live(), C.c_void_p(src.ctypes.data), fs, n, C.c_void_p(dst.ctypes.data), dst.size, ds)
    assert r < (1 << 63), r
    return list(ds)


def begin_end_call(c, src, sizes, dst, caps):
    """The items cut in two, on two slots, both begun before either ends (the pipelined form)."""
    n = len(sizes)
    h = max(n // 2, 1) if n > 1 else n
    so = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    do = np.concatenate([[0], np.cumsum(caps)]).astype(np.int64)
    parts = [(0, h), (h, n)] if n > 1 else [(0, n)]
    keep, out = [], []
    for slot, (a, b) in zip((2, 3), parts):
        fs, ds = (C.c_size_t * (b - a))(*sizes[a:b]), (C.c_size_t * (b - a))(*caps[a:b])
        r = L.zstdb200_decompress_frames_begin(c._live(), slot, C.c_void_p(src.ctypes.data + int(so[a])), fs, b - a,
                                               C.c_void_p(dst.ctypes.data + int(do[a])), int(do[b] - do[a]), ds)
        assert r < (1 << 63), r
        keep.append((slot, fs, ds, b - a))
    for slot, fs, ds, m in keep:
        res = (C.c_size_t * m)()
        assert L.zstdb200_decompress_frames_end(c._live(), slot, res) < (1 << 63)
        out += list(res)
    return out


def batch_call(c, src, sizes, dst, caps):
    n = len(sizes)
    so = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    do = np.concatenate([[0], np.cumsum(caps)]).astype(np.int64)
    sp = (C.c_void_p * n)(*[src.ctypes.data + int(x) for x in so[:-1]])
    dp = (C.c_void_p * n)(*[dst.ctypes.data + int(x) for x in do[:-1]])
    res = (C.c_size_t * n)()
    r = L.zstdb200_decompress_batch(c._live(), n, sp, (C.c_size_t * n)(*sizes), dp, (C.c_size_t * n)(*caps), res)
    assert r < (1 << 63), r
    return list(res)


def device_call(c, src, sizes, dst, caps):
    import torch
    dev = torch.device("cuda:0")
    so = torch.from_numpy(np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)).to(dev)
    do = torch.from_numpy(np.concatenate([[0], np.cumsum(caps)]).astype(np.int64)).to(dev)
    d_src = torch.from_numpy(src).to(dev)
    d_dst = torch.empty(dst.size, dtype=torch.uint8, device=dev)
    d_res = torch.zeros(len(sizes), dtype=torch.int64, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    assert L.zstdb200_decompress_device(c.handle, len(sizes), d_src.data_ptr(), so.data_ptr(), d_dst.data_ptr(), do.data_ptr(), d_res.data_ptr(), st) == 0
    torch.cuda.synchronize()
    t = time.perf_counter() - t0
    dst[:] = d_dst.cpu().numpy()
    return [int(x) for x in d_res.cpu().numpy()], t


def timed(call, c, src, sizes, dst, caps, want: np.ndarray, reps=3, warm=True):
    """Best of `reps` after one warm-up run (when `warm`); the output is compared with `want` after every run."""
    best = None
    for k in range(0 if warm else 1, reps + 1):
        dst[:] = 0
        t0 = time.perf_counter()
        r = call(c, src, sizes, dst, caps)
        t = time.perf_counter() - t0
        if isinstance(r, tuple):
            r, t = r
        assert sum(r) == want.size and np.array_equal(dst[:want.size], want), call.__name__
        if k:
            best = t if best is None else min(best, t)
    return best


def report(rows, name, nbytes, t_new, t_old, old_note=""):
    rows.append({"workload": name, "bytes": nbytes, "this_GBps": round(nbytes / t_new / 1e9, 3),
                 "dec_pipeline0_GBps": round(t_old[0] / t_old[1] / 1e9, 4) if t_old else None, "note": old_note})
    print(json.dumps(rows[-1]), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    rows = [{"card": card()}]
    print(json.dumps(rows[0]), flush=True)
    new = ctx(1)
    old = ctx(0)

    # ---- one 1 GiB streaming frame of many blocks
    data = corpus.corpus(8192, size=131072).reshape(-1)
    z = np.frombuffer(ref_stream_compress(data.tobytes(), 3), dtype=np.uint8)
    zs = pinned(z.size); zs[:] = z
    dst = pinned(data.size)
    small = data[:64 << 20]
    zsm = np.frombuffer(ref_stream_compress(small.tobytes(), 3), dtype=np.uint8).copy()
    dsm = np.zeros(small.size, dtype=np.uint8)
    t_old = timed(frames_call, old, zsm, [zsm.size], dsm, [small.size], small, reps=1, warm=False)
    for call in (frames_call, begin_end_call):
        report(rows, f"stream-1GiB/{call.__name__}", data.size, timed(call, new, zs, [z.size], dst, [data.size], data), (small.size, t_old),
               "dec_pipeline 0 timed on a 64 MiB frame of the same kind, one run")

    # device memory a new context holds after a 1 GiB streaming frame on work sets 0, 0-1, 0-2 and 0-3 (input, output and segment
    # workspaces of each set)
    import torch
    fresh = ctx(1)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    grown = []
    for slot in range(4):
        fs, ds = (C.c_size_t * 1)(z.size), (C.c_size_t * 1)(data.size)
        assert L.zstdb200_decompress_frames_begin(fresh._live(), slot, C.c_void_p(zs.ctypes.data), fs, 1, C.c_void_p(dst.ctypes.data), dst.size, ds) < (1 << 63)
        assert L.zstdb200_decompress_frames_end(fresh._live(), slot, None) < (1 << 63)
        grown.append((free0 - torch.cuda.mem_get_info()[0]) / GiB)
    assert np.array_equal(dst, data)
    fresh.close()
    rows.append({"device_memory_GiB_after_slots_0_to_3": [round(g, 3) for g in grown]})
    print(json.dumps(rows[-1]), flush=True)
    del z, zs

    # ---- 128 items of 64 concatenated 128 KB level-3 frames
    stream, sizes = new.compressChunks(data, 131072, 3)
    stream = stream.copy()
    fsz = sizes.astype(np.int64)
    items = [int(fsz[k * 64:(k + 1) * 64].sum()) for k in range(128)]
    src = pinned(stream.size); src[:] = stream
    caps = [64 * 131072] * 128
    for call in (frames_call, begin_end_call):
        t = timed(call, new, src, items, dst, caps, data)
        t_old = timed(call, old, src, items, dst, caps, data, reps=1)
        report(rows, f"concat-128x64/{call.__name__}", data.size, t, (data.size, t_old), "dec_pipeline 0: one run")

    # ---- the host time of one _begin on 8192 128 KB frames (bench.py's end-to-end leg)
    one = [int(x) for x in fsz]
    fs, ds = (C.c_size_t * 8192)(*one), (C.c_size_t * 8192)(*([131072] * 8192))
    for k in range(4):
        t0 = time.perf_counter()
        assert L.zstdb200_decompress_frames_begin(new._live(), 2, C.c_void_p(src.ctypes.data), fs, 8192, C.c_void_p(dst.ctypes.data), dst.size, ds) < (1 << 63)
        tb = time.perf_counter() - t0
        assert L.zstdb200_decompress_frames_end(new._live(), 2, None) < (1 << 63)
    assert np.array_equal(dst, data)
    rows.append({"begin_host_ms_8192_frames": round(tb * 1e3, 3)})
    print(json.dumps(rows[-1]), flush=True)

    # ---- 8192 x 128 KB magicless frames
    newm, oldm = ctx(1, 1), ctx(0, 1)
    newm_c = ZstdBatchContext(0)
    newm_c.setOption("magicless", 1)
    stream, sizes = newm_c.compressChunks(data, 131072, 3)
    newm_c.close()
    src = pinned(stream.size); src[:] = stream
    one = [int(x) for x in sizes]
    caps = [131072] * 8192
    for call in (batch_call, frames_call, begin_end_call, device_call):
        t = timed(call, newm, src, one, dst, caps, data)
        t_old = timed(call, oldm, src, one, dst, caps, data)
        report(rows, f"magicless-8192/{call.__name__}", data.size, t, (data.size, t_old))
    if args.out:
        Path(args.out).write_text(json.dumps(rows, indent=1))


if __name__ == "__main__":
    main()
