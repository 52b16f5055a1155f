"""Rate of ZSTD_decompressStream on one reference-made frame of many blocks, host memory in and out.

Runs the frame through ZSTD_decompressStream (as the direct-buffer stream drives it) and ZstdInputStream, best of 3 after a warm-up, and
the reference's ZSTD_decompressStream on one host thread; reports the growth of the process's resident memory during the timed runs (the
stream's own host memory, measured after a warm-up run), and prints one JSON line with the card's name and power limit.
    python scripts/gpu_stream_decode.py [--level 1] [--mb 1024] [--lib path/to/libzstdb200.so] [--cap-mb 0]
--lib measures another build of the library (an earlier commit; ZSTD_decompressStream only); --cap-mb feeds only that much input.
"""
from __future__ import annotations

import argparse
import ctypes as C
import io
import json
import os
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def text(n: int, seed: int) -> bytes:
    import numpy as np
    rnd = np.random.default_rng(seed)
    words = rnd.integers(97, 123, size=(4000, 8), dtype=np.uint8)
    words[:, 7] = 32
    return words[rnd.zipf(1.4, size=n // 8 + 1) % 4000].tobytes()[:n]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--level", type=int, default=1)
    ap.add_argument("--mb", type=int, default=1024)
    ap.add_argument("--lib", default="")
    ap.add_argument("--cap-mb", type=int, default=0)
    a = ap.parse_args()
    if a.lib:
        os.environ["ZSTDB200_LIBRARY"] = a.lib
    import threading

    from tests.oracle_util import ERR_MAX, ref, ref_stream_compress
    from zstd_jni_b200 import _native
    data = text(a.mb << 20, a.level)
    frame = ref_stream_compress(data, a.level, 8 << 20, False)
    if a.cap_mb:
        frame = frame[: a.cap_mb << 20]
    if a.lib:
        L = C.CDLL(a.lib)
        for n, r, args in (("ZSTD_createDStream", C.c_void_p, []), ("ZSTD_initDStream", C.c_size_t, [C.c_void_p]),
                           ("ZSTD_freeDStream", C.c_size_t, [C.c_void_p]), ("ZSTD_decompressStream", C.c_size_t, [C.c_void_p] * 3)):
            getattr(L, n).restype = r; getattr(L, n).argtypes = args
    else:
        L = _native.lib()
    R = ref()
    if R is not None:
        for n, r, args in (("ZSTD_createDCtx", C.c_void_p, []), ("ZSTD_freeDCtx", C.c_size_t, [C.c_void_p]),
                           ("ZSTD_decompressStream", C.c_size_t, [C.c_void_p] * 3)):
            getattr(R, n).restype = r; getattr(R, n).argtypes = args

    def rss():
        with open("/proc/self/statm") as f:
            return int(f.read().split()[1]) * os.sysconf("SC_PAGE_SIZE")

    peak = [0]
    stop = threading.Event()

    def sample():
        while not stop.is_set():
            peak[0] = max(peak[0], rss())
            time.sleep(0.002)

    def run_stream(lib=None):
        lib = lib or L
        z = lib.ZSTD_createDCtx() if lib is R else lib.ZSTD_createDStream()
        out = C.create_string_buffer(1 << 17)
        src = C.create_string_buffer(frame, len(frame))
        n = 0
        ib = _native.InBuffer(C.cast(src, C.c_void_p), len(frame), 0)
        t = time.perf_counter()
        while True:
            ob = _native.OutBuffer(C.cast(out, C.c_void_p), 1 << 17, 0)
            r = lib.ZSTD_decompressStream(z, C.byref(ob), C.byref(ib))
            assert r <= ERR_MAX, r
            n += ob.pos
            if r == 0 or (ib.pos == ib.size and ob.pos == 0):
                break
        dt = time.perf_counter() - t
        lib.ZSTD_freeDCtx(z) if lib is R else lib.ZSTD_freeDStream(z)
        return n, dt

    def run_input_stream():
        from zstd_jni_b200.zstd import ZstdInputStream
        t = time.perf_counter()
        s = ZstdInputStream(io.BytesIO(frame))
        n = 0
        while True:
            b = s.read(8 << 20)
            if not b:
                break
            n += len(b)
        return n, time.perf_counter() - t

    res = {"level": a.level, "content_mb": a.mb, "compressed_bytes": len(frame), "library": a.lib or "this tree"}
    runs = [("ZSTD_decompressStream", run_stream)] + ([] if a.lib else [("ZstdInputStream", run_input_stream)])
    for name, fn in runs:
        fn()                                  # warm-up: the CUDA context and the pooled batch contexts are made here
        base = rss(); peak[0] = base; stop.clear()
        th = threading.Thread(target=sample); th.start()
        times = [fn() for _ in range(3)]
        stop.set(); th.join()
        n, best = times[0][0], min(t for _, t in times)
        res[name] = {"bytes_out": n, "GBps": round(n / best / 1e9, 4), "best_s": round(best, 3), "host_memory_growth_mb": round((peak[0] - base) / 2**20, 1)}
    if R is not None:
        n, dt = run_stream(R)
        res["reference_ZSTD_decompressStream_one_thread"] = {"bytes_out": n, "GBps": round(n / dt / 1e9, 4)}
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    res["gpu"] = q.stdout.strip()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
