"""Rate of the one-shot decoder on a stream of many frames, and of batches of checksummed frames, host memory in and out.

  one-shot: ZSTD_decompress of one stream of `--mb` MB cut into 128 KB level-3 frames (what zstdb200_compress_chunks, the NCCL gather
            and ZSTD_compressStream2 write), best of 3 after a warm-up, output compared with the input; the drop of the device's free
            memory over the one-shot runs (cudaMemGetInfo, device-wide: other processes on the card move it too; the decoder's
            workspaces only grow and are kept by the pooled context); the reference's ZSTD_decompress on one host thread, also best of
            3 after a warm-up.
  batch:    zstdb200_decompress_batch of the same frames as 8192-item batches, with and without checksum, best of 3; then the average
            time of every kernel over 3 more calls (option "timing").
Prints one JSON line with the card's name and power limit.
    python scripts/gpu_multiframe_decode.py [--mb 1024] [--oneshot-mb 0] [--lib path/to/libzstdb200.so]
--lib measures another build of the library (an earlier commit); --oneshot-mb times the one-shot call on only that much of the stream
(an earlier build decodes such a stream with one warp).
"""
from __future__ import annotations

import argparse
import ctypes as C
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
    ap.add_argument("--mb", type=int, default=1024)
    ap.add_argument("--oneshot-mb", type=int, default=0)
    ap.add_argument("--lib", default="")
    a = ap.parse_args()
    if a.lib:
        os.environ["ZSTDB200_LIBRARY"] = a.lib
    import numpy as np

    from tests.oracle_util import ERR_MAX, ref
    from zstd_jni_b200 import _native
    from zstd_jni_b200.zstd import ZstdBatchContext
    L = _native.lib()
    data = text(a.mb << 20, 3)
    res = {"content_mb": a.mb, "library": a.lib or "this tree"}
    streams = {}
    ctx = ZstdBatchContext(0)
    for ck in (0, 1):
        ctx.setOption("checksum", ck)
        s, sizes = ctx.compressChunks(np.frombuffer(data, dtype=np.uint8), 131072, 3)
        streams[ck] = (s.tobytes(), [int(x) for x in sizes])
    ctx.close()
    res["frames"] = len(streams[0][1])

    def device_free_mb():
        """Free device memory (cudaMemGetInfo): device-wide, so other processes on the card move it too."""
        import torch
        return torch.cuda.mem_get_info()[0] // 2**20

    def best_of(fn, k=3):
        fn()
        ts = []
        for _ in range(k):
            t = time.perf_counter(); fn(); ts.append(time.perf_counter() - t)
        return min(ts)

    # ---- one-shot ZSTD_decompress of one stream
    stream, sizes = streams[0]
    nf = len(sizes) if not a.oneshot_mb else min(len(sizes), (a.oneshot_mb << 20) // 131072)
    one = stream[: sum(sizes[:nf])]
    content = min(len(data), nf * 131072)
    out = np.empty(content, dtype=np.uint8)
    got = [0]

    def oneshot():
        got[0] = L.ZSTD_decompress(C.c_void_p(out.ctypes.data), content, one, len(one))
    free0 = device_free_mb()
    dt = best_of(oneshot)
    free1 = device_free_mb()
    assert got[0] <= ERR_MAX and got[0] == content and out.tobytes() == data[:content], got[0]
    res["ZSTD_decompress_stream"] = {"content_mb": round(content / 2**20, 1), "frames": nf, "GBps": round(content / dt / 1e9, 4),
                                     "best_s": round(dt, 4), "device_free_drop_mb": free0 - free1}
    R = ref()
    if R is not None:
        rout = C.create_string_buffer(content)
        rn = [0]

        def reference():
            rn[0] = R.ZSTD_decompress(rout, content, one, len(one))
        rdt = best_of(reference)
        assert rn[0] == content
        res["reference_ZSTD_decompress_one_thread"] = {"GBps": round(content / rdt / 1e9, 4), "best_s": round(rdt, 4)}
    # ---- batches of 8192 single frames, with and without checksum
    ctx = ZstdBatchContext(0)
    for ck in (0, 1):
        stream, sizes = streams[ck]
        n = len(sizes)
        offs = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        sb = np.frombuffer(stream, dtype=np.uint8)
        src = (C.c_void_p * n)(*[sb.ctypes.data + int(offs[i]) for i in range(n)])
        ssz = (C.c_size_t * n)(*sizes)
        outb = np.empty(n * 131072, dtype=np.uint8)
        dst = (C.c_void_p * n)(*[outb.ctypes.data + i * 131072 for i in range(n)])
        dcap = (C.c_size_t * n)(*([131072] * n))
        dsz = (C.c_size_t * n)()
        rc = [0]

        def batch():
            rc[0] = L.zstdb200_decompress_batch(ctx._live(), n, src, ssz, dst, dcap, dsz)
        dt = best_of(batch)
        assert rc[0] == 0 and outb[: len(data)].tobytes() == data
        ctx.setOption("timing", 1)
        ctx.kernelTimes()
        for _ in range(3):
            batch()
        kt = ctx.kernelTimes()
        ctx.setOption("timing", 0)
        res[f"decompress_batch_checksum{ck}"] = {"GBps": round(len(data) / dt / 1e9, 4), "best_s": round(dt, 4),
                                                 "kernel_ms": {k: round(v[0], 4) for k, v in kt.items()}}
    ctx.close()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    res["gpu"] = q.stdout.strip()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
