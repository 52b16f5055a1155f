"""Rate of zstdb200_decompress_device (device memory in and out) on multi-block and multi-frame items, against the host-memory call and
against the fused kernel alone (dec_pipeline 0).  Warm, best of 3, outputs compared with the input.

  frame-L3 / frame-L1: one `--mb` MB reference-made frame at level 3 / 1: the device call, and zstdb200_decompress_frames on the same
                       frame (host memory in and out) in the same session
  frame-L3-xxh:        the level-3 frame with a checksum: the device call, whose difference to frame-L3 is the cost of the device XXH64
  items-64x128K:       128 items of 64 concatenated 128 KB level-3 frames: the device call with dec_pipeline 1 and 0
  singles-128K:        8192 items of one 128 KB level-3 frame: the device call
  files-256K:          8192 items of one 256 KB level-3 frame (two blocks, as the zstd tool writes such a file): the device call
  items-2to4x128K:     4096 items of 2-4 concatenated 128 KB level-3 frames: the device call
The one-frame items go to the staged decoder, the two-block files to the fused kernel (many short items), the long frames to the
segment loop; the items of several one-block frames are cut into their frames for the staged decoder.  Prints one JSON line with the
card's name and power limit.
    python scripts/gpu_device_decode.py [--mb 1024] [--lib path/to/libzstdb200.so] [--many-only] [--items]
--lib measures another build of the library (an earlier commit); --many-only times only the many-item workloads (an earlier build
decodes the long items with one warp each, minutes per GiB).  --items also times, on every device workload, alternating with the device
call on host-planned offsets: zstdb200_decompress_items_device, which finds the rooms on the GPU ("items"), and
zstdb200_decompress_bound_device alone ("plan_ms"); plan_share is plan_ms over the items call's time.
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
    ap.add_argument("--lib", default="")
    ap.add_argument("--many-only", action="store_true")
    ap.add_argument("--items", action="store_true")
    args = ap.parse_args()
    if args.lib:
        os.environ["ZSTDB200_LIBRARY"] = args.lib
    import numpy as np
    import torch
    from tests.oracle_util import ref_compress_flags
    from zstd_jni_b200 import _native
    from zstd_jni_b200.zstd import ZstdBatchContext
    L = _native.lib()
    dev = torch.device("cuda:0")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()

    def device_rate(ctx, items, contents):
        n = len(items)
        so = np.concatenate([[0], np.cumsum([len(x) for x in items])]).astype(np.int64)
        do = np.concatenate([[0], np.cumsum([len(x) for x in contents])]).astype(np.int64)
        d_src = torch.from_numpy(np.frombuffer(b"".join(items), dtype=np.uint8).copy()).to(dev)
        d_so, d_do = torch.from_numpy(so).to(dev), torch.from_numpy(do).to(dev)
        d_dst = torch.zeros(int(do[-1]), dtype=torch.uint8, device=dev)
        d_res = torch.zeros(n, dtype=torch.int64, device=dev)
        d_plan = torch.zeros(n + 1, dtype=torch.int64, device=dev)
        d_bounds = torch.zeros(n, dtype=torch.int64, device=dev)
        s = torch.cuda.Stream()
        calls = {"device": lambda: L.zstdb200_decompress_device(ctx.handle, n, d_src.data_ptr(), d_so.data_ptr(), d_dst.data_ptr(),
                                                                d_do.data_ptr(), d_res.data_ptr(), s.cuda_stream)}
        if args.items:
            calls["items"] = lambda: L.zstdb200_decompress_items_device(ctx.handle, n, d_src.data_ptr(), d_so.data_ptr(), d_dst.data_ptr(),
                                                                        int(do[-1]), d_plan.data_ptr(), d_res.data_ptr(), s.cuda_stream)
            calls["plan"] = lambda: L.zstdb200_decompress_bound_device(ctx.handle, n, d_src.data_ptr(), d_so.data_ptr(), d_plan.data_ptr(),
                                                                       d_bounds.data_ptr(), s.cuda_stream)
        best, ok = {}, {}
        for rep in range(4):
            for name, call in calls.items():      # alternating, so that drift on the card touches every call alike
                d_dst.zero_(); d_plan.zero_(); torch.cuda.synchronize()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(s)
                assert call() == 0
                b.record(s); s.synchronize()
                if rep:
                    best[name] = min(best.get(name, 1e9), a.elapsed_time(b))
                if name == "plan":
                    ok[name] = d_plan.cpu().tolist() == do.tolist()
                else:
                    ok[name] = d_res.cpu().tolist() == [len(x) for x in contents] and bytes(d_dst.cpu().numpy()) == b"".join(contents)
                    ok[name] = ok[name] and (name == "device" or d_plan.cpu().tolist() == do.tolist())
        rate = lambda k: {"GBps": round(int(do[-1]) / best[k] / 1e6, 3), "ms": round(best[k], 3), "ok": ok[k]}
        out = rate("device")
        if args.items:
            out["items"] = rate("items")
            out["plan_ms"], out["plan_ok"] = round(best["plan"], 4), ok["plan"]
            out["plan_share"] = round(best["plan"] / best["items"], 5)
        return out

    def frames_rate(ctx, frame, content):
        out = C.create_string_buffer(len(content))
        best = None
        for rep in range(4):
            sizes, fs = (C.c_size_t * 1)(len(content)), (C.c_size_t * 1)(len(frame))
            t = time.perf_counter()
            r = L.zstdb200_decompress_frames(ctx.handle, frame, fs, 1, out, len(content), sizes)
            dt = (time.perf_counter() - t) * 1e3
            if rep:
                best = min(best or 1e9, dt)
        return {"GBps": round(len(content) / best / 1e6, 3), "ms": round(best, 3), "ok": r == 0 and out.raw == content}

    res = {"card": card}
    data = text(args.mb << 20, 1)
    chunk = 128 << 10
    with ZstdBatchContext(0) as ctx:
        # many short items: 64 distinct frames / items, repeated (the decoding work per item is the same)
        parts = [text(2 * chunk, 300 + k) for k in range(64)]
        frames = [ref_compress_flags(p, 3) for p in parts]
        res["files-256K"] = {"device": device_rate(ctx, [frames[i % 64] for i in range(8192)], [parts[i % 64] for i in range(8192)])}
        small = [text(chunk, 400 + k) for k in range(64)]
        sframes = [ref_compress_flags(p, 3) for p in small]
        res["singles-128K"] = {"device": device_rate(ctx, [sframes[i % 64] for i in range(8192)], [small[i % 64] for i in range(8192)])}
        groups = [[(g * 7 + j) % 64 for j in range(2 + g % 3)] for g in range(64)]
        res["items-2to4x128K"] = {"device": device_rate(ctx, [b"".join(sframes[j] for j in groups[i % 64]) for i in range(4096)],
                                                        [b"".join(small[j] for j in groups[i % 64]) for i in range(4096)])}
        if args.many_only:
            print(json.dumps(res))
            return
        for name, level, ck in (("frame-L3", 3, False), ("frame-L1", 1, False), ("frame-L3-xxh", 3, True)):
            f = ref_compress_flags(data, level, checksum=ck)
            res[name] = {"device": device_rate(ctx, [f], [data])}
            if not ck:
                res[name]["frames"] = frames_rate(ctx, f, data)
        items, contents = [], []
        for i in range(128):
            part = text(64 * chunk, 100 + i)
            items.append(b"".join(ref_compress_flags(part[k * chunk:(k + 1) * chunk], 3) for k in range(64)))
            contents.append(part)
        res["items-64x128K"] = {"device": device_rate(ctx, items, contents)}
        ctx.setOption("dec_pipeline", 0)
        res["items-64x128K"]["device-fused"] = device_rate(ctx, items, contents)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
