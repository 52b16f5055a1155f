"""Time of zstdb200_decompress_ranges_device against what a caller does without it: zstdb200_decompress_items_device of the whole items,
then a gather of the slices.  Warm, best of 3 by CUDA events, every output compared with the input.

  4k-random:    64 items of 16 MB (compress_items_device, level 3, 128 KB chunks), 100 000 random 4 KB ranges
  1m-random:    the same items, 10 000 random 1 MB ranges
  whole-items:  the same items, one range per whole item
  1g-tail:      one 1 GiB item (level 3, 128 KB chunks), 1 000 random 4 KB ranges in its last 16 MB: the walk over 8192 frames

For each: ranges_ms (the call), whole_ms (decompress every item whole, then gather), and locate_ms -- k_range_locate, the walk that finds
every request's frames -- with locate_share its part of the call, from one more call with kernel timing on.  Prints one JSON line with
the card's name and power limit.

With --seek-table the items are compressed with seek tables, and every workload is timed twice, alternating: walked (option off; the
walk passes the tables as skippable frames) and located through the tables (seek_ranges_ms, seek_locate_ms, seek_locate_share).
    python scripts/gpu_device_ranges.py [--seek-table]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

BLOCK = 128 << 10


def text(n: int, seed: int) -> bytes:
    import numpy as np
    rnd = np.random.default_rng(seed)
    words = rnd.integers(97, 123, size=(4000, 8), dtype=np.uint8)
    words[:, 7] = 32
    return words[rnd.zipf(1.4, size=n // 8 + 1) % 4000].tobytes()[:n]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seek-table", action="store_true")
    args = ap.parse_args()
    import numpy as np
    import torch
    from zstd_jni_b200 import _native
    from zstd_jni_b200.zstd import ZstdBatchContext
    L = _native.lib()
    dev = torch.device("cuda:0")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    s = torch.cuda.Stream()      # (the calls and the events on one stream)

    def i64(v):
        return torch.as_tensor(np.asarray(v, dtype=np.int64), device=dev)

    def best(f, reps=3):
        f()
        ts = []
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(s)
            f()
            b.record(s)
            torch.cuda.synchronize()
            ts.append(a.elapsed_time(b))
        return min(ts)

    def compress(ctx, d_in, sizes):
        n = len(sizes)
        d_so = i64(np.concatenate([[0], np.cumsum(sizes)]))
        ccap = sum(x + (x >> 7) + 1024 * (x // BLOCK + 1) for x in sizes)
        d_c = torch.empty(ccap, dtype=torch.uint8, device=dev)
        d_co = torch.zeros(n + 1, dtype=torch.int64, device=dev)
        d_res = torch.zeros(n, dtype=torch.int64, device=dev)
        assert L.zstdb200_compress_items_device(ctx.handle, 3, BLOCK, n, d_in.data_ptr(), d_so.data_ptr(), d_c.data_ptr(), ccap, d_co.data_ptr(),
                                                d_res.data_ptr(), s.cuda_stream) == 0
        torch.cuda.synchronize()
        assert (d_res >= 0).all()
        return d_c, d_co

    def workload(name, ctx, d_in, sizes, d_c, d_co, items, begins, length, sctx=None):
        n, m = len(sizes), len(items)
        item_at = np.concatenate([[0], np.cumsum(sizes)])
        starts = i64(item_at[items] + begins)
        d_items, d_begins = i64(items), i64(begins)
        d_do = i64(np.arange(m + 1) * length)
        d_out = torch.empty(m * length, dtype=torch.uint8, device=dev)
        d_res = torch.zeros(m, dtype=torch.int64, device=dev)
        total = int(item_at[-1])
        d_full = torch.empty(total, dtype=torch.uint8, device=dev)
        d_fo = torch.zeros(n + 1, dtype=torch.int64, device=dev)
        d_fres = torch.zeros(n, dtype=torch.int64, device=dev)

        def ranges(c=ctx):
            assert L.zstdb200_decompress_ranges_device(c.handle, n, d_c.data_ptr(), d_co.data_ptr(), m, d_items.data_ptr(), d_begins.data_ptr(),
                                                       d_out.data_ptr(), d_do.data_ptr(), d_res.data_ptr(), s.cuda_stream) == 0

        gathered = {}

        def whole():
            assert L.zstdb200_decompress_items_device(ctx.handle, n, d_c.data_ptr(), d_co.data_ptr(), d_full.data_ptr(), total, d_fo.data_ptr(),
                                                      d_fres.data_ptr(), s.cuda_stream) == 0
            with torch.cuda.stream(s):
                gathered["out"] = d_full.unfold(0, length, 1)[starts].reshape(-1)

        want = d_in.unfold(0, length, 1)[starts].reshape(-1)

        def timed(c):
            c.setOption("timing", 1)
            c.kernelTimes()
            ranges(c)
            torch.cuda.synchronize()
            times = c.kernelTimes()
            c.setOption("timing", 0)
            return times.get("k_range_locate", (0.0, 0))[0], times.get("k_range_parts", (0.0, 0))[0]

        if sctx is None:
            ranges_ms, whole_ms = best(ranges), best(whole)
        else:      # walked and through the tables, alternating
            ranges(), ranges(sctx)
            walk, seek = [], []
            for _ in range(3):
                walk.append(best(ranges, 1))
                seek.append(best(lambda: ranges(sctx), 1))
            ranges_ms, seek_ms, whole_ms = min(walk), min(seek), best(whole)
            d_out.zero_()
            ranges(sctx)
            torch.cuda.synchronize()
            seek_ok = bool((d_res == length).all()) and torch.equal(d_out, want)
            seek_locate, seek_parts = timed(sctx)
        d_out.zero_()
        ranges()
        torch.cuda.synchronize()
        ok = bool((d_res == length).all()) and torch.equal(d_out, want) and torch.equal(gathered["out"], want) and torch.equal(d_full, d_in)
        locate, parts = timed(ctx)
        del d_out, d_full, gathered
        torch.cuda.empty_cache()
        row = {"workload": name, "requests": m, "bytes": m * length, "ranges_ms": round(ranges_ms, 3), "whole_ms": round(whole_ms, 3),
               "speedup": round(whole_ms / ranges_ms, 3), "locate_ms": round(locate, 3), "parts_ms": round(parts, 3),
               "locate_share": round(locate / ranges_ms, 4), "ok": ok}
        if sctx is not None:
            row.update({"seek_ranges_ms": round(seek_ms, 3), "seek_locate_ms": round(seek_locate, 3), "seek_parts_ms": round(seek_parts, 3),
                        "seek_locate_share": round(seek_locate / seek_ms, 4), "ok": ok and seek_ok})
        return row

    rows = []
    rnd = np.random.default_rng(7)
    with ZstdBatchContext(0) as ctx, ZstdBatchContext(0) as sctx:
        if args.seek_table:
            ctx.setOption("seek_table", 1)      # (compress with tables; the walk below runs with the option off)
        size = 16 << 20
        sizes = [size] * 64
        d_in = torch.from_numpy(np.frombuffer(text(64 * size, 1), dtype=np.uint8).copy()).to(dev)
        d_c, d_co = compress(ctx, d_in, sizes)
        ctx.setOption("seek_table", 0)
        sc = None
        if args.seek_table:
            sctx.setOption("seek_table", 1)
            sc = sctx
        for name, m, length in (("4k-random", 100_000, 4096), ("1m-random", 10_000, 1 << 20), ("whole-items", 64, size)):
            if name == "whole-items":
                items, begins = np.arange(64), np.zeros(64, dtype=np.int64)
            else:
                items, begins = rnd.integers(0, 64, m), rnd.integers(0, size - length + 1, m)
            rows.append(workload(name, ctx, d_in, sizes, d_c, d_co, items, begins, length, sc))
        del d_in, d_c, d_co
        torch.cuda.empty_cache()
        big = 1 << 30
        d_in = torch.from_numpy(np.frombuffer(text(big, 2), dtype=np.uint8).copy()).to(dev)
        ctx.setOption("seek_table", int(args.seek_table))
        d_c, d_co = compress(ctx, d_in, [big])
        ctx.setOption("seek_table", 0)
        begins = rnd.integers(big - (16 << 20), big - 4096 + 1, 1000)
        rows.append(workload("1g-tail", ctx, d_in, [big], d_c, d_co, np.zeros(1000, dtype=np.int64), begins, 4096, sc))
    print(json.dumps({"card": card, "workloads": rows, "ok": all(r["ok"] for r in rows)}))


if __name__ == "__main__":
    main()
