"""Rates of the optimal-parser levels (13, 16, 19, 22) on an H100 through the batch API, next to the reference on the CPU.

For 16 KB and 64 KB chunks of the corpus: GPU compression GB/s (synchronised host clock around compressBatch, after a warm-up
call, best of the timed calls), compression ratio, the reference's CPU rate on the same chunks (oracle/_ref, one context per host
thread), a byte-for-byte parity count against the reference on a sample of the frames, and the residency sweep of the
optimal-parser kernel (opt_blocks_per_sm 4 / 6 / 8).  The card name and power limit are read in the same run.
Prints the results as one JSON line; --out also writes them to a file.

  python scripts/gpu_opt_levels.py [--mb 64] [--levels 13,16,19,22] [--sweep-level 19]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:      # noqa: BLE001
        return f"unknown ({e})"


def chunks_of(size: int, total: int):
    from zstd_jni_b200 import corpus
    n = max(1, total // size)
    per = 131072 // size
    return [corpus.chunk(k // per).tobytes()[(k % per) * size:(k % per + 1) * size] for k in range(n)]


def gpu_rate(ctx, chunks, level, reps):
    ctx.compressBatch(chunks[: min(len(chunks), 256)], level)      # warm-up (module load, workspaces)
    best, frames = None, None
    for _ in range(reps):
        t0 = time.perf_counter()
        frames = ctx.compressBatch(chunks, level)
        dt = time.perf_counter() - t0
        best = dt if best is None or dt < best else best
    return best, frames


def cpu_rate(chunks, level):
    from tests.oracle_util import ref_compress
    threads = os.cpu_count() or 1
    t0 = time.perf_counter()
    with ThreadPoolExecutor(threads) as ex:
        list(ex.map(lambda c: ref_compress(c, level), chunks))
    return time.perf_counter() - t0, threads


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mb", type=int, default=64, help="input MB per batch")
    ap.add_argument("--levels", default="13,16,19,22")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--sweep-level", type=int, default=19)
    ap.add_argument("--sample", type=int, default=64, help="frames per batch compared with the reference")
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    from tests.oracle_util import ref, ref_compress
    from zstd_jni_b200.zstd import ZstdBatchContext
    out = {"card": card(), "rows": [], "sweep": []}
    print("card:", out["card"], flush=True)
    with ZstdBatchContext(0) as ctx:
        for size in (16384, 65536):
            chunks = chunks_of(size, args.mb << 20)
            total = sum(map(len, chunks))
            for r in (4, 6, 8):      # residency sweep of k_parse<32, R, ONLY_OPT>
                ctx.setOption("opt_blocks_per_sm", r)
                dt, _ = gpu_rate(ctx, chunks, args.sweep_level, 1)
                row = {"chunk": size, "level": args.sweep_level, "blocks_per_sm": r, "gpu_s": dt, "gpu_GBps": total / dt / 1e9}
                out["sweep"].append(row); print(row, flush=True)
            best_r = min((s for s in out["sweep"] if s["chunk"] == size), key=lambda s: s["gpu_s"])["blocks_per_sm"]
            ctx.setOption("opt_blocks_per_sm", best_r)
            for level in [int(x) for x in args.levels.split(",")]:
                dt, frames = gpu_rate(ctx, chunks, level, args.reps)
                comp = sum(map(len, frames))
                row = {"chunk": size, "level": level, "frames": len(chunks), "input_MB": total / 1e6, "blocks_per_sm": best_r,
                       "gpu_s": dt, "gpu_GBps": total / dt / 1e9, "ratio": total / comp}
                if ref() is not None:
                    cdt, threads = cpu_rate(chunks, level)
                    step = max(1, len(chunks) // args.sample)
                    sample = range(0, len(chunks), step)
                    row.update(cpu_threads=threads, cpu_s=cdt, cpu_GBps=total / cdt / 1e9,
                               parity=f"{sum(frames[k] == ref_compress(chunks[k], level) for k in sample)}/{len(sample)}")
                out["rows"].append(row); print(row, flush=True)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(out, indent=1) + "\n")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
