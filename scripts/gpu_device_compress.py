#!/usr/bin/env python
"""gpu_device_compress.py -- zstdb200_compress_items_device against the host-planned pair on one GPU.

    python scripts/gpu_device_compress.py [--out DIR] [--reps 3]

Three workloads from the synthetic corpus (zstd_jni_b200.corpus), input and output in device memory, level 1 and 3:
  1. 8192 items of 128 KB;  2. 64 items of 16 MB;  3. 20 000 items of 0-300 KB (seeded).
For each: the new call (items in, packed multi-frame streams out, the chunks planned on the GPU) against zstdb200_compress_device plus
zstdb200_compact_device on the same 128 KB chunks, their offsets planned on the host beforehand (not timed).  Both write the same
packed stream, which is compared byte for byte.  Times are CUDA events around each call on one stream, best of `reps` warm runs.
Prints the card's name and power limit, read in the same run, and one JSON line per workload.
With --seek-table the call is also timed with option seek_table on (tables_ms, alternating with the other two), and its output checked
to be the option-off streams each followed by its table.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
CHUNK = 131072


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def bound(x):
    return x + (x >> 8) + (((CHUNK - x) >> 11) if x < CHUNK else 0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--levels", default="1,3")
    ap.add_argument("--seek-table", action="store_true")
    args = ap.parse_args()
    import torch
    from zstd_jni_b200 import _native, corpus
    from zstd_jni_b200.zstd import ZstdBatchContext
    L = _native.lib()
    dev = torch.device("cuda:0")
    gpu = card()
    print("card:", gpu, flush=True)
    base = torch.from_numpy(corpus.corpus(8192).reshape(-1)).to(dev)          # 1 GiB
    rng = np.random.default_rng(20261018)
    mixed = [int(x) for x in rng.integers(0, 300 << 10, size=20_000)]
    workloads = [("8192 x 128 KB", [CHUNK] * 8192), ("64 x 16 MB", [16 << 20] * 64), ("20000 x 0-300 KB", mixed)]
    lines = []
    with ZstdBatchContext(0) as ctx, ZstdBatchContext(0) as tctx:
        tctx.setOption("seek_table", 1)
        s = torch.cuda.Stream()
        for name, sizes in workloads:
            total = sum(sizes)
            src = base.repeat((total + base.numel() - 1) // base.numel())[:total].contiguous()
            so = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
            chunks = [(int(so[i]) + q * CHUNK, int(so[i]) + min((q + 1) * CHUNK, n)) for i, n in enumerate(sizes) for q in range(max(1, -(-n // CHUNK)))]
            co = np.array([a for a, _ in chunks] + [chunks[-1][1]], dtype=np.int64)
            m = len(chunks)
            cap = sum(bound(b - a) for a, b in chunks)
            stride = (bound(CHUNK) + 32 + 63) // 64 * 64
            d_so, d_co = torch.from_numpy(so).to(dev), torch.from_numpy(co).to(dev)
            out_new = torch.zeros(cap, dtype=torch.uint8, device=dev)
            out_old = torch.zeros(cap, dtype=torch.uint8, device=dev)
            do = torch.zeros(len(sizes) + 1, dtype=torch.int64, device=dev)
            res = torch.zeros(len(sizes), dtype=torch.int64, device=dev)
            slots = torch.empty(m * stride, dtype=torch.uint8, device=dev)
            fsz = torch.zeros(m, dtype=torch.int64, device=dev)
            coff = torch.zeros(m + 1, dtype=torch.int64, device=dev)
            ks = [max(1, -(-n // CHUNK)) for n in sizes]
            tcap = cap + sum(17 + 8 * k for k in ks)
            out_tab = torch.zeros(tcap if args.seek_table else 1, dtype=torch.uint8, device=dev)
            dot = torch.zeros(len(sizes) + 1, dtype=torch.int64, device=dev)
            rest = torch.zeros(len(sizes), dtype=torch.int64, device=dev)
            for level in [int(x) for x in args.levels.split(",")]:
                def new():
                    assert L.zstdb200_compress_items_device(ctx.handle, level, CHUNK, len(sizes), src.data_ptr(), d_so.data_ptr(), out_new.data_ptr(),
                                                            cap, do.data_ptr(), res.data_ptr(), s.cuda_stream) == 0

                def old():
                    assert L.zstdb200_compress_device(ctx.handle, level, m, src.data_ptr(), d_co.data_ptr(), slots.data_ptr(), stride, fsz.data_ptr(),
                                                      s.cuda_stream) == 0
                    assert L.zstdb200_compact_device(ctx.handle, m, slots.data_ptr(), stride, fsz.data_ptr(), out_old.data_ptr(), coff.data_ptr(),
                                                     s.cuda_stream) == 0

                def tables():
                    assert L.zstdb200_compress_items_device(tctx.handle, level, CHUNK, len(sizes), src.data_ptr(), d_so.data_ptr(), out_tab.data_ptr(),
                                                            tcap, dot.data_ptr(), rest.data_ptr(), s.cuda_stream) == 0

                times = {"new": [], "pair": [], "tables": []}
                calls = (("new", new), ("pair", old)) + ((("tables", tables),) if args.seek_table else ())
                for rep in range(args.reps + 1):                  # the first round warms up (and builds the graph)
                    for key, f in calls:
                        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        a.record(s)
                        f()
                        b.record(s)
                        s.synchronize()
                        if rep:
                            times[key].append(a.elapsed_time(b))
                n_new, n_old = int(do[-1].item()), int(coff[-1].item())
                same = n_new == n_old and bool(torch.equal(out_new[:n_new], out_old[:n_old]))
                ok = bool((res >= 0).all().item()) and bool((fsz >= 0).all().item())
                line = {"workload": name, "level": level, "items": len(sizes), "chunks": m, "bytes": total, "card": gpu,
                        "new_ms": min(times["new"]), "pair_ms": min(times["pair"]), "new_GBps": total / min(times["new"]) / 1e6,
                        "pair_GBps": total / min(times["pair"]) / 1e6, "new_all_ms": times["new"], "pair_all_ms": times["pair"],
                        "same_output": same, "no_errors": ok, "ratio": total / max(n_new, 1)}
                if args.seek_table:      # every item: the option-off stream, then 8 + 8 k + 9 bytes of table
                    a, b = do.cpu().numpy(), dot.cpu().numpy()
                    tables_ok = bool((rest >= 0).all().item()) and all(int(b[i + 1] - b[i]) == int(a[i + 1] - a[i]) + 17 + 8 * ks[i] for i in range(len(sizes)))
                    step = max(1, len(sizes) // 64)
                    tables_ok = tables_ok and all(torch.equal(out_tab[int(b[i]):int(b[i]) + int(a[i + 1] - a[i])], out_new[int(a[i]):int(a[i + 1])])
                                                  for i in range(0, len(sizes), step))
                    line.update({"tables_ms": min(times["tables"]), "tables_all_ms": times["tables"], "tables_ok": tables_ok})
                    line["no_errors"] = ok and tables_ok
                print(json.dumps(line), flush=True)
                lines.append(line)
            del src, slots, out_new, out_old, out_tab
            torch.cuda.empty_cache()
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / "device_compress.json").write_text(json.dumps(lines, indent=1))
    assert all(x["same_output"] and x["no_errors"] for x in lines)


if __name__ == "__main__":
    main()
