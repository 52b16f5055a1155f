"""Input-stream counters of the level-3 dfast parse, per corpus class, on the 32-lane emulator (CPU only; counts, not times).

Builds the host instantiation of the kernel source with -DZB_STATS into a temporary directory and parses corpus.corpus(N):
  batches/fr   search batches per frame
  coldHead%    batches whose input load reaches a 32-byte sector beyond everything the frame has read forward so far
  wcRounds/fr  rounds of wcount (forward match extension), and wcCold% of them reaching past that mark
  fetch/fr     per-lane candidate and repcode fetches, then the cumulative share at offsets < 1 / 2 / 4 / 6 KB
usage: python scripts/parse_input_stats.py [chunks=64] [level=3]"""
import ctypes as C
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from zstd_jni_b200 import corpus  # noqa: E402

FIELDS = ["batches", "probes", "useful", "candL", "candS", "matches", "bytes", "frames", "coldHeads", "wcReads", "wcCold",
          "n1k", "n2k", "n4k", "n6k", "nfar"]


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 64
    level = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    with tempfile.TemporaryDirectory() as tmp:
        so = os.path.join(tmp, "libzb_stats.so")
        subprocess.run(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-DZB_STATS", "-Wno-unused-function", "-x", "c++",
                        os.path.join(ROOT, "tests", "hostsim", "zb_hostsim.cpp"), "-o", so], check=True)
        L = C.CDLL(so)
    L.zbe_compress.restype = C.c_size_t
    L.zbe_compress.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int]
    data = corpus.corpus(n)
    dst = (C.c_ubyte * (2 * corpus.CHUNK))()
    st = (C.c_ulonglong * len(FIELDS))()
    L.zbh_parse_stats(st, 1)
    per = {}
    for i in range(n):
        x = data[i].tobytes()
        L.zbe_compress(dst, len(dst), x, len(x), level)
        L.zbh_parse_stats(st, 1)
        acc = per.setdefault(i % corpus.N_CLASSES, np.zeros(len(FIELDS), dtype=np.int64))
        acc += np.array(st[:], dtype=np.int64)
    print("class frames batches/fr coldHead% wcRounds/fr wcCold% fetch/fr   <1K   <2K   <4K   <6K  seq/fr")
    for cls in sorted(per) + ["all"]:
        a = dict(zip(FIELDS, per[cls] if cls != "all" else sum(per.values())))
        fr = max(a["frames"], 1)
        near = np.array([a["n1k"], a["n2k"], a["n4k"], a["n6k"], a["nfar"]])
        cum = np.cumsum(near)[:4] / max(near.sum(), 1) * 100
        print(f"{cls!s:5} {a['frames']:6d} {a['batches'] / fr:10.0f} {100 * a['coldHeads'] / max(a['batches'], 1):9.1f} "
              f"{a['wcReads'] / fr:11.0f} {100 * a['wcCold'] / max(a['wcReads'], 1):7.1f} {near.sum() / fr:8.0f} "
              + " ".join(f"{c:5.1f}" for c in cum) + f" {a['matches'] / fr:7.0f}")


if __name__ == "__main__":
    main()
