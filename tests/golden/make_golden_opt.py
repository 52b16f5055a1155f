"""Generates tests/golden/opt.json from the reference compiled in place: frames of the optimal-parser levels 13..22 (btopt,
btultra, btultra2) on inputs of at most 64 KB, with frame flags and explicit strategies -- size and SHA-256 per case, plus the
refusals (-40) of the sizes and rows this build does not serve.
Run in the dev container:  python -m tests.golden.make_golden_opt
"""
from __future__ import annotations

import hashlib
import json
import random
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent.parent))

FLAG_SETS = ({"checksum": True}, {"content_size": False}, {"magicless": True}, {"checksum": True, "content_size": False, "magicless": True})


def cases():
    rnd = random.Random(20261015)
    inputs = [{"kind": "corpus", "index": 0, "size": 9}, {"kind": "corpus", "index": 1, "size": 1000}, {"kind": "corpus", "index": 2, "size": 16384},
              {"kind": "corpus", "index": 3, "size": 16385}, {"kind": "corpus", "index": 4, "size": 40000}, {"kind": "corpus", "index": 5, "size": 65536},
              {"kind": "tokens", "seed": 3, "vocab": 40, "width": 5, "size": 30000}, {"kind": "alphabet", "seed": 4, "alpha": 3, "size": 20000}]
    out = []
    for level in range(13, 23):
        for spec in inputs:
            out.append((spec, level, {}, {}))
        out.append(({"kind": "corpus", "index": 6, "size": 65537}, level, {}, {}))            # refused: the reference splits the block
    for level in (13, 16, 19):
        for flags in FLAG_SETS:
            out.append((inputs[4], level, {}, flags))
    out += [(inputs[1], 11, {}, {}), (inputs[2], 12, {}, {})]                                 # rows 11 / 12 of the <= 16 KB table: refused
    for strat in (7, 8, 9):
        for level in (1, 3, 9):
            params = {"strategy": strat}
            for k, rng in (("hashLog", (6, 20)), ("chainLog", (6, 20)), ("searchLog", (1, 9)), ("minMatch", (3, 7)), ("targetLength", (0, 999))):
                if rnd.random() < 0.4:
                    params[k] = rnd.randint(*rng)
            out.append((rnd.choice(inputs[1:]), level, params, {}))
        out.append(({"kind": "corpus", "index": 7, "size": 70000}, 3, {"strategy": strat}, {}))   # refused: window > 64 KB
    return out


def reference_frame(data: bytes, level: int, params: dict, flags: dict):
    from tests.oracle_util import ref_compress_flags, ref_compress_params
    if params:
        return ref_compress_params(data, level, params)
    return ref_compress_flags(data, level, **flags)


def main():
    from tests.golden.make_golden import regenerate_input
    out = []
    for spec, level, params, flags in cases():
        z = reference_frame(regenerate_input(spec), level, params, flags)
        e = {"input": spec, "level": level, "params": params, "flags": flags}
        served = len(regenerate_input(spec)) <= 65536 and not (level in (11, 12) and not params)
        if served:
            e.update(supported=True, size=len(z), sha256=hashlib.sha256(z).hexdigest())
        else:
            e.update(supported=False)
        out.append(e)
    (HERE / "opt.json").write_text(json.dumps({"cases": out}, indent=1) + "\n")
    print(len(out), "cases")


if __name__ == "__main__":
    main()
