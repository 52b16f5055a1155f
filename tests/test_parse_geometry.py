"""Every k_parse instance and launch geometry the batch options select must write the reference's bytes.

Most of the compressor is compiled into k_parse<LANES, MIN_BLOCKS, ONLY> instances (zb_capi.cu) that plan_parse picks from the
context's options; the other options change only the grid, the order in which frames are parsed and which frames share a group's
tables.  None of them may change a byte.

| instance | reached by | run by |
|---|---|---|
| k_parse<32,8,S_fast>, <32,8,S_dfast> | levels <= 3, defaults | test_gpu_parity.py; here the geometry tests |
| k_parse<32,8,0> (all parsers in one) | level 4, defaults | test_gpu_parity.py; here the geometry tests |
| k_parse<32,6,ONLY_LAZY> | levels 5 ... 10, defaults (11 and 12 run <32,8,0>: their 16 KB rows are refused) | test_gpu_parity.py; here the geometry tests |
| k_parse<32,4,ONLY_OPT> | levels 13 ... 22, defaults | test_opt_levels.py |
| k_parse<4,8,0>, <8,8,0>, <16,8,0> | parse_lanes 4 / 8 / 16, ZSTDB200_PARSE_LANES | test_sub_warp_groups, test_parse_lanes_from_the_environment |
| k_parse<32,10,0>, <32,12,0>, <32,16,0> | parse_blocks_per_sm >= 10 | test_parse_residency |
| k_parse<32,8,0> as the parser for lazy levels | parse_blocks_per_sm 1 ... 7 or 9 at levels >= 5 | test_parse_residency |
| k_parse<32,4,ONLY_LAZY>, <32,8,ONLY_LAZY> | lazy_blocks_per_sm 4 / 8 | test_lazy_residency |
| k_parse<32,6,ONLY_OPT>, <32,8,ONLY_OPT> | opt_blocks_per_sm 6 / 8 | test_opt_residency |

Sub-warp groups are not the full-warp code under another name: their collectives are shifted and masked (GroupDev), several groups of
one warp diverge onto different frames, and some parser code depends on the group width (wcount's first probe width, the probe widths
of the double-fast parser, the iteration batching of the fast parser, the array hash cache and the serial row walk of the row finder
below 32 lanes).  The residency instances are the same source under register caps of 128 down to 32.

CPU: the kernel source with the parse on an emulated group of 4, 8 and 16 lanes (tests/hostsim/zb_hostsim_lanes.cpp, compiled by this module)
against the oracle at every parser family, and with explicit parameters against the compiled reference.

GPU (-m gpu): one test per row of the table.  Each compresses a stale batch at the same level, then a batch of distinct inputs larger
than the frames its grid parses at once (so groups are reused and the ordered path runs), and checks the launch count and every frame.
Parse tables cost groups x (8 << tabLog) bytes, and _GRID_BUDGET bounds what any batch here asks for: with parse_lanes 4 a CTA holds
32 groups, so a level-9 batch on the default grid of 8 CTAs per SM would ask for 33 GB; enc_warps_per_sm shrinks the grid instead.
"""
import ctypes as C
import random
import subprocess
from pathlib import Path

import numpy as np
import pytest

from tests import cases
from tests.oracle_util import (CPARAM_ORDER, ERR_MAX, oracle_compress, oracle_decompress, ref, ref_compress,
                               ref_compress_params)

# ------------------------------------------------------------------------------------------------ CPU
LANES = [4, 8, 16]
CPU_LEVELS = [-5, 1, 2, 3, 4, 5, 7, 9, 10, 12]          # fast, dfast, the all-in-one dispatch at 4 and 12 (btlazy2 above 16 KB), the row finder
CPU_SIZES = [7, 8, 64, 4096, 4097, 16384, 16385, 65536, 131072]


@pytest.fixture(scope="module")
def emu_compress_lanes(tmp_path_factory):
    """tests/hostsim/zb_hostsim_lanes.cpp, compiled for this module: compress(data, level, lanes, params=None) -> frame or negative
    error code, with the parse on an emulated group of `lanes` lanes and the entropy stage on 32."""
    src = Path(__file__).parent / "hostsim" / "zb_hostsim_lanes.cpp"
    so = tmp_path_factory.mktemp("hostsim_lanes") / "libzb_hostsim_lanes.so"
    subprocess.run(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-Wall", "-Wno-unused-function", "-x", "c++", str(src), "-o", str(so)],
                   check=True, cwd=str(src.parent))
    L = C.CDLL(str(so))
    L.zbl_compress.restype = C.c_size_t
    L.zbl_compress.argtypes = [C.c_void_p, C.c_size_t, C.c_char_p, C.c_size_t, C.c_int, C.c_uint, C.POINTER(C.c_uint), C.c_int]

    def compress(data: bytes, level: int, lanes: int, params: dict | None = None):
        ov = (C.c_uint * 7)(*[int(params.get(k, 0)) for k in CPARAM_ORDER]) if params else None
        cap = len(data) + (len(data) >> 8) + 1024
        out = C.create_string_buffer(cap)
        n = L.zbl_compress(out, cap, data, len(data), level, 0, ov, lanes)
        return out.raw[:n] if n <= ERR_MAX else -((1 << 64) - n)
    return compress


def _fit(data: bytes, n: int) -> bytes:
    """`data` cut or repeated to n bytes."""
    return (data * (n // len(data) + 1))[:n]


def _row_finder_inputs():
    """The inputs of test_hostsim.test_emulated_row_parser_batches_match_oracle: long runs of equal hashes and long matches -- lanes
    that hit the same row, rows that wrap inside one batch of insertions, the 384-position skip rule."""
    from zstd_jni_b200 import corpus
    rng = np.random.default_rng(77)
    out = [("corpus-5-50k", corpus.chunk(5)[:50000].tobytes()), ("corpus-23-40k", corpus.chunk(7 + 8 * 2)[:40000].tobytes()),
           ("corpus-0-30k", corpus.chunk(0)[:30000].tobytes())]
    z = np.zeros(50000, dtype=np.uint8); z[rng.integers(0, 50000, 30)] = 9; out.append(("sparse-nines-50k", z.tobytes()))
    for per in (3, 33):
        b = np.tile(rng.integers(0, 256, per, dtype=np.uint8), 40000 // per + 1)[:40000].copy()
        m = rng.random(40000) < 0.01; b[m] = rng.integers(0, 256, int(m.sum()), dtype=np.uint8); out.append((f"period-{per}-noisy-40k", b.tobytes()))
    return out


def _stressors():
    """The cooperative-path stressors of cases.special_cases() and the row-finder inputs."""
    special = dict(cases.special_cases())
    return [(k, special[k]) for k in ("zeros-128k", "period-3", "long-match", "long-literal-run")] + _row_finder_inputs()


@pytest.mark.parametrize("lanes", LANES)
def test_emulated_group_width_matches_oracle(lanes, emu_compress_lanes):
    """Every parser family on a parse group of `lanes` lanes: each level at every size, each (level, size) on four of the ten
    stressors, a different four from cell to cell."""
    pool = _stressors()
    for li, level in enumerate(CPU_LEVELS):
        for si, n in enumerate(CPU_SIZES):
            for j in range(4):
                name, data = pool[(3 * li + si + 3 * j) % len(pool)]
                data = _fit(data, n)
                exp = oracle_compress(data, level)
                assert emu_compress_lanes(data, level, lanes) == exp, (lanes, level, n, name, exp if isinstance(exp, int) else len(exp))


def _param_sweep(seed, count=None, rounds=1):
    """Explicit parameters (strategy x minMatch in full, `rounds` times, the rest drawn): searchLog 1 ... 8 (rowLog 4 / 5 / 6), hashLog
    6 ... 18, targetLength 0 ... 150, windowLog 14 (serial hash chain) or 15 (row finder); inputs no larger than the window."""
    rnd = random.Random(seed)
    pool = _stressors()
    out = []
    for strategy in list(range(1, 6)) * rounds:
        for mm in range(3, 8):
            wl = rnd.choice([14, 15])
            params = {"strategy": strategy, "minMatch": mm, "searchLog": rnd.randint(1, 8), "hashLog": rnd.randint(6, 18),
                      "targetLength": rnd.randint(0, 150), "windowLog": wl}
            n = rnd.choice([7, 64, 1000, 4097, 16384] + ([16385, 32768] if wl == 15 else []))
            name, data = rnd.choice(pool)
            out.append((rnd.choice([1, 3, 5, 9]), params, name, _fit(data, n)))
    rnd.shuffle(out)
    return out[:count]


@pytest.mark.skipif(ref() is None, reason="oracle/_ref not built")
@pytest.mark.parametrize("lanes", LANES)
def test_emulated_group_width_explicit_parameters_match_reference(lanes, emu_compress_lanes):
    for level, params, name, data in _param_sweep(lanes, rounds=4):
        exp = ref_compress_params(data, level, params)
        assert emu_compress_lanes(data, level, lanes, params) == exp, (lanes, level, params, name, len(data))


# ------------------------------------------------------------------------------------------------ GPU
_GRID_BUDGET = 17 << 28           # 4.25 GiB: the most parse tables (and optimal-parser workspaces) one batch here may ask for
_OPT_WORK = 512 << 10             # the optimal parser's workspace per warp (enc_opt_work_bytes, ~410 KB), rounded up


def _table_bytes(level):
    """8 << tabLog per group, tabLog the largest hashLog / chainLog of the level's 16 KB and 128 KB rows (plan_parse)."""
    tab_log = 13 if level < 1 else 15 if level <= 2 else 16 if level == 3 else 17 if level <= 11 else 18
    return (8 << tab_log) + (_OPT_WORK if level >= 13 else 0)


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _grid(level, lanes=32, parse_bps=8, lazy_bps=6, opt_bps=4, enc_warps=0):
    """Frames k_parse parses at once, as plan_parse sizes its grid: CTAs per SM = the instance's residency, fewer when enc_warps_per_sm
    asks for it; 128 / lanes groups per CTA (one warp per frame at the optimal-parser levels)."""
    if level >= 13:
        residency, per_cta = opt_bps, 4
    elif lanes == 32 and parse_bps == 8 and 5 <= level <= 10:
        # the lazy kernel; levels 11 and 12 keep the all-in-one one: their 16 KB rows are refused, so no strategy covers every size
        residency, per_cta = lazy_bps, 4
    else:
        residency, per_cta = parse_bps, 128 // lanes
    ctas = min(-(-enc_warps // 4), residency) if enc_warps > 0 else min(parse_bps, residency)
    return ctas * per_cta * _sms()


def _enc_warps_within_budget(level, per_cta, ctas):
    """enc_warps_per_sm that keeps the grid's tables within _GRID_BUDGET: at most `ctas` CTAs per SM."""
    fit = _GRID_BUDGET // (_table_bytes(level) * per_cta * _sms())
    return 4 * max(1, min(ctas, fit))


_cache = {}


def _batch(level, n, small=(8, 20000)):
    """n distinct inputs (test_gpu_parity._distinct_inputs over its boundary sizes) and their expected frames: the oracle's up to level
    12, the compiled reference's (or the optimal parser's on the host, without it) above."""
    from tests.test_gpu_parity import _GRID_SIZES, _distinct_inputs
    key = (level, n, small)
    if key not in _cache:
        sizes = _GRID_SIZES if level < 13 else [s for s in _GRID_SIZES if s <= 4096] + [16385, 40000, 65536]
        datas = _distinct_inputs(n, sizes, 60 + level, small=small)
        if level < 13:
            exp = [oracle_compress(d, level) for d in datas]
        elif ref() is not None:
            exp = [ref_compress(d, level) for d in datas]
        else:
            from tests.test_opt_levels import host
            exp = [host(d, level) for d in datas]
        _cache[key] = (datas, exp)
    return _cache[key]


def _stale(n):
    from zstd_jni_b200 import corpus
    pool = [corpus.chunk(500 + j)[: (131072, 40000, 7000, 300)[j % 4]].tobytes() for j in range(16)]
    return [pool[k % 16] for k in range(n)]


def _differences(got, exp):
    bad = [k for k in range(len(exp)) if got[k] != exp[k]]
    return len(bad), bad[:8]


def _run(opts, level, datas, exp, launches, failures, what):
    """A context with `opts`: a stale batch at `level`, then `datas`; the launch count of the second and every frame are checked."""
    from zstd_jni_b200.zstd import ZstdBatchContext
    with ZstdBatchContext(0) as c:
        for k, v in opts.items():
            c.setOption(k, v)
        c.compressBatch(_stale(len(datas)), level, raise_on_error=False)
        before = c.kernelLaunches()
        got = c.compressBatch(datas, level, raise_on_error=False)
        ran = c.kernelLaunches() - before
    wrong, first = _differences(got, exp)
    if ran != launches or wrong:
        failures.append(f"{what}, level {level}, {len(datas)} frames: {ran} launches (expected {launches}), {wrong} frames differ, first at {first}")
    return got


def _past_the_grid(level, grid):
    """A batch size past `grid` (ordered: estimate, order, parse + entropy = 4 launches) when its tables fit _GRID_BUDGET; otherwise as
    many frames as fit (every frame starts at once: parse + entropy = 2)."""
    per_group = _table_bytes(level)
    if grid * per_group <= _GRID_BUDGET:
        return grid + max(300, grid // 4), 4
    return _GRID_BUDGET // per_group * 15 // 16, 2


@pytest.mark.gpu
@pytest.mark.parametrize("lanes", LANES)
def test_sub_warp_groups(lanes):
    """parse_lanes 4 / 8 / 16: plan_parse picks k_parse<lanes, 8, 0>, every parser in one kernel, 128 / lanes frames per CTA, at every
    level below 13.  enc_warps_per_sm 1 bounds the grid to one CTA per SM (lanes 4, level 9: 4224 groups x 1 MB of tables); level 12
    at 4 lanes (2 MB per group) runs a batch that fits the budget instead of one past the grid.  Then a sample of the explicit-parameter
    sweep through the c_* options, against the compiled reference."""
    failures = []
    grid = _grid(1, lanes=lanes, enc_warps=1)
    for level in (-5, 1, 3, 4, 5, 9, 12):
        n, launches = _past_the_grid(level, grid)
        datas, exp = _batch(level, n)
        _run({"parse_lanes": lanes, "enc_warps_per_sm": 1}, level, datas, exp, launches, failures, f"parse_lanes {lanes}")
    if ref() is not None:
        from zstd_jni_b200.zstd import ZstdBatchContext
        with ZstdBatchContext(0) as c:
            c.setOption("parse_lanes", lanes)
            sweep = _param_sweep(100 + lanes, 12)
            for level, params, name, data in sweep:
                for k in CPARAM_ORDER:
                    c.setOption("c_" + k, params.get(k, 0))
                datas = [data] + [_fit(d, len(data)) for _, d in _stressors()]
                exp = [ref_compress_params(d, level, params) for d in datas]
                before = c.kernelLaunches()
                got = c.compressBatch(datas, level, raise_on_error=False)
                ran = c.kernelLaunches() - before
                wrong, first = _differences(got, exp)
                if ran != 2 or wrong:
                    failures.append(f"parse_lanes {lanes}, level {level}, {params}, {len(data)} B: {ran} launches, {wrong} frames differ, first at {first}")
    assert not failures, failures


@pytest.mark.gpu
@pytest.mark.parametrize("bps", [1, 2, 7, 10, 12, 16])
def test_parse_residency(bps):
    """parse_blocks_per_sm: 10 / 12 / 16 select k_parse<32, bps, 0> at every level; 1 / 2 / 7 keep k_parse<32, 8, S_fast> at level 1,
    <32, 8, S_dfast> at 3, and make <32, 8, 0> (all parsers in one) the parser of levels 4 and 9 -- the lazy kernel runs only at the
    default of 8.  The grid is bps CTAs per SM, fewer (enc_warps_per_sm) where the tables would pass the budget."""
    failures = []
    for level in (1, 3, 4, 9):
        opts = {"parse_blocks_per_sm": bps}
        if _grid(level, parse_bps=bps) * _table_bytes(level) > _GRID_BUDGET:
            opts["enc_warps_per_sm"] = _enc_warps_within_budget(level, 4, bps)
        grid = _grid(level, parse_bps=bps, enc_warps=opts.get("enc_warps_per_sm", 0))
        assert grid * _table_bytes(level) <= _GRID_BUDGET
        datas, exp = _batch(level, grid + max(300, grid // 4))
        _run(opts, level, datas, exp, 4, failures, f"parse_blocks_per_sm {bps}, {opts}")
    assert not failures, failures


@pytest.mark.gpu
@pytest.mark.parametrize("lbps", [4, 8])
def test_lazy_residency(lbps):
    """lazy_blocks_per_sm 4 / 8: k_parse<32, lbps, ONLY_LAZY> at levels 5 and 9, on inputs of 16 KB or less (the hash-chain finder)
    and above (the row finder).  Level 12 (btlazy2 above 16 KB, refused at or below) stays on k_parse<32, 8, 0> whatever the option
    says: plan_parse picks the lazy kernel only where both of a level's rows are served; its grid (8 CTAs per SM) shows in the launch
    count."""
    failures = []
    for level in (5, 9, 12):
        opts = {"lazy_blocks_per_sm": lbps}
        if _grid(level, lazy_bps=lbps) * _table_bytes(level) > _GRID_BUDGET:
            opts["enc_warps_per_sm"] = _enc_warps_within_budget(level, 4, lbps)
        grid = _grid(level, lazy_bps=lbps, enc_warps=opts.get("enc_warps_per_sm", 0))
        datas, exp = _batch(level, grid + max(300, grid // 4))
        assert sum(len(d) <= 16384 for d in datas) > 1000 and sum(len(d) > 16384 for d in datas) > 300
        _run(opts, level, datas, exp, 4, failures, f"lazy_blocks_per_sm {lbps}, {opts}")
    assert not failures, failures


@pytest.mark.gpu
@pytest.mark.parametrize("obps", [6, 8])
def test_opt_residency(obps):
    """opt_blocks_per_sm 6 / 8: k_parse<32, obps, ONLY_OPT>, one warp per frame, at levels 13, 19 and 22 on inputs of at most 64 KB,
    most of them 4 KB or less (the optimal parse of a frame is serial).  enc_warps_per_sm keeps tables and workspaces in the budget."""
    failures = []
    for level in (13, 19, 22):
        opts = {"opt_blocks_per_sm": obps, "enc_warps_per_sm": _enc_warps_within_budget(level, 4, obps)}
        grid = _grid(level, opt_bps=obps, enc_warps=opts["enc_warps_per_sm"])
        datas, exp = _batch(level, grid + max(300, grid // 4), small=(8, 4097))
        assert max(map(len, datas)) <= 65536 and not any(isinstance(e, int) for e in exp)
        _run(opts, level, datas, exp, 4, failures, f"opt_blocks_per_sm {obps}, {opts}")
    assert not failures, failures


@pytest.mark.gpu
@pytest.mark.parametrize("enc_warps", [1, 5])
def test_enc_warps_per_sm(enc_warps):
    """enc_warps_per_sm 1 / 5: the default instances on a grid of 1 / 2 CTAs per SM, with the entropy stage beside the parse (estimate,
    order, parse + entropy) and behind it (estimate, order, parse, order, entropy)."""
    failures = []
    for level in (1, 3, 9):
        grid = _grid(level, enc_warps=enc_warps)
        datas, exp = _batch(level, grid + max(300, grid // 4))
        for overlap, launches in ((1, 4), (0, 5)):
            _run({"enc_warps_per_sm": enc_warps, "entropy_overlap": overlap}, level, datas, exp, launches, failures,
                 f"enc_warps_per_sm {enc_warps}, entropy_overlap {overlap}")
    assert not failures, failures


@pytest.mark.gpu
@pytest.mark.parametrize("est", [256, 257, 65536])
def test_parse_est_bytes(est):
    """parse_est_bytes: the estimate pass parses an est-byte prefix of the frames longer than 2 x est into the same tables and sequence
    records the real parse then uses; frames of 2 x est and 2 x est + 1 bytes sit on both sides of that cut."""
    failures = []
    cut = [s for s in (2 * est - 1, 2 * est, 2 * est + 1, 2 * est + 2) if s <= 131072]
    for level in (3, 9):
        grid = _grid(level)
        base, base_exp = _batch(level, grid + max(300, grid // 4))
        datas, exp = list(base), list(base_exp)
        for k in range(0, len(datas), 7):              # every 7th input cut to one of the boundary sizes
            s = cut[k // 7 % len(cut)]
            datas[k] = _fit(datas[k] or b"\x01", s)
            exp[k] = oracle_compress(datas[k], level)
        _run({"parse_est_bytes": est}, level, datas, exp, 4, failures, f"parse_est_bytes {est}")
    assert not failures, failures


@pytest.mark.gpu
@pytest.mark.parametrize("level", [3, 9])
def test_parse_order_from_measured_costs(level):
    """parse_order 2: the first call on a batch orders it by the estimate (estimate, order, parse, order, entropy: the entropy stage
    is not overlapped), the second by the parse times the first measured (order, parse, order, entropy)."""
    from zstd_jni_b200.zstd import ZstdBatchContext
    grid = _grid(level)
    datas, exp = _batch(level, grid + max(300, grid // 4))
    with ZstdBatchContext(0) as c:
        c.compressBatch(_stale(len(datas)), level, raise_on_error=False)
        c.setOption("parse_order", 2)
        for call, launches in ((1, 5), (2, 4)):
            before = c.kernelLaunches()
            got = c.compressBatch(datas, level, raise_on_error=False)
            ran = c.kernelLaunches() - before
            assert ran == launches and _differences(got, exp) == (0, []), (call, ran, _differences(got, exp))


@pytest.mark.gpu
@pytest.mark.parametrize("dec_warps", [1, 4, 7])
def test_dec_warps_per_sm(dec_warps):
    """dec_warps_per_sm 1 / 4 / 7 shrink the fused decoder's grid and its scratch: multi-block items, the staged decoder's mix and
    damaged frames, repeated past the fused kernel's warps, must give the oracle's bytes or error code with the staged and segment
    decoders in front of the fused kernel (dec_pipeline 1: prepare, two orders, chains, exec, fused, and the segment kernels) and
    without them (dec_pipeline 0: the fused kernel alone)."""
    from tests.golden.make_golden import multiblock_corruptions
    from tests.test_gpu_parity import _multi_block_items, _staged_decoder_items
    from zstd_jni_b200.zstd import ZstdBatchContext
    zero, small = _staged_decoder_items()
    items = [(z, cap, e) for _, z, cap, e in _multi_block_items()] + zero + small
    items += [(z, cap, oracle_decompress(z, cap)) for _, z, cap, _ in multiblock_corruptions(3)[::4]]
    rng = np.random.default_rng(dec_warps)
    reps = 8 * _sms() // len(items) + 1                  # more items than the fused kernel's warps at 7 per SM
    batch = [items[int(k)] for k in rng.permutation(np.arange(reps * len(items)) % len(items))]
    blobs, caps, exp = [t[0] for t in batch], [t[1] for t in batch], [t[2] for t in batch]
    with ZstdBatchContext(0) as c:
        c.setOption("dec_warps_per_sm", dec_warps)
        c.setOption("host_slices_dec", 1)
        for pipeline in (1, 0):
            c.setOption("dec_pipeline", pipeline)
            before = c.kernelLaunches()
            got = c.decompressBatch(blobs, caps, raise_on_error=False)
            ran = c.kernelLaunches() - before
            assert (ran >= 6) if pipeline else (ran == 1), (pipeline, ran)
            assert _differences(got, exp) == (0, []), (pipeline, _differences(got, exp))


@pytest.mark.gpu
def test_parse_lanes_from_the_environment(monkeypatch):
    """ZSTDB200_PARSE_LANES=8 reaches the context: a level-1 batch past the 32-lane grid (8 CTAs x 4 groups per SM) but within the 8-lane
    one (16 groups per CTA) runs ordered by default (4 launches) and at once with 8 lanes (2), and both give the oracle's frames."""
    from zstd_jni_b200.zstd import ZstdBatchContext
    level = 1
    grid = _grid(level)
    datas, exp = _batch(level, grid + 600, small=(8, 4097))
    assert len(datas) < _grid(level, lanes=8)

    def run(env, opts):
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        try:
            with ZstdBatchContext(0) as c:
                for k, v in opts.items():
                    c.setOption(k, v)
                before = c.kernelLaunches()
                got = c.compressBatch(datas, level, raise_on_error=False)
                return c.kernelLaunches() - before, got
        finally:
            for k in env:
                monkeypatch.delenv(k)

    n_default, frames = run({}, {})
    n_env, frames_env = run({"ZSTDB200_PARSE_LANES": "8"}, {})
    n_opt, frames_opt = run({}, {"parse_lanes": 8})
    assert (n_default, n_env, n_opt) == (4, 2, 2)
    assert frames == exp and frames_env == frames_opt == frames
