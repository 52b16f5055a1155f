"""The encoder's entropy stage on both sides of every threshold it copies from the reference (tests/entropy_families.py).

Each family moves one statistic -- literal count, sequence count, most frequent symbol, compressibility -- across one decision of
compress_literals, select_encoding*, the normalisation or the raw-block fallback.  The compiled reference says at which k its frame
switches sides; k - 1, k and k + 1 must then come out byte for byte the same from:
  CPU: the host instantiation of the kernel source (one lane), the emulated warp with 32- and 8-lane parse groups, and the plain-C
       restatement where it covers the level (fast and dfast);
  GPU (-m gpu): compressBatch at every level and with explicit strategies, with and without checksum, next to corpus chunks, and
       zstdb200_compress_items_device; every frame decodes again through decompressBatch.
test_each_family_switches_sides reads the side of every frame from its bytes, so a generator that drifts off its threshold fails.

Decisions no input of at most 128 KB reaches with a supported parameter set, and so are not tested here:
  - LONGNBSEQ (32512 sequences, the 3-byte count): the fast to btlazy2 parsers take matches of at least 4 bytes, so 32512 sequences
    need 130048 bytes of matches without a literal between them -- more than a 128 KB block leaves once every distinct 4-byte
    token has appeared once as literals; the optimal parsers (3-byte matches) are served up to 64 KB, at most 21845 sequences.
  - raw literals below 8 literals for btultra2: fewer than 13 literals always fail hSize + 12 >= n first, so both sides of 7 / 8
    are raw (the 8-literal RLE frame of rle_literals_strategy9 covers the n >= 8 side).
  - the mostFrequent < nbSeq >> (log - 1) test for LL and OF (ML: ml_most_frequent_*).  From the minimum nbSeq on, mostFrequent below
    nbSeq >> 5 needs more distinct LL codes than the 36 there are, unless codes of 64 KB literals and more occur several times.  For
    OF, mostFrequent < nbSeq >> 4 needs more than 16 distinct codes; below lazy the parsers write no offset code 1 (their repeat
    matches are all offBase 1), real offsets below 2^17 give codes 2 .. 16, and code 17 (offsets from 131069) fits once at most.
  - direct weights refused above maxSymbolValue 128: the FSE description is chosen unless it is at most one byte or at least
    maxSymbolValue / 2 bytes.  One byte means equal written weights, which 129 symbols next to a last one cannot have (Kraft sum);
    64.5 bytes would need about 4 bits of entropy per weight, while at most 15 of them can take the four largest values.  Seeded
    weight spreads at 129 gave descriptions of at most 55 bytes.  huffman_direct_weights_at_128 writes the largest direct table.
  - an offset code above DefaultMaxOff (28): offsets of 2^28.
  - a four-stream Huffman stream above 65535 bytes: 128 KB of literals gives at most 32 KB per stream.
Not reached by any family here, though not shown unreachable:
  - lastCountSize + streamSize below 4 (the raw-block fallback of entropy_compress): seeded searches over blocks of 2 to 6
    sequences at the lazy to btultra2 levels found no sum below 5.
  - inside fse_normalize_m2 (which fse_normalize_m2_ml enters): the second low-count pass, and the cases where every symbol is
    low (distributed == maxSymbolValue + 1, total == 0).  Those need all counts at most 1.5 total / 2^tableLog, while the table log
    fse_optimal_log picks for sequence codes exceeds log2(nbSeq) or the alphabet, and Huffman weights take at most 12 values.
"""
from __future__ import annotations

import ctypes as C
import functools

import pytest

from tests import entropy_families as ef
from tests.oracle_util import CPARAM_ORDER, ERR_MAX, ROOT, oracle_compress, ref, ref_compress_params

needs_ref = pytest.mark.skipif(ref() is None, reason="oracle/_ref not built on this machine")
NAMES = [f.name for f in ef.FAMILIES]
BY_NAME = {f.name: f for f in ef.FAMILIES}

_lib = None


def host(data: bytes, level: int, params: dict | None = None, checksum: bool = False, emu: bool = False):
    """Frame or negative error code from the kernel source on the host (libzb_hostsim_opt.so: every level and strategy)."""
    global _lib
    if _lib is None:
        path = ROOT / "tests" / "hostsim" / "libzb_hostsim_opt.so"
        if not path.exists():
            raise RuntimeError(f"{path} missing: run __graft_entry__.build()")
        _lib = C.CDLL(str(path))
        _lib.zbo_compress.restype = C.c_size_t
        _lib.zbo_compress.argtypes = [C.c_void_p, C.c_size_t, C.c_char_p, C.c_size_t, C.c_int, C.c_uint, C.c_void_p, C.c_int]
    ov = (C.c_uint * 7)(*[int((params or {}).get(k, 0)) for k in CPARAM_ORDER])
    cap = len(data) + (len(data) >> 8) + 1024
    out = C.create_string_buffer(cap)
    n = _lib.zbo_compress(out, cap, data, len(data), level, 1 if checksum else 0, ov, 1 if emu else 0)
    return out.raw[:n] if n <= ERR_MAX else -((1 << 64) - n)


def reference(data: bytes, level: int, params: dict | None = None, checksum: bool = False):
    return ref_compress_params(data, level, params or {}, checksum=checksum)


@functools.lru_cache(maxsize=None)
def rows(name: str):
    """(k, [(k', input, explicit parameters, the reference's frame) for k' = k - 1, k, k + 1]) of a family; every k' in lo..hi for
    the families without a single threshold."""
    fam = BY_NAME[name]
    k = ef.find_boundary(fam, reference)
    ks = [k - 1, k, k + 1] if fam.boundary else list(range(fam.lo, fam.hi + 1))
    out = []
    for kk in ks:
        data = fam.gen(kk, fam.seed)
        params = fam.params_at(kk)
        out.append((kk, data, params, reference(data, fam.level, params)))
    return k, out


def restated(fam) -> bool:
    """Whether the plain-C restatement (fast and dfast, levels only) covers the family's parameter set."""
    return not fam.params_at(fam.lo) and fam.level in (-5, -1, 1, 2, 3)


# ------------------------------------------------------------------------------------------------ CPU
@needs_ref
def test_each_family_switches_sides():
    """From the bytes of the reference's frames: every family's k - 1 and k + 1 lie on different sides of its decision, and where
    the decision is on a count the frame shows, k lands on the threshold itself."""
    short = {}
    for name in NAMES:
        fam = BY_NAME[name]
        if not fam.boundary:
            continue
        k, r = rows(name)
        sides = [fam.side(ef.block(z)) for _, _, _, z in r]
        if not (sides[0] != sides[2] and sides[1] == sides[2]):
            short[name] = sides
        if fam.exact and not fam.exact(ef.block(r[1 + fam.exact_at][3])):
            short[name] = ("k is not on the threshold", k)
    assert not short, short


@needs_ref
def test_fixed_families_reach_their_choices():
    """The families without one threshold reach what they are for: Huffman logs cut below the tree's depth, FSE-compressed
    weights at maxSymbolValue 125 .. 131, compressed literals for the sort ties, and ML tables normalised through
    fse_normalize_m2 (recomputed from the frames' sequences)."""
    logs = {z and ef.huf_log(ef.block(z)) for _, _, _, z in rows("huffman_depth_limit_log11")[1]}
    assert 11 in logs, logs
    small = {ef.huf_log(ef.block(z)) for _, _, _, z in rows("huffman_depth_limit_small_log")[1]}
    assert min(small) < 11, small
    fmts = {ef.weight_format(ef.block(z)) for _, _, _, z in rows("huffman_weights_maxsv")[1]}
    assert fmts == {"fse"}, fmts
    for name in ("huffman_sort_ties", "huffman_sort_ties_strategy8", "huffman_depth_limit_repair"):
        assert {ef.lit_kind(ef.block(z)) for _, _, _, z in rows(name)[1]} == {"huf4"}, name
    fmts = [ef.weight_format(ef.block(z)) for _, _, _, z in rows("huffman_direct_weights_at_128")[1]]
    assert fmts == ["fse", "direct", "fse"], fmts
    m2 = [ef.ml_table_enters_m2(ef.block(z)) for _, _, _, z in rows("fse_normalize_m2_ml")[1]]
    assert sum(m2) >= 4, m2


@needs_ref
@pytest.mark.parametrize("name", NAMES)
def test_host_instantiation_matches_reference(name):
    fam = BY_NAME[name]
    for kk, data, params, want in rows(name)[1]:
        assert host(data, fam.level, params) == want, (name, kk)
        assert host(data, fam.level, params, checksum=True) == reference(data, fam.level, params, checksum=True), (name, kk, "checksum")


@needs_ref
@pytest.mark.parametrize("lanes", ["32", "8"])
@pytest.mark.parametrize("name", NAMES)
def test_emulated_warp_matches_reference(name, lanes, monkeypatch):
    """The cooperative entropy code (hist_warp, w.sum / w.exscan sizing, atomic_or32 row packing) on the emulated 32-lane warp,
    behind a 32- or an 8-lane parse group (the 8-lane group only for the levels libzb_hostsim.so serves without explicit parameters)."""
    from tests.oracle_util import emu_compress
    fam = BY_NAME[name]
    if lanes == "8" and (fam.params_at(fam.lo) or fam.level > 12):
        pytest.skip("the 8-lane parse group runs levels 1..12 without explicit parameters")
    monkeypatch.setenv("ZB_EMU_PARSE_LANES", lanes)
    for kk, data, params, want in rows(name)[1]:
        got = host(data, fam.level, params, emu=True) if lanes == "32" else emu_compress(data, fam.level)
        assert got == want, (name, kk, lanes)


@needs_ref
@pytest.mark.parametrize("name", [n for n in NAMES if restated(BY_NAME[n])])
def test_restatement_matches_reference(name):
    fam = BY_NAME[name]
    for kk, data, _, want in rows(name)[1]:
        assert oracle_compress(data, fam.level) == want, (name, kk)


# ------------------------------------------------------------------------------------------------ GPU
GPU_LEVELS = [-5, -1] + list(range(1, 23))


def _served(level: int, n: int) -> bool:
    """Levels 11 and 12 are served above 16 KB, the optimal levels up to 64 KB."""
    return not ((level in (11, 12) and n <= 16384) or (level >= 13 and n > 65536))


def _level_inputs(level: int):
    """Every family input the level serves; levels 19..22 only those of the families whose decision depends on the strategy."""
    out = []
    for name in NAMES:
        if level >= 19 and not BY_NAME[name].strategy_dependent:
            continue
        out += [d for _, d, _, _ in rows(name)[1] if _served(level, len(d))]
    return out


def _with_corpus(inputs, level):
    from zstd_jni_b200 import corpus
    chunks = [corpus.chunk(i).tobytes()[:65536 if level >= 13 else 131072] for i in range(6)]
    mixed = []
    for i, d in enumerate(inputs):
        mixed.append(d)
        if i % max(1, len(inputs) // len(chunks)) == 0 and chunks:
            mixed.append(chunks.pop())
    return mixed + chunks


def _check_batch(ctx, batch, frames, want):
    for i, (d, f) in enumerate(zip(batch, frames)):
        assert f == want(d), (i, len(d))
    assert ctx.decompressBatch(frames, [len(d) for d in batch]) == batch


@needs_ref
@pytest.mark.gpu
@pytest.mark.parametrize("level", GPU_LEVELS)
def test_gpu_every_level(level):
    """All families' inputs at one level in one batch, between corpus chunks, so boundary frames share warps and CTAs with ordinary
    ones; with a checksum on the odd levels."""
    from zstd_jni_b200.zstd import ZstdBatchContext
    batch = _with_corpus(_level_inputs(level), level)
    checksum = level % 2 != 0
    with ZstdBatchContext(0) as ctx:
        ctx.setOption("checksum", int(checksum))
        frames = ctx.compressBatch(batch, level)
        _check_batch(ctx, batch, frames, lambda d: reference(d, level, checksum=checksum))


@needs_ref
@pytest.mark.gpu
@pytest.mark.parametrize("checksum", [False, True])
def test_gpu_explicit_parameters(checksum):
    """Every family with explicit parameters (strategies 1..9 through c_strategy, targetLength) at its own parameter set."""
    from zstd_jni_b200.zstd import ZstdBatchContext
    groups = {}
    for name in NAMES:
        fam = BY_NAME[name]
        for _, d, params, _ in rows(name)[1]:
            if params:
                groups.setdefault((fam.level, tuple(sorted(params.items()))), []).append(d)
    assert {dict(p).get("strategy") for _, p in groups} >= set(range(1, 10))
    for (level, params), batch in groups.items():
        with ZstdBatchContext(0) as ctx:
            ctx.setOption("checksum", int(checksum))
            for k in CPARAM_ORDER:
                ctx.setOption("c_" + k, dict(params).get(k, 0))
            frames = ctx.compressBatch(batch, level)
            _check_batch(ctx, batch, frames, lambda d: reference(d, level, dict(params), checksum=checksum))


@needs_ref
@pytest.mark.gpu
def test_gpu_device_items():
    """One zstdb200_compress_items_device call at level 3 whose items are the families' inputs, each one chunk of the call."""
    import numpy as np
    import torch
    from zstd_jni_b200 import _native
    from zstd_jni_b200.zstd import ZstdBatchContext
    level, cs = 3, 131072
    items = _level_inputs(level)
    L = _native.lib()
    dev = torch.device("cuda:0")
    so = np.concatenate([[0], np.cumsum([len(x) for x in items])]).astype(np.int64)
    cap = sum(L.ZSTD_compressBound(len(x)) + 32 for x in items)
    d_src = torch.from_numpy(np.frombuffer(b"".join(items), dtype=np.uint8).copy()).to(dev)
    d_so = torch.from_numpy(so).to(dev)
    d_dst = torch.zeros(cap, dtype=torch.uint8, device=dev)
    d_do = torch.full((len(items) + 1,), -1, dtype=torch.int64, device=dev)
    d_res = torch.zeros(len(items), dtype=torch.int64, device=dev)
    with ZstdBatchContext(0) as ctx:
        s = torch.cuda.Stream()
        r = L.zstdb200_compress_items_device(ctx.handle, level, cs, len(items), d_src.data_ptr(), d_so.data_ptr(), d_dst.data_ptr(), cap,
                                             d_do.data_ptr(), d_res.data_ptr(), s.cuda_stream)
        assert r == 0, r
        s.synchronize()
        do = [int(x) for x in d_do.cpu().numpy()]
        res = [int(x) for x in d_res.cpu().numpy()]
        assert res == [do[i + 1] - do[i] for i in range(len(items))], "per-item results are the stream sizes"
        out = d_dst.cpu().numpy()
        frames = [out[do[i]:do[i + 1]].tobytes() for i in range(len(items))]
        _check_batch(ctx, items, frames, lambda d: reference(d, level))
