"""The optimal-parser levels 13..22 (btopt, btultra, btultra2) on inputs of at most 64 KB: frames must be the compiled reference's
bytes, and everything outside that scope must be refused with parameter_unsupported (40) -- inputs above 64 KB (the reference
splits such blocks after the parse), rows 11 / 12 of the <= 16 KB table, explicit strategies 7..9 on inputs above 64 KB.

CPU: the kernel source on one lane and on the emulated 32-lane warp (tests/hostsim/zb_hostsim_opt.cpp) against tests/golden/opt.json
(made by the compiled reference) and, when oracle/_ref is built, against the reference itself.  GPU (-m gpu): the batch API, the
libzstd layer, begin/end, device memory and launch splits.
"""
import ctypes as C
import hashlib
import json
import random
from pathlib import Path

import numpy as np
import pytest

from tests import cases
from tests.golden.make_golden import regenerate_input
from tests.oracle_util import CPARAM_ORDER, ERR_MAX, ROOT, ref, ref_compress, ref_compress_flags, ref_compress_params, oracle_decompress

GOLDEN = json.loads((Path(__file__).parent / "golden" / "opt.json").read_text())["cases"]
OPT_LEVELS = list(range(13, 23))
EDGE = [0, 1, 7, 8, 9, 64, 1000, 1024, 4096, 16383, 16384, 16385, 40000, 65535, 65536]
needs_ref = pytest.mark.skipif(ref() is None, reason="oracle/_ref not built on this machine")

_lib = None


def _hostsim():
    global _lib
    if _lib is None:
        path = ROOT / "tests" / "hostsim" / "libzb_hostsim_opt.so"
        if not path.exists():
            raise RuntimeError(f"{path} missing: run __graft_entry__.build()")
        _lib = C.CDLL(str(path))
        _lib.zbo_compress.restype = C.c_size_t
        _lib.zbo_compress.argtypes = [C.c_void_p, C.c_size_t, C.c_char_p, C.c_size_t, C.c_int, C.c_uint, C.c_void_p, C.c_int]
    return _lib


def host(data: bytes, level: int, params: dict | None = None, flags: dict | None = None, emu: bool = False):
    """Frame (bytes) or negative error code from the kernel source on the host (1 lane, or the 32-lane emulator)."""
    flags = flags or {}
    f = (1 if flags.get("checksum") else 0) | (0 if flags.get("content_size", True) else 2) | (4 if flags.get("magicless") else 0)
    ov = (C.c_uint * 7)(*[int((params or {}).get(k, 0)) for k in CPARAM_ORDER])
    cap = len(data) + (len(data) >> 8) + 1024
    out = C.create_string_buffer(cap)
    n = _hostsim().zbo_compress(out, cap, data, len(data), level, f, ov, 1 if emu else 0)
    return out.raw[:n] if n <= ERR_MAX else -((1 << 64) - n)


def _check_golden(e, z):
    if e["supported"]:
        assert not isinstance(z, int) and len(z) == e["size"] and hashlib.sha256(z).hexdigest() == e["sha256"], (e["input"], e["level"], e["params"], e["flags"])
    else:
        assert z == -40, (e["input"], e["level"], e["params"], z if isinstance(z, int) else len(z))


# ------------------------------------------------------------------------------------------------ CPU
def test_hostsim_matches_golden():
    for e in GOLDEN:
        _check_golden(e, host(regenerate_input(e["input"]), e["level"], e["params"], e["flags"]))


def test_emulated_warp_matches_golden():
    for e in GOLDEN[::3]:
        _check_golden(e, host(regenerate_input(e["input"]), e["level"], e["params"], e["flags"], emu=True))


@needs_ref
@pytest.mark.parametrize("level", OPT_LEVELS)
def test_every_level_matches_reference(level):
    todo = cases.special_cases() + cases.corpus_cases(8) + cases.edge_cases(classes=(0, 2, 4, 5), sizes=EDGE)
    for name, data in todo:
        data = data[:65536]
        assert host(data, level) == ref_compress(data, level), (name, len(data), level)
    for name, data in (cases.special_cases()[::3] + cases.edge_cases(classes=(0, 4), sizes=[0, 9, 1000, 16385, 65536])):      # cooperative stages
        data = data[:65536]
        assert host(data, level, emu=True) == ref_compress(data, level), (name, len(data), level)


def test_boundaries_are_refused():
    big = [corpus_bytes(1, 65537), corpus_bytes(2, 131072)]
    for level in OPT_LEVELS:
        for data in big:
            assert host(data, level) == -40, (level, len(data))
    for level in (11, 12):
        for n in (0, 9, 1000, 16384):
            assert host(corpus_bytes(3, n), level) == -40, (level, n)
            assert host(corpus_bytes(3, n), level, {"strategy": 6}) == -40, (level, n)
    for strat in (7, 8, 9):
        for data in big + [corpus_bytes(5, 70000)]:
            assert host(data, 3, {"strategy": strat}) == -40, (strat, len(data))
            assert host(data, 3, {"strategy": strat, "windowLog": 16}) == -40, (strat, len(data))    # a window smaller than the input


def corpus_bytes(i, n):
    from zstd_jni_b200 import corpus
    return corpus.chunk(i)[:n].tobytes() if n <= 131072 else b""


@needs_ref
def test_explicit_strategies_match_reference():
    rnd = random.Random(77)
    inputs = [corpus_bytes(i, n) for i, n in ((0, 65536), (1, 20000), (2, 5000), (3, 16384), (4, 900), (6, 40000))] + [(b"abcd" * 9000)[:36000]]
    for trial in range(45):
        strat = (7, 8, 9)[trial % 3]
        level = (1, 3, 9)[(trial // 3) % 3]
        params = {"strategy": strat}
        for k, rng in (("windowLog", (10, 24)), ("hashLog", (6, 22)), ("chainLog", (6, 22)), ("searchLog", (1, 9)), ("minMatch", (3, 7)),
                       ("targetLength", (0, 999))):
            if rnd.random() < 0.4:
                params[k] = rnd.randint(*rng)
        data = rnd.choice(inputs)
        exp = ref_compress_params(data, level, params)
        got = host(data, level, params, emu=trial % 5 == 0)
        if params.get("windowLog", 30) < 30 and (1 << params["windowLog"]) < len(data):
            assert got == -40, (trial, level, params, len(data))      # the window must cover the input
        else:
            assert got == exp, (trial, level, params, len(data))


@needs_ref
def test_frame_flags_match_reference():
    todo = cases.edge_cases(classes=(0, 5), sizes=[0, 1, 9, 300, 5000, 16385, 65536]) + [("period-3", (b"abc" * 20000)[:60000])]
    for level in (13, 16, 19):
        for flags in ({"checksum": True}, {"content_size": False}, {"magicless": True}, {"checksum": True, "content_size": False, "magicless": True}):
            for name, data in todo:
                assert host(data, level, flags=flags) == ref_compress_flags(data, level, **flags), (name, level, flags)


@needs_ref
def test_btultra2_two_passes_and_early_stop_inputs():
    """Inputs where the statistics of btultra2's first pass decide the second (short repeats, a shift of the alphabet half way),
    and inputs that reach btopt's early stop and the cooperative pricing: long runs, many nested matches, targetLength 999."""
    rng = np.random.default_rng(5)
    a = rng.integers(0, 6, 30000, dtype=np.uint8); a[15000:] += 100
    nested = b"".join(bytes(range(k, k + 40)) * 3 for k in range(0, 200, 3))
    inputs = [a.tobytes(), nested, b"\x07" * 50000 + b"\x08" * 15000, (b"xyzw" * 4000 + b"xyz") * 3,
              np.resize(rng.integers(0, 256, 700, dtype=np.uint8), 60000).tobytes(), corpus_bytes(9, 65536)]
    for data in inputs:
        for level in (13, 15, 18, 19, 22):
            assert host(data, level) == ref_compress(data, level), (len(data), level)
        for level, params in ((3, {"strategy": 7, "targetLength": 999}), (3, {"strategy": 9, "targetLength": 999, "searchLog": 9})):
            exp = ref_compress_params(data, level, params)
            assert host(data, level, params) == exp and host(data, level, params, emu=True) == exp, (len(data), params)


@needs_ref
def test_randomised_optimal_levels_and_sizes():
    """Seeded fuzz over levels 13..22 and inputs of at most 64 KB in the style of test_hostsim.test_randomised_levels_and_sizes."""
    from zstd_jni_b200 import corpus
    rng = np.random.default_rng(1313)

    def make(kind, n):
        if kind == 0:
            return corpus.chunk(int(rng.integers(0, 64))).tobytes()[:n]
        if kind == 1:
            a = np.resize(rng.integers(0, 256, int(rng.integers(3, 300)), dtype=np.uint8), n).copy()
            k = int(n * rng.random() * 0.05)
            if k:
                a[rng.integers(0, n, k)] = rng.integers(0, 256, k, dtype=np.uint8)
            return a.tobytes()
        if kind == 2:
            return rng.integers(0, int(rng.integers(2, 40)), n, dtype=np.uint8).tobytes()
        parts, left = [], n
        while left > 0:
            ln = min(left, int(rng.integers(1, 20000)))
            parts.append(make(int(rng.integers(0, 3)), ln)); left -= ln
        return b"".join(parts)

    for it in range(40):
        n = int(rng.choice([rng.integers(0, 300), rng.integers(300, 16385), rng.integers(16385, 65537), 65536]))
        data = make(int(rng.integers(0, 4)), n)
        level = int(rng.integers(13, 23))
        assert host(data, level, emu=it % 4 == 0) == ref_compress(data, level), (it, n, level)


# ------------------------------------------------------------------------------------------------ GPU
def _mixed_batch():
    small = [d[:65536] for _, d in cases.special_cases()[::2]] + [d for _, d in cases.edge_cases(classes=(0, 4), sizes=EDGE)]
    large = [corpus_bytes(3, 65537), corpus_bytes(4, 100000), corpus_bytes(5, 131072)]
    return small[:3] + large[:1] + small[3:] + large[1:]


@pytest.mark.gpu
@pytest.mark.parametrize("level", OPT_LEVELS)
def test_gpu_batch_per_level(level):
    from zstd_jni_b200.zstd import ZstdBatchContext
    batch = _mixed_batch()
    with ZstdBatchContext(0) as ctx:
        frames = ctx.compressBatch(batch, level, raise_on_error=False)
        assert ctx.kernelLaunches() > 0
        for data, f in zip(batch, frames):
            if len(data) > 65536:
                assert f == -40, (level, len(data))
            else:
                assert f == ref_compress(data, level) if ref() is not None else not isinstance(f, int), (level, len(data))
        small = [(d, f) for d, f in zip(batch, frames) if len(d) <= 65536]
        assert ctx.decompressBatch([f for _, f in small], [len(d) for d, _ in small]) == [d for d, _ in small]
        for d, f in small[::4]:
            assert oracle_decompress(f, len(d)) == d


@pytest.mark.gpu
def test_gpu_golden_and_libzstd_layer():
    from zstd_jni_b200.zstd import Zstd, ZstdBatchContext, ZstdCompressCtx, ZstdException
    for e in GOLDEN:
        if e["params"] or e["flags"]:
            continue
        with ZstdBatchContext(0) as ctx:
            out = ctx.compressBatch([regenerate_input(e["input"])], e["level"], raise_on_error=False)[0]
        _check_golden(e, out)
    data = corpus_bytes(2, 40000)
    with ZstdCompressCtx() as c:
        c.setLevel(19); c.setChecksum(True); c.setMagicless(True)
        z = c.compress(data)
        assert z == host(data, 19, flags={"checksum": True, "magicless": True})
        if ref() is not None:
            assert z == ref_compress_flags(data, 19, checksum=True, magicless=True)
        with pytest.raises(ZstdException) as ei:
            c.compress(corpus_bytes(2, 70000))
        assert ei.value.getErrorCode() == 40
    z22 = Zstd.compress(data, 22)
    assert z22 == host(data, 22) and Zstd.decompress(z22, len(data)) == data
    for e in GOLDEN:
        if not e["params"]:
            continue
        with ZstdBatchContext(0) as ctx:
            for k in CPARAM_ORDER:
                ctx.setOption("c_" + k, e["params"].get(k, 0))
            out = ctx.compressBatch([regenerate_input(e["input"])], e["level"], raise_on_error=False)[0]
        _check_golden(e, out)


@pytest.mark.gpu
def test_gpu_scale_begin_end_and_device_memory():
    """More than 16384 frames of <= 4 KB at one optimal level (launch parts, more frames than resident warps), the asynchronous
    begin/end pair on two slots, and compression of device-resident chunks."""
    import torch
    from zstd_jni_b200 import corpus
    from zstd_jni_b200 import _native as N
    from zstd_jni_b200.zstd import ZstdBatchContext
    base = corpus.chunk(11)[:65536].tobytes()
    n = 16384 + 700
    chunks = [base[(k * 577) % 60000:(k * 577) % 60000 + 1 + (k * 131) % 4096] for k in range(n)]
    uniq = {}
    with ZstdBatchContext(0) as ctx:
        frames = ctx.compressBatch(chunks, 16)
        for k in range(0, n, 97):
            exp = uniq.setdefault(chunks[k], host(chunks[k], 16))
            assert frames[k] == exp, k
        assert ctx.decompressBatch(frames, [len(c) for c in chunks]) == chunks
        # begin/end on two slots
        a = np.frombuffer(corpus.chunk(12).tobytes() * 4, dtype=np.uint8).copy()
        b = np.frombuffer(corpus.chunk(13).tobytes()[:200000], dtype=np.uint8).copy()
        cs = 32768
        ctx.compressChunksBegin(0, a, cs, 19)
        ctx.compressChunksBegin(1, b, cs, 19)
        for src, slot in ((a, 0), (b, 1)):
            nf = -(-src.size // cs)
            dst = np.empty(nf * (cs + 1024), dtype=np.uint8)
            fs = (C.c_size_t * nf)()
            total = ctx.compressChunksEnd(slot, dst, fs)
            off = 0
            for k in range(nf):
                piece = src[k * cs:(k + 1) * cs].tobytes()
                assert dst[off:off + fs[k]].tobytes() == host(piece, 19), (slot, k)
                off += fs[k]
            assert off == total
        # device memory (zstdb200_compress_device)
        L = N.lib()
        pieces = [corpus.chunk(20 + k).tobytes()[: 1000 + 9000 * k] for k in range(7)]
        src = torch.tensor(np.frombuffer(b"".join(pieces), dtype=np.uint8).copy(), device="cuda:0")
        offs = np.cumsum([0] + [len(p) for p in pieces]).astype(np.uint64)
        d_off = torch.tensor(offs.astype(np.int64), device="cuda:0")
        stride = ((L.ZSTD_compressBound(max(map(len, pieces))) + 32 + 63) // 64) * 64
        slots = torch.empty(len(pieces) * stride, dtype=torch.uint8, device="cuda:0")
        sizes = torch.zeros(len(pieces), dtype=torch.int64, device="cuda:0")
        torch.cuda.synchronize()
        r = L.zstdb200_compress_device(ctx.handle, 19, len(pieces), C.c_void_p(src.data_ptr()), C.c_void_p(d_off.data_ptr()), C.c_void_p(slots.data_ptr()),
                                       stride, C.c_void_p(sizes.data_ptr()), None)
        assert not N.is_error(r)
        assert not N.is_error(L.zstdb200_sync(ctx.handle, None))
        hs = sizes.cpu().numpy().astype(np.uint64); hslots = slots.cpu().numpy()
        for k, p in enumerate(pieces):
            assert hslots[k * stride:k * stride + int(hs[k])].tobytes() == host(p, 19), k
