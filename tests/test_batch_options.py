"""The option contract of a batch context (-m gpu): which values `zstdb200_set_option` accepts for every name, and the options that
`zstdb200_create` reads from ZSTDB200_* environment variables."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

_ANY = [-(1 << 63), -1, 0, 1, 7, (1 << 63) - 1]
_ON_OFF = [0, 1, -1, 2, 1 << 40]

# name -> (accepted values, rejected values): the boundary values of every rule and the values just outside them
CONTRACT = {
    "enc_warps_per_sm": (_ANY, []),
    "dec_warps_per_sm": (_ANY, []),
    "parse_order": (_ANY, []),
    "chain_roles": (_ANY, []),
    "skip_entropy": (_ON_OFF, []),
    "kernel_fifo": (_ON_OFF, []),
    "entropy_overlap": (_ON_OFF, []),
    "dec_pipeline": (_ON_OFF, []),
    "timing": (_ON_OFF, []),
    "checksum": (_ON_OFF, []),
    "content_size": (_ON_OFF, []),
    "magicless": (_ON_OFF, []),
    "parse_lanes": ([4, 8, 16, 32], [0, 1, 3, 5, 7, 9, 15, 17, 31, 33, 64, -4, (1 << 32) + 4]),
    "parse_est_bytes": ([256, 257, 2048, 65535, 65536], [0, 255, 65537, -256, (1 << 32) + 256]),
    "opt_blocks_per_sm": ([4, 6, 8], [0, 3, 5, 7, 9, (1 << 32) + 4]),
    "lazy_blocks_per_sm": ([4, 6, 8], [0, 3, 5, 7, 9, (1 << 32) + 4]),
    "parse_blocks_per_sm": ([1, 2, 15, 16], [0, 17, -1, (1 << 32) + 1]),
    "host_slices": ([1, 2, 63, 64], [0, 65, -1, (1 << 32) + 1]),
    "host_slices_dec": ([1, 2, 63, 64], [0, 65, -1, (1 << 32) + 1]),
    "l2_fetch_granularity": ([32, 128, 64], [0, 31, 33, 63, 65, 127, 129, 256, (1 << 32) + 64]),
}
# explicit compression parameters: 0 (from the level) or within ZSTD_cParam_getBounds
for _name, (_lo, _hi) in {"c_windowLog": (10, 31), "c_hashLog": (6, 30), "c_chainLog": (6, 30), "c_searchLog": (1, 30),
                          "c_minMatch": (3, 7), "c_targetLength": (0, 131072), "c_strategy": (1, 9)}.items():
    CONTRACT[_name] = ([0, _lo, _hi], [v for v in (_lo - 1, _hi + 1, (1 << 32) + _lo) if v != 0])


@pytest.fixture(scope="module")
def lib():
    from zstd_jni_b200 import _native
    return _native.lib()


@pytest.mark.parametrize("name", sorted(CONTRACT))
def test_option_accepts_its_range(lib, name):
    accepted, rejected = CONTRACT[name]
    ctx = lib.zstdb200_create(0)
    assert ctx, lib.zstdb200_last_error().decode()
    try:
        for v in rejected:
            assert lib.zstdb200_set_option(ctx, name.encode(), v) == -1, (name, v)
        for v in accepted:
            assert lib.zstdb200_set_option(ctx, name.encode(), v) == 0, (name, v)
    finally:
        lib.zstdb200_free(ctx)


def test_unknown_option_is_rejected(lib):
    ctx = lib.zstdb200_create(0)
    assert ctx, lib.zstdb200_last_error().decode()
    try:
        for name in [b"", b"nope", b"PARSE_LANES", b"parse_lanes ", b"c_windowlog", b"l2_fetch", b"ZSTDB200_HOST_SLICES", b"c_"]:
            assert lib.zstdb200_set_option(ctx, name, 1) == -1, name
        assert lib.zstdb200_set_option(ctx, None, 1) == -1
        assert lib.zstdb200_set_option(None, b"timing", 1) == -1
    finally:
        lib.zstdb200_free(ctx)


def _launches(ctx, call):
    before = ctx.kernelLaunches()
    out = call()
    return ctx.kernelLaunches() - before, out


def test_environment_reaches_the_context(monkeypatch):
    """ZSTDB200_ENTROPY_OVERLAP=0: a batch smaller than the resident parse grid runs parse, order and entropy (3 launches) instead of
    the overlapped pair (2).  ZSTDB200_HOST_SLICES=2: compress_chunks on 512 chunks runs as two slices, each with its own parse, entropy,
    scan and compaction; an out-of-range value (65) leaves the default of one slice."""
    from zstd_jni_b200 import corpus
    from zstd_jni_b200.zstd import ZstdBatchContext
    datas = [corpus.chunk(i, 3000).tobytes() for i in range(64)]
    flat = np.concatenate([corpus.chunk(100 + i, 1024) for i in range(512)])

    def run(env):
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        try:
            with ZstdBatchContext(0) as c:
                batch = _launches(c, lambda: c.compressBatch(datas, 3))
                chunks = _launches(c, lambda: c.compressChunks(flat, 1024, 3))
        finally:
            for k in env:
                monkeypatch.delenv(k)
        return batch, chunks

    (nb, frames), (nc, (stream, sizes)) = run({})
    assert nb == 2 and nc == 4, (nb, nc)
    (nb0, frames0), _ = run({"ZSTDB200_ENTROPY_OVERLAP": "0"})
    assert nb0 == 3 and frames0 == frames
    _, (nc2, (stream2, sizes2)) = run({"ZSTDB200_HOST_SLICES": "2"})
    assert nc2 == 2 * nc and stream2.tobytes() == stream.tobytes() and list(sizes2) == list(sizes)
    _, (nc65, (stream65, _s)) = run({"ZSTDB200_HOST_SLICES": "65"})
    assert nc65 == nc and stream65.tobytes() == stream.tobytes()
