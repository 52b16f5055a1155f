"""The segment decoder for frames of many blocks (zb_decode_segment.cuh).

CPU: the host instantiation of its stages (tests/hostsim/libzb_hostsim_seg.so) with the blocks in shuffled order, segment cuts at
every block boundary and the carried state passed between them, against the oracle; corrupted frames either decode to the fused
decoder's bytes or are deferred to it; the repcode summaries against the serial walk.
GPU: the batch API routes such frames to the segment decoder (dec_pipeline 1) and must give the bytes / error codes of the fused
kernel (dec_pipeline 0), with segments as small as one block.
"""
from __future__ import annotations

import ctypes as C
import random
from pathlib import Path

import pytest

from tests.oracle_util import ERR_MAX, hostsim_decompress, oracle_decompress, ref, ref_stream_compress

ROOT = Path(__file__).resolve().parent.parent
GOLDEN = ROOT / "tests" / "golden"
SEG_PATH = ROOT / "tests" / "hostsim" / "libzb_hostsim_seg.so"
MB = sorted(p for p in GOLDEN.glob("mb_*.zst"))


def _seg():
    L = C.CDLL(str(SEG_PATH))
    L.zbs_decompress.restype = C.c_size_t
    L.zbs_decompress.argtypes = [C.c_void_p, C.c_size_t, C.c_char_p, C.c_size_t, C.c_uint, C.c_uint, C.c_int, C.POINTER(C.c_int)]
    L.zbs_rep_check.restype = C.c_uint
    L.zbs_rep_check.argtypes = [C.c_uint, C.c_uint, C.c_uint]
    return L


def seg_decompress(frame: bytes, cap: int, seg_blocks: int = 0, seed: int = 0, emu: bool = False):
    """(status, bytes): status 0 decoded, 1 deferred to the fused decoder, 2 not a frame of many blocks."""
    out = C.create_string_buffer(max(cap, 1))
    st = C.c_int(-1)
    n = _seg().zbs_decompress(out, cap, frame, len(frame), seg_blocks, seed, 1 if emu else 0, C.byref(st))
    assert n <= ERR_MAX
    return st.value, out.raw[:n]


def _blocks(frame: bytes) -> int:
    """Number of blocks of an item that is exactly one frame (0 otherwise)."""
    fhd = frame[4]
    did, single, fcs = fhd & 3, (fhd >> 5) & 1, fhd >> 6
    pos = 5 + (not single) + (4 if did == 3 else did) + ((1 << fcs) if fcs else 0) + (1 if single and not fcs else 0)
    n = 0
    while pos + 3 <= len(frame):
        bh = int.from_bytes(frame[pos:pos + 3], "little")
        pos += 3 + (1 if (bh >> 1) & 3 == 1 else bh >> 3)
        n += 1
        if bh & 1:
            return n if pos + 4 * ((fhd >> 2) & 1) == len(frame) else 0
    return 0


def _cases():
    out = []
    for p in MB:
        out.append((p.name, p.read_bytes()))
    return out


def _content(frame: bytes) -> int:
    r = oracle_decompress(frame, 1 << 24)
    return len(r) if isinstance(r, bytes) else 1 << 20


@pytest.mark.parametrize("name,frame", _cases(), ids=[c[0] for c in _cases()])
def test_golden_multiblock_every_cut(name, frame):
    want = oracle_decompress(frame, 1 << 24)
    n = _blocks(frame)
    if not isinstance(want, bytes) or n < 2:
        st, _ = seg_decompress(frame, 1 << 24)
        assert st in (1, 2)        # not taken, or deferred to the fused decoder
        return
    cuts = sorted({1, 2, 3, max(1, n // 2), n - 1, n, 0}) if n > 8 else range(0, n + 1)
    for k, seg in enumerate(cuts):
        st, got = seg_decompress(frame, len(want), seg, seed=k)
        assert st == 0 and got == want, (name, seg, st)


@pytest.mark.parametrize("level", [1, 3, 9, 19])
@pytest.mark.parametrize("checksum", [False, True])
def test_reference_stream_frames(level, checksum):
    if ref() is None:
        pytest.skip("oracle/_ref not built")
    rnd = random.Random(level)
    words = [bytes(rnd.choice(b"abcdefghij") for _ in range(rnd.randint(2, 9))) for _ in range(300)]
    data = b" ".join(rnd.choice(words) for _ in range(120000))[:700000]
    frame = ref_stream_compress(data, level, 50000, checksum)
    assert _blocks(frame) >= 4
    for seg, seed in ((0, 1), (1, 2), (3, 3)):
        st, got = seg_decompress(frame, len(data), seg, seed)
        assert st == 0 and got == data


def test_emulated_warp_stages():
    frame = (GOLDEN / "mb_L3_xxh.zst").read_bytes()
    want = oracle_decompress(frame, 1 << 24)
    st, got = seg_decompress(frame, len(want), 2, 7, emu=True)
    assert st == 0 and got == want


def test_small_capacity_defers():
    frame = (GOLDEN / "mb_L1.zst").read_bytes()
    want = oracle_decompress(frame, 1 << 24)
    st, _ = seg_decompress(frame, len(want) - 1, 0)
    assert st == 1


@pytest.mark.parametrize("name", ["mb_L1.zst", "mb_L19.zst", "mb_L3_w10_raw_rle.zst", "mb_L3_xxh.zst"])
def test_corruptions_match_fused_or_defer(name):
    frame = (GOLDEN / name).read_bytes()
    cap = _content(frame)
    rnd = random.Random(name)
    for _ in range(60):
        b = bytearray(frame)
        i = rnd.randrange(6, len(b))
        b[i] ^= 1 << rnd.randrange(8)
        b = bytes(b)
        st, got = seg_decompress(b, cap, rnd.choice([0, 1, 2]), rnd.randrange(1 << 30))
        if st == 0:
            assert got == hostsim_decompress(b, cap), i


@pytest.mark.parametrize("seed", range(8))
def test_repcode_summaries_compose_like_the_serial_walk(seed):
    assert _seg().zbs_rep_check(seed, 200, 40) == 0


# ---------------------------------------------------------------- GPU: the batch API
def _ctx(pipeline: int, seg_blocks: int = 0):
    from zstd_jni_b200 import _native
    from zstd_jni_b200.zstd import ZstdBatchContext
    ctx = ZstdBatchContext(0)
    assert _native.lib().zstdb200_set_option(ctx._live(), b"dec_pipeline", pipeline) == 0
    if seg_blocks:
        assert _native.lib().zstdb200_set_option(ctx._live(), b"dec_segment_blocks", seg_blocks) == 0
    return ctx


def _segment_frames(ctx):
    """(decoded, deferred): frames the segment decoder regenerated / handed to the fused kernel so far."""
    from zstd_jni_b200 import _native
    L = _native.lib()
    return L.zstdb200_segment_frames(ctx._live(), 0), L.zstdb200_segment_frames(ctx._live(), 1)


def _batch(ctx, frames, caps):
    return ctx.decompressBatch(frames, caps, raise_on_error=False)


def _decoded_on_segments(ctx, frames, caps):
    """Decodes valid frames of many blocks and checks that the segment decoder itself regenerated every one of them."""
    d0, f0 = _segment_frames(ctx)
    out = ctx.decompressBatch(frames, caps)
    assert _segment_frames(ctx) == (d0 + len(frames), f0)
    return out


def _text(n: int, seed: int) -> bytes:
    import numpy as np
    rnd = np.random.default_rng(seed)
    words = rnd.integers(97, 123, size=(4000, 8), dtype=np.uint8)
    words[:, 7] = 32
    return words[rnd.zipf(1.4, size=n // 8 + 1) % 4000].tobytes()[:n]


@pytest.mark.gpu
@pytest.mark.parametrize("seg_blocks", [0, 1, 3])
def test_gpu_golden_segments(seg_blocks):
    """Every valid one-frame fixture of many blocks is regenerated by the segment decoder itself, in one segment or cut after every
    block, and gives the oracle's bytes; the rest of the fixtures give the fused kernel's results."""
    frames = [p.read_bytes() for p in MB]
    caps = [_content(f) for f in frames]
    valid = [(f, cap) for f, cap in zip(frames, caps) if _blocks(f) >= 2 and isinstance(oracle_decompress(f, cap), bytes)]
    assert len(valid) >= 10
    with _ctx(1, seg_blocks) as a, _ctx(0) as b:
        for f, cap in valid:
            assert _decoded_on_segments(a, [f], [cap]) == [oracle_decompress(f, cap)]
        assert _batch(a, frames, caps) == _batch(b, frames, caps)


@pytest.mark.gpu
@pytest.mark.parametrize("level", [1, 3, 9, 19])
def test_gpu_reference_stream_frames(level):
    if ref() is None:
        pytest.skip("oracle/_ref not built")
    from zstd_jni_b200.zstd import Zstd
    data = _text(8 << 20, level)
    for checksum in (False, True):
        frame = ref_stream_compress(data, level, 1 << 20, checksum)
        for seg_blocks in (0, 5):
            with _ctx(1, seg_blocks) as a:
                assert _decoded_on_segments(a, [frame], [len(data)]) == [data]
        assert Zstd.decompress(frame, len(data)) == data


@pytest.mark.gpu
@pytest.mark.parametrize("window_log", [17, 20, 24, 27])
def test_gpu_window_logs(window_log):
    """One-shot reference frames of many blocks at windowLog 17 ... 27, checksummed at the even ones."""
    if ref() is None:
        pytest.skip("oracle/_ref not built")
    from tests.oracle_util import ref_compress_params
    data = _text(6 << 20, window_log)
    data = data[: 3 << 20] + data[: 3 << 20]          # repeats from 3 MB back: only the larger windows reach them
    params = {"windowLog": window_log}
    frame = ref_compress_params(data, 3, params, checksum=window_log % 2 == 0)
    assert isinstance(frame, bytes) and _blocks(frame) > 2
    with _ctx(1, 7) as a:
        assert _decoded_on_segments(a, [frame], [len(data)]) == [data]


@pytest.mark.gpu
def test_gpu_large_frame_many_segments_with_checksum():
    if ref() is None:
        pytest.skip("oracle/_ref not built")
    data = _text(160 << 20, 11)                       # 1280 blocks: three segments of the default 512
    frame = ref_stream_compress(data, 1, 4 << 20, True)
    with _ctx(1) as a:
        assert _decoded_on_segments(a, [frame], [len(data)]) == [data]
    bad = bytearray(frame)
    bad[-1] ^= 1                                       # the checksum: verified on the host, the fused kernel gives the error code
    with _ctx(1) as a, _ctx(0) as b:
        d0, f0 = _segment_frames(a)
        assert _batch(a, [bytes(bad)], [len(data)]) == _batch(b, [bytes(bad)], [len(data)])
        assert _segment_frames(a) == (d0, f0 + 1)


@pytest.mark.gpu
def test_gpu_corruptions_match_the_compiled_reference():
    """Damaged multi-block fixtures through the segment decoder (two blocks per segment), judged by the compiled reference: a result may
    differ only in a class frame_info.reference_difference computes (DESIGN.md section 5)."""
    if ref() is None:
        pytest.skip("oracle/_ref not built")
    from collections import Counter

    from tests.golden.frame_info import reference_difference
    from tests.golden.make_golden import multiblock_corruptions
    from tests.oracle_util import ref_decompress
    todo = multiblock_corruptions(5)
    exp = [ref_decompress(z, cap) for _, z, cap, _ in todo]
    with _ctx(1, 2) as a:
        got = _batch(a, [t[1] for t in todo], [t[2] for t in todo])
        decoded, deferred = _segment_frames(a)
    assert decoded > 0 and deferred > 0
    allowed = Counter()
    for (fn, z, cap, k), e, g in zip(todo, exp, got):
        if e == g:
            continue
        cls = reference_difference((GOLDEN / fn).read_bytes(), z, cap, e, g) if k is not None else None
        assert cls, (fn, k, e if isinstance(e, int) else "bytes", g if isinstance(g, int) else "bytes")
        allowed[cls] += 1
    assert sum(allowed.values()) <= len(todo) // 4, allowed


@pytest.mark.gpu
def test_gpu_bit_flips_equal_fused():
    rnd = random.Random(5)
    with _ctx(1, 2) as a, _ctx(0) as b:
        for name in ("mb_L1.zst", "mb_L9.zst", "mb_L19.zst", "mb_L3_xxh.zst", "mb_L3_w10_raw_rle.zst"):
            frame = (GOLDEN / name).read_bytes()
            cap = _content(frame)
            items = []
            for _ in range(80):
                x = bytearray(frame)
                i = rnd.randrange(6, len(x))
                x[i] ^= 1 << rnd.randrange(8)
                items.append(bytes(x))
            assert _batch(a, items, [cap] * len(items)) == _batch(b, items, [cap] * len(items))
