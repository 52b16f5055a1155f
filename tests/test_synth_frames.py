"""Every decoder on legal frames written with encoding choices the reference's encoder never makes (tests/frame_writer.py).

The writer's frames carry window mantissas, wide content-size and dictionary-ID fields, literal headers wider than needed, 1-stream
Huffman literals past 255 bytes and 4-stream ones below 256, Huffman table logs 1 ... 12, alphabets of 2 ... 256 symbols, FSE tables at
every accuracy bound, RLE tables on the largest codes, tables and Huffman trees repeated blocks later across raw, RLE and sequence-free
blocks, an RLE first block, the most sequences a block holds, the largest length codes, offsets of exactly the window and windows of 2^27.

CPU: each frame decodes to its content with the compiled reference and the restatement, and with the kernel source on the host: the fused
decoder (1 lane and the emulated warp), the staged decoder (which must take every one-block frame it can), the segment decoder, the
device-call loop, the frame stream and the decode list.  A coverage check reads every intended feature back from the bytes
(tests/frame_reader.py, on frame_info's walk).
Structured illegal variants give the compiled reference's error code (or its bytes, where it accepts the frame).
GPU: the same frames through decompressBatch (default and fused-only contexts), the frame-list calls, the device call, ZSTD_decompressStream
and a magicless context.
"""
from __future__ import annotations

import ctypes as C
import os
import random
import subprocess
import sys
from functools import lru_cache
from pathlib import Path

import pytest

from tests.frame_writer import FEATURES, Block, Frame, FrameWriter, Lit, Tab, generate, text
from tests.frame_reader import walk_item
from tests.oracle_util import (ERR_MAX, emu_decompress, hostsim_decompress, hostsim_decompress_magicless, oracle_decompress, ref,
                               ref_decompress, ref_decompress_magicless, staged_decompress)

ROOT = Path(__file__).resolve().parent.parent
U64 = C.c_ulonglong
SEG_WINDOW_MAX = 1 << 27         # zb_decode_segment.cuh: the segment decoders take frames whose window is at most this


@lru_cache(maxsize=None)
def cases():
    """[(name, item, content)] of every feature at two seeds."""
    out = []
    for f in FEATURES:
        for seed in (0, 1):
            for k, (z, c) in enumerate(generate(f, seed)):
                out.append((f"{f}-{seed}-{k}", z, c))
    return out


def _frames(z):
    return [p for p in walk_item(z) if not isinstance(p, tuple)]


def _huf_log(weights):
    return (sum(1 << (w - 1) for w in weights if w)).bit_length() - 1


def _single_frames():
    return [(n, z, c) for n, z, c in cases() if len(walk_item(z)) == 1 and len(_frames(z)[0].blocks) == 1]


def _multi_block():
    return [(n, z, c) for n, z, c in cases() if len(walk_item(z)) == 1 and len(_frames(z)[0].blocks) > 1]


def _multi_frame():
    return [(n, z, c) for n, z, c in cases() if len(walk_item(z)) > 1]


def _strip_magic(z):
    return z[4:]


def _build(tmp_path_factory, name):
    so = tmp_path_factory.mktemp(name) / f"lib{name}.so"
    subprocess.run(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-Wall", "-Wno-unused-function", "-x", "c++",
                    str(ROOT / "tests" / "hostsim" / f"{name}.cpp"), "-o", str(so)], check=True)
    return C.CDLL(str(so))


@pytest.fixture(scope="module")
def loop_lib(tmp_path_factory):
    L = _build(tmp_path_factory, "zb_hostsim_loop")
    L.zbl_loop.restype = C.c_uint
    L.zbl_loop.argtypes = [C.c_char_p, C.POINTER(U64), C.c_size_t, C.c_char_p, C.POINTER(U64), C.POINTER(U64), C.POINTER(C.c_int),
                           C.c_uint, C.c_int, C.c_uint, C.c_int]
    return L


@pytest.fixture(scope="module")
def items_lib(tmp_path_factory):
    L = _build(tmp_path_factory, "zb_hostsim_items")
    L.zbi_item_walk.restype = C.c_uint
    L.zbi_item_walk.argtypes = [C.c_char_p, C.c_size_t, C.c_ulonglong, C.POINTER(C.c_ulonglong), C.c_uint, C.POINTER(C.c_int)]
    L.zbi_staged_mode.restype = C.c_uint
    L.zbi_staged_mode.argtypes = [C.c_char_p, C.c_size_t, C.c_size_t]
    return L


# ---------------------------------------------------------------------------------------------------------------------- coverage
# feature -> (frames it must have, predicate on (frame walk, item) from the bytes)
def _any_block(pred):
    return lambda fr, z: any(pred(b, fr) for b in fr.blocks)


def _repeat_after_gap(fr, z):
    """A repeated table whose source block lies two or more blocks back, with a raw, RLE or sequence-free block in between."""
    src = None
    for k, b in enumerate(fr.blocks):
        if "repeat" in b.modes and src is not None and k - src >= 2:
            between = fr.blocks[src + 1:k]
            if any(x.block_type < 2 or x.nb_seq == 0 for x in between):
                return True
        if b.nb_seq:
            src = k
    return False


def _repeat_of(mode):
    def pred(fr, z):
        last = [None] * 3
        for b in fr.blocks:
            if b.nb_seq:
                for t in range(3):
                    if b.modes[t] == "repeat" and last[t] == mode:
                        return True
                    if b.modes[t] != "repeat":
                        last[t] = b.modes[t]
        return False
    return pred


def _treeless_after_plain(fr, z):
    seen = False
    for b in fr.blocks:
        if b.lit_mode == 3 and seen:
            return True
        seen |= b.block_type < 2 or b.lit_mode in (0, 1)
    return False


def _rep_over_seq_free(fr, z):
    gap = False
    for b in fr.blocks:
        if b.first_rep and gap:
            return True
        gap = gap or (b.block_type < 2 or b.nb_seq == 0)
        if b.nb_seq and not b.first_rep:
            gap = False
    return False


def _min_lit_header(b):
    if b.lit_mode < 2:
        return 1 if b.lit_size < 32 else 2 if b.lit_size < 4096 else 3
    return 3 if max(b.lit_size, b.lit_payload[1] - b.lit_payload[0]) < 1024 else 4 if max(b.lit_size, b.lit_payload[1] - b.lit_payload[0]) < 16384 else 5


def _minus1_beside_one(b, fr):
    return any(n is not None and sum(1 for c in n if c > 0) == 1 and -1 in n for n in b.norms)


def _zero_run(b, fr):
    """A normalization whose zeros need chained repeat flags: a run of more than 3 zeros followed by a present symbol."""
    for n in b.norms:
        if n is None:
            continue
        last = max(i for i, c in enumerate(n) if c)
        run = 0
        for c in n[:last + 1]:
            run = run + 1 if c == 0 else 0
            if run > 3:
                return True
    return False


COVERAGE = {
    "window mantissa, window < 128 KB": (6, lambda fr, z: fr.window_mantissa and fr.window_size < 1 << 17 and len(fr.blocks) > 1),
    "window 2^27 mantissa 0": (2, lambda fr, z: fr.window_size == 1 << 27),
    "window 2^27 mantissa 1": (2, lambda fr, z: fr.window_size == (1 << 27) + (1 << 24)),
    "content-size field wider than needed": (4, lambda fr, z: fr.content_size is not None and fr.fcs_bytes > (
        1 if fr.single_segment and fr.content_size < 256 else 2 if fr.content_size < 65792 else 4)),
    "dictionary-ID field, value 0": (4, lambda fr, z: fr.did_bytes > 0),
    "raw / RLE literal header wider than needed": (4, _any_block(lambda b, fr: b.lit_mode in (0, 1) and b.lit_header > _min_lit_header(b))),
    "compressed literal header wider than needed": (3, _any_block(lambda b, fr: b.lit_mode >= 2 and b.lit_header > _min_lit_header(b))),
    "1 stream, 256 ... 1023 literals": (5, _any_block(lambda b, fr: b.lit_streams == 1 and 256 <= b.lit_size <= 1023)),
    "4 streams, 6 ... 255 literals": (6, _any_block(lambda b, fr: b.lit_streams == 4 and 6 <= b.lit_size <= 255)),
    "4 streams, the 4th one empty": (2, _any_block(lambda b, fr: b.lit_streams == 4 and b.lit_size == 3 * ((b.lit_size + 3) // 4))),
    "Huffman table log 12": (2, _any_block(lambda b, fr: b.huf_weights and _huf_log(b.huf_weights) == 12)),
    "compressed literals larger than their content": (2, _any_block(lambda b, fr: b.lit_payload and b.lit_payload[1] - b.lit_payload[0] > b.lit_size)),
    "compressed block larger than its content": (2, _any_block(lambda b, fr: b.block_type == 2 and b.size > b.regen)),
    "compressed block regenerating 0 bytes": (2, _any_block(lambda b, fr: b.block_type == 2 and b.regen == 0)),
    "FSE LL / ML log 5": (2, _any_block(lambda b, fr: b.modes[:1] == ("fse",) and b.table_logs[0] == 5 and b.table_logs[2] == 5)),
    "FSE LL / ML log 9": (2, _any_block(lambda b, fr: b.modes and b.modes[0] == b.modes[2] == "fse" and b.table_logs[0] == b.table_logs[2] == 9)),
    "FSE OF log 8": (2, _any_block(lambda b, fr: b.modes and b.modes[1] == "fse" and b.table_logs[1] == 8)),
    "FSE OF log 5": (2, _any_block(lambda b, fr: b.modes and b.modes[1] == "fse" and b.table_logs[1] == 5)),
    "-1 cells beside one large cell": (2, _any_block(_minus1_beside_one)),
    "zero runs with chained repeat flags": (2, _any_block(_zero_run)),
    "RLE LL 35": (2, _any_block(lambda b, fr: b.rle_codes and b.rle_codes[0] == 35)),
    "RLE ML 52": (2, _any_block(lambda b, fr: b.rle_codes and b.rle_codes[2] == 52)),
    "RLE OF >= 18": (2, _any_block(lambda b, fr: b.rle_codes and (b.rle_codes[1] or 0) >= 18)),
    "repeat two or more blocks after the table, across plain blocks": (6, _repeat_after_gap),
    "repeat of a predefined table": (2, _repeat_of("predefined")),
    "repeat of an RLE table": (2, _repeat_of("rle")),
    "treeless literals after raw / RLE literals": (4, _treeless_after_plain),
    "repcode carried over sequence-free blocks": (2, _rep_over_seq_free),
    "sequence count in a longer form": (4, _any_block(lambda b, fr: b.nb_seq_bytes == 2 and b.nb_seq < 128)),
    "RLE first block": (3, lambda fr, z: fr.blocks[0].block_type == 1),
    "43 690 sequences in one block": (2, _any_block(lambda b, fr: b.nb_seq == 43690 and b.nb_seq_bytes == 3)),
    "offset equal to the window": (4, _any_block(lambda b, fr: not fr.single_segment and b.max_offset == fr.window_size)),
    "offset reaching the frame's first byte": (2, _any_block(lambda b, fr: b.reaches_start)),
}


def _huffman_alphabet_rows(found):
    sizes = {}
    odd_direct, logs = 0, set()
    for n, z, c in cases():
        for fr in _frames(z):
            for b in fr.blocks:
                if b.huf_weights:
                    k = sum(1 for w in b.huf_weights if w)
                    sizes[k] = sizes.get(k, 0) + 1
                    logs.add(_huf_log(b.huf_weights))
                    payload = z[b.lit_payload[0]]
                    if payload >= 128 and (payload - 127) % 2 == 1:
                        odd_direct += 1
    for k in (2, 3, 127, 128, 255, 256):
        found[f"alphabet of {k}"] = sizes.get(k, 0)
    found["direct weights, odd count"] = odd_direct
    found["table logs 1 ... 12"] = len(logs & set(range(1, 13)))


def test_coverage_from_the_bytes():
    found = {k: 0 for k in COVERAGE}
    for n, z, c in cases():
        for fr in _frames(z):
            for k, (_, pred) in COVERAGE.items():
                if pred(fr, z):
                    found[k] += 1
    _huffman_alphabet_rows(found)
    need = {k: v[0] for k, v in COVERAGE.items()}
    need.update({f"alphabet of {k}": 2 for k in (2, 3, 127, 128, 255, 256)})
    need["direct weights, odd count"] = 3
    need["table logs 1 ... 12"] = 12
    items = [walk_item(z) for _, z, _ in cases()]
    found["item of several frames, second frame opens with a repcode"] = sum(
        1 for parts in items if sum(1 for p in parts if not isinstance(p, tuple)) > 1
        and any(not isinstance(p, tuple) and p.blocks[0].nb_seq for p in parts[1:]))
    need["item of several frames, second frame opens with a repcode"] = 4
    found["skippable magics"] = len({z[p[1]] & 15 for parts, (_, z, _) in zip(items, cases()) for p in parts if isinstance(p, tuple)})
    need["skippable magics"] = 16
    short = {k: (found[k], v) for k, v in need.items() if found[k] < v}
    assert not short, short


def test_second_frames_start_from_the_initial_repcodes():
    """Each later frame of a multi-frame item opens with offsets 8 and 4 written as repcodes of the history {1, 4, 8}."""
    for n, z, c in _multi_frame():
        frames = _frames(z)
        assert len(frames) > 1
        for fr in frames[1:]:
            b = fr.blocks[0]
            assert b.nb_seq and b.state_in[1] == [1, 4, 8]
            assert z[b.seq_section[0]] and not b.first_rep      # the repcodes come from the initial history, not from a block


# ---------------------------------------------------------------------------------------------------------------------- CPU decoders
def test_writer_frames_decode_with_the_reference_and_the_restatement():
    for n, z, c in cases():
        assert oracle_decompress(z, len(c)) == c, n
        if ref() is not None:
            assert ref_decompress(z, len(c)) == c, n


@pytest.mark.parametrize("emu", [False, True])
def test_fused_decoder(emu):
    dec = emu_decompress if emu else hostsim_decompress
    for n, z, c in cases():
        if emu and len(c) > 300_000:
            continue
        assert dec(z, len(c)) == c, n
        assert dec(z, len(c) + 777) == c, n


def test_staged_decoder_takes_every_frame_it_can(items_lib):
    taken = 0
    for n, z, c in _single_frames():
        fr = _frames(z)[0]
        b = fr.blocks[0]
        can = (fr.content_size is not None and fr.content_size <= 1 << 17 and (not b.huf_weights or _huf_log(b.huf_weights) <= 11)
               and b.nb_seq <= 43776)
        mode = items_lib.zbi_staged_mode(z, len(z), len(c))
        assert bool(mode) == can, (n, mode)
        taken += bool(mode)
        for emu, mis in ((False, 0), (False, 3), (True, 1), (True, 14)):
            if emu and len(c) > 70_000:
                continue
            assert staged_decompress(z, len(c), emu=emu, misalign=mis) == c, (n, emu, mis)
    assert taken >= 40


def test_segment_decoder():
    from tests.test_frame_segments import seg_decompress
    checked = 0
    for n, z, c in _multi_block():
        fr = _frames(z)[0]
        for k, seg in enumerate((0, 1, 2, 3)):
            st, got = seg_decompress(z, len(c), seg, seed=17 * k + len(n))
            if fr.window_size <= SEG_WINDOW_MAX:
                assert st == 0 and got == c, (n, seg, st)
                checked += 1
            else:
                assert st in (1, 2), (n, seg, st)
    assert checked >= 4 * 25


@pytest.mark.parametrize("B", [1, 2, 3, 7])
def test_device_call_loop(loop_lib, B):
    from tests.test_device_segment_loop import run_loop
    mb = [(z, c) for _, z, c in _multi_block() + _multi_frame()]
    rnd = random.Random(B)
    plain = [(z, c) for _, z, c in _single_frames()]
    items, want = [], []
    for z, c in mb:
        items.append(z); want.append(c)
        z2, c2 = rnd.choice(plain)
        items.append(z + z2); want.append(c + c2)
    got = run_loop(loop_lib, items, [len(w) for w in want], B, seed=B)
    routed = 0
    for k, ((st, b), w, z) in enumerate(zip(got, want, items)):
        big = any(f.window_size > SEG_WINDOW_MAX for f in _frames(z))
        if st != 2:
            routed += 1
            assert (st, b) == (0, w) or big and st == 1, (k, st)
    assert routed >= len(items) // 2


def test_frame_stream_resumes():
    from tests.test_stream_frames import stream_decode
    for n, z, c in _multi_block():
        nb = len(_frames(z)[0].blocks)
        if _frames(z)[0].window_size > SEG_WINDOW_MAX:
            continue
        for k in sorted({0, 1, nb // 2, nb - 1}):
            for stream in (False, True):
                st, got = stream_decode(z, len(c), 2, resume_from=k, stream=stream)
                assert st == 0 and got == c, (n, k, stream)


def test_decode_list_splits_multi_frame_items(items_lib):
    from tests.test_multiframe_items import item_walk
    for n, z, c in _multi_frame():
        frames, split = item_walk(items_lib, z, len(c))
        zs = [f for f in frames if not f[3]]
        assert len(zs) == len(_frames(z)), n
        assert split == all(f[2] is not None for f in zs[:-1]), n


def test_magicless_copies():
    for n, z, c in cases():
        if len(walk_item(z)) != 1 or len(c) > 300_000:
            continue
        m = _strip_magic(z)
        assert hostsim_decompress_magicless(m, len(c)) == c, n
        if ref() is not None:
            assert ref_decompress_magicless(m, len(c)) == c, n


# ---------------------------------------------------------------------------------------------------------------------- illegal
def _w(content, frame, seed=0):
    return FrameWriter().frame(content, frame, random.Random(seed))


def illegal_variants():
    """[(name, item, capacity)]: one-field edits of generated frames."""
    rnd = random.Random(5)
    t = text(rnd, 6000)
    out = []
    one = _w(t, Frame([Block(size=len(t), lit=Lit("huf"))], window_log=13))
    fw = _frames(one)[0]
    b = fw.blocks[0]
    modes_at = b.seq_section[0] + b.nb_seq_bytes
    x = bytearray(one); x[modes_at] |= 0xC0
    out.append(("repeat LL table in the first block", bytes(x), len(t)))
    x = bytearray(one); x[b.offset + 3] |= 3
    out.append(("treeless literals in the first block", bytes(x), len(t)))
    second = _w(t, Frame([Block(size=len(t), lit=Lit("huf"))], window_log=13))
    x = bytearray(second); x[modes_at] = (x[modes_at] & 0x3F) | 0xC0
    out.append(("repeat LL table in the second frame", one + bytes(x), 2 * len(t)))
    x = bytearray(second); x[b.offset + 3] |= 3
    out.append(("treeless literals in the second frame", one + bytes(x), 2 * len(t)))
    x = bytearray(one); x[modes_at + 1] = (x[modes_at + 1] & 0xF0) | 5
    out.append(("LL accuracy log 10", bytes(x), len(t)))
    x = bytearray(one); x[modes_at] |= 1
    out.append(("modes byte reserved bit", bytes(x), len(t)))
    rle = _w(b"abc" + b"c" * 900, Frame([Block(size=903, seqs=[(3, 900, 1)], lit=Lit("raw"), tabs=(Tab("rle"),) * 3)], window_log=10))
    rb = _frames(rle)[0].blocks[0]
    p = rb.seq_section[0] + rb.nb_seq_bytes + 1
    for k, (name, mx) in enumerate((("LL", 35), ("OF", 31), ("ML", 52))):
        x = bytearray(rle); x[p + k] = mx + 1
        out.append((f"RLE {name} symbol {mx + 1}", bytes(x), 903))
    small = [z for n, z, c in cases() if n.startswith("huf_4stream_small") and _frames(z)[0].blocks[0].lit_size == 6][0]
    sb = _frames(small)[0].blocks[0]
    x = bytearray(small); h = int.from_bytes(x[sb.offset + 3:sb.offset + 6], "little")
    h = (h & ~(0x3FF << 4)) | (5 << 4)
    x[sb.offset + 3:sb.offset + 6] = h.to_bytes(3, "little")
    out.append(("4 streams of 5 literals", bytes(x), 100))
    wide = _w(t[:900], Frame([Block(size=900, seqs=[], lit=Lit("huf", header=4, streams=4))], window_log=10))
    wb = _frames(wide)[0].blocks[0]
    x = bytearray(wide); h = int.from_bytes(x[wb.offset + 3:wb.offset + 7], "little")
    h = (h & ~(0x3FFF << 4)) | (1100 << 4)
    x[wb.offset + 3:wb.offset + 7] = h.to_bytes(4, "little")
    out.append(("literals above the block size max of a 1 KB window", bytes(x), 2000))
    raw = bytes(_w(t[:1024], Frame([Block("raw", 1024)], window_log=10)))
    rbk = _frames(raw)[0].blocks[0]
    hdr = ((1100 << 3) | 1).to_bytes(3, "little")
    out.append(("raw block above the block size max", raw[:rbk.offset - 4] + (1100).to_bytes(4, "little") + hdr + t[:1100], 2000))
    rep0 = _w(b"xy" * 100, Frame([Block(size=200, seqs=[(2, 10, 2, 4), (0, 8, 1, 3)], lit=Lit("raw"))][:1], window_log=10))
    out.append(("repcode rep1 - 1 = 0", rep0, 400))
    c = text(rnd, 3000)
    before = _w(c, Frame([Block(size=3000, seqs=[(100, 200, 500, 503)], lit=Lit("huf"))], window_log=12))
    out.append(("offset before the frame", one + before, len(t) + 3000))
    c = bytes(rnd.randrange(256) for _ in range(1500)) + b"\0" * 500
    c = c[:1500] + c[:500]
    beyond = _w(c, Frame([Block(size=1000, lit=Lit("raw")), Block(size=1000, seqs=[(500, 500, 1500)], lit=Lit("raw"))], window_log=10))
    out.append(("offset beyond the window inside the frame", beyond, 2000))
    return out


def test_illegal_variants_against_the_reference(loop_lib):
    if ref() is None:
        pytest.skip("oracle/_ref not built")
    from tests.test_device_segment_loop import run_loop
    from tests.test_frame_segments import seg_decompress
    todo = illegal_variants()
    assert len(todo) >= 12
    for name, z, cap in todo:
        want = ref_decompress(z, cap)
        assert hostsim_decompress(z, cap) == want, name
        assert emu_decompress(z, cap) == want, name
        st, got = seg_decompress(z, cap, 1, 3)
        assert st != 0 or got == want, name
        (st, got), = run_loop(loop_lib, [z], [cap], 2)
        assert st != 0 or got == want, name


def test_offset_beyond_the_window_is_deferred_by_the_segment_paths(loop_lib):
    """The reference's one-shot decoder accepts a match beyond the window but inside the frame (it checks against the frame's start);
    the segment decoder and the loop must not decode it themselves from a history they do not keep."""
    from tests.test_device_segment_loop import run_loop
    from tests.test_frame_segments import seg_decompress
    name, z, cap = [v for v in illegal_variants() if v[0] == "offset beyond the window inside the frame"][0]
    fused = hostsim_decompress(z, cap)
    assert isinstance(fused, bytes)
    for seg in (0, 1):
        st, got = seg_decompress(z, cap, seg, 1)
        assert st == 1 or got == fused
    (st, got), = run_loop(loop_lib, [z], [cap], 1)
    assert st == 1 or got == fused


# ---------------------------------------------------------------------------------------------------------------------- GPU
def _ctx(pipeline=1, seg_blocks=0, magicless=0):
    from zstd_jni_b200 import _native
    from zstd_jni_b200.zstd import ZstdBatchContext
    ctx = ZstdBatchContext(0)
    ctx.setOption("dec_pipeline", pipeline)
    if magicless:
        ctx.setOption("magicless", 1)
    if seg_blocks:
        assert _native.lib().zstdb200_set_option(ctx.handle, b"dec_segment_blocks", seg_blocks) == 0
    return ctx


def _counters(ctx, which):
    from zstd_jni_b200 import _native
    f = getattr(_native.lib(), which)
    return f(ctx.handle, 0), f(ctx.handle, 1)


@pytest.mark.gpu
def test_gpu_batch_single_block_frames_mixed_with_encoder_frames():
    singles = [(z, c) for _, z, c in _single_frames()]
    rnd = random.Random(3)
    plain = [text(rnd, rnd.randrange(100, 60000)) for _ in range(64)]
    with _ctx() as ctx:
        enc = ctx.compressBatch(plain, 3)
    items, want = [], []
    for i in range(3000):
        z, c = singles[i % len(singles)] if i % 2 == 0 else (enc[i % 64], plain[i % 64])
        items.append(z); want.append(c)
    caps = [len(w) for w in want]
    for pipeline in (1, 0):
        with _ctx(pipeline) as ctx:
            assert ctx.decompressBatch(items, caps) == want, pipeline


def _frame_list(ctx, items, caps):
    """zstdb200_decompress_frames and the begin / end pair."""
    from tests.test_decode_list_calls import call_begin_end, call_frames
    return call_frames(ctx, items, caps, 2), call_begin_end(ctx, items, caps)


@pytest.mark.gpu
@pytest.mark.parametrize("seg_blocks", [1, 3, 0])
def test_gpu_multi_block_and_multi_frame_items(seg_blocks):
    mb = [(z, c) for _, z, c in _multi_block()]
    mf = [(z, c) for _, z, c in _multi_frame()]
    with _ctx(1, seg_blocks) as ctx:
        d0 = _counters(ctx, "zstdb200_segment_frames")
        s0 = _counters(ctx, "zstdb200_split_items")
        for group in (mb, mf, mb + mf):
            items, want = [z for z, _ in group], [c for _, c in group]
            assert ctx.decompressBatch(items, [len(w) for w in want]) == want
        taken = [z for z, c in mb if _frames(z)[0].window_size <= SEG_WINDOW_MAX]
        assert _counters(ctx, "zstdb200_segment_frames")[1] == d0[1]          # nothing the segment decoder takes was deferred
        assert _counters(ctx, "zstdb200_segment_frames")[0] == d0[0] + 2 * len(taken)     # mb and mb + mf
        assert _counters(ctx, "zstdb200_split_items")[1] == s0[1]
    with _ctx(1, seg_blocks) as ctx:
        items, want = [z for z, _ in mb + mf], [c for _, c in mb + mf]
        a, b = _frame_list(ctx, items, [len(w) for w in want])
        assert a == want and b == want


@pytest.mark.gpu
@pytest.mark.parametrize("seg_blocks", [1, 4, 0])
def test_gpu_device_call(seg_blocks):
    from tests.test_device_segment_loop import call_device
    everything = [(z, c) for _, z, c in cases()]
    items, want = [z for z, _ in everything], [c for _, c in everything]
    with _ctx(1, seg_blocks) as ctx:
        assert call_device(ctx, items, [len(w) for w in want]) == want


@pytest.mark.gpu
def test_gpu_magicless_context():
    todo = [(_strip_magic(z), c) for _, z, c in cases() if len(walk_item(z)) == 1]
    with _ctx(1, magicless=1) as ctx:
        assert ctx.decompressBatch([z for z, _ in todo], [len(c) for _, c in todo]) == [c for _, c in todo]


@pytest.mark.gpu
def test_gpu_illegal_variants():
    if ref() is None:
        pytest.skip("oracle/_ref not built")
    from tests.test_device_segment_loop import call_device
    todo = illegal_variants()
    want = [ref_decompress(z, cap) for _, z, cap in todo]
    for seg_blocks in (1, 0):
        with _ctx(1, seg_blocks) as ctx:
            assert ctx.decompressBatch([z for _, z, _ in todo], [cap for _, _, cap in todo], raise_on_error=False) == want
            assert call_device(ctx, [z for _, z, _ in todo], [cap for _, _, cap in todo]) == want


_STREAM_CHILD = r"""
import random, sys
sys.path.insert(0, sys.argv[1])
from tests.test_synth_frames import _multi_block, _frames
from tests.test_stream_frames import _dstream
rnd = random.Random(7)
for n, z, c in _multi_block():
    if _frames(z)[0].window_size > 1 << 27:
        continue
    code, got, _ = _dstream(z, rnd.randrange(1, 200000), rnd.randrange(1, 140000))
    assert code == 0 and got == c, n
print("ok")
"""


@pytest.mark.gpu
def test_gpu_decompress_stream_past_one_segment():
    """ZSTD_decompressStream with 4-block segments, input pieces and output buffers of random sizes."""
    env = dict(os.environ, ZSTDB200_DEC_SEGMENT_BLOCKS="4")
    r = subprocess.run([sys.executable, "-c", _STREAM_CHILD, str(ROOT)], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "ok" in r.stdout, r.stderr[-3000:]


@pytest.mark.gpu
def test_gpu_decompress_stream_large_window_like_the_reference():
    """Windows of 2^27 plus a mantissa exceed the default windowLogMax of the streaming decoder: frameParameter_windowTooLarge, as the
    reference's ZSTD_decompressStream says; 2^27 itself streams."""
    from tests.test_stream_frames import _dstream, _ref_stream_lib
    for n, z, c in _multi_block():
        ws = _frames(z)[0].window_size
        if ws < 1 << 27:
            continue
        code, got, _ = _dstream(z, 65536, 131072)
        if ws == 1 << 27:
            assert code == 0 and got == c, n
        else:
            assert code == -16, n                 # frameParameter_windowTooLarge
            if ref() is not None:
                assert code == _dstream(z, 65536, 131072, lib=_ref_stream_lib())[0], n
