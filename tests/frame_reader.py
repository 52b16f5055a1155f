"""More of a frame's choices, read from its bytes on top of tests/golden/frame_info.py's walk (test infrastructure only).

frame_info.walk_item gives every frame's blocks, their sections and the state each compressed block starts from.  walk_item here
returns the same walk with the fields that frames written by tests/frame_writer.py vary and the reference's encoder does not:
  frame:  window_mantissa, fcs_bytes (content-size field width), did_bytes (dictionary-ID field width);
  block:  lit_header, lit_size, lit_streams, nb_seq_bytes, table_logs / rle_codes / norms per (LL, OF, ML), huf_weights (the block's
          own Huffman tree, the implied last weight included), reaches_start (some match copies the frame's first byte).
Everything is parsed from the bytes with frame_info's readers, independently of the writer.
"""
from __future__ import annotations

from tests.golden import frame_info as fi


def huffman_weights(payload: bytes) -> list:
    """Weights of a Huffman tree description (RFC 8878 4.2.1), the implied last weight included.  FSE-compressed weights are decoded
    with two interleaved states until an update reads past the start of their stream."""
    hb = payload[0]
    if hb >= 128:
        w = [(payload[1 + i // 2] >> (4 if i % 2 == 0 else 0)) & 15 for i in range(hb - 127)]
    else:
        norm, log, used = fi._read_ncount(payload, 1, 15)
        table = fi._build_table(norm, log)
        bs = fi._Backward(payload[1 + used:1 + hb], strict=False)
        st = [bs.read(log), bs.read(log)]
        w, k = [], 0
        while True:
            s, nb, base = table[st[k]]
            w.append(s)
            st[k] = base + bs.read(nb)
            if bs.under:
                w.append(table[st[1 - k]][0])
                break
            k = 1 - k
            if len(w) > 255:
                raise ValueError("too many Huffman weights")
    total = sum(1 << (x - 1) for x in w if x)
    rest = (1 << total.bit_length()) - total
    if rest & (rest - 1):
        raise ValueError("Huffman weights do not complete a tree")
    return w + [rest.bit_length()]


def _table_norms(blk: bytes, modes: tuple, p: int) -> tuple:
    out = []
    for mode, max_sym in zip(modes, (35, 31, 52)):
        if mode == "fse":
            norm, _, used = fi._read_ncount(blk, p, max_sym)
            out.append(norm); p += used
        else:
            out.append(None); p += mode == "rle"
    return tuple(out)


def _frame_fields(z: bytes, f: fi.FrameWalk):
    at = f.offset
    fhd = z[at + 4]
    single, did_flag, fcs_flag = (fhd >> 5) & 1, fhd & 3, fhd >> 6
    f.window_mantissa = 0 if single else z[at + 5] & 7
    f.did_bytes = (0, 1, 2, 4)[did_flag]
    f.fcs_bytes = (1 if single else 0) if fcs_flag == 0 else (2, 4, 8)[fcs_flag - 1]


def _block_fields(z: bytes, b: fi.BlockInfo):
    b.lit_header = b.lit_size = b.lit_streams = b.nb_seq_bytes = 0
    b.table_logs = b.norms = b.rle_codes = ()
    b.huf_weights, b.reaches_start = None, False
    if b.block_type != 2:
        return
    blk = z[b.offset + 3:b.offset + 3 + b.size]
    h = fi.FrameInfo(0, False, False, 0, None, 2, b.size, False, False)
    fi._block_headers(blk, h)
    b.lit_header, b.lit_size, b.lit_streams, b.nb_seq_bytes = h.lit_header, h.lit_size, h.lit_streams, h.nb_seq_bytes
    if h.lit_mode == 2:
        b.huf_weights = huffman_weights(z[b.lit_payload[0]:b.lit_payload[1]])
    if not h.nb_seq:
        return
    out, rep, prev = b.state_in
    seqs, tables = fi._block_sequences(blk, h.nb_seq, h.modes, h.seq_header_end, prev)
    b.table_logs = tuple(t[1] for t in tables)
    b.rle_codes = tuple(t[0][0][0] if m == "rle" else None for t, m in zip(tables, h.modes))
    b.norms = _table_norms(blk, h.modes, h.seq_header_end)
    cur = out
    for ll, ml, of, _ in seqs:
        cur += ll
        off, rep = fi._resolve_offset(of, ll, rep)
        b.reaches_start |= off == cur
        cur += ml


def walk_item(z: bytes) -> list:
    """frame_info.walk_item(z), its frames and blocks carrying the fields above."""
    parts = fi.walk_item(z)
    for f in parts:
        if isinstance(f, tuple):
            continue
        _frame_fields(z, f)
        for b in f.blocks:
            _block_fields(z, b)
    return parts
