"""Header parser for single-block zstd frames (RFC 8878), test infrastructure only.

parse_frame() reads the frame header, the block header, the literals section header and the sequences section header
of a frame that holds exactly one block.  decode_sequences() walks the sequence bitstream of a compressed block
(FSE tables, predefined / RLE / compressed modes) and returns the sequences as (litLength, matchLength, offsetValue,
mlCode).  features() turns both into the tags that tests/golden/manifest.json stores for its decode-only frames.
"""
from __future__ import annotations

from dataclasses import dataclass

MAGIC = 0xFD2FB528
MODES = ("predefined", "rle", "fse", "repeat")

# RFC 8878 3.1.1.3.2.2: predefined distributions (accuracy logs 6 / 5 / 6)
LL_DEFAULT = [4, 3, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 1, 1, 1, 2, 2, 2, 2, 2, 2, 2, 2, 2, 3, 2, 1, 1, 1, 1, 1, -1, -1, -1, -1]
ML_DEFAULT = [1, 4, 3, 2, 2, 2, 2, 2, 2] + [1] * 37 + [-1] * 7
OF_DEFAULT = [1, 1, 1, 1, 1, 1, 2, 2, 2] + [1] * 15 + [-1] * 5
LL_BASE = list(range(16)) + [16, 18, 20, 22, 24, 28, 32, 40, 48, 64, 128, 256, 512, 1024, 2048, 4096, 8192, 16384, 32768, 65536]
LL_BITS = [0] * 16 + [1, 1, 1, 1, 2, 2, 3, 3, 4, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16]
ML_BASE = [c + 3 for c in range(32)] + [35, 37, 39, 41, 43, 47, 51, 59, 67, 83, 99, 131, 259, 515, 1027, 2051, 4099, 8195, 16387, 32771, 65539]
ML_BITS = [0] * 32 + [1, 1, 1, 1, 2, 2, 3, 3, 4, 4, 5, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16]
FAST_MAXS = 43776        # zb_decode_fast.cuh: the staged decoder takes at most this many sequences per frame


@dataclass
class FrameInfo:
    header_size: int
    single_segment: bool
    checksum: bool
    dict_id: int
    content_size: int | None
    block_type: int              # 0 raw, 1 rle, 2 compressed
    block_size: int
    last_block: bool
    one_block: bool              # the frame is exactly this one last block
    lit_mode: int = -1           # 0 raw, 1 rle, 2 compressed (Huffman), 3 treeless
    lit_size: int = 0            # regenerated literal bytes
    lit_streams: int = 0         # Huffman streams (1 or 4), 0 for raw / rle literals
    lit_header: int = 0          # bytes of the literals section header
    lit_section: int = 0         # bytes of the whole literals section (header included)
    nb_seq: int = 0
    nb_seq_bytes: int = 0        # width of the sequence count (1, 2 or 3 bytes)
    modes: tuple = ()            # (LL, OF, ML) table modes, names from MODES; () when nb_seq == 0
    seq_header_end: int = 0      # offset (inside the block content) of the first table description

    @property
    def staged(self) -> bool:
        """What the staged batch decoder takes itself (dec_prepare): magic, content size <= 128 KB, no checksum, no dictionary ID,
        exactly one block and at most FAST_MAXS sequences."""
        return (self.content_size is not None and self.content_size <= 131072 and not self.checksum and self.dict_id == 0 and self.one_block
                and self.nb_seq <= FAST_MAXS)


def parse_frame(z: bytes) -> FrameInfo:
    if int.from_bytes(z[:4], "little") != MAGIC:
        raise ValueError("no zstd magic number")
    fhd = z[4]
    single, checksum, did_flag, fcs_flag = (fhd >> 5) & 1, (fhd >> 2) & 1, fhd & 3, fhd >> 6
    pos = 5 + (0 if single else 1)
    did_len = (0, 1, 2, 4)[did_flag]
    dict_id = int.from_bytes(z[pos:pos + did_len], "little"); pos += did_len
    fcs_len = (1 if single else 0) if fcs_flag == 0 else (2, 4, 8)[fcs_flag - 1]
    content = int.from_bytes(z[pos:pos + fcs_len], "little") + (256 if fcs_len == 2 else 0) if fcs_len else None
    pos += fcs_len
    bh = int.from_bytes(z[pos:pos + 3], "little")
    btype, bsize = (bh >> 1) & 3, bh >> 3
    payload = 1 if btype == 1 else bsize
    info = FrameInfo(header_size=pos, single_segment=bool(single), checksum=bool(checksum), dict_id=dict_id, content_size=content,
                     block_type=btype, block_size=bsize, last_block=bool(bh & 1),
                     one_block=bool(bh & 1) and pos + 3 + payload + (4 if checksum else 0) == len(z))
    if btype != 2:
        return info
    blk = z[pos + 3:pos + 3 + bsize]
    b0 = blk[0]; lt, sf = b0 & 3, (b0 >> 2) & 3
    if lt < 2:
        if sf in (0, 2): lh, size = 1, b0 >> 3
        elif sf == 1: lh, size = 2, (b0 >> 4) | (blk[1] << 4)
        else: lh, size = 3, (b0 >> 4) | (blk[1] << 4) | (blk[2] << 12)
        info.lit_section = lh + (size if lt == 0 else 1)
        info.lit_streams = 0
    else:
        lh, bits = ((3, 10), (3, 10), (4, 14), (5, 18))[sf]
        v = int.from_bytes(blk[:lh], "little") >> 4
        size, csize = v & ((1 << bits) - 1), (v >> bits) & ((1 << bits) - 1)
        info.lit_section = lh + csize
        info.lit_streams = 1 if sf == 0 else 4
    info.lit_mode, info.lit_size, info.lit_header = lt, size, lh
    p = info.lit_section
    s0 = blk[p]
    if s0 == 0: info.nb_seq, info.nb_seq_bytes = 0, 1
    elif s0 < 128: info.nb_seq, info.nb_seq_bytes = s0, 1
    elif s0 < 255: info.nb_seq, info.nb_seq_bytes = ((s0 - 128) << 8) + blk[p + 1], 2
    else: info.nb_seq, info.nb_seq_bytes = blk[p + 1] + (blk[p + 2] << 8) + 0x7F00, 3
    p += info.nb_seq_bytes
    if info.nb_seq:
        m = blk[p]
        info.modes = (MODES[m >> 6], MODES[(m >> 4) & 3], MODES[(m >> 2) & 3])
        p += 1
    info.seq_header_end = p
    return info


def literal_payload(z: bytes):
    """(first, end) byte range of the compressed-literals payload (Huffman tree description + streams) of a one-block frame, or
    None when the block is not compressed or its literals are raw / rle."""
    info = parse_frame(z)
    if info.block_type != 2 or info.lit_mode < 2:
        return None
    blk = info.header_size + 3
    return blk + info.lit_header, blk + info.lit_section


# ---- sequences
class _Forward:
    def __init__(self, data: bytes, pos: int):
        self.v = int.from_bytes(data[pos:pos + 512], "little"); self.bit = 0

    def peek(self, n): return (self.v >> self.bit) & ((1 << n) - 1)

    def skip(self, n): self.bit += n


def _read_ncount(data: bytes, pos: int, max_sym: int):
    """FSE table description (RFC 8878 4.1.1): (normalized counts, accuracy log, bytes used)."""
    r = _Forward(data, pos)
    log = r.peek(4) + 5; r.skip(4)
    remaining, threshold, nb = (1 << log) + 1, 1 << log, log + 1
    norm = []
    while remaining > 1 and len(norm) <= max_sym:
        mx = (2 * threshold - 1) - remaining
        v = r.peek(nb)
        if (v & (threshold - 1)) < mx:
            count = v & (threshold - 1); r.skip(nb - 1)
        else:
            count = v & (2 * threshold - 1)
            if count >= threshold:
                count -= mx
            r.skip(nb)
        count -= 1
        remaining -= abs(count)
        norm.append(count)
        if count == 0:
            while True:
                rep = r.peek(2); r.skip(2)
                norm.extend([0] * rep)
                if rep != 3:
                    break
        while remaining < threshold:
            nb -= 1; threshold >>= 1
    if remaining != 1 or len(norm) > max_sym + 1:
        raise ValueError("bad FSE table description")
    return norm + [0] * (max_sym + 1 - len(norm)), log, (r.bit + 7) >> 3


def _build_table(norm, log):
    """Decode table: per state (symbol, nbBits, baseline)."""
    size = 1 << log
    syms = [0] * size
    high = size - 1
    for s, c in enumerate(norm):
        if c == -1:
            syms[high] = s; high -= 1
    step, pos = (size >> 1) + (size >> 3) + 3, 0
    for s, c in enumerate(norm):
        for _ in range(max(c, 0)):
            syms[pos] = s
            pos = (pos + step) & (size - 1)
            while pos > high:
                pos = (pos + step) & (size - 1)
    nxt = [1 if c == -1 else c for c in norm]
    table = []
    for u in range(size):
        s = syms[u]; x = nxt[s]; nxt[s] += 1
        nbits = log - (x.bit_length() - 1)
        table.append((s, nbits, (x << nbits) - size))
    return table


class _Backward:
    def __init__(self, data: bytes):
        if not data or data[-1] == 0:
            raise ValueError("sequence bitstream without end mark")
        self.d = data; self.pos = (len(data) - 1) * 8 + data[-1].bit_length() - 1

    def read(self, n):
        if n == 0:
            return 0
        self.pos -= n
        if self.pos < 0:
            raise ValueError("sequence bitstream overrun")
        lo = self.pos >> 3
        return (int.from_bytes(self.d[lo:(self.pos + n + 7) >> 3], "little") >> (self.pos & 7)) & ((1 << n) - 1)


def decode_sequences(z: bytes):
    """Sequences of a one-block compressed frame: list of (litLength, matchLength, offsetValue, mlCode); offsetValue 1..3 are
    repcodes.  Raises ValueError when the stream does not end exactly on its first bit or the sequences do not add up to the
    frame's content size."""
    info = parse_frame(z)
    if info.block_type != 2 or not info.nb_seq:
        return []
    blk = z[info.header_size + 3:info.header_size + 3 + info.block_size]
    p = info.seq_header_end
    tables = []
    for mode, default, dlog, max_sym in zip(info.modes, (LL_DEFAULT, OF_DEFAULT, ML_DEFAULT), (6, 5, 6), (35, 31, 52)):
        if mode == "predefined":
            tables.append((_build_table(default, dlog), dlog))
        elif mode == "rle":
            tables.append(([(blk[p], 0, 0)], 0)); p += 1
        elif mode == "fse":
            norm, log, used = _read_ncount(blk, p, max_sym)
            tables.append((_build_table(norm, log), log)); p += used
        else:
            raise ValueError("repeat mode in a single-block frame")
    (tLL, lLL), (tOF, lOF), (tML, lML) = tables
    bs = _Backward(blk[p:])
    sLL, sOF, sML = bs.read(lLL), bs.read(lOF), bs.read(lML)
    out = []
    for i in range(info.nb_seq):
        llc, ofc, mlc = tLL[sLL][0], tOF[sOF][0], tML[sML][0]
        of = (1 << ofc) + bs.read(ofc)
        ml = ML_BASE[mlc] + bs.read(ML_BITS[mlc])
        ll = LL_BASE[llc] + bs.read(LL_BITS[llc])
        out.append((ll, ml, of, mlc))
        if i + 1 < info.nb_seq:          # state updates: LL, ML, OF
            sLL = tLL[sLL][2] + bs.read(tLL[sLL][1])
            sML = tML[sML][2] + bs.read(tML[sML][1])
            sOF = tOF[sOF][2] + bs.read(tOF[sOF][1])
    if bs.pos != 0:
        raise ValueError("sequence bitstream not consumed exactly")
    if sum(s[0] for s in out) > info.lit_size or info.content_size is not None and info.lit_size + sum(s[1] for s in out) != info.content_size:
        raise ValueError("sequences do not add up to the content size")
    return out


# ---- tags of the decode-only fixtures
EDGE_NBSEQ = (1, 2, 15, 16, 17, 31, 32, 33)       # around the 16-deep walk -> value link and the 32-wide k_order bucket
NEAR_MAX_NBSEQ = 42000          # near FAST_MAXS: the reference writes 42397 sequences for 131070 bytes of random 3-byte tokens
REQUIRED_FEATURES = frozenset(
    [f"nbseq_{n}" for n in EDGE_NBSEQ] + ["nbseq_3byte", "nbseq_near_max", "nbseq_0_huf", "huf_lit_8_63", "huf_lit_255", "huf_lit_256",
                                          "huf_lit_ge_1k", "raw_lit_with_seq", "rle_lit_with_seq", "ml_code_0", "rep_ll0"]
    + [f"{t}_{m}" for t in ("LL", "OF", "ML") for m in ("predefined", "rle", "fse")])


def features(z: bytes) -> list:
    """Sorted tags of a one-block frame, derived from its bytes alone."""
    info = parse_frame(z)
    tags = set()
    if not info.single_segment:
        tags.add("window_desc")
    if info.block_type == 2:
        n = info.nb_seq
        if n in EDGE_NBSEQ: tags.add(f"nbseq_{n}")
        if info.nb_seq_bytes == 3: tags.add("nbseq_3byte")
        if n >= NEAR_MAX_NBSEQ: tags.add("nbseq_near_max")
        if info.lit_mode == 2:
            tags.add(f"huf_{info.lit_streams}stream")
            if n == 0: tags.add("nbseq_0_huf")
            if 8 <= info.lit_size <= 63: tags.add("huf_lit_8_63")
            if info.lit_size in (255, 256): tags.add(f"huf_lit_{info.lit_size}")
            if info.lit_size >= 1024: tags.add("huf_lit_ge_1k")
        if n and info.lit_mode == 0: tags.add("raw_lit_with_seq")
        if n and info.lit_mode == 1: tags.add("rle_lit_with_seq")
        for t, m in zip(("LL", "OF", "ML"), info.modes):
            tags.add(f"{t}_{m}")
        seqs = decode_sequences(z)
        if any(mlc == 0 for _, _, _, mlc in seqs): tags.add("ml_code_0")
        if any(of <= 3 and ll == 0 for ll, _, of, _ in seqs): tags.add("rep_ll0")
    return sorted(tags)
