"""A zstd frame writer written from RFC 8878, test infrastructure only.

It makes no compression decisions: the caller's plan fixes the frame header fields, every block's type, its sequences, the literals'
mode, header width, stream count and Huffman code lengths, the weight description, and each sequence table's mode, accuracy log and
normalization.  So it writes the legal frames that the reference's encoder never writes (wide header fields, window mantissas, 1-stream
Huffman literals past 255 bytes, table log 12, repeat of a predefined or RLE table, an RLE first block, ...), and the decoders can be
tested on them.  The code tables, predefined distributions and the FSE spread come from tests/golden/frame_info.py.

generate(feature, seed) turns a feature name (FEATURES) and a seed into (item, content) pairs.
"""
from __future__ import annotations

import random
from dataclasses import dataclass, field

from tests.golden.frame_info import LL_BASE, LL_BITS, LL_DEFAULT, MAGIC, ML_BASE, ML_BITS, ML_DEFAULT, OF_DEFAULT, _build_table

BLOCK_MAX = 1 << 17
SKIPPABLE = 0x184D2A50


# ---------------------------------------------------------------- bit writers
class ForwardBits:
    """Little-endian bit writer, first field in the lowest bits (FSE table descriptions)."""

    def __init__(self):
        self.v, self.n = 0, 0

    def add(self, value: int, nbits: int):
        assert 0 <= value < 1 << nbits or nbits == 0 and value == 0
        self.v |= value << self.n
        self.n += nbits

    def bytes(self) -> bytes:
        return self.v.to_bytes((self.n + 7) >> 3, "little")


class BackwardBits:
    """Bitstream read from its end (Huffman and sequence streams).  Fields are added in the order the decoder reads them; the last one
    read sits at bit 0, and a 1 bit above the first one read marks the end."""

    def __init__(self):
        self.fields = []

    def add(self, value: int, nbits: int):
        assert 0 <= value < 1 << nbits or nbits == 0 and value == 0
        if nbits:
            self.fields.append((value, nbits))

    def bytes(self) -> bytes:
        v, n = 0, 0
        for value, nbits in reversed(self.fields):
            v |= value << n
            n += nbits
        v |= 1 << n
        return v.to_bytes((n >> 3) + 1, "little")


# ---------------------------------------------------------------- FSE
@dataclass
class Fse:
    """An FSE table built from a normalization: the decode table of frame_info._build_table, and per symbol the state whose range
    holds a given next state (the encoder walks the symbols backwards)."""
    norm: list
    log: int
    table: list = None
    enc: dict = None

    def __post_init__(self):
        if self.table is None:
            self.table = _build_table(self.norm, self.log)
        size = 1 << self.log
        self.enc = {}
        for u, (s, nb, base) in enumerate(self.table):
            arr = self.enc.setdefault(s, [None] * size)
            for t in range(base, base + (1 << nb)):
                arr[t] = u

    def first_state(self, sym: int, want_bits: bool = False) -> int:
        states = [u for u, e in enumerate(self.table) if e[0] == sym]
        if want_bits:
            states = [u for u in states if self.table[u][1]] or states
        return states[0]

    def prev_state(self, sym: int, nxt: int) -> int:
        return self.enc[sym][nxt]

    def bits(self, state: int, nxt: int):
        _, nb, base = self.table[state]
        return nxt - base, nb


def rle_table(sym: int) -> Fse:
    return Fse(norm=None, log=0, table=[(sym, 0, 0)])


def ncount_bytes(norm: list, log: int) -> bytes:
    """FSE table description (RFC 8878 4.1.1) of a normalization that sums to 2^log, -1 counting as one cell."""
    assert sum(abs(c) for c in norm) == 1 << log and any(norm)
    last = max(i for i, c in enumerate(norm) if c)
    w = ForwardBits()
    w.add(log - 5, 4)
    remaining, threshold, nb = (1 << log) + 1, 1 << log, log + 1
    s = 0
    while s <= last:
        c = norm[s] + 1
        mx = 2 * threshold - 1 - remaining
        if c < mx:
            w.add(c, nb - 1)
        elif c < threshold:
            w.add(c, nb)
        else:
            w.add(c + mx, nb)
        remaining -= abs(norm[s])
        s += 1
        if c == 1:
            z = 0
            while s + z <= last and norm[s + z] == 0:
                z += 1
            s += z
            while z >= 3:
                w.add(3, 2); z -= 3
            w.add(z, 2)
        while remaining < threshold:
            nb -= 1; threshold >>= 1
    assert remaining == 1
    return w.bytes()


def normalize(counts: dict, log: int, max_sym: int, low: str = "one") -> list:
    """A normalization of symbol counts at accuracy `log`: every present symbol gets at least one cell; with low="minus1" the symbols
    that would get one cell are written as -1 (less than one); the largest symbol takes what is left."""
    total = sum(counts.values())
    size = 1 << log
    assert len(counts) <= size
    norm = [0] * (max_sym + 1)
    for s, c in counts.items():
        norm[s] = max(1, c * size // total)
    big = max(counts, key=lambda s: (counts[s], -s))
    while sum(norm) > size:
        k = max((s for s in counts if s != big and norm[s] > 1), key=lambda s: norm[s], default=None)
        if norm[big] > 1 and (k is None or norm[big] >= norm[k]):
            norm[big] -= 1
        else:
            norm[k] -= 1
    norm[big] += size - sum(norm)
    if low == "minus1":
        for s in counts:
            if s != big and norm[s] == 1:
                norm[s] = -1
    return norm


# ---------------------------------------------------------------- Huffman
def code_lengths(symbols: list, max_bits: int, rnd: random.Random) -> dict:
    """A Kraft-complete set of code lengths for `symbols` (in order of falling frequency) whose longest code is exactly max_bits:
    a chain to max_bits, then random leaves split until every symbol has one."""
    n = len(symbols)
    assert max_bits + 1 <= n <= 1 << max_bits or n == 2 and max_bits == 1
    lens = [l for l in range(1, max_bits)] + [max_bits, max_bits]
    lens = lens[:n] if n < len(lens) else lens
    while len(lens) < n:
        cand = [i for i, l in enumerate(lens) if l < max_bits]
        i = rnd.choice(cand)
        l = lens.pop(i)
        lens += [l + 1, l + 1]
    lens.sort()
    return dict(zip(symbols, lens))


def canonical_codes(lengths: dict) -> dict:
    """zstd's canonical prefix codes (RFC 8878 4.2.1.3): longest codes first from 0, same length in symbol order."""
    codes, code, prev = {}, 0, None
    for s in sorted(lengths, key=lambda s: (-lengths[s], s)):
        l = lengths[s]
        if prev is not None and l < prev:
            code >>= prev - l
        codes[s] = code
        code += 1
        prev = l
    return codes


def huffman_weights(lengths: dict) -> list:
    max_bits = max(lengths.values())
    last = max(lengths)
    return [max_bits + 1 - lengths[s] if s in lengths else 0 for s in range(last)]


def weights_description(weights: list, how: str, wlog: int = 6, wnorm: list = None) -> bytes:
    """Huffman tree description: direct 4-bit weights, or FSE-compressed with two interleaved states (RFC 8878 4.2.1.2)."""
    if how == "direct":
        assert len(weights) <= 128
        ws = weights + [0] * (len(weights) & 1)
        return bytes([127 + len(weights)]) + bytes((ws[i] << 4) | ws[i + 1] for i in range(0, len(ws), 2))
    n = len(weights)
    assert n >= 2
    counts = {}
    for x in weights:
        counts[x] = counts.get(x, 0) + 1
    norm = wnorm or normalize(counts, wlog, 12)
    f = Fse(norm, wlog)
    x = [0] * n
    x[n - 1] = f.first_state(weights[n - 1])
    x[n - 2] = f.first_state(weights[n - 2], want_bits=True)
    assert f.table[x[n - 2]][1], "the last update of the weight stream must read past its start"
    for i in range(n - 3, -1, -1):
        x[i] = f.prev_state(weights[i], x[i + 2])
    bw = BackwardBits()
    bw.add(x[0], wlog); bw.add(x[1], wlog)
    for i in range(n - 2):
        bw.add(*f.bits(x[i], x[i + 2]))
    body = ncount_bytes(norm[:max(i for i, c in enumerate(norm) if c) + 1], wlog) + bw.bytes()
    assert len(body) < 128
    return bytes([len(body)]) + body


def huffman_stream(data: bytes, codes: dict, lengths: dict) -> bytes:
    bw = BackwardBits()
    for b in data:
        bw.add(codes[b], lengths[b])
    return bw.bytes()


# ---------------------------------------------------------------- plans
@dataclass
class Lit:
    mode: str = "raw"            # raw, rle, huf (fresh tree), treeless (the frame's last tree)
    header: int = 0              # header bytes; 0 = the smallest that holds the sizes
    streams: int = 0             # 1 or 4 (huf / treeless); 0 = 1 below 256 literals, 4 from there
    max_bits: int = 0            # Huffman table log; 0 = the smallest that takes the literal alphabet
    extra_symbols: int = 0       # symbols with a code that the literals do not use
    alphabet: bytes = b""        # ... and these too (so that later treeless literals can use them)
    weights: str = "auto"        # direct, fse, or auto: direct when the highest symbol is at most 128
    wlog: int = 6


@dataclass
class Tab:
    mode: str = "fse"            # predefined, rle, fse, repeat
    log: int = 0                 # fse: accuracy log, 0 = 6 (LL / ML) or 5 (OF)
    low: str = "one"             # fse: "one" or "minus1" (rare symbols as -1 cells)
    norm: list = None            # fse: an explicit normalization (overrides log / low)
    full: bool = False           # fse: a cell for every code of the alphabet, so that later blocks can repeat the table


@dataclass
class Block:
    kind: str = "comp"           # raw, rle, comp
    size: int = 0                # bytes the block regenerates
    seqs: list = None            # comp: [(litLength, matchLength, offset)], offsets as distances, or (litLength, matchLength, offset,
                                 # offsetValue) to write that value whatever it means; None = plan them
    lit: Lit = field(default_factory=Lit)
    tabs: tuple = None           # comp: (LL, OF, ML) Tab; None = three FSE tables
    count_bytes: int = 0         # width of the sequence count; 0 = the shortest
    reps: bool = True            # write repcodes where the history allows
    last: bool = None


@dataclass
class Frame:
    blocks: list
    magic: bool = True
    single: bool = False
    window_log: int = 17
    mantissa: int = 0
    fcs_bytes: int = -1          # -1 = the narrowest field; 0 = none; 1 (single segment only), 2, 4, 8
    did_bytes: int = 0           # dictionary-ID field width (value 0)
    checksum: bool = False

    @property
    def window(self) -> int:
        return (1 << self.window_log) + ((1 << self.window_log) >> 3) * self.mantissa


# ---------------------------------------------------------------- XXH64
_P1, _P2, _P3, _P4, _P5 = 11400714785074694791, 14029467366897019727, 1609587929392839161, 9650029242287828579, 2870177450012600261
_M = (1 << 64) - 1


def _rotl(x, r):
    return ((x << r) | (x >> (64 - r))) & _M


def _round(acc, lane):
    return (_rotl((acc + lane * _P2) & _M, 31) * _P1) & _M


def xxh64(data: bytes, seed: int = 0) -> int:
    n, p = len(data), 0
    if n >= 32:
        v = [(seed + _P1 + _P2) & _M, (seed + _P2) & _M, seed, (seed - _P1) & _M]
        while p + 32 <= n:
            for i in range(4):
                v[i] = _round(v[i], int.from_bytes(data[p + 8 * i:p + 8 * i + 8], "little"))
            p += 32
        h = (_rotl(v[0], 1) + _rotl(v[1], 7) + _rotl(v[2], 12) + _rotl(v[3], 18)) & _M
        for x in v:
            h = ((h ^ _round(0, x)) * _P1 + _P4) & _M
    else:
        h = (seed + _P5) & _M
    h = (h + n) & _M
    while p + 8 <= n:
        h = (_rotl(h ^ _round(0, int.from_bytes(data[p:p + 8], "little")), 27) * _P1 + _P4) & _M; p += 8
    if p + 4 <= n:
        h = (_rotl(h ^ (int.from_bytes(data[p:p + 4], "little") * _P1 & _M), 23) * _P2 + _P3) & _M; p += 4
    while p < n:
        h = (_rotl(h ^ (data[p] * _P5 & _M), 11) * _P1) & _M; p += 1
    h = ((h ^ (h >> 33)) * _P2) & _M
    h = ((h ^ (h >> 29)) * _P3) & _M
    return h ^ (h >> 32)


# ---------------------------------------------------------------- sequences
def _code(v: int, base: list, bits: list) -> int:
    c = max(i for i, b in enumerate(base) if b <= v)
    assert v < base[c] + (1 << bits[c])
    return c


def ll_code(ll: int) -> int:
    return ll if ll < 16 else _code(ll, LL_BASE, LL_BITS)


def ml_code(ml: int) -> int:
    return ml - 3 if ml < 35 else _code(ml, ML_BASE, ML_BITS)


def offset_value(off: int, ll: int, rep: list, use_reps: bool):
    """(offsetValue, new history) for a match at distance `off` (RFC 8878 3.1.2.5)."""
    if use_reps:
        cands = [(1, rep[0]), (2, rep[1]), (3, rep[2])] if ll else [(1, rep[1]), (2, rep[2]), (3, rep[0] - 1)]
        for ov, d in cands:
            if d == off:
                idx = ov - 1 + (ll == 0)
                if idx == 0:
                    return ov, rep
                if idx == 3:
                    return ov, [rep[0] - 1, rep[0], rep[1]]
                return ov, [rep[idx], rep[0], rep[2] if idx == 1 else rep[1]]
    return off + 3, [off, rep[0], rep[1]]


def plan_sequences(buf: bytes, start: int, end: int, frame_start: int, window: int, rnd: random.Random, min_match: int = 4,
                   hash_from: int = None) -> list:
    """Greedy hash matches for buf[start:end] against buf[frame_start:], distances at most `window`.  The last match's distance is
    tried first (a repcode), and a match may overlap its own output (distance below its length)."""
    seqs, pos, lit0 = [], start, start
    table = {}
    h0 = frame_start if hash_from is None else hash_from
    for p in range(max(h0, start - window), start - min_match + 1):
        table[buf[p:p + min_match]] = p
    last_off = None
    while pos + min_match <= end:
        key = buf[pos:pos + min_match]
        cand = table.get(key)
        table[key] = pos
        off = None
        if last_off and pos - last_off >= frame_start and buf[pos - last_off:pos - last_off + min_match] == key:
            off = last_off                                       # a repcode
        elif cand is not None and pos - cand <= window:
            off = pos - cand
        if off is None:
            pos += 1
            continue
        ml = min_match
        while pos + ml < end and buf[pos + ml] == buf[pos + ml - off]:
            ml += 1
        seqs.append((pos - lit0, ml, off))
        last_off = off
        for q in range(pos + 1, min(pos + ml, end - min_match + 1)):
            table[buf[q:q + min_match]] = q
        pos += ml
        lit0 = pos
    return seqs


# ---------------------------------------------------------------- the writer
class FrameWriter:
    def __init__(self):
        self.tables = None            # (LL, OF, ML) Fse of the frame's last block with sequences
        self.huf = None               # (codes, lengths) of the frame's last Huffman tree
        self.rep = [1, 4, 8]

    def literals(self, lits: bytes, L: Lit, rnd: random.Random) -> bytes:
        n = len(lits)
        if L.mode in ("raw", "rle"):
            t = 0 if L.mode == "raw" else 1
            hdr = L.header or (1 if n < 32 else 2 if n < 4096 else 3)
            assert n < (32, 4096, 1 << 20)[hdr - 1]
            h = (t | (n << 3)) if hdr == 1 else (t | (1 << 2) | (n << 4)) if hdr == 2 else (t | (3 << 2) | (n << 4))
            body = lits if t == 0 else lits[:1]
            assert t == 0 or len(set(lits)) == 1 and n
            return h.to_bytes(hdr, "little") + body
        streams = L.streams or (1 if n < 256 else 4)
        if L.mode == "huf":
            syms = sorted(set(lits), key=lambda s: (-lits.count(s), s))
            syms += sorted(set(L.alphabet) - set(syms))
            syms += [s for s in range(256) if s not in syms][:max(0, 2 - len(syms))]     # a tree has at least two symbols
            extra = [s for s in rnd.sample(range(256), 256) if s not in syms][:L.extra_symbols]
            syms += extra
            mb = L.max_bits or max(1, (len(syms) - 1).bit_length())
            lengths = code_lengths(syms, mb, rnd)
            codes = canonical_codes(lengths)
            weights = huffman_weights(lengths)
            how = L.weights if L.weights != "auto" else "direct" if len(weights) <= 128 else "fse"
            tree = weights_description(weights, how, L.wlog)
            self.huf = (codes, lengths)
            t = 2
        else:
            codes, lengths = self.huf
            tree = b""
            t = 3
        if streams == 1:
            payload = huffman_stream(lits, codes, lengths)
        else:
            seg = (n + 3) // 4
            parts = [lits[:seg], lits[seg:2 * seg], lits[2 * seg:3 * seg], lits[3 * seg:]]
            ss = [huffman_stream(p, codes, lengths) for p in parts]
            payload = b"".join(len(s).to_bytes(2, "little") for s in ss[:3]) + b"".join(ss)
        csize = len(tree) + len(payload)
        hdr = L.header or (3 if max(n, csize) < 1024 else 4 if max(n, csize) < 16384 else 5)
        sf = {3: 0 if streams == 1 else 1, 4: 2, 5: 3}[hdr]
        assert streams == 4 or sf == 0
        bits = (10, 10, 14, 18)[sf]
        assert n < 1 << bits and csize < 1 << bits
        h = t | (sf << 2) | (n << 4) | (csize << (4 + bits))
        return h.to_bytes(hdr, "little") + tree + payload

    def sequences(self, seqs: list, B: Block) -> bytes:
        n = len(seqs)
        cb = B.count_bytes or (1 if n < 128 else 2 if n < 0x7F00 else 3)
        if cb == 1:
            out = bytes([n]); assert n < 128
        elif cb == 2:
            assert n < 0x7F00
            out = bytes([128 + (n >> 8), n & 255])
        else:
            assert n >= 0x7F00
            out = bytes([255]) + (n - 0x7F00).to_bytes(2, "little")
        if not n:
            return out
        codes = [[ll_code(ll) for ll, _, _ in seqs], [ov.bit_length() - 1 for _, _, ov in seqs], [ml_code(ml) for _, ml, _ in seqs]]
        tabs = B.tabs or (Tab(), Tab(), Tab())
        modes, descs, fses = 0, b"", []
        for k, (T, default, dlog, max_sym) in enumerate(zip(tabs, (LL_DEFAULT, OF_DEFAULT, ML_DEFAULT), (6, 5, 6), (35, 31, 52))):
            mode = ("predefined", "rle", "fse", "repeat").index(T.mode)
            modes |= mode << (6 - 2 * k)
            if T.mode == "predefined":
                fses.append(Fse(default, dlog))
            elif T.mode == "rle":
                assert len(set(codes[k])) == 1
                descs += bytes([codes[k][0]]); fses.append(rle_table(codes[k][0]))
            elif T.mode == "fse":
                if T.norm:
                    norm = T.norm
                    log = sum(abs(c) for c in norm).bit_length() - 1
                else:
                    counts = {}
                    for c in codes[k]:
                        counts[c] = counts.get(c, 0) + 1
                    if T.full:
                        counts = {c: counts.get(c, 0) + 1 for c in range(max_sym + 1)}
                    log = T.log or (5 if k == 1 else 6)
                    norm = normalize(counts, log, max_sym, T.low)
                descs += ncount_bytes(norm[:max(i for i, c in enumerate(norm) if c) + 1], log)
                fses.append(Fse(norm + [0] * (max_sym + 1 - len(norm)), log))
            else:
                fses.append(self.tables[k])
        self.tables = tuple(fses)
        fLL, fOF, fML = fses
        st = [[0] * n for _ in range(3)]
        for k, f in ((0, fLL), (1, fOF), (2, fML)):
            st[k][n - 1] = f.first_state(codes[k][n - 1])
            for i in range(n - 2, -1, -1):
                st[k][i] = f.prev_state(codes[k][i], st[k][i + 1])
        bw = BackwardBits()
        bw.add(st[0][0], fLL.log); bw.add(st[1][0], fOF.log); bw.add(st[2][0], fML.log)
        for i, (ll, ml, ov) in enumerate(seqs):
            llc, ofc, mlc = codes[0][i], codes[1][i], codes[2][i]
            bw.add(ov - (1 << ofc), ofc)
            bw.add(ml - ML_BASE[mlc], ML_BITS[mlc])
            bw.add(ll - LL_BASE[llc], LL_BITS[llc])
            if i + 1 < n:
                bw.add(*fLL.bits(st[0][i], st[0][i + 1]))
                bw.add(*fML.bits(st[2][i], st[2][i + 1]))
                bw.add(*fOF.bits(st[1][i], st[1][i + 1]))
        return out + bytes([modes]) + descs + bw.bytes()

    def block(self, content: bytes, at: int, B: Block, frame_start: int, window: int, rnd: random.Random) -> bytes:
        data = content[at:at + B.size]
        if B.kind == "raw":
            return data, 0
        if B.kind == "rle":
            assert len(set(data)) <= 1
            return data[:1] or b"\0", 1
        seqs = B.seqs if B.seqs is not None else plan_sequences(content, at, at + B.size, frame_start, window, rnd)
        lits, p, ovs = bytearray(), at, []
        for ll, ml, off, *forced in seqs:
            lits += content[p:p + ll]
            p += ll
            ov, self.rep = offset_value(off, ll, self.rep, B.reps)
            if forced:
                ov = forced[0]
            else:
                assert off <= p - frame_start and all(content[p + i] == content[p + i - off] for i in range(ml)), "bad match"
            ovs.append((ll, ml, ov))
            p += ml
        lits += content[p:at + B.size]
        return self.literals(bytes(lits), B.lit, rnd) + self.sequences(ovs, B), 2

    def frame(self, content: bytes, F: Frame, rnd: random.Random, at: int = 0) -> bytes:
        """The frame of content[at:at + sum of block sizes]; earlier bytes of `content` are not part of it."""
        self.tables, self.huf, self.rep = None, None, [1, 4, 8]
        size = sum(b.size for b in F.blocks)
        fcs = F.fcs_bytes
        if fcs == -1:
            fcs = 1 if size < 256 else 2 if size < 65536 + 256 else 4 if size < 1 << 32 else 8
            fcs = 4 if fcs == 1 and not F.single else fcs
        flag = {0: 0, 1: 0, 2: 1, 4: 2, 8: 3}[fcs]
        assert not (fcs == 1 and not F.single) and not (fcs == 0 and F.single)
        did = {0: 0, 1: 1, 2: 2, 4: 3}[F.did_bytes]
        out = bytearray(MAGIC.to_bytes(4, "little") if F.magic else b"")
        out.append((flag << 6) | (F.single << 5) | (F.checksum << 2) | did)
        if not F.single:
            out.append(((F.window_log - 10) << 3) | F.mantissa)
        out += bytes(F.did_bytes)
        if fcs:
            out += (size - 256 if fcs == 2 else size).to_bytes(fcs, "little")
        window = size if F.single else F.window
        bmax = min(window, BLOCK_MAX)
        p = at
        for k, B in enumerate(F.blocks):
            body, t = self.block(content, p, B, at, window, rnd)
            last = B.last if B.last is not None else k == len(F.blocks) - 1
            bs = B.size if t == 1 else len(body)
            assert B.size <= bmax
            out += ((bs << 3) | (t << 1) | last).to_bytes(3, "little") + body
            p += B.size
        if F.checksum:
            out += (xxh64(content[at:p]) & 0xFFFFFFFF).to_bytes(4, "little")
        return bytes(out)


def skippable(n: int, low: int = 0) -> bytes:
    return (SKIPPABLE + low).to_bytes(4, "little") + n.to_bytes(4, "little") + bytes((i * 29 + low) & 0xFF for i in range(n))


# ---------------------------------------------------------------- the generator
TEXT = b"abcdefgh ijklmno"


def text(rnd: random.Random, n: int, alphabet: bytes = TEXT, words: int = 60) -> bytes:
    """Word soup over `alphabet`: repeats for the matcher, skewed bytes for Huffman."""
    ws = [bytes(rnd.choice(alphabet) for _ in range(rnd.randrange(2, 9))) for _ in range(words)]
    out = bytearray()
    while len(out) < n:
        out += rnd.choice(ws[:rnd.randrange(1, words)])
    return bytes(out[:n])


def _write(content: bytes, F: Frame, rnd: random.Random) -> bytes:
    return FrameWriter().frame(content, F, rnd)


def _window_mantissa(rnd):
    out = []
    for wl, m in ((10, 1), (11, 7), (12, 3), (14, 5), (16, 2), (16, 7)):
        F = Frame([], window_log=wl, mantissa=m, checksum=m & 1 == 1)
        w = F.window
        sizes = [w, w, w // 3 + 1, rnd.randrange(1, w)]
        content = text(rnd, sum(sizes))
        F.blocks = [Block(size=s, lit=Lit("huf", alphabet=TEXT)) for s in sizes]
        F.blocks[2] = Block("raw", sizes[2])
        out.append((_write(content, F, rnd), content))
    return out


def _wide_header(rnd):
    out = []
    for k, (single, fcs, did) in enumerate(((True, 8, 1), (True, 4, 0), (False, 8, 2), (False, 4, 4), (True, 2, 4), (False, 2, 1))):
        n = 300 + 157 * k
        content = text(rnd, n)
        out.append((_write(content, Frame([Block(size=n, lit=Lit("huf"))], single=single, fcs_bytes=fcs, did_bytes=did, checksum=k == 2), rnd),
                    content))
    return out


def _lit_header_wide(rnd):
    out = []
    for k, (mode, hdr, n) in enumerate((("raw", 2, 5), ("raw", 3, 20), ("rle", 2, 7), ("rle", 3, 31), ("raw", 3, 1000),
                                        ("huf", 4, 40), ("huf", 5, 300), ("huf", 4, 900), ("huf", 5, 6))):
        content = text(rnd, n) if mode != "rle" else bytes([97 + k]) * n
        out.append((_write(content, Frame([Block(size=n, seqs=[], lit=Lit(mode, header=hdr, streams=4 if mode == "huf" else 0))], window_log=10),
                           rnd), content))
    return out


def _huf_streams(rnd, streams, sizes):
    out = []
    for n in sizes:
        content = text(rnd, n)
        out.append((_write(content, Frame([Block(size=n, seqs=[], lit=Lit("huf", streams=streams))], window_log=10 + (n & 1)), rnd), content))
    return out


def _huf_logs(rnd):
    out = []
    for L in range(1, 13):
        nsym = rnd.randrange(L + 1, min(256, 1 << L) + 1)
        direct = nsym <= 129 and (L % 2 or nsym <= 20)
        alpha = bytes(rnd.sample(range(129 if direct else 256), nsym))
        n = rnd.randrange(200, 3000)
        content = bytes(rnd.choice(alpha) for _ in range(n))
        lit = Lit("huf", max_bits=L, alphabet=alpha, weights="direct" if direct else "fse")
        out.append((_write(content, Frame([Block(size=n, seqs=[], lit=lit)], window_log=12), rnd), content))
    return out


def _huf_alphabets(rnd):
    out = []
    for nsym in (2, 3, 127, 128, 255, 256):
        for how in ("direct", "fse"):
            if how == "direct" and nsym > 129 or how == "fse" and nsym < 20:
                continue
            alpha = bytes(rnd.sample(range(129 if how == "direct" else 256), nsym))
            n = rnd.randrange(nsym, 4 * nsym + 300)
            content = bytes(rnd.choice(alpha) for _ in range(n))
            lit = Lit("huf", alphabet=alpha, weights=how, max_bits=max(1, (nsym - 1).bit_length()) + (nsym > 3))
            out.append((_write(content, Frame([Block(size=n, seqs=[], lit=lit)], window_log=12, checksum=nsym & 1 == 1), rnd), content))
    return out


def _expand(rnd):
    out = []
    content = bytes(rnd.randrange(256) for _ in range(700))       # literals Huffman makes larger
    out.append((_write(content, Frame([Block(size=700, seqs=[], lit=Lit("huf", max_bits=9))], window_log=10), rnd), content))
    content = bytes(rnd.randrange(256) for _ in range(40))        # a block larger than its content
    out.append((_write(content, Frame([Block(size=40, seqs=[], lit=Lit("huf", max_bits=11, header=5, streams=4))], window_log=10), rnd), content))
    content = text(rnd, 3000)
    F = Frame([Block(size=1000, lit=Lit("huf")), Block(size=0, seqs=[], lit=Lit("raw")), Block(size=2000, lit=Lit("treeless")),
               Block(size=0, seqs=[], lit=Lit("raw", header=3), count_bytes=2)], window_log=12)
    out.append((_write(content, F, rnd), content))                 # compressed blocks that regenerate nothing, the last one too
    return out


def _fse_bounds(rnd):
    out = []
    for k, (ll, of, ml, low) in enumerate(((5, 5, 5, "one"), (9, 8, 9, "one"), (9, 5, 5, "minus1"), (5, 8, 9, "minus1"), (6, 6, 7, "minus1"))):
        content = text(rnd, 20000 + 999 * k)
        F = Frame([Block(size=len(content), lit=Lit("huf"), tabs=(Tab("fse", ll, low), Tab("fse", of, low), Tab("fse", ml, low)))],
                  window_log=15)
        out.append((_write(content, F, rnd), content))
    # only -1 cells beside one large cell, and zero runs that need chained repeat flags
    for log in (5, 6, 9):
        content = text(rnd, 9000)
        seqs = plan_sequences(content, 0, len(content), 0, 1 << 15, rnd)
        llc = sorted({ll_code(s[0]) for s in seqs})
        mlc = sorted({ml_code(s[1]) for s in seqs})
        def lone(codes, lg, width):
            norm = [0] * (width + 1)
            for c in codes:
                norm[c] = -1
            norm[codes[0]] = (1 << lg) - (len(codes) - 1)
            return norm
        norm_ml = [0] * 53
        for c in mlc:
            norm_ml[c] = -1
        norm_ml[52] = -1                                           # a long zero run before the last symbol
        norm_ml[mlc[-1]] = (1 << log) - len(mlc)
        F = Frame([Block(size=len(content), seqs=seqs, lit=Lit("huf"), tabs=(Tab("fse", norm=lone(llc, log, 35)), Tab("fse", 5),
                                                                                   Tab("fse", norm=norm_ml)))], window_log=15)
        out.append((_write(content, F, rnd), content))
    return out


def _rle_max_codes(rnd):
    out = []
    base = text(rnd, 70000)
    # LL code 35 for every sequence, ML code 52 for every sequence, OF codes of the window's order
    c1 = base[:65600] + base[100:2100]
    c2 = b"abc" + b"c" * 70000
    c3 = base[:20000] + bytes(rnd.randrange(256) for _ in range(300000)) + base[:20000]
    cases = [
        (c1, [Block(size=len(c1), seqs=[(65600, 2000, 65500)], lit=Lit("huf"), tabs=(Tab("rle"), Tab("rle"), Tab("rle")))], 17),
        (c2, [Block(size=len(c2), seqs=[(3, len(c2) - 3, 1)],
                    lit=Lit("raw"), tabs=(Tab("rle"), Tab("rle"), Tab("rle")))], 17),
        (c3, [Block("raw", 131072), Block("raw", 131072), Block("raw", len(c3) - 262144 - 20000),
              Block(size=20000, seqs=[(0, 20000, 320000)], lit=Lit("raw"), tabs=(Tab("rle"), Tab("rle"), Tab("rle")))], 19),
    ]
    for content, blocks, wl in cases:
        out.append((_write(content, Frame(blocks, window_log=wl), rnd), content))
    return out


def _cross_block(rnd):
    """Repeated tables two and more blocks after they were set, with raw, RLE and sequence-free blocks between; repeats of predefined
    and RLE tables; treeless literals after raw / RLE literals; repcodes carried over sequence-free blocks."""
    out = []
    for k in range(6):
        n = 4000 + 1000 * k
        chunk = text(rnd, n)
        mode = ("fse", "predefined", "fse", "predefined", "fse", "fse")[k]
        first = (Tab(mode, 6 + k % 3, full=True), Tab(mode, full=True), Tab(mode, full=True)) if mode == "fse" else (Tab(mode),) * 3
        rep = (Tab("repeat"),) * 3
        blocks, parts = [], []
        def add(b, data):
            blocks.append(b); parts.append(data)
        add(Block(size=n, lit=Lit("huf", alphabet=TEXT), tabs=first), chunk)
        if k % 2:
            add(Block("raw", 500), text(rnd, 500))
        add(Block("rle", 300 + k), b"x" * (300 + k))
        add(Block(size=600, seqs=[], lit=Lit(("raw", "rle", "treeless")[k % 3])), b"y" * 600 if k % 3 == 1 else text(rnd, 600))
        add(Block(size=n, lit=Lit("treeless" if k % 2 else "raw"), tabs=rep), chunk)
        add(Block(size=200, seqs=[], lit=Lit("rle")), b"z" * 200)
        add(Block(size=n, lit=Lit("huf", alphabet=TEXT), tabs=(Tab("repeat"), Tab("fse", 5, full=True), Tab("repeat"))), chunk[::-1])
        add(Block(size=n, lit=Lit("treeless"), tabs=rep), chunk)
        content = b"".join(parts)
        out.append((_write(content, Frame(blocks, window_log=17, checksum=k == 3), rnd), content))
    # repcodes carried over a raw block and a sequence-free compressed block
    for k in range(2):
        unit = text(rnd, 8 + k)
        d = len(unit)
        content = bytearray(unit * 21 + text(rnd, 50) + text(rnd, 30) + text(rnd, 5))
        for _ in range(40 + k):
            content.append(content[-d])
        content = bytes(content)
        blocks = [Block(size=21 * d, seqs=[(d, 20 * d, d)], lit=Lit("huf")), Block("raw", 50), Block(size=30, seqs=[], lit=Lit("raw")),
                  Block(size=45 + k, seqs=[(5, 40 + k, d)], lit=Lit("raw"), tabs=(Tab("predefined"),) * 3)]
        out.append((_write(content, Frame(blocks, window_log=12), rnd), content))
    # a repeat of an RLE table two blocks later: every sequence of both blocks has the same codes
    unit = text(rnd, 8)
    content = bytearray(unit * 201 + b"q" * 100 + b"L")
    for _ in range(1199):
        content.append(content[-8])
    content = bytes(content)
    b0 = Block(size=1608, seqs=[(8, 1600, 8)], lit=Lit("raw"), tabs=(Tab("rle"),) * 3, reps=False)
    b2 = Block(size=1200, seqs=[(1, 1199, 8)], lit=Lit("raw"), tabs=(Tab("rle"), Tab("repeat"), Tab("repeat")), reps=False)
    out.append((_write(content, Frame([b0, Block("rle", 100), b2], window_log=14), rnd), content))
    return out


def _nbseq_long(rnd):
    out = []
    for k in range(3):
        content = text(rnd, 500 + 200 * k)
        seqs = plan_sequences(content, 0, len(content), 0, 1 << 12, rnd)[:120]
        content = content[:sum(s[0] + s[1] for s in seqs) + 7]
        out.append((_write(content, Frame([Block(size=len(content), seqs=seqs, lit=Lit("huf"), count_bytes=2)], window_log=12), rnd), content))
    content = text(rnd, 200)
    out.append((_write(content, Frame([Block(size=200, seqs=[], lit=Lit("huf"), count_bytes=2)], single=True), rnd), content))
    return out


def _rle_first(rnd):
    out = []
    for k in range(3):
        head = bytes([rnd.randrange(256)]) * (1000 + 3000 * k)
        tail = text(rnd, 5000)
        content = head + tail
        F = Frame([Block("rle", len(head)), Block(size=len(tail), lit=Lit("huf"))], window_log=13 + k, checksum=k == 1)
        out.append((_write(content, F, rnd), content))
    return out


def _max_seqs(rnd):
    """The most sequences a 128 KB block holds: 2 literals, then 43 690 matches of 3 bytes."""
    content = (b"ab" * 65536)
    seqs = [(2, 3, 2)] + [(0, 3, 2)] * 43689
    F = Frame([Block(size=131072, seqs=seqs, lit=Lit("raw"), tabs=(Tab("predefined"), Tab("rle"), Tab("fse", 5)), reps=False)], window_log=17)
    return [(_write(content, F, rnd), content)]


def _max_extra(rnd):
    """Literal length code 35 and match length code 52 with the largest extra values a 128 KB block leaves room for."""
    lits = text(rnd, 131069)
    c1 = lits + lits[:3]
    c2 = b"Q" * 131072
    return [(_write(c1, Frame([Block(size=131072, seqs=[(131069, 3, 131069)], lit=Lit("huf"))], window_log=17), rnd), c1),
            (_write(c2, Frame([Block(size=131072, seqs=[(1, 131071, 1)], lit=Lit("raw"))], window_log=17), rnd), c2)]


def _window_offsets(rnd):
    out = []
    for wl, m in ((10, 0), (12, 5), (16, 1), (17, 0)):
        F = Frame([], window_log=wl, mantissa=m)
        w = F.window
        head = text(rnd, w, alphabet=bytes(range(32, 127)), words=400)
        body = head[:64] + text(rnd, 300)
        content = head + body
        bmax = min(w, BLOCK_MAX)
        blocks, pos = [], 0
        while pos < w:
            s = min(bmax, w - pos)
            blocks.append(Block(size=s, lit=Lit("huf", alphabet=bytes(range(32, 127)))))
            pos += s
        seqs = [(0, 64, w)] + plan_sequences(content, w + 64, len(content), 0, w, rnd)
        blocks.append(Block(size=len(body), seqs=seqs, lit=Lit("huf", alphabet=bytes(range(32, 127)))))
        F.blocks = blocks
        out.append((_write(content, F, rnd), content))
    # offsets that reach the frame's first byte, in a later frame of the item (history must not reach the earlier frame)
    a = text(rnd, 3000)
    b = text(rnd, 2000)
    c2 = b[:100] * 11 + b[:100] * 11
    seqs2 = [(100, 1000, 100), (0, 1100, 1100)]
    z1 = _write(a, Frame([Block(size=len(a), lit=Lit("huf"))], window_log=12), rnd)
    z2 = _write(c2, Frame([Block(size=len(c2), seqs=seqs2, lit=Lit("raw"))], window_log=12), rnd)
    out.append((z1 + z2, a + c2))
    return out


def _big_window(rnd):
    out = []
    for m in (0, 1, 0, 1):
        content = text(rnd, 400_000 + 50_000 * m)
        sizes = [131072, 131072, 131072, len(content) - 3 * 131072]
        F = Frame([Block(size=s, lit=Lit("huf")) for s in sizes], window_log=27, mantissa=m, checksum=len(out) >= 2)
        out.append((_write(content, F, rnd), content))
    return out


def _multi_frame(rnd):
    """Items of several generated frames with skippable frames of all 16 magic values between them; every frame after the first opens
    with repcode matches (history {1, 4, 8} again at each frame)."""
    out = []
    for k in range(4):
        parts, content = [], b""
        for j in range(3 + k):
            pre = text(rnd, 16)
            body = pre + pre[-8:] + pre[-4:] + pre[-1:] * 5 + text(rnd, 1500 + 300 * j)
            seqs = [(16, 8, 8), (0, 4, 4), (0, 5, 1)] + plan_sequences(body, 33, len(body), 0, 4096, rnd)
            F = Frame([Block(size=len(body), seqs=seqs, lit=Lit("huf")), Block("raw", 0)][: 1 + (j % 2)], window_log=12,
                      checksum=j % 3 == 2, single=j % 4 == 3)
            parts.append(_write(body, F, rnd))
            content += body
            low = (4 * k + j) % 16
            parts.append(skippable((0, 1, 37)[(k + j) % 3], low))
        if k == 3:
            parts += [skippable(n, low) for low, n in zip(range(16), [0, 5] * 8)]
        out.append((b"".join(parts), content))
    return out


def _plain(rnd):
    """Single-block frames of ordinary shape (4 streams, FSE tables), a backdrop for the batch tests."""
    out = []
    for k in range(4):
        content = text(rnd, rnd.randrange(500, 60000))
        out.append((_write(content, Frame([Block(size=len(content), lit=Lit("huf"))], single=k % 2 == 0, window_log=16), rnd), content))
    return out


FEATURES = {
    "window_mantissa": _window_mantissa,
    "wide_header": _wide_header,
    "lit_header_wide": _lit_header_wide,
    "huf_1stream_large": lambda rnd: _huf_streams(rnd, 1, (256, 300, 511, 777, 1023)),
    "huf_4stream_small": lambda rnd: _huf_streams(rnd, 4, (6, 7, 9, 10, 33, 100, 254, 255)),
    "huf_logs": _huf_logs,
    "huf_alphabets": _huf_alphabets,
    "expand": _expand,
    "fse_bounds": _fse_bounds,
    "rle_max_codes": _rle_max_codes,
    "cross_block": _cross_block,
    "nbseq_long": _nbseq_long,
    "rle_first": _rle_first,
    "max_seqs": _max_seqs,
    "max_extra": _max_extra,
    "window_offsets": _window_offsets,
    "big_window": _big_window,
    "multi_frame": _multi_frame,
    "plain": _plain,
}


def generate(feature: str, seed: int = 0) -> list:
    """[(item, content)] of one feature of FEATURES, deterministic in the seed."""
    return FEATURES[feature](random.Random(f"{feature}/{seed}"))
