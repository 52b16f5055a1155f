"""Inputs that land on each side of the encoder's entropy-stage decisions (test infrastructure only).

Every family is a generator gen(k, seed) -> bytes in which the integer k moves one statistic -- a literal count, a sequence
count, the count of the most frequent symbol -- across one threshold of the entropy stage (zb_encode.cuh: compress_literals,
the huf_* functions, select_encoding*, fse_normalize*, entropy_compress and the raw-block fallback of encode_stage).  side()
reads which way a frame went from its bytes alone (tests/frame_reader.py): literal type, Huffman stream count, literal header
width, sequence-count width, table modes, -1 cells in the normalised counts, weight format, block type.  find_boundary() asks
the compiled reference for the k at which its frame switches sides.

The generators control the parse by planting exact copies of earlier random spans into random bytes: a copy of length m at
distance d is one sequence with match length m and offset d, because the bytes just before and just after it are chosen to differ
from the bytes around its source, so the match can be neither extended nor found longer elsewhere.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Callable

import numpy as np

from tests import frame_reader
from tests.golden import frame_info

S_FAST, S_DFAST, S_GREEDY, S_LAZY, S_LAZY2, S_BTLAZY2, S_BTOPT, S_BTULTRA, S_BTULTRA2 = range(1, 10)


class Planter:
    """Random literals with planted exact copies of earlier spans."""

    def __init__(self, seed: int):
        self.rng = np.random.default_rng(seed)
        self.buf = bytearray()
        self.avoid = None          # the byte the next literal must not be (it would extend the last copy)

    def lits(self, data) -> "Planter":
        data = bytearray(data)
        if data and self.avoid is not None and data[0] == self.avoid:
            data[0] = (data[0] + 1) & 0xFF
        self.avoid = None
        self.buf += data
        return self

    def rand(self, n: int, alphabet: int = 256, base: int = 0) -> "Planter":
        return self.lits((self.rng.integers(0, alphabet, n) + base).astype(np.uint8).tobytes())

    def copy(self, dist: int, length: int) -> "Planter":
        start = len(self.buf) - dist
        assert 0 < dist <= len(self.buf) and length > 0
        if start > 0 and self.buf[-1] == self.buf[start - 1]:
            self.buf[-1] = (self.buf[-1] + 1) & 0xFF       # a literal before the copy: keep the match from growing backwards
        for i in range(length):
            self.buf.append(self.buf[start + i])
        self.avoid = self.buf[start + length] if start + length < len(self.buf) - length else None
        return self

    def bytes(self) -> bytes:
        return bytes(self.buf)


def de_bruijn(k: int, n: int) -> list:
    """The de Bruijn sequence of order n over 0 .. k-1: every n-symbol string once (so no prefix repeats one)."""
    a, seq = [0] * k * n, []

    def db(t, p):
        if t > n:
            if n % p == 0:
                seq.extend(a[1:p + 1])
        else:
            a[t] = a[t - p]
            db(t + 1, p)
            for j in range(a[t - p] + 1, k):
                a[t] = j
                db(t + 1, t)
    db(1, 1)
    return seq


def with_counts(rng, counts: dict) -> bytes:
    """The symbols of `counts` ({byte: occurrences}) in a random order."""
    a = np.concatenate([np.full(c, s, dtype=np.uint8) for s, c in counts.items() if c])
    return rng.permutation(a).tobytes()


# ------------------------------------------------------------------------------------------------ generators
def repeated_literals(lits: bytes, times: int = 4) -> bytes:
    """`lits` followed by times-1 copies of itself: the literals of the frame are `lits`, behind one long match."""
    return lits * times


def lit_run(k: int, seed: int, alphabet: int = 128) -> bytes:
    """k literals drawn uniformly from `alphabet` values (k - 1 of them a prefix of the k-literal run), behind one long match."""
    rng = np.random.default_rng(seed)
    return repeated_literals(rng.integers(0, alphabet, 1 << 17).astype(np.uint8)[:k].tobytes())


def skewed_run(k: int, seed: int) -> bytes:
    """k literals of a skewed 32-symbol distribution, behind one long match."""
    rng = np.random.default_rng(seed)
    p = 0.8 ** np.arange(32); p /= p.sum()
    return repeated_literals(rng.choice(np.arange(32, dtype=np.uint8), 1 << 17, p=p)[:k].tobytes())


def sample_size(k: int, seed: int) -> bytes:
    """Literals only: 4096 random bytes, k - 8192 bytes of a 128-value alphabet, 4096 random bytes.  From 40960 literals the encoder
    looks at the two random ends first and stores the literals raw; below it the 7-bit middle makes Huffman coding pay."""
    rng = np.random.default_rng(seed)
    return (rng.integers(0, 256, 4096).astype(np.uint8).tobytes() + rng.integers(0, 128, 1 << 17).astype(np.uint8)[:k - 8192].tobytes()
            + rng.integers(0, 256, 4096).astype(np.uint8).tobytes())


def sample_ratio(k: int, seed: int) -> bytes:
    """4096 random literals, k sequences of 18 literals of a 128-value alphabet and one planted 8-byte copy, 4096 random literals.
    The random ends are looked at (and make the literals raw) only while litSize / nbSeq >= 20, i.e. up to k = 4096."""
    p = Planter(seed)
    p.rand(4096).copy(4096, 600)          # a long first match, so the parser's step is back to 1 for the short copies
    for _ in range(k):
        p.rand(18, 128)
        p.copy(int(p.rng.integers(8, 19)), 8)
    p.rand(4096)
    return p.bytes()


def sample_total(k: int, seed: int) -> bytes:
    """Literals only: two 4096-byte ends whose most frequent bytes occur 34 and k - 34 times (every other byte at most 16 times)
    around 40000 bytes of a 128-value alphabet.  largestTotal = k: at most 68 stores the literals raw."""
    rng = np.random.default_rng(seed)

    def end(top):
        counts = {s: 16 for s in range(256)}
        counts[0] = top
        extra = sum(counts.values()) - 4096
        for s in range(1, 256):
            d = min(extra, 16)
            counts[s] -= d; extra -= d
        return with_counts(rng, counts)
    return end(34) + rng.integers(0, 128, 40000).astype(np.uint8).tobytes() + end(k - 34)


def rle_literals(k: int, seed: int) -> bytes:
    """Eight equal bytes (too short for any match of the optimal parser: all eight are literals), then k - 1 other bytes."""
    return b"Z" * 8 + b"Y" * max(0, k - 1)


def largest_count(k: int, seed: int) -> bytes:
    """200 literals: byte 0 k times, the rest spread over 40 other values at most 5 times each, behind one long match.  Literals
    whose most frequent byte occurs at most (200 >> 7) + 4 = 5 times are stored raw."""
    rng = np.random.default_rng(seed)
    counts = {0: k}
    left = 200 - k
    for s in range(1, 41):
        counts[s + 60] = min(5, max(left, 0))
        left -= counts[s + 60]
    return repeated_literals(with_counts(rng, counts))


def mixed_run(k: int, seed: int, n: int = 2000) -> bytes:
    """n literals, the first k of them random bytes and the rest of a 128-value alphabet, behind one long match: the larger k, the
    less Huffman coding saves."""
    rng = np.random.default_rng(seed)
    a = rng.integers(0, 128, n).astype(np.uint8)
    a[:k] = rng.integers(0, 256, k).astype(np.uint8)
    return repeated_literals(a.tobytes())


def mixed_literals_only(k: int, seed: int, n: int = 3000) -> bytes:
    """As mixed_run, without the match: the whole block is the literals section, so the block's own gain test decides."""
    rng = np.random.default_rng(seed)
    a = rng.integers(0, 128, n).astype(np.uint8)
    a[:k] = rng.integers(0, 256, k).astype(np.uint8)
    return a.tobytes()


def sequences(k: int, seed: int, pick) -> bytes:
    """k sequences, each a run of literals of a 128-value alphabet and one copy from inside that run: pick(i, rng) gives sequence
    i's (literal run, offset, match length) with offset <= run.  Every source position lies less than 256 bytes behind the last match,
    where the fast parsers still look at every position, so each copy is found as planted.  Offsets that equal one of the last
    three are moved to the nearest other one, so no copy turns into a repeat code."""
    p = Planter(seed)
    recent = [1, 4, 8]
    for i in range(k):
        r, off, ml = pick(i, p.rng)
        if off in recent:
            off = min((o for o in range(ml, r + 1) if o not in recent), key=lambda o: abs(o - off))
        recent = [off] + recent[:2]
        p.rand(r, 128)
        p.copy(off, ml)
    p.rand(16, 128)
    return p.bytes()


def copies(k: int, seed: int) -> bytes:
    """k sequences of 70 literals and an 8-byte copy at distance 29..60."""
    return sequences(k, seed, lambda i, rng: (70, int(rng.integers(29, 61)), 8))


def code_pairs(table: int, k: int, seed: int) -> bytes:
    """k sequences whose codes are constant in two of the three tables and alternate between two values in `table` (0 LL, 1 OF,
    2 ML): LL codes 25 / 23 (70 / 40 literals), OF codes 5 / 6 (distance 29..60 / 61..70), ML codes 5 / 37 (8 / 40 bytes)."""
    def pick(i, rng):
        alt = i % 2
        r = 40 if table == 0 and alt else 70
        off = int(rng.integers(61, 71)) if table == 1 and alt else int(rng.integers(40 if table == 2 else 29, 41 if table == 0 and alt else 61))
        ml = 40 if table == 2 and alt else 8
        return r, off, ml
    return sequences(k, seed, pick)


def same_codes(k: int, seed: int) -> bytes:
    """k sequences with the same LL, OF and ML codes (100..127 literals, distance 61..100, 20 bytes): predefined tables up to
    nbSeq 2, RLE tables from 3."""
    return sequences(k, seed, lambda i, rng: (int(rng.integers(100, 128)), int(rng.integers(61, 101)), 20))


def low_prob(k: int, seed: int, last_common: bool = True) -> bytes:
    """k sequences of 16 literals and an 8-byte copy (ML code 5) but for eight rare ones of 9..11 bytes (codes 6..8, each at most
    three times, below total >> tableLog): their normalised counts are -1 only from nbSeq_1 = 2048.  With last_common the last
    sequence's code is the common one, whose count the encoder lowers by one before normalising (nbSeq_1 = nbSeq - 1); otherwise
    it is a 12-byte copy (code 9) of its own."""
    rare = set(range(100, 100 + 8 * 211, 211))

    def pick(i, rng):
        ml = 9 + i % 3 if i in rare else 8
        if i == k - 1 and not last_common:
            ml = 12
        return 16, int(rng.integers(ml, 17)), ml
    return sequences(k, seed, pick)


def fibonacci_literals(k: int, seed: int, scale: float = 1.0, times: int = 1) -> bytes:
    """Literals whose counts follow the Fibonacci numbers fib(1) .. fib(k) (times `scale`, at least 1), in a random order: their
    Huffman tree is k - 1 deep, deeper than the table log, so huf_set_max_height has to cut it down."""
    rng = np.random.default_rng(seed)
    f = [1, 1]
    while len(f) < k:
        f.append(f[-1] + f[-2])
    counts = {40 + 3 * i: max(1, int(c * scale)) for i, c in enumerate(f[:k])}
    return repeated_literals(with_counts(rng, counts), times)


def perturbed_fibonacci(k: int, seed: int) -> bytes:
    """Fibonacci counts fib(1) .. fib(k) times 0.3, each scaled by a random factor in 0.6 .. 1.6, and up to 29 byte values 1 .. 3
    times: trees whose cut leaves no symbol one level above the target, the rankLast[1] == noSymbol repair of huf_set_max_height."""
    rng = np.random.default_rng(seed)
    f = [1, 1]
    while len(f) < k:
        f.append(f[-1] + f[-2])
    counts = {40 + 3 * i: max(1, int(c * 0.3 * rng.uniform(0.6, 1.6))) for i, c in enumerate(f)}
    for j in range(int(rng.integers(0, 30))):
        counts[150 + j] = int(rng.integers(1, 4))
    return repeated_literals(with_counts(rng, counts), 2)


def weight_spread(k: int, seed: int) -> bytes:
    """Literals over the byte values 0 .. k with counts 2^u, u uniform in 0..9: Huffman weights spread over ten values, so that the
    FSE-compressed weights come out near maxSymbolValue / 2 bytes and the direct (4-bit) form competes with them up to 128."""
    rng = np.random.default_rng(seed)
    counts = {s: int(1 << int(rng.integers(0, 10))) for s in range(k + 1)}
    return repeated_literals(with_counts(rng, counts), 2)


def sort_ties(k: int, seed: int) -> bytes:
    """Literal counts around HUF_DISTINCT_CUTOFF (165): 24 byte values with counts k - 2 .. k + 2, several of each, so the ties sit
    inside one rank bucket and across the boundary between the distinct buckets and the log buckets."""
    rng = np.random.default_rng(seed)
    counts = {10 + 7 * i: k - 2 + i % 5 for i in range(24)}
    counts[1] = 3 * k
    return repeated_literals(with_counts(rng, counts), 2)


def ml_code_sequences(codes, seed: int, run: int = 48) -> bytes:
    """One sequence per entry of `codes`: `run` literals and a copy of the shortest length of that ML code (codes 3 .. 36: 6 .. 43
    bytes)."""
    return sequences(len(codes), seed, lambda i, rng: (run, int(rng.integers(frame_info.ML_BASE[codes[i]], run + 1)),
                                                       frame_info.ML_BASE[codes[i]]))


def ml_most_frequent(k: int, seed: int, n: int = 1024) -> bytes:
    """n sequences over the 34 ML codes 3 .. 36: code 3 k times, the other 33 codes share the rest evenly (at most 31 times each
    from k = 1 on).  Below lazy the ML table stays predefined while mostFrequent < n >> 5 = 32."""
    rng = np.random.default_rng(seed)
    return ml_code_sequences(rng.permutation([3] * k + [4 + i % 33 for i in range(n - k)]).tolist(), seed)


def ml_flat(k: int, seed: int) -> bytes:
    """k sequences whose ML codes are drawn uniformly from the 27 codes 3 .. 29: 5 to 12 of each, so that FSE_normalizeCount's
    rounding hands out more than the table holds and fse_normalize_m2 redistributes it."""
    rng = np.random.default_rng(seed)
    return ml_code_sequences(rng.integers(3, 30, k).tolist(), seed)


def equal_weights(k: int, seed: int) -> bytes:
    """Byte values 0 .. k-1 16 times each and byte k 16 k + 64 times, alternating with them (64 of them twice in a row), in an
    order without a repeated 4-byte string, so all of it is literals.  Byte k gets a 1-bit code; at k = 128 the
    others all get 8-bit codes, so the 128 written weights are equal, their FSE description would be one byte, and the weights are
    written directly, the largest alphabet that can be.  At 127 and 129 the codes are 7 or 8 (8 or 9) bits long, and the weights
    are FSE-compressed."""
    from math import gcd
    steps = [d for d in range(1, k) if gcd(d, k) == 1][:16]
    others, x = [], seed % k
    for d in steps:                  # 16 rounds, each a full cycle x -> x + d: no two neighbouring pairs repeat, nor any 4-byte string
        for _ in range(k):
            x = (x + d) % k
            others.append(x)
    out = bytearray()
    for i, o in enumerate(others):
        out += bytes([k, k, o] if i < 64 else [k, o])
    return repeated_literals(bytes(out), 2)


# ------------------------------------------------------------------------------------------------ FSE_normalizeCount's decision
_RTB = (0, 473195, 504333, 520860, 550000, 700000, 750000, 830000)


def fse_optimal_log(max_log: int, n: int, max_sv: int, minus: int) -> int:
    """FSE_optimalTableLog_internal (RFC-independent: the reference's choice of an accuracy log for n symbols up to max_sv)."""
    hb = lambda x: x.bit_length() - 1
    log = min(max_log, hb(n - 1) - minus)
    log = max(log, min(hb(n) + 1, hb(max_sv) + 2))
    return max(5, min(12, log))


def enters_m2(count: list, total: int, log: int) -> bool:
    """Whether FSE_normalizeCount leaves the rounded counts to FSE_normalizeM2: the counts it rounds up overshoot the table by at
    least half the largest one."""
    scale, still, low = 62 - log, 1 << log, total >> log
    step, vstep = (1 << 62) // total, 1 << (62 - log - 20)
    largest = 0
    for c in count:
        if c == 0:
            continue
        if c <= low:
            still -= 1
            continue
        p = (c * step) >> scale
        if p < 8:
            p += ((c * step) - (p << scale)) > vstep * _RTB[p]
        largest = max(largest, p)
        still -= p
    return -still >= largest >> 1


def ml_table_enters_m2(b) -> bool:
    """From a frame's bytes: its ML table is described (FSE) and was normalised through fse_normalize_m2.  As the encoder does, the
    count of the last sequence's code is lowered by one first when it is above one."""
    if b.block_type != 2 or not b.nb_seq or b.modes[2] != "fse":
        return False
    codes = [m for _, _, _, m in frame_info.decode_sequences(b.frame)]
    count = [codes.count(c) for c in range(max(codes) + 1)]
    total = len(codes)
    if count[codes[-1]] > 1:
        count[codes[-1]] -= 1
        total -= 1
    return enters_m2(count, total, fse_optimal_log(9, len(codes), max(codes), 2))


def ml_most_frequent_count(b) -> int:
    codes = [m for _, _, _, m in frame_info.decode_sequences(b.frame)]
    return max(codes.count(c) for c in set(codes))


# ------------------------------------------------------------------------------------------------ sides
def block(z: bytes):
    b = frame_reader.walk_item(z)[0].blocks[0]
    b.frame = z
    return b


def lit_kind(b) -> str:
    if b.block_type != 2:
        return "raw block"
    return ("raw", "rle", "huf%d" % b.lit_streams, "treeless")[b.lit_mode]


def huf_log(b) -> int:
    w = b.huf_weights or []
    total = sum(1 << (x - 1) for x in w if x)
    return total.bit_length() - 1


def weight_format(b) -> str:
    if b.block_type != 2 or b.lit_mode != 2:
        return lit_kind(b)
    return "direct" if b.frame[b.lit_payload[0]] >= 128 else "fse"


def has_low_prob(b, t: int) -> bool:
    return b.block_type == 2 and b.nb_seq > 0 and b.norms[t] is not None and -1 in b.norms[t]


@dataclass
class Family:
    name: str
    decision: str                          # the comparison in zb_encode.cuh whose two sides k crosses
    gen: Callable[[int, int], bytes]
    side: Callable                         # side(block) of frame_reader's walk
    lo: int                                # side(lo) != side(hi) for the reference's frames
    hi: int
    level: int = 1
    params: Callable[[int], dict] | dict | None = None
    seed: int = 1
    exact: Callable | None = None          # exact(block): the statistic lands on the threshold itself ...
    exact_at: int = 0                      # ... in the frame of k + exact_at (-1: the threshold is visible only below k)
    boundary: bool = True                  # False: no single threshold; every k in lo..hi is compared

    def params_at(self, k: int) -> dict | None:
        return self.params(k) if callable(self.params) else self.params

    @property
    def strategy_dependent(self) -> bool:
        """Explicit strategy, or an optimal-parser level of its own: the decision depends on the strategy."""
        return "strategy" in (self.params_at(self.lo) or {}) or self.level >= 13


def _lits(n: int) -> Callable:
    return lambda b: b.block_type == 2 and b.lit_size == n


def _strategy(s: int) -> dict:
    return {"strategy": s}


FAMILIES: list = []
for s in range(1, 10):
    thr = 8 << min(9 - s, 3)
    # btultra: 16 literals compress only with a 2-byte tree description, i.e. three symbols 0..2 without a repeated 3-byte
    # string; btultra2: from 8 equal literals (all of them literals for the optimal parser) an RLE literals section
    gen = {S_BTULTRA: lambda k, seed: repeated_literals(bytes(de_bruijn(3, 3)[:k])), S_BTULTRA2: lambda k, seed: b"Z" * k}.get(
        s, lambda k, seed: skewed_run(k, seed))
    FAMILIES.append(Family(f"raw_below_min_literals_strategy{s}", f"n < 8 << min(9 - strategy, 3) = {thr} stores raw literals",
                           gen, lit_kind, max(thr - 8, 1) if s < S_BTULTRA2 else 5, thr + 8 if s < S_BTULTRA2 else 9, level=3,
                           params=_strategy(s), exact=_lits(thr)))
FAMILIES += [
    Family("literal_compression_disabled", "fast with targetLength > 0 stores raw literals", lambda k, seed: skewed_run(600, seed),
           lit_kind, 0, 2, level=1, params=lambda k: {"strategy": S_FAST, "targetLength": k} if k else {"strategy": S_FAST}),
    Family("uncompressible_sample_size", "the sample of the two ends is taken from n >= 40960 literals", sample_size, lit_kind,
           40950, 40970, exact=_lits(40959), exact_at=-1),
    Family("uncompressible_sample_ratio", "the sample is taken while litSize / nbSeq >= 20", sample_ratio, lit_kind, 4000, 4200),
    Family("uncompressible_sample_total", "largestTotal <= 68 stores raw literals", sample_total, lit_kind, 60, 76),
    Family("rle_literals_strategy9", "largest == n writes RLE literals", rle_literals, lit_kind, 0, 3, level=3, params=_strategy(S_BTULTRA2)),
    Family("raw_when_tree_description_is_large_strategy8", "hSize + 12 >= n stores raw literals",
           lambda k, seed: repeated_literals(bytes(x if x < 2 else k for x in de_bruijn(3, 3)[:16])), lit_kind, 2, 12, level=3,
           params=_strategy(S_BTULTRA)),
    Family("raw_when_no_symbol_dominates", "largest <= (n >> 7) + 4 stores raw literals", largest_count, lit_kind, 2, 10),
    Family("literal_gain_strategy3", "cLit >= n - min_gain(n, strategy) stores raw literals", mixed_run, lit_kind, 0, 2000, level=3,
           params=_strategy(S_GREEDY)),
    Family("literal_gain_strategy8", "cLit >= n - min_gain(n, strategy), btultra's shift", mixed_run, lit_kind, 0, 2000, level=3,
           params=_strategy(S_BTULTRA)),
    Family("literal_gain_strategy9", "cLit >= n - min_gain(n, strategy), btultra2's shift", mixed_run, lit_kind, 0, 2000, level=3,
           params=_strategy(S_BTULTRA2)),
    Family("one_or_four_streams", "n < 256 writes one Huffman stream", lambda k, seed: lit_run(k, seed, 16), lit_kind, 250, 262,
           exact=_lits(256)),
    Family("literal_header_1024", "n >= 1024 widens the literal header", lambda k, seed: lit_run(k, seed), lambda b: (lit_kind(b), b.lit_header),
           1018, 1030, exact=_lits(1024)),
    Family("literal_header_16384", "n >= 16384 widens the literal header", lambda k, seed: lit_run(k, seed), lambda b: (lit_kind(b), b.lit_header),
           16378, 16390, exact=_lits(16384)),
    Family("block_gain_strategy1", "cSize >= srcSize - min_gain(srcSize, strategy) stores a raw block", mixed_literals_only,
           lambda b: b.block_type, 0, 3000, level=1),
    Family("block_gain_strategy8", "cSize >= srcSize - min_gain, btultra's shift", mixed_literals_only, lambda b: b.block_type, 0, 3000,
           level=3, params=_strategy(S_BTULTRA), seed=2),
    # sequences
    Family("nbseq_header_128", "nbSeq >= 128 widens the sequence count", copies, lambda b: b.nb_seq_bytes, 120, 136,
           exact=lambda b: b.nb_seq == 128),
    Family("rle_tables_at_3_sequences_strategy1", "mostFrequent == nbSeq: predefined up to nbSeq 2, RLE from 3", same_codes,
           lambda b: b.modes, 1, 5, level=1),
    Family("rle_tables_at_3_sequences_strategy2", "mostFrequent == nbSeq: predefined up to nbSeq 2, RLE from 3", same_codes,
           lambda b: b.modes, 1, 5, level=3),
    Family("rle_tables_at_3_sequences_strategy3", "mostFrequent == nbSeq: predefined up to nbSeq 2, RLE from 3", same_codes,
           lambda b: b.modes, 1, 5, level=3, params=_strategy(S_GREEDY)),
]
for s, level in ((S_FAST, 1), (S_DFAST, 3), (S_GREEDY, 3)):
    FAMILIES.append(Family(f"ml_most_frequent_strategy{s}", "mostFrequent < nbSeq >> (6 - 1) keeps the predefined ML table",
                           ml_most_frequent, lambda b: b.modes[2], 26, 38, level=level, params=_strategy(s),
                           exact=lambda b: ml_most_frequent_count(b) == b.nb_seq >> 5))
for s, level in ((S_FAST, 1), (S_DFAST, 3), (S_GREEDY, 3)):
    for t, tname in enumerate(("LL", "OF", "ML")):
        lo = ((64 if t != 1 else 32) * (10 - s)) >> 3
        FAMILIES.append(Family(f"dynamic_fse_min_{tname}_strategy{s}", f"nbSeq < dynamicFse_nbSeq_min = {lo} keeps the predefined {tname} table",
                               (lambda t: lambda k, seed: code_pairs(t, k, seed))(t), (lambda t: lambda b: b.modes[t])(t),
                               lo - 6, lo + 6, level=level, params=_strategy(s), exact=(lambda lo: lambda b: b.nb_seq == lo)(lo)))
for t, tname in enumerate(("LL", "OF", "ML")):
    FAMILIES.append(Family(f"cost_choice_{tname}_strategy4", "basicCost <= compressedCost keeps the predefined table (lazy and up)",
                           (lambda t: lambda k, seed: code_pairs(t, k, seed))(t), (lambda t: lambda b: b.modes[t])(t), 2, 60, level=7))
FAMILIES += [
    Family("huffman_depth_limit_log11", "huf_set_max_height cuts trees 11 to 23 deep to log 11", fibonacci_literals, huf_log, 12, 24,
           level=1, boundary=False),
    Family("huffman_depth_limit_small_log", "huf_set_max_height cuts to the smaller logs fse_optimal_log picks for few literals",
           lambda k, seed: fibonacci_literals(k, seed, 0.02, 4), huf_log, 12, 20, level=1, boundary=False),
    Family("huffman_depth_limit_strategy9", "huf_optimal_depth (btultra2) over Fibonacci counts",
           lambda k, seed: fibonacci_literals(k, seed, 0.5), huf_log, 12, 20, level=19, boundary=False),
    Family("huffman_depth_limit_repair", "huf_set_max_height's rankLast[1] == noSymbol repair (btultra2)", perturbed_fibonacci, huf_log,
           14, 19, level=19, seed=18, boundary=False),
    Family("huffman_weights_maxsv", "spread weights at maxSymbolValue 125 .. 131: the FSE-compressed ones are shorter",
           weight_spread, weight_format, 125, 131, level=1, boundary=False),
    Family("huffman_direct_weights_at_128", "direct weights up to maxSymbolValue 128, when their FSE description is one byte",
           equal_weights, weight_format, 127, 129, level=1, boundary=False),
    Family("fse_normalize_m2_ml", "-still >= norm[largest] >> 1 hands the ML counts to fse_normalize_m2", ml_flat,
           ml_table_enters_m2, 200, 215, level=1, seed=4, boundary=False),
    Family("huffman_weights_direct_or_fse", "FSE-compressed weights only when shorter than maxSymbolValue / 2", weight_spread,
           weight_format, 38, 125, level=1),
    Family("huffman_sort_ties", "huf_sort's distinct buckets end at HUF_DISTINCT_CUTOFF = 165", sort_ties, lit_kind, 160, 170,
           level=1, boundary=False),
    Family("huffman_sort_ties_strategy8", "huf_sort ties under huf_optimal_depth (btultra)", sort_ties, lit_kind, 163, 167,
           level=3, params=_strategy(S_BTULTRA), boundary=False),
    Family("low_prob_cells_2049", "nbSeq_1 >= 2048 writes -1 cells (last code's count lowered)", low_prob, lambda b: has_low_prob(b, 2),
           2040, 2056, exact=lambda b: b.nb_seq == 2049),
    Family("low_prob_cells_2048", "nbSeq_1 >= 2048 writes -1 cells (last code unique)", lambda k, seed: low_prob(k, seed, False),
           lambda b: has_low_prob(b, 2), 2040, 2056, exact=lambda b: b.nb_seq == 2048),
]


def find_boundary(fam: Family, compress) -> int:
    """The smallest k in (lo, hi] whose frame is on the other side from lo's, by bisection; `compress(data, level, params)`.
    Families without a single threshold give lo + 1."""
    if not fam.boundary:
        return fam.lo + 1
    side = lambda k: fam.side(block(compress(fam.gen(k, fam.seed), fam.level, fam.params_at(k))))
    a, b = fam.lo, fam.hi
    sa = side(a)
    assert side(b) != sa, (fam.name, "no switch in range", sa)
    while b - a > 1:
        m = (a + b) // 2
        if side(m) == sa:
            a = m
        else:
            b = m
    return b
