"""A plain LZ4 block writer and format checker for the block-edge tests (test_block_edges_dev.py / _sim.py).

encode() builds a block from explicit sequences, so a test can put the last match at any distance from the end of the
block and pair it with any final literal run; no compressor ever writes most of those streams.  strict_check() applies
the format's end-of-block rules to a compressor's output.  Neither says what a decoder must return for a stream: the
tests take that from the CPU checker (the reference's own C, or the pinned port).

The case menus (grid_cases, random_streams, compress_inputs) live here too so the GPU file and its emulator twin
run the same streams."""
from __future__ import annotations

import random

MINMATCH = 4
LAST_LITERALS = 5          # the last 5 bytes of a block are literals
MFLIMIT = 12               # the last match starts at least 12 bytes before the end of the block
MAX_OFFSET = 65535


def _chain(n: int) -> bytes:
    """the 255-chain of a length field that overflowed its nibble by n (n >= 0): 255 x k, then the rest (which may be 0)"""
    return b"\xff" * (n // 255) + bytes([n % 255])


def encode(seqs, last_literals: bytes) -> bytes:
    """seqs: (literals, offset, match_len) triples, match_len >= 4 and 1 <= offset <= 65535; then the final literal run.
    A nibble of 15 is always followed by its chain, so lengths 15 / 19 / 270 / 274 end in a 0 extension byte."""
    out = bytearray()
    for lit, off, ml in seqs:
        assert ml >= MINMATCH and 0 < off <= MAX_OFFSET, (ml, off)
        L, M = len(lit), ml - MINMATCH
        out.append((min(L, 15) << 4) | min(M, 15))
        if L >= 15:
            out += _chain(L - 15)
        out += lit
        out += bytes([off & 255, off >> 8])
        if M >= 15:
            out += _chain(M - 15)
    L = len(last_literals)
    out.append(min(L, 15) << 4)
    if L >= 15:
        out += _chain(L - 15)
    out += last_literals
    return bytes(out)


def decoded_size(seqs, last_literals: bytes) -> int:
    return sum(len(lit) + ml for lit, _, ml in seqs) + len(last_literals)


def _length(c: bytes, ip: int, nib: int):
    n = nib
    if nib == 15:
        while True:
            if ip >= len(c):
                return None, ip
            b = c[ip]; ip += 1; n += b
            if b != 255:
                break
    return n, ip


def strict_check(stream: bytes, n: int):
    """None when `stream` is a block of the format that decodes to n bytes and keeps every end rule; otherwise what is
    wrong.  Rules: the last sequence is literals only; the last match starts at or before n - 12 and ends at or before
    n - 5 (so a block under 13 bytes is literals only); 0 < offset <= position and offset <= 65535."""
    c = bytes(stream)
    ip = op = 0
    last_start = last_end = None
    while True:
        if ip >= len(c):
            return f"stream ends inside a sequence at {ip}"
        tok = c[ip]; ip += 1
        L, ip = _length(c, ip, tok >> 4)
        if L is None or ip + L > len(c):
            return f"literal run of sequence at {ip} runs past the stream"
        ip += L; op += L
        if ip == len(c):
            if tok & 15:
                return "the last sequence has a match nibble"
            break
        if ip + 2 > len(c):
            return f"offset cut at {ip}"
        off = c[ip] | (c[ip + 1] << 8); ip += 2
        M, ip = _length(c, ip, tok & 15)
        if M is None:
            return f"match length chain cut at {ip}"
        M += MINMATCH
        if off == 0 or off > op or off > MAX_OFFSET:
            return f"offset {off} at position {op}"
        last_start, op = op, op + M
        last_end = op
    if op != n:
        return f"decodes to {op} bytes, not {n}"
    if last_start is not None:
        if n < MFLIMIT + 1:
            return f"a {n}-byte block has a match"
        if last_start > n - MFLIMIT:
            return f"last match starts at {last_start} > n - 12 = {n - MFLIMIT}"
        if last_end > n - LAST_LITERALS:
            return f"last match ends at {last_end} > n - 5 = {n - LAST_LITERALS}"
    return None


# ------------------------------------------------------------------------------------------------ decoder cases
GRID_MATCH_LENS = list(range(4, 22)) + [273, 274, 275, 276]
GRID_FINAL_RUNS = list(range(0, 17))
PREFIX_LITS = [0, 14, 15, 16, 269, 270, 271]


def _prefix(rng: random.Random, kind: str):
    """the sequences in front of the tail, and the position where they end.
    p20 / p70: one / three short sequences; p700: ~40 sequences over every prefix literal length (the stream is long
    enough for the batched decoder's window, so decode_batch runs in front of the tail); far: a 65 600-byte run that
    makes offset 65535 reachable."""
    seqs = []
    if kind == "p20":
        seqs.append((rng.randbytes(20), 20, 4))
    elif kind == "p70":
        seqs += [(rng.randbytes(30), 7, 9), (rng.randbytes(15), 33, 15), (rng.randbytes(14), 1, 19)]
    elif kind == "p700":
        pos = 0
        for k in range(40):
            L = PREFIX_LITS[k % len(PREFIX_LITS)]
            if pos + L == 0:
                L = 8
            ml = [4, 5, 15, 18, 19, 20, 40][k % 7]
            off = [1, 3, 8, 16, 17, pos + L, rng.randrange(1, pos + L + 1)][(k * 3) % 7]
            seqs.append((rng.randbytes(L), max(1, min(off, pos + L, MAX_OFFSET)), ml))
            pos += L + ml
    elif kind == "far":
        seqs += [(rng.randbytes(40), 1, 65600), (rng.randbytes(270), 65535, 300)]
    else:
        raise ValueError(kind)
    return seqs, sum(len(lit) + ml for lit, _, ml in seqs)


def grid_cases(prefixes=("p20", "p70", "p700", "far"), match_lens=None, final_runs=None, seed=1):
    """(name, stream, decoded size) for the end-of-block grid: a prefix, one last match and a final literal run.  Offsets 1-8 (the
    overlap paths), 15, 16, 17, 32 and offset = position for every prefix; 65535 where the prefix reaches that far."""
    rng = random.Random(seed)
    match_lens = GRID_MATCH_LENS if match_lens is None else match_lens
    final_runs = GRID_FINAL_RUNS if final_runs is None else final_runs
    out = []
    for kind in prefixes:
        pre, pos = _prefix(rng, kind)
        for ml in match_lens:
            for fr in final_runs:
                lit = rng.randbytes(3)                      # the last match's own literals: position = pos + 3
                offs = [1, 2, 3, 4, 5, 6, 7, 8, 15, 16, 17, 32, pos + 3] if kind != "far" else [65535, pos + 3 if pos + 3 <= MAX_OFFSET else 65534]
                for off in offs:
                    seqs, last = pre + [(lit, off, ml)], rng.randbytes(fr)
                    out.append((f"{kind}/ml{ml}/fr{fr}/off{off}", encode(seqs, last), decoded_size(seqs, last)))
    return out


def random_streams(count: int, seed: int):
    """`count` multi-sequence streams drawn from the same menus (1 to 120 sequences, lengths around every nibble and
    chain boundary, offsets short, near and = position), some long enough for the batched decoder's window"""
    rng = random.Random(seed)
    out = []
    for t in range(count):
        seqs, pos = [], 0
        for _ in range(rng.choice([1, 2, 5, 40, 120])):
            L = rng.choice(PREFIX_LITS + [1, 3, 7, 17, 31, 32, 33, rng.randrange(0, 80)])
            if pos + L == 0:
                L = rng.choice([1, 8, 20])
            ml = rng.choice([4, 5, 8, 15, 16, 17, 18, 19, 20, 33, 64, 273, 274, 275, rng.randrange(4, 300)])
            off = rng.choice([1, 2, 3, 4, 5, 7, 8, 9, 15, 16, 17, 31, 32, pos + L, rng.randrange(1, pos + L + 1)])
            seqs.append((rng.randbytes(L), max(1, min(off, pos + L, MAX_OFFSET)), ml))
            pos += L + ml
        last = rng.randbytes(rng.choice([0, 1, 4, 5, 6, 11, 12, 13, 15, 16, 40]))
        out.append((f"rand{t}", encode(seqs, last), decoded_size(seqs, last)))
    return out


# ------------------------------------------------------------------------------------------------ compressor inputs
FAMILIES = ("zeros", "two", "period3", "tailrep", "random")


def family(kind: str, n: int, seed: int = 0) -> bytes:
    rng = random.Random(seed * 7919 + n)
    if kind == "zeros":
        return bytes(n)
    if kind == "two":
        return bytes(rng.getrandbits(1) * 0x41 for _ in range(n)) if n < 4096 else \
            bytes((b & 1) * 0x41 for b in rng.randbytes(n))
    if kind == "period3":
        return (b"abc" * (n // 3 + 1))[:n]
    if kind == "tailrep":                           # random bytes whose second half repeats the first
        h = rng.randbytes(n // 2)
        return (h + h + rng.randbytes(2))[:n]
    if kind == "random":
        return rng.randbytes(n)
    raise ValueError(kind)


def compress_inputs(lengths):
    return [(f"{kind}_{n}", family(kind, n)) for n in lengths for kind in FAMILIES]
