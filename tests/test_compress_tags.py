"""The <= 64 KiB fast compressor with hash tags (TAG_BITS = 1, 2, 4, 8 bits per table slot) on the CPU emulator
(tests/simt): the tags only skip verify loads of candidates that cannot match, so every width must emit exactly the bytes
of the untagged table (TAG_BITS = 0), in both warp builds, at every source alignment and under every output capacity."""
import ctypes
import hashlib
import json
import os
import random

import numpy as np
import pytest

import corpus
from test_kernel_logic_cpu import PAD, _build

HERE = os.path.dirname(os.path.abspath(__file__))
WIDTHS = (1, 2, 4, 8)
SHIFTS = (0, 1, 3, 8, 13)          # source alignment within the 16-byte words the verify loads read


@pytest.fixture(scope="module")
def wsim():
    lib = _build("tag_harness.cpp", "libtagsim.so")
    lib.sim_compress_wide.restype = ctypes.c_int
    lib.sim_compress_wide.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int]
    return lib


def compress(wsim, d, cap, nw, tag_bits, shift=0):
    a = np.zeros(len(d) + 2 * PAD + 16, dtype=np.uint8)
    a[PAD + shift:PAD + shift + len(d)] = np.frombuffer(d, dtype=np.uint8)
    o = np.full(max(cap, 0) + 2 * PAD, 0x55, dtype=np.uint8)
    r = wsim.sim_compress_wide(a.ctypes.data + PAD + shift, len(d), o.ctypes.data + PAD, cap, nw, tag_bits)
    assert (o[:PAD] == 0x55).all() and (o[PAD + max(cap, 0):] == 0x55).all(), "wrote outside [dst, dst+cap)"
    return r, o[PAD:PAD + max(r, 0)].tobytes()


def _inputs(port):
    return [(name, d) for name, d in corpus.blocks(port) if len(d) < 65536 + 11]


@pytest.mark.parametrize("nw", [3, 2])
@pytest.mark.parametrize("tag_bits", WIDTHS)
def test_tagged_streams_equal_untagged(wsim, port, tag_bits, nw):
    gold = json.load(open(os.path.join(HERE, "golden", "fast_streams.json")))["streams"]
    for name, d in _inputs(port):
        cap = port.compress_bound(len(d))
        for shift in SHIFTS:
            want = compress(wsim, d, cap, nw, 0, shift)
            got = compress(wsim, d, cap, nw, tag_bits, shift)
            assert got == want, (name, shift)
            if shift == 0 and name in gold:
                assert (got[0], hashlib.sha256(got[1]).hexdigest()) == (gold[name]["c"], gold[name]["sha256"]), name


@pytest.mark.parametrize("nw", [3, 2])
@pytest.mark.parametrize("tag_bits", WIDTHS)
def test_tagged_limited_output_equals_untagged(wsim, port, tag_bits, nw):
    rng = random.Random(7)
    for d in [d for _, d in corpus.blocks(port, big=False)][::5]:
        full, _ = compress(wsim, d, port.compress_bound(len(d)), nw, 0)
        for cap in sorted({-1, 0, 1, full - 1, full, full + 1, max(0, full // 2), max(0, full - 17), rng.randrange(0, full + 20)}):
            assert compress(wsim, d, cap, nw, tag_bits) == compress(wsim, d, cap, nw, 0), (len(d), cap)
