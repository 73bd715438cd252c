"""ctypes loader for libb200lz4.so (include/b200lz4.h).  No fallback: if the CUDA library is
missing or no H100 (sm_90) is usable, callers get an exception, never a CPU path."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# The one library the package loads.  No environment switch here: tests/conftest.py and tools/_variant.py (development
# infrastructure, outside the package) may point SO_PATH at another BUILD of the same library before first use — a
# sanitizer / A-B variant build, or the emulator build of tests/simt — via B200LZ4_TEST_SO.
SO_PATH = os.path.join(_HERE, "libb200lz4.so")

E_NODEVICE, E_CUDA, E_ARG = -2147483647, -2147483646, -2147483645      # INT_MIN + 1..3: below every -(offset)-1 a decoder can return

# every symbol include/b200lz4.h declares: (name, restype, argtypes)
_vp, _i, _sz, _u32, _u64, _i32 = C.c_void_p, C.c_int, C.c_size_t, C.c_uint32, C.c_uint64, C.c_int32
_BATCH = [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _sz]
SYMBOLS = [
    ("b200lz4_version", _i, []),
    ("b200lz4_device_count", _i, []),
    ("b200lz4_set_device", _i, [_i]),
    ("b200lz4_last_error", C.c_char_p, []),
    ("b200lz4_last_status", _i, []),
    ("b200lz4_host_register", _i, [_vp, _sz]),
    ("b200lz4_host_unregister", _i, [_vp]),
    ("b200lz4_compressBound", _i, [_i]),
    ("b200lz4_compress_default", _i, [_vp, _vp, _i, _i]),
    ("b200lz4_compress_HC", _i, [_vp, _vp, _i, _i, _i]),
    ("b200lz4_decompress_safe", _i, [_vp, _vp, _i, _i]),
    ("b200lz4_decompress_fast_bounded", _i, [_vp, _i, _vp, _i]),
    ("b200xxh32", _u32, [_vp, _sz, _u32]),
    ("b200xxh64", _u64, [_vp, _sz, _u64]),
    ("b200xxh32_create", _vp, [_u32]),
    ("b200xxh32_reset", None, [_vp, _u32]),
    ("b200xxh32_update", _i, [_vp, _vp, _sz]),
    ("b200xxh32_digest", _u32, [_vp]),
    ("b200xxh32_free", None, [_vp]),
    ("b200xxh64_create", _vp, [_u64]),
    ("b200xxh64_reset", None, [_vp, _u64]),
    ("b200xxh64_update", _i, [_vp, _vp, _sz]),
    ("b200xxh64_digest", _u64, [_vp]),
    ("b200xxh64_free", None, [_vp]),
    ("b200lz4_compress_fast_batch_dev", _i, _BATCH + [_i, _vp]),
    ("b200lz4_compress_hc_batch_dev", _i, _BATCH + [_i, _vp]),
    ("b200lz4_decompress_safe_batch_dev", _i, _BATCH + [_vp]),
    ("b200lz4_decompress_fast_batch_dev", _i, _BATCH + [_vp]),
    ("b200xxh32_batch_dev", _i, [_vp, _vp, _vp, _u32, _vp, _sz, _vp]),
    ("b200xxh64_batch_dev", _i, [_vp, _vp, _vp, _u64, _vp, _sz, _vp]),
    ("b200lz4_compact_dev", _i, [_vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    ("b200lz4_stitch_shards_dev", _i, [_vp, _vp, _vp, _i, _vp, _i, _sz, _vp]),
    ("b200lz4_compress_fast_batch_host", _i, _BATCH + [_i]),
    ("b200lz4_compress_hc_batch_host", _i, _BATCH + [_i]),
    ("b200lz4_decompress_safe_batch_host", _i, _BATCH),
    ("b200lz4_decompress_fast_batch_host", _i, _BATCH),
    ("b200xxh32_batch_host", _i, [_vp, _vp, _vp, _u32, _vp, _sz]),
    ("b200xxh64_batch_host", _i, [_vp, _vp, _vp, _u64, _vp, _sz]),
    ("b200lz4_compress_fast_batch_host_multi", _i, _BATCH + [_i, _vp, _i]),
    ("b200lz4_compress_fast_compact_host_multi", _i, [_vp, _vp, _vp, _vp, _sz, _vp, _vp, _sz, _i, _vp, _i, _vp, _vp]),
    ("b200lz4_compress_hc_batch_host_multi", _i, _BATCH + [_i, _vp, _i]),
    ("b200lz4_decompress_safe_batch_host_multi", _i, _BATCH + [_vp, _i]),
    ("b200lz4_decompress_fast_batch_host_multi", _i, _BATCH + [_vp, _i]),
    ("b200xxh32_batch_host_multi", _i, [_vp, _vp, _vp, _u32, _vp, _sz, _vp, _i]),
    ("b200xxh64_batch_host_multi", _i, [_vp, _vp, _vp, _u64, _vp, _sz, _vp, _i]),
    ("b200lz4_compress_fast_compact_host", _i, [_vp, _vp, _vp, _vp, _sz, _vp, _vp, _sz, _i, _vp]),
    ("b200lz4f_decompress_host", C.c_int64, [_vp, _sz, _vp, _sz]),
    ("b200lz4f_index_create", _vp, [_vp, _sz, _vp, _vp]),
    ("b200lz4f_index_create_single", _vp, [_vp, _sz, _vp, _vp, _vp]),
    ("b200lz4f_decompress_host_single", C.c_int64, [_vp, _sz, _vp, _sz, _vp]),
    ("b200lz4f_expected_content_size", _i, [_vp, _sz, _vp]),
    ("b200lz4f_index_frames", _sz, [_vp]),
    ("b200lz4f_index_blocks", _sz, [_vp]),
    ("b200lz4f_index_block_offsets", None, [_vp, _vp]),
    ("b200lz4f_decode_dev", C.c_int64, [_vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    ("b200lz4f_index_free", None, [_vp]),
    ("b200lz4f_index_create_dev", _vp, [_vp, _sz, _i, _vp, _sz, _vp, _vp, _vp, _vp]),
    ("b200lz4f_decompress_dev", C.c_int64, [_vp, _sz, _vp, _sz, _i, _vp, _sz, _vp, _vp]),
    ("b200lz4f_decompress_streams_dev", _i, [_vp, _vp, _vp, _sz, _vp, _vp, _vp, _i, _vp, _vp, _vp, _vp]),
    ("b200lz4f_reader_create", _vp, [_sz, _i, _vp]),
    ("b200lz4f_reader_read_dev", _i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    ("b200lz4f_reader_free", None, [_vp]),
    ("b200lz4f_compress_dev", C.c_int64, [_vp, _vp, _vp, _sz, _vp, _sz, _vp, _vp, _i, _i, _i, _vp]),
    ("b200lz4f_writer_create", _vp, [_sz, _i, _i, _i, _vp, _vp]),
    ("b200lz4f_writer_write_dev", _i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    ("b200lz4f_writer_free", None, [_vp]),
    ("b200lz4f_compress_bound", _sz, [_sz, _i]),
    ("b200lz4f_compress_host", C.c_int64, [_vp, _sz, _vp, _sz, _i, _i]),
    ("b200lz4f_compress_host_hc", C.c_int64, [_vp, _sz, _vp, _sz, _i, _i, _i]),
    ("b200lz4block_compress_bound", _sz, [_sz, _i]),
    ("b200lz4block_compress_host", C.c_int64, [_vp, _sz, _vp, _sz, _i]),
    ("b200lz4block_compress_host_hc", C.c_int64, [_vp, _sz, _vp, _sz, _i, _i]),
    ("b200lz4block_decompress_host", C.c_int64, [_vp, _sz, _vp, _sz, C.c_int, _vp]),
    ("b200lz4block_compress_dev", C.c_int64, [_vp, _vp, _vp, _sz, _vp, _sz, _vp, _vp, _i, _i, _vp]),
    ("b200lz4block_decompress_dev", _i, [_vp, _vp, _vp, _sz, _vp, _vp, _vp, _i, _vp, _vp, _vp, _vp]),
    ("b200lz4block_writer_create", _vp, [_sz, _i, _i, _vp]),
    ("b200lz4block_writer_write_dev", _i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    ("b200lz4block_writer_free", None, [_vp]),
    ("b200lz4block_reader_create", _vp, [_sz, _i, _vp]),
    ("b200lz4block_reader_read_dev", _i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    ("b200lz4block_reader_free", None, [_vp]),
    ("b200lz4_compress_with_length", _i, [_vp, _vp, _i, _i]),
    ("b200lz4_decompressed_length", _i, [_vp]),
    ("b200lz4_decompress_with_length", _i, [_vp, _i, _vp, _i]),
    ("b200lz4_decompress_with_length_safe", _i, [_vp, _i, _vp, _i]),
    ("b200lz4_compress_with_length_dev", C.c_int64, [_vp, _vp, _vp, _sz, _vp, _sz, _vp, _vp, _i, _vp]),
    ("b200lz4_decompress_with_length_dev", _i, [_vp, _vp, _vp, _sz, _vp, _vp, _vp, _i, _vp, _vp, _vp]),
    ("b200lz4_launch_count", _u64, []),
    ("b200lz4_launch_count_reset", None, []),
    ("b200lz4_context_count", _i, []),
]

_lib = None


class B200Error(RuntimeError):
    """The CUDA backend failed (no device, CUDA error, bad batch layout).  Never swallowed."""


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(SO_PATH):
            raise ImportError(
                f"{SO_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(make -C lz4-java_b200/csrc).  There is no CPU fallback.")
        L = C.CDLL(SO_PATH)
        for name, res, args in SYMBOLS:
            f = getattr(L, name)          # AttributeError here == ABI/header mismatch
            f.restype = res
            f.argtypes = args
        _lib = L
    return _lib


def check(rc: int) -> int:
    if rc in (E_NODEVICE, E_CUDA, E_ARG):
        raise B200Error(f"libb200lz4: {lib().b200lz4_last_error().decode()} (code {rc})")
    return rc


def checked_value(v: int) -> int:
    """for the entry points that return a hash value: raise if the call left an error status (see b200lz4_last_status)"""
    rc = lib().b200lz4_last_status()
    if rc:
        raise B200Error(f"libb200lz4: {lib().b200lz4_last_error().decode()} (code {rc})")
    return v


def last_error() -> str:
    return lib().b200lz4_last_error().decode()
