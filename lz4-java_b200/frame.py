"""LZ4 Frame batch decoding on the B200 backend — the semantics of LZ4FrameInputStream.read()
(src/java/net/jpountz/lz4/LZ4FrameInputStream.java:132-321) for whole buffers of concatenated frames.

The reference's stream class decodes one block per native call; here one call indexes the container on
the host and decodes every block of every frame in batched GPU launches, verifying the header, block
and content XXH32 checksums on the device."""
from __future__ import annotations

import numpy as np

from . import _native as N
from .lz4 import _view

ERRORS = {
    -1: "Stream ended prematurely",                 # LZ4FrameInputStream.PREMATURE_EOS
    -2: "Stream unsupported (invalid magic bytes)",  # NOT_SUPPORTED
    -3: "Stream frame descriptor corrupted",         # DESCRIPTOR_HASH_MISMATCH
    -4: "Block size exceeded max",
    -5: "Block checksum mismatch",                   # BLOCK_HASH_MISMATCH
    -6: "Error decoding block",
    -7: "Content checksum mismatch",
    -8: "Size check mismatch",
    -9: "destination too small",
    -10: "unsupported frame descriptor",
}


class LZ4FrameError(IOError):
    """what LZ4FrameInputStream throws as java.io.IOException"""

    def __init__(self, code: int):
        super().__init__(ERRORS.get(code, f"B200 backend error {code}"))
        self.code = code


def decompress_frames(src, max_decoded: int, read_single_frame: bool = False) -> bytes:
    """decode every frame in `src` (concatenated / skippable frames allowed) -> the decoded stream;
    read_single_frame: stop behind the first non-skippable frame like LZ4FrameInputStream(in, true) (:83-91)"""
    s = _view(src)
    out = np.empty(max(max_decoded, 1), dtype=np.uint8)
    if read_single_frame:
        r = N.lib().b200lz4f_decompress_host_single(s.ctypes.data, len(s), out.ctypes.data, max_decoded, None)
    else:
        r = N.lib().b200lz4f_decompress_host(s.ctypes.data, len(s), out.ctypes.data, max_decoded)
    N.check(r)
    if r < 0:
        raise LZ4FrameError(int(r))
    return out[:r].tobytes()


def expected_content_size(src) -> int:
    """LZ4FrameInputStream.getExpectedContentSize (:416-428): the content size the first non-skippable frame declares, -1 if none"""
    import ctypes
    s = _view(src)
    size = ctypes.c_int64(-1)
    r = N.lib().b200lz4f_expected_content_size(s.ctypes.data, len(s), ctypes.byref(size))
    N.check(r)
    if r < 0:
        raise LZ4FrameError(int(r))
    return int(size.value)


def compress_frame(src, block_size_code: int = 4, content_checksum=True, block_checksum=False, content_size=False, hc_level: int = 0) -> bytes:
    """one LZ4 frame as LZ4FrameOutputStream writes it (LZ4FrameOutputStream.java:178-251), whole buffer at once;
    hc_level: the stream's compressor argument (:132-133) -- 0 = fastCompressor(), 1..17 = highCompressor(level)"""
    s = _view(src)
    flags = (1 if content_checksum else 0) | (2 if block_checksum else 0) | (4 if content_size else 0)
    L = N.lib()
    cap = L.b200lz4f_compress_bound(len(s), block_size_code)
    if cap == 0:
        raise ValueError("block_size_code must be 4..7 (64 KiB .. 4 MiB)")
    out = np.empty(cap, dtype=np.uint8)
    r = L.b200lz4f_compress_host_hc(s.ctypes.data, len(s), out.ctypes.data, cap, block_size_code, flags, hc_level)
    N.check(r)
    if r < 0:
        raise LZ4FrameError(int(r))
    return out[:r].tobytes()


def compress_frames_dev(src, src_off, src_len, block_size_code: int = 4, content_checksum=True, block_checksum=False,
                        content_size=False, hc_level: int = 0, out=None):
    """independent LZ4 frames of bytes already in device memory, written on the device (b200lz4f_compress_dev): frame f is
    src[src_off[f] : src_off[f] + src_len[f]], byte for byte what compress_frame writes for the same bytes at the same 16-byte
    phase.  src: a uint8 CUDA tensor; src_off / src_len: host sequences; out: a uint8 CUDA tensor on src's device (default: a
    new one of the summed frame bounds).  Runs on torch's current stream and returns when the frames are written.
    -> (out[:total], frame_off, frame_len), the last two np.uint64 arrays (where each frame lies in out)"""
    import torch
    off = np.ascontiguousarray(np.asarray(src_off, dtype=np.uint64).reshape(-1))
    ln = np.ascontiguousarray(np.asarray(src_len, dtype=np.uint64).reshape(-1))
    if len(off) != len(ln):
        raise ValueError("src_off and src_len must have the same length")
    if src.dtype != torch.uint8 or not src.is_cuda or not src.is_contiguous():
        raise ValueError("src must be a contiguous uint8 CUDA tensor")
    if len(ln) and int((off + ln).max()) > src.numel():
        raise ValueError("a frame reaches past the end of src")
    if not 4 <= block_size_code <= 7:
        raise ValueError("block_size_code must be 4..7 (64 KiB .. 4 MiB)")
    L = N.lib()
    bounds = [L.b200lz4f_compress_bound(int(n), block_size_code) for n in ln]
    if out is None:
        out = torch.empty(max(sum(bounds), 1), dtype=torch.uint8, device=src.device)
    elif out.dtype != torch.uint8 or out.device != src.device or not out.is_contiguous():
        raise ValueError("out must be a contiguous uint8 tensor on src's device")
    flags = (1 if content_checksum else 0) | (2 if block_checksum else 0) | (4 if content_size else 0)
    frame_off, frame_len = np.zeros(len(ln), dtype=np.uint64), np.zeros(len(ln), dtype=np.uint64)
    r = L.b200lz4f_compress_dev(src.data_ptr(), off.ctypes.data, ln.ctypes.data, len(ln), out.data_ptr(), out.numel(),
                                frame_off.ctypes.data, frame_len.ctypes.data, block_size_code, flags, hc_level,
                                torch.cuda.current_stream(src.device).cuda_stream)
    N.check(r)
    if r < 0:
        raise LZ4FrameError(int(r))
    return out[:r], frame_off, frame_len


def decompress_frames_dev(src, max_decoded: int, read_single_frame: bool = False, frame_hints=None, out=None):
    """decompress_frames for a container already in device memory, decoded into device memory (b200lz4f_decompress_dev):
    no byte of the container or the content crosses to the host.  src: a contiguous uint8 CUDA tensor; out: a contiguous
    uint8 CUDA tensor on src's device (default: a new one of max_decoded bytes); at most min(max_decoded, out.numel())
    bytes are decoded.  frame_hints: offsets where frames are believed to start (compress_frames_dev's frame_off), which
    lets the container be indexed in parallel; wrong hints cost time, never a different result.  Runs on torch's current
    stream and returns out[:total] when it is written."""
    import torch
    if not isinstance(src, torch.Tensor) or src.dtype != torch.uint8 or not src.is_cuda or not src.is_contiguous():
        raise ValueError("src must be a contiguous uint8 CUDA tensor")
    if out is None:
        out = torch.empty(max(max_decoded, 1), dtype=torch.uint8, device=src.device)
    elif not isinstance(out, torch.Tensor) or out.dtype != torch.uint8 or out.device != src.device or not out.is_contiguous():
        raise ValueError("out must be a contiguous uint8 tensor on src's device")
    hints = np.ascontiguousarray(np.asarray([] if frame_hints is None else frame_hints, dtype=np.uint64).reshape(-1))
    r = N.lib().b200lz4f_decompress_dev(src.data_ptr(), src.numel(), out.data_ptr(), min(max_decoded, out.numel()),
                                        int(bool(read_single_frame)), hints.ctypes.data if len(hints) else None, len(hints),
                                        None, torch.cuda.current_stream(src.device).cuda_stream)
    N.check(r)
    if r < 0:
        raise LZ4FrameError(int(r))
    return out[:r]


def decompress_frame_streams_dev(src, src_off, src_len, out, dst_off, dst_cap, read_single_frame: bool = False):
    """many independent LZ4 frame streams in device memory, each read as its own LZ4FrameInputStream(in, readSingleFrame) into
    device memory (b200lz4f_decompress_streams_dev): stream s is src[src_off[s] : src_off[s] + src_len[s]], decoded to
    out[dst_off[s]:] with room for dst_cap[s] bytes.  No byte of the streams or the content crosses to the host.  src, out:
    contiguous uint8 CUDA tensors on one device; the offsets and lengths: host sequences.  Runs on torch's current stream and
    returns when the results are on the host.  -> (result, src_consumed, content_len), np.int64 / np.uint64 / np.uint64
    arrays: per stream what decompress_frames would return (decoded bytes, or the LZ4FrameError code -1 .. -10), where the
    reader stopped (0 on an error), and what it decodes to when room is not the limit.  Raises only on a backend error."""
    import torch
    off, ln = _dev_streams(src, src_off, src_len, "stream")
    doff, dcap = _dev_ranges(src, out, dst_off, dst_cap, len(ln), "stream")
    result = np.zeros(len(ln), dtype=np.int64)
    consumed, content = np.zeros(len(ln), dtype=np.uint64), np.zeros(len(ln), dtype=np.uint64)
    N.check(N.lib().b200lz4f_decompress_streams_dev(src.data_ptr(), off.ctypes.data, ln.ctypes.data, len(ln), out.data_ptr(),
                                                    doff.ctypes.data, dcap.ctypes.data, int(bool(read_single_frame)),
                                                    result.ctypes.data, consumed.ctypes.data, content.ctypes.data,
                                                    torch.cuda.current_stream(src.device).cuda_stream))
    return result, consumed, content


MORE_INPUT, MORE_ROOM, DONE = 0, 1, 2
WRITE, FLUSH, CLOSE = 0, 1, 2


def _eofs(eof):
    return np.ascontiguousarray(np.asarray(eof, dtype=bool).reshape(-1)).astype(np.uint8)


def _ops(op):
    return np.ascontiguousarray(np.asarray(op, dtype=np.int64).reshape(-1))


class _Incremental:
    """what the incremental readers and writers share: the argument checks of a call, the handle's lifetime (close(), the
    context manager), torch's current stream.  _h: the handle; _free: the C call that frees it; _what: "reader" or "writer"."""
    _h = None

    def _call(self, fn, src, src_off, src_len, out, dst_off, dst_cap, last, last_name):
        """last: eof or op, converted by _eofs or _ops; the checks run in the order FrameReader and FrameWriter always had"""
        import torch
        if not self._h:
            raise ValueError(f"the {self._what} is closed")
        off, ln = _dev_streams(src, src_off, src_len, "piece")
        if not isinstance(out, torch.Tensor) or out.dtype != torch.uint8 or out.device != src.device or not out.is_contiguous():
            raise ValueError("out must be a contiguous uint8 tensor on src's device")
        doff = np.ascontiguousarray(np.asarray(dst_off, dtype=np.uint64).reshape(-1))
        dcap = np.ascontiguousarray(np.asarray(dst_cap, dtype=np.uint64).reshape(-1))
        last = (_ops if last_name == "op" else _eofs)(last)
        if len(ln) != self.ns or len(doff) != self.ns or len(dcap) != self.ns or len(last) != self.ns:
            raise ValueError(f"src_off, src_len, dst_off, dst_cap and {last_name} must have one entry per stream ({self.ns})")
        if last_name == "op":
            if ((last < WRITE) | (last > CLOSE)).any():
                raise ValueError("op must be WRITE, FLUSH or CLOSE")
            last = last.astype(np.uint8)
        if self.ns and int((doff + dcap).max()) > out.numel():
            raise ValueError("a destination range reaches past the end of out")
        status = np.zeros(self.ns, dtype=np.int32)
        consumed, produced, need = (np.zeros(self.ns, dtype=np.uint64) for _ in range(3))
        N.check(fn(self._h, src.data_ptr(), off.ctypes.data, ln.ctypes.data, last.ctypes.data, out.data_ptr(), doff.ctypes.data,
                   dcap.ctypes.data, status.ctypes.data, consumed.ctypes.data, produced.ctypes.data, need.ctypes.data,
                   torch.cuda.current_stream(src.device).cuda_stream))
        return status, consumed, produced, need

    def close(self):
        if self._h:
            getattr(N.lib(), self._free)(self._h)
            self._h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class FrameReader(_Incremental):
    """ns LZ4 frame streams read piece by piece in device memory, each one LZ4FrameInputStream(in, readSingleFrame) whose
    bytes arrive over time (b200lz4f_reader_*).  The reader is host data, the streams' carried state; not thread-safe.

        with FrameReader(ns) as rd:
            status, consumed, produced, need = rd.read(src, src_off, src_len, out, dst_off, dst_cap, eof)

    A call takes the complete units at the start of stream s's piece src[src_off[s] : src_off[s] + src_len[s]] and packs their
    content into out[dst_off[s] : dst_off[s] + produced[s]], never past dst_cap[s].  The next piece of stream s must start
    at byte consumed[s] of this one.  status[s]: MORE_INPUT (need[s]: bytes the next unit takes), MORE_ROOM (need[s]: the room
    the next block takes), DONE, or the LZ4FrameError code -1 .. -10, after the content in front of the failing unit was
    delivered.  eof[s] true: the piece ends the stream.  DONE and errors are latched.  src, out: contiguous uint8 CUDA tensors
    on one device; the rest: host sequences.  Runs on torch's current stream and returns when the results are on the host.
    -> (status, consumed, produced, need): np.int32 / np.uint64 arrays."""

    def __init__(self, ns: int, read_single_frame: bool = False):
        import ctypes
        err = ctypes.c_int(0)
        self.ns = int(ns)
        self._h = N.lib().b200lz4f_reader_create(self.ns, int(bool(read_single_frame)), ctypes.byref(err))
        if not self._h:
            N.check(err.value)
            raise MemoryError("b200lz4f_reader_create")

    _free, _what = "b200lz4f_reader_free", "reader"

    def read(self, src, src_off, src_len, out, dst_off, dst_cap, eof):
        return self._call(N.lib().b200lz4f_reader_read_dev, src, src_off, src_len, out, dst_off, dst_cap, eof, "eof")


class FrameWriter(_Incremental):
    """ns LZ4 frame streams written piece by piece in device memory, each one LZ4FrameOutputStream whose content arrives over
    time (b200lz4f_writer_*).  The writer is host data, the streams' carried state; not thread-safe.

        with FrameWriter(ns, block_size_code=4) as wr:
            status, consumed, produced, need = wr.write(src, src_off, src_len, out, dst_off, dst_cap, op)

    A call writes stream s's header on its first call, then takes whole blocks from the start of its piece
    src[src_off[s] : src_off[s] + src_len[s]]; op[s] FLUSH also takes the rest as a short block (flush()), CLOSE then writes the
    EndMark and content checksum (close()).  The frame bytes go to out[dst_off[s] : dst_off[s] + produced[s]], never past
    dst_cap[s].  The rest of the piece, past consumed[s], must start stream s's next piece.  status[s]: MORE_INPUT (need[s]:
    the bytes missing for the next whole block), MORE_ROOM (need[s]: the room the next unit takes), DONE (latched).
    known_size: the streams' declared content sizes (one int or one per stream; None: not declared).  src, out: contiguous
    uint8 CUDA tensors on one device; the rest: host sequences.  Runs on torch's current stream and returns when the results
    are on the host.  -> (status, consumed, produced, need): np.int32 / np.uint64 arrays."""

    def __init__(self, ns: int, block_size_code: int = 4, content_checksum=True, block_checksum=False, known_size=None,
                 hc_level: int = 0):
        import ctypes
        if not 4 <= block_size_code <= 7:
            raise ValueError("block_size_code must be 4..7 (64 KiB .. 4 MiB)")
        self.ns = int(ns)
        flags = (1 if content_checksum else 0) | (2 if block_checksum else 0) | (4 if known_size is not None else 0)
        known = None
        if known_size is not None:
            known = np.ascontiguousarray(np.broadcast_to(np.asarray(known_size, dtype=np.int64).reshape(-1), (self.ns,)))
            if (known < 0).any():
                raise ValueError("known_size must be >= 0")
        err = ctypes.c_int(0)
        self._h = N.lib().b200lz4f_writer_create(self.ns, block_size_code, flags, hc_level,
                                                 known.ctypes.data if known is not None else None, ctypes.byref(err))
        if not self._h:
            N.check(err.value)
            raise MemoryError("b200lz4f_writer_create")

    _free, _what = "b200lz4f_writer_free", "writer"

    def write(self, src, src_off, src_len, out, dst_off, dst_cap, op):
        return self._call(N.lib().b200lz4f_writer_write_dev, src, src_off, src_len, out, dst_off, dst_cap, op, "op")


# ---- lz4-java's private "LZ4Block" container (LZ4BlockOutputStream / LZ4BlockInputStream)
def compress_lz4block(src, block_size: int = 1 << 16, hc_level: int = 0) -> bytes:
    s = _view(src)
    L = N.lib()
    cap = L.b200lz4block_compress_bound(len(s), block_size)
    if cap == 0:
        raise ValueError("blockSize must be >= 64 and <= 32 MiB")            # LZ4BlockOutputStream.java:58-66
    out = np.empty(cap, dtype=np.uint8)
    r = L.b200lz4block_compress_host_hc(s.ctypes.data, len(s), out.ctypes.data, cap, block_size, hc_level)
    N.check(r)
    if r < 0:
        raise LZ4FrameError(int(r))
    return out[:r].tobytes()


def decompress_lz4block(src, max_decoded: int, stop_on_empty_block: bool = True) -> bytes:
    """LZ4BlockInputStream(in, stopOnEmptyBlock) read to its end (LZ4BlockInputStream.java:60-72, default true :100-104)."""
    s = _view(src)
    out = np.empty(max(max_decoded, 1), dtype=np.uint8)
    r = N.lib().b200lz4block_decompress_host(s.ctypes.data, len(s), out.ctypes.data, max_decoded, int(bool(stop_on_empty_block)), None)
    N.check(r)
    if r == -1:
        raise EOFError("Stream ended prematurely")                           # LZ4BlockInputStream.java:197
    if r < 0:
        raise IOError("Stream is corrupted" if r == -2 else f"error {r}")    # LZ4BlockInputStream.java:203,...
    return out[:r].tobytes()


def _dev_streams(src, src_off, src_len, what):
    """the host offset / length arrays of a device call over streams of src, checked against it"""
    import torch
    off = np.ascontiguousarray(np.asarray(src_off, dtype=np.uint64).reshape(-1))
    ln = np.ascontiguousarray(np.asarray(src_len, dtype=np.uint64).reshape(-1))
    if len(off) != len(ln):
        raise ValueError("src_off and src_len must have the same length")
    if not isinstance(src, torch.Tensor) or src.dtype != torch.uint8 or not src.is_cuda or not src.is_contiguous():
        raise ValueError("src must be a contiguous uint8 CUDA tensor")
    if len(ln) and int((off + ln).max()) > src.numel():
        raise ValueError(f"a {what} reaches past the end of src")
    return off, ln


def _dev_ranges(src, out, dst_off, dst_cap, n, what):
    """the host destination offset / capacity arrays of a device call over n streams (or records) of src, checked against out"""
    import torch
    if not isinstance(out, torch.Tensor) or out.dtype != torch.uint8 or out.device != src.device or not out.is_contiguous():
        raise ValueError("out must be a contiguous uint8 tensor on src's device")
    doff = np.ascontiguousarray(np.asarray(dst_off, dtype=np.uint64).reshape(-1))
    dcap = np.ascontiguousarray(np.asarray(dst_cap, dtype=np.uint64).reshape(-1))
    if len(doff) != n or len(dcap) != n:
        raise ValueError(f"dst_off and dst_cap must have one entry per {what}")
    if n and int((doff + dcap).max()) > out.numel():
        raise ValueError("a destination range reaches past the end of out")
    return doff, dcap


def compress_lz4block_dev(src, src_off, src_len, block_size: int = 1 << 16, hc_level: int = 0, out=None):
    """independent LZ4Block streams of bytes already in device memory, written on the device (b200lz4block_compress_dev):
    stream s is src[src_off[s] : src_off[s] + src_len[s]], byte for byte what compress_lz4block writes for the same bytes at
    the same 16-byte phase.  src: a uint8 CUDA tensor; src_off / src_len: host sequences; out: a uint8 CUDA tensor on src's
    device (default: a new one of the summed stream bounds).  Runs on torch's current stream and returns when the streams
    are written.  -> (out[:total], stream_off, stream_len), the last two np.uint64 arrays (where each stream lies in out)"""
    import torch
    off, ln = _dev_streams(src, src_off, src_len, "stream")
    L = N.lib()
    if L.b200lz4block_compress_bound(0, block_size) == 0:
        raise ValueError("blockSize must be >= 64 and <= 32 MiB")            # LZ4BlockOutputStream.java:58-66
    bound = sum(L.b200lz4block_compress_bound(int(n), block_size) for n in ln)
    if out is None:
        out = torch.empty(max(bound, 1), dtype=torch.uint8, device=src.device)
    elif not isinstance(out, torch.Tensor) or out.dtype != torch.uint8 or out.device != src.device or not out.is_contiguous():
        raise ValueError("out must be a contiguous uint8 tensor on src's device")
    stream_off, stream_len = np.zeros(len(ln), dtype=np.uint64), np.zeros(len(ln), dtype=np.uint64)
    r = L.b200lz4block_compress_dev(src.data_ptr(), off.ctypes.data, ln.ctypes.data, len(ln), out.data_ptr(), out.numel(),
                                    stream_off.ctypes.data, stream_len.ctypes.data, block_size, hc_level,
                                    torch.cuda.current_stream(src.device).cuda_stream)
    N.check(r)
    if r < 0:
        raise LZ4FrameError(int(r))
    return out[:r], stream_off, stream_len


def decompress_lz4block_dev(src, src_off, src_len, out, dst_off, dst_cap, stop_on_empty_block: bool = True):
    """many LZ4Block streams in device memory, each read as its own LZ4BlockInputStream(in, stopOnEmptyBlock) into device
    memory (b200lz4block_decompress_dev): stream s is src[src_off[s] : src_off[s] + src_len[s]], decoded to out[dst_off[s]:]
    with room for dst_cap[s] bytes.  No byte of the streams or the content crosses to the host.  src, out: contiguous uint8
    CUDA tensors on one device; the offsets and lengths: host sequences.  Runs on torch's current stream and returns when the
    results are on the host.  -> (result, src_consumed, content_len), np.int64 / np.uint64 / np.uint64 arrays: per stream
    what decompress_lz4block would return (decoded bytes, or -1 premature end, -2 corrupted, -9 room too small), how far it
    read (0 on an error), and what it decodes to when room is not the limit.  Raises only on a backend error."""
    import torch
    off, ln = _dev_streams(src, src_off, src_len, "stream")
    doff, dcap = _dev_ranges(src, out, dst_off, dst_cap, len(ln), "stream")
    result = np.zeros(len(ln), dtype=np.int64)
    consumed, content = np.zeros(len(ln), dtype=np.uint64), np.zeros(len(ln), dtype=np.uint64)
    N.check(N.lib().b200lz4block_decompress_dev(src.data_ptr(), off.ctypes.data, ln.ctypes.data, len(ln), out.data_ptr(),
                                                doff.ctypes.data, dcap.ctypes.data, int(bool(stop_on_empty_block)),
                                                result.ctypes.data, consumed.ctypes.data, content.ctypes.data,
                                                torch.cuda.current_stream(src.device).cuda_stream))
    return result, consumed, content


class LZ4BlockWriter(_Incremental):
    """ns LZ4Block streams written piece by piece in device memory, each one LZ4BlockOutputStream(out, blockSize, compressor,
    checksum, syncFlush=True) whose content arrives over time (b200lz4block_writer_*).  The writer is host data, whether each
    stream is closed; not thread-safe.

        with LZ4BlockWriter(ns, block_size=1 << 16) as wr:
            status, consumed, produced, need = wr.write(src, src_off, src_len, out, dst_off, dst_cap, op)

    A call takes whole blocks from the start of stream s's piece src[src_off[s] : src_off[s] + src_len[s]]; op[s] FLUSH also
    takes the rest as a short block (flush()), CLOSE then writes the empty end block (finish()).  The stream bytes go to
    out[dst_off[s] : dst_off[s] + produced[s]], never past dst_cap[s].  The rest of the piece, past consumed[s], must start
    stream s's next piece.  status[s]: MORE_INPUT (need[s]: the bytes missing for the next whole block), MORE_ROOM (need[s]:
    the room the next unit takes, 21 + its length), DONE (latched).  hc_level 0: the fast compressor, 1..17: HC.  src, out:
    contiguous uint8 CUDA tensors on one device; the rest: host sequences.  Runs on torch's current stream and returns when
    the results are on the host.  -> (status, consumed, produced, need): np.int32 / np.uint64 arrays."""
    _free, _what = "b200lz4block_writer_free", "writer"

    def __init__(self, ns: int, block_size: int = 1 << 16, hc_level: int = 0):
        import ctypes
        if not 64 <= block_size <= 1 << 25:
            raise ValueError("blockSize must be >= 64 and <= 32 MiB")            # LZ4BlockOutputStream.java:58-66
        self.ns = int(ns)
        err = ctypes.c_int(0)
        self._h = N.lib().b200lz4block_writer_create(self.ns, block_size, hc_level, ctypes.byref(err))
        if not self._h:
            N.check(err.value)
            raise MemoryError("b200lz4block_writer_create")

    def write(self, src, src_off, src_len, out, dst_off, dst_cap, op):
        return self._call(N.lib().b200lz4block_writer_write_dev, src, src_off, src_len, out, dst_off, dst_cap, op, "op")


class LZ4BlockReader(_Incremental):
    """ns LZ4Block streams read piece by piece in device memory, each one LZ4BlockInputStream(in, stopOnEmptyBlock) whose
    bytes arrive over time (b200lz4block_reader_*).  The reader is host data, each stream's latched status; not thread-safe.

        with LZ4BlockReader(ns) as rd:
            status, consumed, produced, need = rd.read(src, src_off, src_len, out, dst_off, dst_cap, eof)

    A call takes the complete blocks at the start of stream s's piece and decodes them into out[dst_off[s] : dst_off[s] +
    produced[s]], never past dst_cap[s].  The next piece of stream s must start at byte consumed[s] of this one.  status[s]:
    MORE_INPUT (need[s]: bytes the next unit takes), MORE_ROOM (need[s]: the next block's original length), DONE, or -1
    (premature end) / -2 (corrupted), after the content in front of the failing unit was delivered.  eof[s] true: the piece
    ends the stream.  DONE and errors are latched.  src, out: contiguous uint8 CUDA tensors on one device; the rest: host
    sequences.  Runs on torch's current stream and returns when the results are on the host.  -> (status, consumed,
    produced, need): np.int32 / np.uint64 arrays."""
    _free, _what = "b200lz4block_reader_free", "reader"

    def __init__(self, ns: int, stop_on_empty_block: bool = True):
        import ctypes
        err = ctypes.c_int(0)
        self.ns = int(ns)
        self._h = N.lib().b200lz4block_reader_create(self.ns, int(bool(stop_on_empty_block)), ctypes.byref(err))
        if not self._h:
            N.check(err.value)
            raise MemoryError("b200lz4block_reader_create")

    def read(self, src, src_off, src_len, out, dst_off, dst_cap, eof):
        return self._call(N.lib().b200lz4block_reader_read_dev, src, src_off, src_len, out, dst_off, dst_cap, eof, "eof")


# ---- LZ4CompressorWithLength / LZ4DecompressorWithLength
def compress_with_length(src) -> bytes:
    s = _view(src)
    cap = len(s) + len(s) // 255 + 16 + 4
    out = np.empty(cap, dtype=np.uint8)
    r = N.lib().b200lz4_compress_with_length(s.ctypes.data if len(s) else None, out.ctypes.data, len(s), cap)
    N.check(r)
    if r <= 0:
        from .lz4 import LZ4Exception
        raise LZ4Exception("maxDestLen is too small")
    return out[:r].tobytes()


def decompress_with_length(src, safe: bool = False) -> bytes:
    """LZ4DecompressorWithLength.decompress(src).  safe=False: the LZ4FastDecompressor flavour, src[4:] is read as far as the
    declared length needs; safe=True: the LZ4SafeDecompressor flavour of lz4-java 1.8 (LZ4DecompressorWithLength.java:148-154),
    src is exactly one record and the decoded bytes are returned, at most the declared length of them."""
    s = _view(src)
    from .lz4 import LZ4Exception
    if len(s) < 4:
        raise LZ4Exception("Error decoding offset 0 of input buffer")
    n = N.lib().b200lz4_decompressed_length(s.ctypes.data)
    if n < 0:
        raise LZ4Exception("negative length")
    out = np.empty(max(n, 1), dtype=np.uint8)
    if safe:
        r = N.lib().b200lz4_decompress_with_length_safe(s.ctypes.data, len(s), out.ctypes.data, n)
        N.check(r)
        if r < 0:
            raise LZ4Exception("Error decoding offset " + str(4 - r) + " of input buffer")   # LZ4JNISafeDecompressor.java:39-41
        return out[:r].tobytes()
    r = N.lib().b200lz4_decompress_with_length(s.ctypes.data, len(s), out.ctypes.data, n)
    N.check(r)
    if r < 0:
        raise LZ4Exception("Error decoding offset " + str(-r) + " of input buffer")
    return out[:n].tobytes()


def compress_with_length_dev(src, src_off, src_len, hc_level: int = 0, out=None):
    """independent length-prefixed records (LZ4CompressorWithLength) of bytes already in device memory, written on the device
    (b200lz4_compress_with_length_dev): record r is src[src_off[r] : src_off[r] + src_len[r]]; with hc_level 0 it is byte for
    byte what compress_with_length writes for the same bytes at the same 16-byte phase, with 1..17 the length and an
    LZ4_compress_HC block of that level.  src: a uint8 CUDA tensor; src_off / src_len: host sequences; out: a uint8 CUDA tensor
    on src's device (default: a new one of the summed record bounds).  Runs on torch's current stream and returns when the
    records are written.  -> (out[:total], rec_off, rec_len), the last two np.uint64 arrays (where each record lies in out)"""
    import torch
    off, ln = _dev_streams(src, src_off, src_len, "record")
    if len(ln) and int(ln.max()) > 0x7E000000:
        raise ValueError("a record is at most 0x7E000000 bytes (LZ4_MAX_INPUT_SIZE)")
    bound = int((ln + ln // 255 + 16 + 4).sum())
    if out is None:
        out = torch.empty(max(bound, 1), dtype=torch.uint8, device=src.device)
    elif not isinstance(out, torch.Tensor) or out.dtype != torch.uint8 or out.device != src.device or not out.is_contiguous():
        raise ValueError("out must be a contiguous uint8 tensor on src's device")
    rec_off, rec_len = np.zeros(len(ln), dtype=np.uint64), np.zeros(len(ln), dtype=np.uint64)
    r = N.lib().b200lz4_compress_with_length_dev(src.data_ptr(), off.ctypes.data, ln.ctypes.data, len(ln), out.data_ptr(),
                                                 out.numel(), rec_off.ctypes.data, rec_len.ctypes.data, hc_level,
                                                 torch.cuda.current_stream(src.device).cuda_stream)
    N.check(r)
    if r < 0:
        raise LZ4FrameError(int(r))
    return out[:r], rec_off, rec_len


def decompress_with_length_dev(src, src_off, src_len, out, dst_off, dst_cap, safe: bool = False):
    """many length-prefixed records in device memory, each read by LZ4DecompressorWithLength into device memory
    (b200lz4_decompress_with_length_dev): record r is src[src_off[r] : src_off[r] + src_len[r]], decoded to out[dst_off[r]:]
    with room for dst_cap[r] bytes.  safe: the LZ4SafeDecompressor flavour (the record is exactly src_len[r] bytes) rather
    than the LZ4FastDecompressor one.  No byte of the records or the content crosses to the host.  src, out: contiguous uint8
    CUDA tensors on one device; the offsets and lengths: host sequences.  Runs on torch's current stream and returns when the
    results are on the host.  -> (result, orig_len), np.int64 arrays: per record what decompress_with_length's host call
    returns (fast: the bytes read including the prefix; safe: the bytes decoded; < 0 on an error), and the declared length
    (-1 when the record is shorter than 4 bytes).  Raises only on a backend error."""
    import torch
    off, ln = _dev_streams(src, src_off, src_len, "record")
    doff, dcap = _dev_ranges(src, out, dst_off, dst_cap, len(ln), "record")
    result, orig_len = np.zeros(len(ln), dtype=np.int64), np.zeros(len(ln), dtype=np.int64)
    N.check(N.lib().b200lz4_decompress_with_length_dev(src.data_ptr(), off.ctypes.data, ln.ctypes.data, len(ln), out.data_ptr(),
                                                       doff.ctypes.data, dcap.ctypes.data, int(bool(safe)), result.ctypes.data,
                                                       orig_len.ctypes.data, torch.cuda.current_stream(src.device).cuda_stream))
    return result, orig_len
