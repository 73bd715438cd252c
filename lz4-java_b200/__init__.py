"""lz4-java_b200 — H100-native LZ4 block codec + XXHash behind the net.jpountz API surface.

The directory name carries a hyphen (it mirrors the reference repo's name), so it is imported
through the root-level alias module `lz4java_b200`.
"""
from . import _native
from ._native import B200Error
from .lz4 import (LZ4Factory, LZ4Compressor, LZ4FastDecompressor, LZ4SafeDecompressor, LZ4Exception,
                  max_compressed_length)
from .xxhash import XXHashFactory, XXHash32, XXHash64, StreamingXXHash32, StreamingXXHash64
from . import batch
from . import frame
from .frame import (decompress_frames, expected_content_size, compress_frame, compress_frames_dev, decompress_frames_dev,
                    decompress_frame_streams_dev, FrameReader, FrameWriter, compress_lz4block,
                    decompress_lz4block, compress_lz4block_dev, decompress_lz4block_dev, LZ4BlockWriter, LZ4BlockReader,
                    compress_with_length, decompress_with_length,
                    compress_with_length_dev, decompress_with_length_dev, LZ4FrameError)

__all__ = ["LZ4Factory", "LZ4Compressor", "LZ4FastDecompressor", "LZ4SafeDecompressor", "LZ4Exception",
           "XXHashFactory", "XXHash32", "XXHash64", "StreamingXXHash32", "StreamingXXHash64",
           "max_compressed_length", "batch", "B200Error", "frame", "decompress_frames", "compress_frame", "compress_frames_dev", "decompress_frames_dev",
           "decompress_frame_streams_dev", "FrameReader", "FrameWriter", "compress_lz4block",
           "decompress_lz4block", "compress_lz4block_dev", "decompress_lz4block_dev", "LZ4BlockWriter", "LZ4BlockReader",
           "expected_content_size", "compress_with_length",
           "decompress_with_length", "compress_with_length_dev", "decompress_with_length_dev", "LZ4FrameError"]
