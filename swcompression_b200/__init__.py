"""swcompression_b200 — H100-native batched decompression engine behind SWCompression's decode API.

`api` mirrors the reference's Swift types (Deflate, BZip2, LZMA, LZMA2, LZ4, GzipArchive, ZlibArchive, XZArchive);
`batch` exposes the batched C-ABI calls on torch CUDA tensors (device memory, streams) for bulk work and benchmarks.
All compute runs in hand-written sm_90a kernels inside libswcgpu.so; there is no CPU fallback."""
from .api import (BZip2, Deflate, ExtraField, GzipArchive, GzipHeader, ZlibHeader, LZ4, LZMA, LZMA2, LZMAProperties, XZArchive, ZlibArchive, ZipContainer, ZipEntry, ZipEntryInfo,  # noqa: F401
                  TarContainer, TarEntry, TarEntryInfo,
                  adler32, bzip2_crc32, crc32, crc64, sha256, xxh32)
from .errors import (BZip2Error, DataError, DeflateError, EngineError, GzipError, LZMA2Error, LZMAError,  # noqa: F401
                     TarError, ZipError,
                     SWCompressionError, XZError, ZlibError)

__all__ = ["Deflate", "BZip2", "LZMA", "LZMA2", "LZMAProperties", "LZ4", "GzipArchive", "GzipHeader", "ZlibArchive", "ZlibHeader", "XZArchive", "ZipContainer", "TarContainer"]
