"""ctypes loader for libswcgpu.so (built in-tree by __graft_entry__.build() / csrc/Makefile).

The product path has no CPU fallback: if the library is missing, or no CUDA device is visible, calls fail loudly."""
import ctypes as C
import os
import re
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.environ.get("SWCGPU_SO") or os.path.join(_HERE, "libswcgpu.so")      # SWCGPU_SO: A/B runs of kernel variants
HEADER = os.path.join(os.path.dirname(_HERE), "include", "swcgpu.h")
_LIB = None

u8p = C.POINTER(C.c_uint8)
u64p = C.POINTER(C.c_uint64)
szp = C.POINTER(C.c_size_t)


def build(force=False, verbose=False):
    """Compile every CUDA source for sm_90a (nvcc cross-compiles without a GPU)."""
    csrc = os.path.join(_HERE, "csrc")
    cmd = ["make", "-C", csrc, "-j8"] + (["-B"] if force else [])
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if verbose or res.returncode:
        print(res.stdout)
    if res.returncode:
        raise RuntimeError("libswcgpu build failed")
    return SO_PATH


def declared_symbols():
    """Every function include/swcgpu.h declares (used by the CPU-side ABI test)."""
    with open(HEADER) as f:
        txt = f.read()
    return sorted(set(re.findall(r"\b(swc_[a-z0-9_]+)\s*\(", txt)))


class Lz4FrameInfo(C.Structure):
    """swc_lz4_frame_info (include/swcgpu.h)"""
    _fields_ = [("status", C.c_int32), ("kind", C.c_uint32), ("n_blocks", C.c_uint64), ("flags", C.c_uint32),
                ("max_block_size", C.c_uint32), ("content_size", C.c_uint64), ("frame_start", C.c_uint64),
                ("frame_end", C.c_uint64)]


class TarEntry(C.Structure):
    """swc_tar_entry (include/swcgpu.h)"""
    _fields_ = ([(f, C.c_uint64) for f in ("header_off", "data_off")]
                + [(f, C.c_int64) for f in ("size", "open_size", "mode", "uid", "gid", "dev_major", "dev_minor", "mtime",
                                            "atime", "ctime")]
                + [(f, C.c_uint64) for f in ("name_off", "name_len", "prefix_off", "prefix_len", "link_off", "link_len",
                                             "uname_off", "uname_len", "gname_off", "gname_len", "charset_off",
                                             "charset_len", "comment_off", "comment_len")]
                + [("pax_time_off", C.c_uint64 * 6), ("pax_time_len", C.c_uint64 * 6)]
                + [(f, C.c_uint64) for f in ("local_off", "local_len", "global_off", "global_len")]
                + [("present", C.c_uint32), ("typeflag", C.c_uint8), ("reserved", C.c_uint8 * 3)])


def tar_record(e):
    """swc_tar_entry -> dict of its fields (arrays as tuples, the reserved bytes dropped)"""
    out = {}
    for name, _ in TarEntry._fields_:
        if name != "reserved":
            v = getattr(e, name)
            out[name] = tuple(v) if hasattr(v, "__len__") else int(v)
    return out


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(SO_PATH):
            raise RuntimeError(f"{SO_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                               "(libswcgpu has no CPU fallback)")
        L = C.CDLL(SO_PATH)
        L.swc_last_error_string.restype = C.c_char_p
        L.swc_status_name.restype = C.c_char_p
        L.swc_status_name.argtypes = [C.c_int32]
        L.swc_alloc.restype = C.c_void_p
        L.swc_alloc_pinned.restype = C.c_void_p
        L.swc_alloc_pinned.argtypes = [C.c_size_t]
        L.swc_free.argtypes = [C.c_void_p]
        L.swc_free_pinned.argtypes = [C.c_void_p]
        L.swc_kernel_launches.restype = C.c_uint64
        L.swc_deflate_batch_scratch_bytes.restype = C.c_size_t
        L.swc_deflate_batch_scratch_bytes.argtypes = [C.c_uint64, C.c_uint64]
        vp, sz, u64, i32, u32 = C.c_void_p, C.c_size_t, C.c_uint64, C.c_int32, C.c_uint32
        L.swc_deflate_decompress.argtypes = [vp, sz, sz, C.POINTER(vp), szp, szp]
        L.swc_deflate_decompress_batch.argtypes = [vp, vp, vp, vp, vp, vp, vp, u64, vp, vp, vp, u64, vp, sz, vp]
        L.swc_deflate_decompress_batch_host.argtypes = [vp, vp, vp, u64, vp, vp, vp, u64, vp, vp, vp, u64]
        L.swc_lz4_decompress.argtypes = [vp, sz, vp, sz, i32, u32, C.POINTER(vp), szp, szp]
        L.swc_lz4_multi_decompress.argtypes = [vp, sz, vp, sz, i32, u32, C.POINTER(vp), szp, C.POINTER(vp), szp]
        L.swc_lz4_block_decompress_batch.argtypes = [vp, vp, vp, vp, u64, vp, vp, vp, vp, vp, u64, vp]
        L.swc_lz4_block_decompress_batch_host.argtypes = [vp, vp, vp, u64, vp, vp, vp, u64, vp, vp, u64]
        L.swc_lz4_frame_batch_scratch_bytes.restype = C.c_size_t
        L.swc_lz4_frame_batch_scratch_bytes.argtypes = [u64, u64, u64]
        L.swc_lz4_frame_decompress_batch.argtypes = [vp, vp, vp, vp, u64, i32, u32, vp, vp, vp, vp, vp, vp, u64, u64, vp, sz, vp]
        L.swc_lz4_frame_info_batch.argtypes = [vp, vp, vp, i32, i32, u32, vp, u64, vp]
        L.swc_lz4_compress.argtypes = [vp, sz, i32, i32, i32, i32, C.c_int64, vp, sz, i32, u32, C.POINTER(vp), szp]
        L.swc_lz4_compress_batch_scratch_bytes.restype = C.c_size_t
        L.swc_lz4_compress_batch_scratch_bytes.argtypes = [C.c_uint64, C.c_uint64]
        L.swc_lz4_block_compress_batch.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, u64, vp, sz, vp]
        L.swc_lz4_frame_compress_max_bytes.restype = C.c_size_t
        L.swc_lz4_frame_compress_max_bytes.argtypes = [u64, C.c_int64, i32, i32, i32, i32]
        L.swc_lz4_frame_compress_batch_scratch_bytes.restype = C.c_size_t
        L.swc_lz4_frame_compress_batch_scratch_bytes.argtypes = [u64, u64, C.c_int64, i32, u64]
        L.swc_lz4_frame_compress_batch.argtypes = [vp, vp, vp, i32, i32, i32, i32, C.c_int64, vp, u64, i32, u32, vp, vp, vp,
                                                   vp, vp, u64, u64, vp, sz, vp]
        L.swc_deflate_compress.argtypes = [vp, sz, C.POINTER(vp), szp]
        L.swc_zlib_archive.argtypes = [vp, sz, C.POINTER(vp), szp]
        L.swc_gzip_archive.argtypes = [vp, sz, vp, C.POINTER(vp), szp]
        L.swc_deflate_compress_batch_scratch_bytes.restype = C.c_size_t
        L.swc_deflate_compress_batch_scratch_bytes.argtypes = [C.c_uint64, C.c_uint64]
        L.swc_deflate_compress_batch.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, u64, vp, sz, vp]
        L.swc_gzip_archive_header.argtypes = [vp, vp, sz, szp]
        L.swc_gzip_archive_max_bytes.restype = C.c_size_t
        L.swc_gzip_archive_max_bytes.argtypes = [u64, u64]
        L.swc_zlib_archive_max_bytes.restype = C.c_size_t
        L.swc_zlib_archive_max_bytes.argtypes = [u64]
        L.swc_archive_compress_batch_scratch_bytes.restype = C.c_size_t
        L.swc_archive_compress_batch_scratch_bytes.argtypes = [u64, u64]
        L.swc_gzip_archive_batch.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, u64, u64, vp, sz, vp]
        L.swc_zlib_archive_batch.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, u64, u64, vp, sz, vp]
        L.swc_bzip2_compress.argtypes = [vp, sz, i32, C.POINTER(vp), szp]
        L.swc_bzip2_compress_max_bytes.restype = C.c_size_t
        L.swc_bzip2_compress_max_bytes.argtypes = [C.c_uint64, i32]
        L.swc_bzip2_compress_batch_scratch_bytes.restype = C.c_size_t
        L.swc_bzip2_compress_batch_scratch_bytes.argtypes = [C.c_uint64, C.c_uint64, i32]
        L.swc_bzip2_compress_batch.argtypes = [vp, vp, vp, i32, vp, vp, vp, vp, vp, u64, vp, sz, vp]
        L.swc_bzip2_decompress.argtypes = [vp, sz, sz, C.POINTER(vp), szp, szp]
        L.swc_bzip2_multi_decompress.argtypes = [vp, sz, C.POINTER(vp), szp, C.POINTER(vp), szp]
        L.swc_bzip2_decompress_batch.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, u64, vp]
        L.swc_bzip2_stream_batch_scratch_bytes.restype = C.c_size_t
        L.swc_bzip2_stream_batch_scratch_bytes.argtypes = [u64, u64, u64]
        L.swc_bzip2_stream_decompress_batch.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, u64, u64, vp, sz, vp]
        L.swc_bzip2_multi_decompress_batch.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, u64, u64, vp, sz, vp]
        L.swc_lzma_decompress.argtypes = [vp, sz, C.POINTER(vp), szp, szp]
        L.swc_lzma_decompress_raw.argtypes = [vp, sz, i32, i32, i32, C.c_int64, C.c_int64, C.POINTER(vp), szp, szp]
        L.swc_lzma2_decompress.argtypes = [vp, sz, C.POINTER(vp), szp, szp]
        L.swc_lzma2_decompress_batch.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, u64, vp]
        L.swc_gzip_unarchive.argtypes = [vp, sz, C.POINTER(vp), szp, szp]
        L.swc_gzip_multi_unarchive.argtypes = [vp, sz, C.POINTER(vp), szp, C.POINTER(vp), szp]
        L.swc_gzip_multi_unarchive_members.argtypes = [vp, sz, C.POINTER(vp), szp, C.POINTER(vp), C.POINTER(vp), szp]
        L.swc_gzip_header_parse.argtypes = [vp, sz, sz, vp]
        L.swc_zlib_header_parse.argtypes = [vp, sz, vp]
        L.swc_lzma_decompress_batch.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, u64, vp]
        L.swc_crc32_batch.argtypes = [vp, vp, vp, vp, vp, u64, vp]
        L.swc_zip_open.argtypes = [vp, sz, C.POINTER(vp), szp, C.POINTER(vp), szp]
        L.swc_zip_info.argtypes = [vp, sz, C.POINTER(vp), szp]
        L.swc_xxh32_batch.argtypes = [vp, vp, vp, vp, u64, vp]
        L.swc_adler32_batch.argtypes = [vp, vp, vp, vp, vp, u64, vp]
        L.swc_unarchive_batch_scratch_bytes.restype = C.c_size_t
        L.swc_unarchive_batch_scratch_bytes.argtypes = [C.c_uint64, C.c_uint64]
        L.swc_gzip_unarchive_batch.argtypes = [vp, vp, vp, vp, vp, vp, u64, vp, vp, vp, vp, u64, vp, sz, vp]
        L.swc_zlib_unarchive_batch.argtypes = [vp, vp, vp, vp, vp, vp, u64, vp, vp, vp, u64, vp, sz, vp]
        L.swc_gzip_member_batch_scratch_bytes.restype = C.c_size_t
        L.swc_gzip_member_batch_scratch_bytes.argtypes = [u64, u64, u64]
        L.swc_gzip_multi_unarchive_batch.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, u64, u64, vp, sz,
                                                     vp]
        L.swc_zlib_unarchive.argtypes = [vp, sz, C.POINTER(vp), szp]
        L.swc_xz_unarchive.argtypes = [vp, sz, C.POINTER(vp), szp]
        L.swc_xz_unarchive_batch.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, u64, vp]
        L.swc_xz_block_batch_scratch_bytes.restype = C.c_size_t
        L.swc_xz_block_batch_scratch_bytes.argtypes = [u64, u64]
        L.swc_xz_block_unarchive_batch.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, u64, u64, vp, sz, vp]
        L.swc_xz_occupancy.argtypes = [vp, vp]
        L.swc_crc64_batch.argtypes = [vp, vp, vp, vp, vp, u64, vp]
        L.swc_xz_split_unarchive.argtypes = [vp, sz, C.POINTER(vp), szp, C.POINTER(vp), szp]
        L.swc_tar_walk_batch.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, u64, vp]
        L.swc_tar_info.argtypes = [vp, sz, C.POINTER(vp), szp]
        L.swc_tar_open.argtypes = [vp, sz, C.POINTER(vp), szp]
        L.swc_tar_format.argtypes = [vp, sz, C.POINTER(i32)]
        for name in ("swc_crc32", "swc_bzip2_crc32", "swc_adler32", "swc_xxh32", "swc_crc64", "swc_sha256"):
            getattr(L, name).argtypes = [vp, sz, vp]
        _LIB = L
    return _LIB


def status_name(code):
    return lib().swc_status_name(code).decode()


def last_error():
    return lib().swc_last_error_string().decode()


def inbuf(data):
    """bytes-like -> (ctypes pointer, length); keeps a reference alive through the returned object."""
    b = data if isinstance(data, bytes) else bytes(data)
    return C.c_char_p(b or b"\0"), len(b)          # zero-copy: c_char_p keeps `b` alive and the library only reads it


def take(ptr, n):
    """Copy an swc_alloc'ed result into bytes and free it."""
    if ptr.value and n.value:
        # string_at() takes a C int; results of 2 GiB and more go through a buffer view instead
        out = C.string_at(ptr.value, n.value) if n.value < (1 << 31) else bytes((C.c_char * n.value).from_address(ptr.value))
    else:
        out = b""
    if ptr.value:
        lib().swc_free(ptr)
    return out


def take_sizes(ptr, n):
    vals = []
    if ptr.value:
        arr = C.cast(ptr, szp)
        vals = [arr[i] for i in range(n.value)]
        lib().swc_free(ptr)
    return vals
