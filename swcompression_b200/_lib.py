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
        L.swc_lz4_compress.argtypes = [vp, sz, i32, i32, i32, i32, C.c_int64, vp, sz, i32, u32, C.POINTER(vp), szp]
        L.swc_lz4_compress_batch_scratch_bytes.restype = C.c_size_t
        L.swc_lz4_compress_batch_scratch_bytes.argtypes = [C.c_uint64, C.c_uint64]
        L.swc_lz4_block_compress_batch.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, u64, vp, sz, vp]
        L.swc_bzip2_decompress.argtypes = [vp, sz, sz, C.POINTER(vp), szp, szp]
        L.swc_bzip2_multi_decompress.argtypes = [vp, sz, C.POINTER(vp), szp, C.POINTER(vp), szp]
        L.swc_bzip2_decompress_batch.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, u64, vp]
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
        L.swc_zlib_unarchive.argtypes = [vp, sz, C.POINTER(vp), szp]
        L.swc_xz_unarchive.argtypes = [vp, sz, C.POINTER(vp), szp]
        L.swc_xz_split_unarchive.argtypes = [vp, sz, C.POINTER(vp), szp, C.POINTER(vp), szp]
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
