"""Batched calls on torch CUDA tensors (torch is plumbing here: device memory + streams).

A `Batch` packs n compressed units into one contiguous device buffer (16-byte aligned unit starts) with the offset /
length tables the C ABI takes, and owns the output buffer + result tables.  `run()` launches the kernels on the
current torch stream through libswcgpu's *_batch entry points (device pointers, asynchronous)."""
import ctypes as C

import numpy as np
import torch

from . import _lib


def _align(v, a=16):
    return (v + a - 1) // a * a


# the most scratch a compress Batch allocates: past it the library runs the batch in slices that fit
COMPRESS_SCRATCH_LIMIT = 16 << 30

# the frame options of LZ4.compress(data:) (LZ4+Compress.swift:16-19), the defaults of an 'lz4_frame_compress' Batch
LZ4_FRAME_DEFAULTS = dict(independentBlocks=True, blockChecksums=False, contentChecksum=True, contentSize=False)
LZ4_FRAME_BLOCK_SIZE = 4 << 20


def compress_scratch_bytes(codec, in_len, dict_len=None, block_size=1):
    """The scratch that runs a compress batch of units of `in_len` bytes in one slice, capped at COMPRESS_SCRATCH_LIMIT.
    `dict_len` are the LZ4 units' dictionary window lengths (None: no dictionaries)."""
    L = _lib.lib()
    lens = np.asarray(in_len, dtype=np.uint64)
    n, total = len(lens), int(lens.sum())
    if codec == "lz4_block_compress":
        if dict_len is not None:
            total += int(np.minimum(np.asarray(dict_len, dtype=np.uint64), np.uint64(65536)).sum())
        nbytes = L.swc_lz4_compress_batch_scratch_bytes(n, total)
    elif codec == "deflate_compress":
        nbytes = L.swc_deflate_compress_batch_scratch_bytes(n, total)
    elif codec == "bzip2_compress":
        nbytes = L.swc_bzip2_compress_batch_scratch_bytes(n, total, max(1, min(9, int(block_size))))
    elif codec in ("gzip_archive", "zlib_archive"):
        nbytes = L.swc_archive_compress_batch_scratch_bytes(n, total)
    else:
        raise ValueError(codec)
    return min(nbytes, COMPRESS_SCRATCH_LIMIT)


def pack_units(units, align=16):
    """list of bytes -> (uint8 numpy buffer, offsets u64, lengths u64)"""
    lens = np.fromiter((len(u) for u in units), dtype=np.uint64, count=len(units))
    padded = (lens + np.uint64(align - 1)) // np.uint64(align) * np.uint64(align)
    offs = np.zeros(len(units), dtype=np.uint64)
    if len(units) > 1:
        offs[1:] = np.cumsum(padded[:-1])
    total = int(padded.sum()) if len(units) else 0
    buf = np.zeros(total + 64, dtype=np.uint8)
    for u, o in zip(units, offs):
        buf[int(o):int(o) + len(u)] = np.frombuffer(u, dtype=np.uint8)
    return buf, offs, lens


class Batch:
    """Device-resident batch for one codec ('deflate', 'lz4_block', 'bzip2', 'bzip2_stream', 'bzip2_multi', 'lzma2', 'gzip', 'zlib', 'xz',
    'xz_blocks', 'gzip_multi', 'lz4_frame', 'lz4_block_compress', 'lz4_frame_compress', 'deflate_compress', 'gzip_archive',
    'zlib_archive', 'bzip2_compress', 'tar').

    'tar' walks one TAR archive per unit (TarContainer.open / info / formatOf, TarContainer.swift:36-261) into a table of
    swc_tar_entry records; `out_cap` is each unit's record capacity (None: in_len // 512 + 1).  results() gives info's
    status and the record count, tar_results() every column, records(i) / entries(i) unit i's records.  Batch.tar_of
    walks another batch's outputs where they lie.  run() reads nothing back (it can be captured in a CUDA graph).

    'bzip2' and 'bzip2_stream' both decode the first .bz2 stream of each unit (BZip2.decompress(data:), BZip2.swift:50-95)
    with the same statuses, bytes and consumed bits.  'bzip2' gives each stream one warp and reads the capacities back
    first; 'bzip2_stream' decodes the blocks of all streams side by side and, on overflow of a stream whose blocks
    validated, reports its exact size.  `max_blocks` is the capacity of its block table: with it the batch owns a scratch
    of swc_bzip2_stream_batch_scratch_bytes (capped at `scratch_bytes`, which the library then runs in slices) and run()
    reads nothing back (it can be captured in a CUDA graph).  None lets the library count the blocks first (one
    synchronisation) and use its pool, or `scratch_bytes` of caller scratch.
    'bzip2_multi' decodes every stream of each unit (BZip2.multiDecompress, BZip2.swift:40-48) with the blocks of all
    streams of all units side by side; results() gives the status, the streams' total size and 0 consumed bytes, streams(i)
    unit i as multiDecompress returns it, stream_table(i) its stream ends and starts, and parallel_streams() how many
    streams of each unit the block stage gave (the rest took the stream kernel).  `stream_cap` is each unit's stream table
    capacity (None: in_len // 14 + 1, always enough); `max_blocks` and `scratch_bytes` work as for 'bzip2_stream'.

    'gzip' / 'zlib' decode one archive per unit (GzipArchive.unarchive, GzipArchive.swift:38-47, 79-100 / ZlibArchive.unarchive,
    ZlibArchive.swift:25-42): the first member only, whose status, size and consumed bytes results() returns.  With
    `headers=True` a 'gzip' batch also fills a device array of swc_gzip_header, which gzip_headers() reads back.
    'xz' decodes one whole .xz file per unit (XZArchive.unarchive, XZArchive.swift:27-50): every stream and block, the outputs
    concatenated.  It takes no scratch and no aux, and reports no consumed bytes (results() gives zeros in that column).
    'xz_blocks' gives the same statuses, sizes and bytes as 'xz' with the blocks of every file decoded side by side (the
    streams' indexes place them); parallel_blocks() tells how many blocks of each unit took that path (0: the whole unit
    was decoded as 'xz' decodes it).  `max_blocks` is the capacity of its block table: with it the batch owns a scratch of
    swc_xz_block_batch_scratch_bytes and run() reads nothing back (it can be captured in a CUDA graph).  None lets the
    library count the blocks first (one synchronisation) and use its pool.
    'gzip_multi' decodes every member of each unit (GzipArchive.multiUnarchive, GzipArchive.swift:52-100) with the members
    of all units side by side; results() gives the status, the members' total size and the consumed bytes (the end of the
    last member returned), members(i) unit i's [GzipArchive.Member] and parallel_members() how many members of each unit
    the parallel spans gave (the rest took the sequential walk).  `member_cap` is each unit's member table capacity (None:
    in_len // 20 + 1, always enough).  `max_members` is the capacity of the candidate table: with it the batch owns a
    scratch of swc_gzip_member_batch_scratch_bytes (or `scratch_bytes`) and run() reads nothing back (it can be captured in
    a CUDA graph).  None lets the library count the candidates first (one synchronisation) and use its pool, or
    `scratch_bytes` of caller scratch.

    'lz4_frame' decodes the first LZ4 frame of each unit (LZ4.decompress(data:dictionary:dictionaryID:), LZ4.swift:73-91):
    `aux` is the dictionary's bytes (None: nil), `dict_id` the dictionary ID (None: nil), and results() gives the consumed
    bytes.  `max_blocks` is the capacity of the batch's block table; with it the batch owns a scratch sized for it and run()
    reads nothing back (it can be captured in a CUDA graph).  None lets the library count the blocks first (one
    synchronisation) and use its pool.

    'lz4_block_compress' compresses each unit into a raw LZ4 block (LZ4+Compress.swift:156-277); `aux` is then an optional
    (dict_off, dict_len) pair of u64 arrays placing each unit's dictionary window inside `in_buf`.
    'lz4_frame_compress' compresses each unit into a whole LZ4 frame, as LZ4.compress(data:independentBlocks:blockChecksums:
    contentChecksum:contentSize:blockSize:dictionary:dictionaryID:) (LZ4+Compress.swift:47-154) does: `frame_flags` takes
    any of LZ4_FRAME_DEFAULTS' keys, `block_size` is the block size (default 4 MiB), `aux` the dictionary's bytes (None: nil)
    and `dict_id` the dictionary ID (None: nil); every option applies to the whole batch.  api.LZ4.max_compressed_size
    gives the output a unit may need.  `max_blocks` works as for 'lz4_frame' (None: the library counts the blocks first,
    one synchronisation); results() gives 0 consumed bytes.
    'deflate_compress' compresses each unit into a raw Deflate stream (Deflate.compress, Deflate+Compress.swift:22-42); a
    unit of n bytes needs at most (9 n + 17) // 8 bytes of output.
    'gzip_archive' / 'zlib_archive' compress each unit into a whole gzip member / zlib stream, as GzipArchive.archive
    (GzipArchive.swift:126-241) / ZlibArchive.archive (ZlibArchive.swift:54-70) do.  `gzip_options` is one dict of
    GzipArchive.archive's keywords for the whole batch, or a list of n of them (identical headers are uploaded once);
    api.GzipArchive.max_archive_size / api.ZlibArchive.max_archive_size give the output a unit may need.
    `max_in_bytes` bounds the batch's input: the batch owns a scratch sized for it and run() reads nothing back (it can be
    captured in a CUDA graph); units past the bound report SWC_ERR_UNSUPPORTED.  None lets the library read the lengths
    back first (one synchronisation) and run in slices of the scratch.
    'bzip2_compress' compresses each unit into a complete .bz2 stream (BZip2.compress(data:blockSize:),
    BZip2+Compress.swift:44-74) with raw blocks of 80 000 x `block_size` bytes; api.BZip2.max_compressed_size gives the
    output a unit may need.
    The compress codecs pass a caller scratch that runs the batch in one slice (compress_scratch_bytes(...) for the raw
    codecs) up to COMPRESS_SCRATCH_LIMIT; `scratch_bytes` caps it lower (the library then runs the batch in slices; a scratch that
    cannot hold the largest unit fails the run with SWC_ERR_INVALID_ARG)."""

    def __init__(self, codec, in_buf, in_off, in_len, out_cap, device="cuda:0", aux=None, scratch_bytes=None, block_size=None,
                 headers=False, dict_id=None, max_blocks=None, frame_flags=None, gzip_options=None, max_in_bytes=None,
                 max_members=None, member_cap=None, stream_cap=None):
        self.codec = codec
        self.device = torch.device(device)
        self.n = len(in_off)
        if codec == "tar":
            t = lambda a: torch.from_numpy(np.ascontiguousarray(np.asarray(a, dtype=np.uint64)).view(np.int64)).to(self.device)
            lens = np.asarray(in_len, dtype=np.uint64)
            self._init_tar(torch.from_numpy(np.array(in_buf, dtype=np.uint8)).to(self.device), t(in_off), t(lens),
                           lens // np.uint64(512) + np.uint64(1) if out_cap is None else out_cap)
            return
        caps = np.asarray(out_cap, dtype=np.uint64)
        if caps.ndim == 0:
            caps = np.full(self.n, int(caps), dtype=np.uint64)
        pc = (caps + np.uint64(15)) // np.uint64(16) * np.uint64(16)
        out_off = np.zeros(self.n, dtype=np.uint64)
        if self.n > 1:
            out_off[1:] = np.cumsum(pc[:-1])
        self.out_total = int(pc.sum())
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.int64) if a.dtype == np.uint64 else a).to(self.device)
        self.d_in = t(np.asarray(in_buf, dtype=np.uint8))
        self.d_in_off, self.d_in_len = t(np.asarray(in_off, dtype=np.uint64)), t(np.asarray(in_len, dtype=np.uint64))
        self.d_out_off, self.d_out_cap = t(out_off), t(caps)
        self.h_out_off, self.h_out_cap = out_off, caps
        self.d_out = torch.empty(self.out_total + 64, dtype=torch.uint8, device=self.device)
        self.d_out_len = torch.zeros(self.n, dtype=torch.int64, device=self.device)
        self.d_consumed = torch.zeros(self.n, dtype=torch.int64, device=self.device)
        self.d_status = torch.full((self.n,), -1, dtype=torch.int32, device=self.device)
        self.d_scratch = None
        self.d_dict_off = self.d_dict_len = None
        self.block_size = int(block_size) if block_size is not None else LZ4_FRAME_BLOCK_SIZE if codec == "lz4_frame_compress" else 1
        self.dict_id, self.max_blocks = dict_id, 0 if max_blocks is None else int(max_blocks)
        if codec in ("bzip2_stream", "bzip2_multi"):
            self.d_aux = None
            if codec == "bzip2_multi":
                self.d_parallel = torch.zeros(self.n, dtype=torch.int32, device=self.device)
                scap = np.asarray(in_len, dtype=np.uint64) // np.uint64(14) + np.uint64(1) if stream_cap is None else stream_cap
                scap = np.broadcast_to(np.asarray(scap, dtype=np.uint64), (self.n,)).copy()
                soff = np.zeros(self.n, dtype=np.uint64)
                if self.n > 1:
                    soff[1:] = np.cumsum(scap[:-1])
                self.h_stream_off, self.h_stream_cap = soff, scap
                self.d_stream_off, self.d_stream_cap = t(soff), t(scap)
                self.d_n_streams = torch.zeros(self.n, dtype=torch.int64, device=self.device)
                slots = max(int(scap.sum()), 1)
                self.d_stream_end = torch.zeros(slots, dtype=torch.int64, device=self.device)
                self.d_stream_in_off = torch.zeros(slots, dtype=torch.int64, device=self.device)
            if self.max_blocks or scratch_bytes is not None:
                nbytes = _lib.lib().swc_bzip2_stream_batch_scratch_bytes(self.n, self.max_blocks, self.out_total)
                if scratch_bytes is not None:
                    nbytes = min(nbytes, int(scratch_bytes))
                self.d_scratch = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        elif codec == "xz_blocks":
            self.d_aux = None
            self.d_parallel = torch.zeros(self.n, dtype=torch.int32, device=self.device)
            if self.max_blocks:
                nbytes = _lib.lib().swc_xz_block_batch_scratch_bytes(self.n, self.max_blocks)
                self.d_scratch = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        elif codec == "gzip_multi":
            self.d_aux = None
            self.d_parallel = torch.zeros(self.n, dtype=torch.int32, device=self.device)
            mcap = np.asarray(in_len, dtype=np.uint64) // np.uint64(20) + np.uint64(1) if member_cap is None else member_cap
            mcap = np.broadcast_to(np.asarray(mcap, dtype=np.uint64), (self.n,)).copy()
            moff = np.zeros(self.n, dtype=np.uint64)
            if self.n > 1:
                moff[1:] = np.cumsum(mcap[:-1])
            self.h_member_off, self.h_member_cap = moff, mcap
            self.d_member_off, self.d_member_cap = t(moff), t(mcap)
            self.d_n_members = torch.zeros(self.n, dtype=torch.int64, device=self.device)
            slots = max(int(mcap.sum()), 1)
            self.d_member_end = torch.zeros(slots, dtype=torch.int64, device=self.device)
            self.d_member_in_off = torch.zeros(slots, dtype=torch.int64, device=self.device)
            self.max_members = 0 if max_members is None else int(max_members)
            if self.max_members or scratch_bytes is not None:
                nbytes = (_lib.lib().swc_gzip_member_batch_scratch_bytes(self.n, self.max_members, self.out_total)
                          if scratch_bytes is None else int(scratch_bytes))
                self.d_scratch = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        elif codec == "lz4_frame":
            # an empty dictionary is still a dictionary: one spare byte keeps its pointer non-null
            self.dict_len = 0 if aux is None else len(aux)
            self.d_aux = None if aux is None else t(np.frombuffer(bytes(aux) + b"\0", dtype=np.uint8).copy())
            if self.max_blocks:
                nbytes = _lib.lib().swc_lz4_frame_batch_scratch_bytes(self.n, int(np.asarray(in_len, dtype=np.uint64).sum()),
                                                                     self.max_blocks)
                self.d_scratch = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        elif codec == "lz4_frame_compress":
            unknown = set(frame_flags or {}) - set(LZ4_FRAME_DEFAULTS)
            if unknown:
                raise ValueError(f"unknown frame flags {sorted(unknown)}")
            self.frame_flags = dict(LZ4_FRAME_DEFAULTS, **(frame_flags or {}))
            self.dict_len = 0 if aux is None else len(aux)
            self.d_aux = None if aux is None else t(np.frombuffer(bytes(aux) + b"\0", dtype=np.uint8).copy())
            bs = self.block_size
            lens = np.asarray(in_len, dtype=np.uint64)
            blocks = self.max_blocks or (max(1, int(((lens + np.uint64(bs - 1)) // np.uint64(bs)).sum())) if bs >= 1 else 1)
            nbytes = min(_lib.lib().swc_lz4_frame_compress_batch_scratch_bytes(
                self.n, blocks, bs, int(bool(self.frame_flags["independentBlocks"])), self.dict_len), COMPRESS_SCRATCH_LIMIT)
            if scratch_bytes is not None:
                nbytes = min(nbytes, int(scratch_bytes))
            self.d_scratch = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        elif codec == "lz4_block_compress":
            self.d_aux = None
            if aux is not None:
                self.d_dict_off, self.d_dict_len = t(np.asarray(aux[0], dtype=np.uint64)), t(np.asarray(aux[1], dtype=np.uint64))
        else:
            self.d_aux = None if aux is None else torch.from_numpy(np.frombuffer(bytes(aux), dtype=np.uint8).copy()).to(self.device)
        self.max_in_bytes = 0 if max_in_bytes is None else int(max_in_bytes)
        if codec == "gzip_archive":
            from .api import GzipArchive
            opts = gzip_options if isinstance(gzip_options, (list, tuple)) else [gzip_options or {}] * self.n
            if len(opts) != self.n:
                raise ValueError(f"gzip_options has {len(opts)} entries for {self.n} units")
            # each distinct header once, back to back
            blob, at, hdr_off, hdr_len = bytearray(), {}, np.zeros(self.n, dtype=np.uint64), np.zeros(self.n, dtype=np.uint64)
            for i, o in enumerate(opts):
                h = GzipArchive.archive_header(**o)
                if h not in at:
                    at[h] = len(blob)
                    blob += h
                hdr_off[i], hdr_len[i] = at[h], len(h)
            self.headers = [bytes(blob[int(o):int(o) + int(ln)]) for o, ln in zip(hdr_off, hdr_len)]
            self.d_hdr = t(np.frombuffer(bytes(blob) + b"\0", dtype=np.uint8).copy())
            self.d_hdr_off, self.d_hdr_len = t(hdr_off), t(hdr_len)
        if codec in ("gzip_archive", "zlib_archive") and self.max_in_bytes:
            nbytes = _lib.lib().swc_archive_compress_batch_scratch_bytes(self.n, self.max_in_bytes)
            if scratch_bytes is not None:
                nbytes = min(nbytes, int(scratch_bytes))
            self.d_scratch = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        elif codec in ("lz4_block_compress", "deflate_compress", "bzip2_compress", "gzip_archive", "zlib_archive"):
            nbytes = compress_scratch_bytes(codec, in_len, None if aux is None else aux[1], self.block_size)
            if scratch_bytes is not None:
                nbytes = min(nbytes, int(scratch_bytes))
            self.d_scratch = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        if codec == "deflate":
            nbytes = _lib.lib().swc_deflate_batch_scratch_bytes(self.n, self.out_total)
            self.d_scratch = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        if codec in ("gzip", "zlib"):
            nbytes = _lib.lib().swc_unarchive_batch_scratch_bytes(self.n, self.out_total)
            self.d_scratch = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        self.d_headers = None
        if headers and codec == "gzip":
            from .api import _CGzipHeader
            self.d_headers = torch.zeros(max(self.n, 1) * C.sizeof(_CGzipHeader), dtype=torch.uint8, device=self.device)

    def _init_tar(self, d_in, d_in_off, d_in_len, entry_cap, d_in_cap=None, d_in_status=None):
        self.d_in, self.d_in_off, self.d_in_len = d_in, d_in_off, d_in_len
        self.d_in_cap, self.d_in_status = d_in_cap, d_in_status
        caps = np.asarray(entry_cap, dtype=np.uint64)
        if caps.ndim == 0:
            caps = np.full(self.n, int(caps), dtype=np.uint64)
        offs = np.zeros(self.n, dtype=np.uint64)
        if self.n > 1:
            offs[1:] = np.cumsum(caps[:-1])
        self.h_entry_off, self.h_entry_cap = offs, caps
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.int64)).to(self.device)
        self.d_entry_off, self.d_entry_cap = t(offs), t(caps)
        self.d_entries = torch.zeros(max(int(caps.sum()), 1) * C.sizeof(_lib.TarEntry), dtype=torch.uint8, device=self.device)
        self.d_out_len = torch.zeros(self.n, dtype=torch.int64, device=self.device)          # n_entries
        self.d_consumed = torch.zeros(self.n, dtype=torch.int64, device=self.device)
        self.d_status = torch.full((self.n,), -1, dtype=torch.int32, device=self.device)     # info's status
        self.d_open_status = torch.full((self.n,), -1, dtype=torch.int32, device=self.device)
        self.d_format = torch.zeros(self.n, dtype=torch.int32, device=self.device)
        self.d_format_status = torch.full((self.n,), -1, dtype=torch.int32, device=self.device)

    @classmethod
    def tar_of(cls, other, entry_cap=None):
        """A 'tar' batch over another batch's device outputs (unit i: other.d_out[out_off[i] ..+ out_len[i]), with no
        copy): a 'gzip' / 'gzip_multi' / 'xz' / 'xz_blocks' / 'bzip2_stream' / 'bzip2_multi' batch of .tar.gz / .tar.xz /
        .tar.bz2 files feeds the walk in the same stream ('gzip_multi' and 'bzip2_multi' outputs are each unit's members or
        streams back to back, so a BGZF .tar.gz or a pbzip2 .tar.bz2 is walked in place).  Each unit is walked over at most other's out_cap bytes (an overflowing decode reports a required size
        past its region), and a unit whose decode failed is not walked: it reports that status in every status column.
        Entry tables default to out_cap // 512 + 1 records, enough for any archive the outputs can hold without a
        negative size."""
        b = cls.__new__(cls)
        b.codec, b.device, b.n = "tar", other.device, other.n
        caps = other.h_out_cap // np.uint64(512) + np.uint64(1) if entry_cap is None else entry_cap
        b._init_tar(other.d_out, other.d_out_off, other.d_out_len, caps, other.d_out_cap, other.d_status)
        return b

    @classmethod
    def from_units(cls, codec, units, out_cap, device="cuda:0", aux=None, scratch_bytes=None, block_size=None, headers=False,
                   dict_id=None, max_blocks=None, frame_flags=None, gzip_options=None, max_in_bytes=None, max_members=None,
                   member_cap=None, stream_cap=None):
        buf, offs, lens = pack_units(units)
        return cls(codec, buf, offs, lens, out_cap, device, aux, scratch_bytes, block_size, headers, dict_id, max_blocks,
                   frame_flags, gzip_options, max_in_bytes, max_members, member_cap, stream_cap)

    def run(self):
        L = _lib.lib()
        stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
        p = lambda t: C.c_void_p(t.data_ptr())
        if self.codec == "deflate":
            st = L.swc_deflate_decompress_batch(p(self.d_in), p(self.d_in_off), p(self.d_in_len), None, p(self.d_out),
                                                p(self.d_out_off), p(self.d_out_cap), self.out_total, p(self.d_out_len),
                                                p(self.d_consumed), p(self.d_status), self.n, p(self.d_scratch),
                                                self.d_scratch.numel(), stream)
        elif self.codec == "gzip":
            st = L.swc_gzip_unarchive_batch(p(self.d_in), p(self.d_in_off), p(self.d_in_len), p(self.d_out), p(self.d_out_off),
                                            p(self.d_out_cap), self.out_total, p(self.d_out_len), p(self.d_consumed),
                                            p(self.d_status), None if self.d_headers is None else p(self.d_headers), self.n,
                                            p(self.d_scratch), self.d_scratch.numel(), stream)
        elif self.codec == "zlib":
            st = L.swc_zlib_unarchive_batch(p(self.d_in), p(self.d_in_off), p(self.d_in_len), p(self.d_out), p(self.d_out_off),
                                            p(self.d_out_cap), self.out_total, p(self.d_out_len), p(self.d_consumed),
                                            p(self.d_status), self.n, p(self.d_scratch), self.d_scratch.numel(), stream)
        elif self.codec == "xz":
            st = L.swc_xz_unarchive_batch(p(self.d_in), p(self.d_in_off), p(self.d_in_len), p(self.d_out), p(self.d_out_off),
                                          p(self.d_out_cap), p(self.d_out_len), p(self.d_status), self.n, stream)
        elif self.codec == "xz_blocks":
            st = L.swc_xz_block_unarchive_batch(p(self.d_in), p(self.d_in_off), p(self.d_in_len), p(self.d_out),
                                                p(self.d_out_off), p(self.d_out_cap), p(self.d_out_len), p(self.d_status),
                                                p(self.d_parallel), self.n, self.max_blocks,
                                                None if self.d_scratch is None else p(self.d_scratch),
                                                0 if self.d_scratch is None else self.d_scratch.numel(), stream)
        elif self.codec == "gzip_multi":
            opt = lambda t: None if t is None else p(t)
            st = L.swc_gzip_multi_unarchive_batch(p(self.d_in), p(self.d_in_off), p(self.d_in_len), p(self.d_out),
                                                  p(self.d_out_off), p(self.d_out_cap), p(self.d_out_len), p(self.d_consumed),
                                                  p(self.d_status), p(self.d_n_members), p(self.d_member_off),
                                                  p(self.d_member_cap), p(self.d_member_end), p(self.d_member_in_off),
                                                  p(self.d_parallel), self.n, self.max_members, opt(self.d_scratch),
                                                  0 if self.d_scratch is None else self.d_scratch.numel(), stream)
        elif self.codec == "lz4_block":
            st = L.swc_lz4_block_decompress_batch(p(self.d_in), p(self.d_in_off), p(self.d_in_len), None, 0, p(self.d_out),
                                                  p(self.d_out_off), p(self.d_out_cap), p(self.d_out_len), p(self.d_status),
                                                  self.n, stream)
        elif self.codec == "lz4_frame":
            opt = lambda t: None if t is None else p(t)
            st = L.swc_lz4_frame_decompress_batch(p(self.d_in), p(self.d_in_off), p(self.d_in_len), opt(self.d_aux), self.dict_len,
                                                  self.dict_id is not None, self.dict_id or 0, p(self.d_out), p(self.d_out_off),
                                                  p(self.d_out_cap), p(self.d_out_len), p(self.d_consumed), p(self.d_status),
                                                  self.n, self.max_blocks, opt(self.d_scratch),
                                                  0 if self.d_scratch is None else self.d_scratch.numel(), stream)
        elif self.codec == "lz4_block_compress":
            opt = lambda t: None if t is None else p(t)
            st = L.swc_lz4_block_compress_batch(p(self.d_in), p(self.d_in_off), p(self.d_in_len), opt(self.d_dict_off),
                                                opt(self.d_dict_len), p(self.d_out), p(self.d_out_off), p(self.d_out_cap),
                                                p(self.d_out_len), p(self.d_status), self.n, p(self.d_scratch),
                                                self.d_scratch.numel(), stream)
        elif self.codec == "lz4_frame_compress":
            fl = self.frame_flags
            st = L.swc_lz4_frame_compress_batch(p(self.d_in), p(self.d_in_off), p(self.d_in_len), int(bool(fl["independentBlocks"])),
                                                int(bool(fl["blockChecksums"])), int(bool(fl["contentChecksum"])),
                                                int(bool(fl["contentSize"])), self.block_size,
                                                None if self.d_aux is None else p(self.d_aux), self.dict_len,
                                                self.dict_id is not None, self.dict_id or 0, p(self.d_out), p(self.d_out_off),
                                                p(self.d_out_cap), p(self.d_out_len), p(self.d_status), self.n, self.max_blocks,
                                                p(self.d_scratch), self.d_scratch.numel(), stream)
        elif self.codec == "deflate_compress":
            st = L.swc_deflate_compress_batch(p(self.d_in), p(self.d_in_off), p(self.d_in_len), p(self.d_out), p(self.d_out_off),
                                              p(self.d_out_cap), p(self.d_out_len), p(self.d_status), self.n, p(self.d_scratch),
                                              self.d_scratch.numel(), stream)
        elif self.codec == "gzip_archive":
            st = L.swc_gzip_archive_batch(p(self.d_in), p(self.d_in_off), p(self.d_in_len), p(self.d_hdr), p(self.d_hdr_off),
                                          p(self.d_hdr_len), p(self.d_out), p(self.d_out_off), p(self.d_out_cap), p(self.d_out_len),
                                          p(self.d_status), self.n, self.max_in_bytes, p(self.d_scratch), self.d_scratch.numel(),
                                          stream)
        elif self.codec == "zlib_archive":
            st = L.swc_zlib_archive_batch(p(self.d_in), p(self.d_in_off), p(self.d_in_len), p(self.d_out), p(self.d_out_off),
                                          p(self.d_out_cap), p(self.d_out_len), p(self.d_status), self.n, self.max_in_bytes,
                                          p(self.d_scratch), self.d_scratch.numel(), stream)
        elif self.codec == "bzip2_compress":
            st = L.swc_bzip2_compress_batch(p(self.d_in), p(self.d_in_off), p(self.d_in_len), self.block_size, p(self.d_out),
                                            p(self.d_out_off), p(self.d_out_cap), p(self.d_out_len), p(self.d_status), self.n,
                                            p(self.d_scratch), self.d_scratch.numel(), stream)
        elif self.codec == "bzip2":
            st = L.swc_bzip2_decompress_batch(p(self.d_in), p(self.d_in_off), p(self.d_in_len), p(self.d_out), p(self.d_out_off),
                                              p(self.d_out_cap), p(self.d_out_len), p(self.d_consumed), p(self.d_status), self.n, stream)
        elif self.codec == "bzip2_stream":
            opt = lambda t: None if t is None else p(t)
            st = L.swc_bzip2_stream_decompress_batch(p(self.d_in), p(self.d_in_off), p(self.d_in_len), p(self.d_out),
                                                     p(self.d_out_off), p(self.d_out_cap), p(self.d_out_len), p(self.d_consumed),
                                                     p(self.d_status), self.n, self.max_blocks, opt(self.d_scratch),
                                                     0 if self.d_scratch is None else self.d_scratch.numel(), stream)
        elif self.codec == "bzip2_multi":
            opt = lambda t: None if t is None else p(t)
            st = L.swc_bzip2_multi_decompress_batch(p(self.d_in), p(self.d_in_off), p(self.d_in_len), p(self.d_out),
                                                    p(self.d_out_off), p(self.d_out_cap), p(self.d_out_len), p(self.d_status),
                                                    p(self.d_n_streams), p(self.d_stream_off), p(self.d_stream_cap),
                                                    p(self.d_stream_end), p(self.d_stream_in_off), p(self.d_parallel), self.n,
                                                    self.max_blocks, opt(self.d_scratch),
                                                    0 if self.d_scratch is None else self.d_scratch.numel(), stream)
        elif self.codec == "tar":
            opt = lambda t: None if t is None else p(t)
            st = L.swc_tar_walk_batch(p(self.d_in), p(self.d_in_off), p(self.d_in_len), opt(self.d_in_cap), opt(self.d_in_status),
                                      p(self.d_entries), p(self.d_entry_off),
                                      p(self.d_entry_cap), p(self.d_out_len), p(self.d_status), p(self.d_open_status),
                                      p(self.d_format), p(self.d_format_status), self.n, stream)
        elif self.codec == "lzma2":
            st = L.swc_lzma2_decompress_batch(p(self.d_in), p(self.d_in_off), p(self.d_in_len), p(self.d_aux), p(self.d_out), p(self.d_out_off),
                                              p(self.d_out_cap), p(self.d_out_len), p(self.d_consumed), p(self.d_status), self.n, stream)
        else:
            raise ValueError(self.codec)
        if st != 0:
            raise RuntimeError(f"{self.codec} batch launch failed: {_lib.status_name(st)} {_lib.last_error()}")

    def results(self):
        """-> (status int32[n], out_len int64[n], consumed int64[n]) on the host (synchronises).  consumed is in bits for
        'deflate', 'bzip2' and 'bzip2_stream', in bytes for 'lzma2', 'gzip', 'zlib' and 'lz4_frame', and 0 for 'xz', 'xz_blocks',
        'bzip2_multi' and the compress codecs."""
        torch.cuda.synchronize(self.device)
        return self.d_status.cpu().numpy(), self.d_out_len.cpu().numpy(), self.d_consumed.cpu().numpy()

    def parallel_blocks(self):
        """-> uint32[n] of an 'xz_blocks' batch: the blocks of each unit decoded block-parallel and accepted (synchronises)"""
        torch.cuda.synchronize(self.device)
        return self.d_parallel.cpu().numpy().view(np.uint32)

    def parallel_members(self):
        """-> uint32[n] of a 'gzip_multi' batch: the members of each unit accepted from the parallel spans (synchronises)"""
        torch.cuda.synchronize(self.device)
        return self.d_parallel.cpu().numpy().view(np.uint32)

    def parallel_streams(self):
        """-> uint32[n] of a 'bzip2_multi' batch: the leading streams of each unit accepted from the block stage
        (synchronises)"""
        torch.cuda.synchronize(self.device)
        return self.d_parallel.cpu().numpy().view(np.uint32)

    def stream_table(self, i):
        """-> (stream ends in the output, stream starts in the unit) of unit i of a 'bzip2_multi' batch, at most its stream
        capacity (synchronises)"""
        torch.cuda.synchronize(self.device)
        k = min(int(self.d_n_streams[i].item()), int(self.h_stream_cap[i]))
        o = int(self.h_stream_off[i])
        return [int(v) for v in self.d_stream_end[o:o + k].cpu()], [int(v) for v in self.d_stream_in_off[o:o + k].cpu()]

    def streams(self, i):
        """unit i of a 'bzip2_multi' batch as BZip2.multiDecompress returns it: a list of bytes, one per stream; raises the
        matching BZip2Error otherwise (on wrongCRC its payload is the failing stream's bytes) (synchronises)"""
        from .errors import error_for
        st, ln, _ = self.results()
        ends, _ = self.stream_table(i)
        out = self.output(i)
        parts, prev = [], 0
        for e in ends:
            parts.append(out[prev:e])
            prev = e
        if int(st[i]) == 0:
            return parts
        if int(st[i]) == 210:                                   # wrongCRC: the failing stream is the table's last
            raise error_for(210, parts[-1:])
        raise error_for(int(st[i]), None)

    def member_table(self, i):
        """-> (member ends in the output, member starts in the unit) of unit i of a 'gzip_multi' batch, at most its member
        capacity (synchronises)"""
        torch.cuda.synchronize(self.device)
        k = min(int(self.d_n_members[i].item()), int(self.h_member_cap[i]))
        o = int(self.h_member_off[i])
        return [int(v) for v in self.d_member_end[o:o + k].cpu()], [int(v) for v in self.d_member_in_off[o:o + k].cpu()]

    def members(self, i):
        """unit i of a 'gzip_multi' batch as GzipArchive.multiUnarchive returns it: [GzipArchive.Member], the headers parsed
        from the unit's bytes at each member's start (synchronises)"""
        from .api import GzipArchive, GzipHeader
        ends, starts = self.member_table(i)
        data, out = self.unit_bytes(i), self.output(i)
        members, prev = [], 0
        for e, s in zip(ends, starts):
            members.append(GzipArchive.Member(GzipHeader(data, _member_off=s), out[prev:e]))
            prev = e
        return members

    def tar_results(self):
        """-> (n_entries, info_status, open_status, format, format_status) of a 'tar' batch, numpy arrays (synchronises)"""
        torch.cuda.synchronize(self.device)
        return (self.d_out_len.cpu().numpy(), self.d_status.cpu().numpy(), self.d_open_status.cpu().numpy(),
                self.d_format.cpu().numpy(), self.d_format_status.cpu().numpy())

    def records(self, i):
        """unit i's swc_tar_entry records as dicts (_lib.tar_record), at most its entry capacity (synchronises)"""
        torch.cuda.synchronize(self.device)
        n = min(int(self.d_out_len[i].item()), int(self.h_entry_cap[i]))
        size, o = C.sizeof(_lib.TarEntry), int(self.h_entry_off[i])
        raw = self.d_entries[o * size:(o + n) * size].cpu().numpy().tobytes()
        return [_lib.tar_record(_lib.TarEntry.from_buffer_copy(raw, k * size)) for k in range(n)]

    def unit_bytes(self, i):
        torch.cuda.synchronize(self.device)
        o, n = int(self.d_in_off[i].item()), int(self.d_in_len[i].item())
        if getattr(self, "d_in_cap", None) is not None:
            n = min(n, int(self.d_in_cap[i].item()))
        return bytes(self.d_in[o:o + n].cpu().numpy())

    def entries(self, i):
        """unit i of a 'tar' batch as TarContainer.info returns it: [TarEntryInfo] (synchronises)"""
        from .api import tar_entry_info
        data = self.unit_bytes(i)
        return [tar_entry_info(data, r) for r in self.records(i)]

    def gzip_headers(self):
        """-> the swc_gzip_header of every unit of a 'gzip' batch made with headers=True (synchronises); offsets are
        relative to the batch's input buffer"""
        from .api import _CGzipHeader
        torch.cuda.synchronize(self.device)
        raw = self.d_headers.cpu().numpy().tobytes()
        size = C.sizeof(_CGzipHeader)
        return [_CGzipHeader.from_buffer_copy(raw, i * size) for i in range(self.n)]

    def output(self, i):
        st, ln, _ = self.results()
        o = int(self.h_out_off[i])
        return bytes(self.d_out[o:o + int(ln[i])].cpu().numpy())

    def outputs(self):
        st, ln, _ = self.results()
        host = self.d_out.cpu().numpy()
        return [bytes(host[int(o):int(o) + int(l)]) for o, l in zip(self.h_out_off, ln)]
