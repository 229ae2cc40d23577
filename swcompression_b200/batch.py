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
    """Device-resident batch for one codec ('deflate', 'lz4_block', 'bzip2', 'lzma2', 'lz4_block_compress').

    'lz4_block_compress' compresses each unit into a raw LZ4 block (LZ4+Compress.swift:156-277); `aux` is then an optional
    (dict_off, dict_len) pair of u64 arrays placing each unit's dictionary window inside `in_buf`."""

    def __init__(self, codec, in_buf, in_off, in_len, out_cap, device="cuda:0", aux=None):
        self.codec = codec
        self.device = torch.device(device)
        self.n = len(in_off)
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
        if codec == "lz4_block_compress":
            self.d_aux = None
            dl = np.zeros(self.n, dtype=np.uint64)
            if aux is not None:
                self.d_dict_off, self.d_dict_len = t(np.asarray(aux[0], dtype=np.uint64)), t(np.asarray(aux[1], dtype=np.uint64))
                dl = np.asarray(aux[1], dtype=np.uint64)
            window = int(np.asarray(in_len, dtype=np.uint64).sum()) + int(np.minimum(dl, np.uint64(65536)).sum())
            # past 16 GiB of scratch the library runs the batch in slices that fit
            nbytes = min(_lib.lib().swc_lz4_compress_batch_scratch_bytes(self.n, window), 16 << 30)
            self.d_scratch = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        else:
            self.d_aux = None if aux is None else torch.from_numpy(np.frombuffer(bytes(aux), dtype=np.uint8).copy()).to(self.device)
        if codec == "deflate":
            nbytes = _lib.lib().swc_deflate_batch_scratch_bytes(self.n, self.out_total)
            self.d_scratch = torch.empty(nbytes, dtype=torch.uint8, device=self.device)

    @classmethod
    def from_units(cls, codec, units, out_cap, device="cuda:0", aux=None):
        buf, offs, lens = pack_units(units)
        return cls(codec, buf, offs, lens, out_cap, device, aux)

    def run(self):
        L = _lib.lib()
        stream = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
        p = lambda t: C.c_void_p(t.data_ptr())
        if self.codec == "deflate":
            st = L.swc_deflate_decompress_batch(p(self.d_in), p(self.d_in_off), p(self.d_in_len), None, p(self.d_out),
                                                p(self.d_out_off), p(self.d_out_cap), self.out_total, p(self.d_out_len),
                                                p(self.d_consumed), p(self.d_status), self.n, p(self.d_scratch),
                                                self.d_scratch.numel(), stream)
        elif self.codec == "lz4_block":
            st = L.swc_lz4_block_decompress_batch(p(self.d_in), p(self.d_in_off), p(self.d_in_len), None, 0, p(self.d_out),
                                                  p(self.d_out_off), p(self.d_out_cap), p(self.d_out_len), p(self.d_status),
                                                  self.n, stream)
        elif self.codec == "lz4_block_compress":
            opt = lambda t: None if t is None else p(t)
            st = L.swc_lz4_block_compress_batch(p(self.d_in), p(self.d_in_off), p(self.d_in_len), opt(self.d_dict_off),
                                                opt(self.d_dict_len), p(self.d_out), p(self.d_out_off), p(self.d_out_cap),
                                                p(self.d_out_len), p(self.d_status), self.n, p(self.d_scratch),
                                                self.d_scratch.numel(), stream)
        elif self.codec == "bzip2":
            st = L.swc_bzip2_decompress_batch(p(self.d_in), p(self.d_in_off), p(self.d_in_len), p(self.d_out), p(self.d_out_off),
                                              p(self.d_out_cap), p(self.d_out_len), p(self.d_consumed), p(self.d_status), self.n, stream)
        elif self.codec == "lzma2":
            st = L.swc_lzma2_decompress_batch(p(self.d_in), p(self.d_in_off), p(self.d_in_len), p(self.d_aux), p(self.d_out), p(self.d_out_off),
                                              p(self.d_out_cap), p(self.d_out_len), p(self.d_consumed), p(self.d_status), self.n, stream)
        else:
            raise ValueError(self.codec)
        if st != 0:
            raise RuntimeError(f"{self.codec} batch launch failed: {_lib.status_name(st)} {_lib.last_error()}")

    def results(self):
        """-> (status int32[n], out_len int64[n], consumed int64[n]) on the host (synchronises)."""
        torch.cuda.synchronize(self.device)
        return self.d_status.cpu().numpy(), self.d_out_len.cpu().numpy(), self.d_consumed.cpu().numpy()

    def output(self, i):
        st, ln, _ = self.results()
        o = int(self.h_out_off[i])
        return bytes(self.d_out[o:o + int(ln[i])].cpu().numpy())

    def outputs(self):
        st, ln, _ = self.results()
        host = self.d_out.cpu().numpy()
        return [bytes(host[int(o):int(o) + int(l)]) for o, l in zip(self.h_out_off, ln)]
