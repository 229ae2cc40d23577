// runtime.cu — library plumbing: error text, launch counter, host/pinned allocators, scratch pool, host <-> device hand-off
// helpers of the C-ABI files, status names.
#include <algorithm>
#include <cstring>
#include <mutex>
#include <thread>
#include <string>
#include <atomic>
#include <vector>
#include <cstdio>
#include <cstdlib>
#include "common.cuh"
#include "../../include/swcgpu.h"
#include "host_util.h"

namespace swc {

static thread_local std::string g_err;
static std::atomic<uint64_t> g_launches{0};

void count_launch(int n) { g_launches.fetch_add((uint64_t)n, std::memory_order_relaxed); }

int cuda_fail(cudaError_t e, const char *where) {
    g_err = std::string(where) + ": " + cudaGetErrorString(e);
    cudaGetLastError();   // clear sticky-less errors
    return e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver ? SWC_ERR_NO_DEVICE : SWC_ERR_CUDA;
}

static DeviceCtx g_ctx[64];
DeviceCtx &device_ctx() {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); dev = 0; }
    return g_ctx[dev & 63];
}

// ---- grow-only scratch pool, one per device ----
struct Pool { void *p = nullptr; size_t bytes = 0; };
static std::mutex g_pool_mu;
static Pool g_pools[64][4];      // [device][slot]: 0 kernel scratch, 1-3 staging arenas of the *_batch_host paths

int scratch_get(size_t bytes, void **p, cudaStream_t stream, bool *kept) { return arena_get(0, bytes, p, stream, kept); }

int arena_get(int slot, size_t bytes, void **p, cudaStream_t stream, bool *kept) {
    int dev = 0;
    SWC_CUDA_TRY(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> lk(g_pool_mu);
    Pool &pool = g_pools[dev & 63][slot & 3];
    if (kept) *kept = pool.p && pool.bytes >= bytes;
    if (pool.bytes < bytes) {
        if (pool.p) {
            SWC_CUDA_TRY(cudaStreamSynchronize(stream));
            SWC_CUDA_TRY(cudaDeviceSynchronize());
            cudaFree(pool.p);
            pool.p = nullptr; pool.bytes = 0;
        }
        size_t want = bytes + (bytes >> 3) + (1 << 20);
        cudaError_t e = cudaMalloc(&pool.p, want);
        if (e != cudaSuccess) { want = bytes; e = cudaMalloc(&pool.p, want); }
        if (e != cudaSuccess) { pool.p = nullptr; return cuda_fail(e, "cudaMalloc(scratch)"); }
        pool.bytes = want;
    }
    *p = pool.p;
    return SWC_OK;
}

// ---- large copies between PAGEABLE host memory and the device ----
// cudaMemcpy on pageable memory is one driver thread staging through one bounce buffer; for a freshly malloc'ed result it
// also takes every first-touch page fault on that thread.  Here T host threads each
// own a slice of the transfer, a stream and two pinned bounce buffers: DMA of chunk k+1 overlaps the memcpy of chunk k, and
// page faults / memcpy bandwidth scale with T.
static std::mutex g_pin_mu;
static void *g_pin = nullptr;
static size_t g_pin_bytes = 0;

int copy_pageable(void *dst, const void *src, size_t bytes, bool to_device) {
    const cudaMemcpyKind kind = to_device ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToHost;
    if (bytes < ((size_t)48 << 20)) {
        if (bytes) SWC_CUDA_TRY(cudaMemcpy(dst, src, bytes, kind));
        return SWC_OK;
    }
    unsigned hw = std::thread::hardware_concurrency();
    const int T = (int)std::min<unsigned>(16, std::max<unsigned>(2, hw / 4));
    const size_t CH = (size_t)8 << 20;
    int dev = 0;
    SWC_CUDA_TRY(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> lk(g_pin_mu);                           // one big transfer at a time owns the bounce buffers
    if (g_pin_bytes < (size_t)T * 2 * CH) {
        if (g_pin) cudaFreeHost(g_pin);
        g_pin = nullptr; g_pin_bytes = 0;
        SWC_CUDA_TRY(cudaMallocHost(&g_pin, (size_t)T * 2 * CH));
        g_pin_bytes = (size_t)T * 2 * CH;
    }
    const size_t slice = ((bytes + T - 1) / T + 4095) & ~(size_t)4095;
    std::atomic<int> err{0};
    std::vector<std::thread> th;
    for (int t = 0; t < T; t++) {
        th.emplace_back([&, t] {
            const size_t beg = std::min(bytes, (size_t)t * slice), end = std::min(bytes, beg + slice);
            if (beg >= end) return;
            cudaStream_t s;
            if (cudaSetDevice(dev) != cudaSuccess || cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking) != cudaSuccess) { err = 1; return; }
            uint8_t *b[2] = {(uint8_t *)g_pin + (size_t)(2 * t) * CH, (uint8_t *)g_pin + (size_t)(2 * t + 1) * CH};
            uint8_t *h = (uint8_t *)(to_device ? const_cast<void *>(src) : dst);
            uint8_t *d = (uint8_t *)(to_device ? dst : const_cast<void *>(src));
            const size_t nch = (end - beg + CH - 1) / CH;
            auto len = [&](size_t k) { return std::min(CH, end - (beg + k * CH)); };
            bool ok = true;
            if (to_device) {
                // memcpy chunk k into a bounce buffer, then DMA it while chunk k+1 is being memcpy'd
                cudaEvent_t ev[2];
                ok = cudaEventCreateWithFlags(&ev[0], cudaEventDisableTiming) == cudaSuccess &&
                     cudaEventCreateWithFlags(&ev[1], cudaEventDisableTiming) == cudaSuccess;
                for (size_t k = 0; k < nch && ok; k++) {
                    if (k >= 2) ok = cudaEventSynchronize(ev[k & 1]) == cudaSuccess;   // DMA k-2 has drained this buffer; DMA k-1 may still fly
                    memcpy(b[k & 1], h + beg + k * CH, len(k));
                    ok = ok && cudaMemcpyAsync(d + beg + k * CH, b[k & 1], len(k), cudaMemcpyHostToDevice, s) == cudaSuccess &&
                         cudaEventRecord(ev[k & 1], s) == cudaSuccess;
                }
                ok = ok && cudaStreamSynchronize(s) == cudaSuccess;
                cudaEventDestroy(ev[0]); cudaEventDestroy(ev[1]);
            } else {
                ok = cudaMemcpyAsync(b[0], d + beg, len(0), cudaMemcpyDeviceToHost, s) == cudaSuccess;
                for (size_t k = 0; k < nch && ok; k++) {
                    ok = cudaStreamSynchronize(s) == cudaSuccess;                // chunk k has landed in b[k&1]
                    if (ok && k + 1 < nch)
                        ok = cudaMemcpyAsync(b[(k + 1) & 1], d + beg + (k + 1) * CH, len(k + 1), cudaMemcpyDeviceToHost, s) == cudaSuccess;
                    if (ok) memcpy(h + beg + k * CH, b[k & 1], len(k));
                }
            }
            cudaStreamDestroy(s);
            if (!ok) err = 1;
        });
    }
    for (auto &x : th) x.join();
    if (err) return cuda_fail(cudaGetLastError(), "copy_pageable");
    return SWC_OK;
}

int upload_input(DevBuf &d, const uint8_t *in, size_t n) {
    int st = d.alloc(round16(n) + 256);
    if (st) return st;
    return copy_pageable(d.p, in, n, true);
}

int to_host_alloc(const void *d, size_t n, uint8_t **out, size_t *out_len) {
    uint8_t *h = (uint8_t *)swc_alloc(n);
    if (!h) return SWC_ERR_OUTPUT_OVERFLOW;
    if (n) {
        int st = copy_pageable(h, d, n, false);
        if (st) { swc_free(h); return st; }
    }
    *out = h;
    *out_len = n;
    return SWC_OK;
}

int give_sizes(const std::vector<size_t> &v, size_t **dst, uint8_t **out, size_t *out_len) {
    *dst = (size_t *)swc_alloc(sizeof(size_t) * (v.size() + 1));
    if (!*dst) {
        swc_free(*out);
        *out = nullptr; *out_len = 0;
        return SWC_ERR_OUTPUT_OVERFLOW;
    }
    if (!v.empty()) memcpy(*dst, v.data(), sizeof(size_t) * v.size());
    return SWC_OK;
}

int check_host_units(const uint64_t *in_off, const uint64_t *in_len, uint64_t in_total, const uint64_t *out_off,
                     const uint64_t *out_cap, uint64_t out_total, uint64_t n, bool *monotone) {
    *monotone = true;
    for (uint64_t i = 0; i < n; i++) {
        if (in_off[i] > in_total || in_len[i] > in_total - in_off[i] || out_off[i] > out_total || out_cap[i] > out_total - out_off[i])
            return SWC_ERR_INVALID_ARG;
        if (out_off[i] & 15) return SWC_ERR_INVALID_ARG;
        if (i && (in_off[i] < in_off[i - 1] + in_len[i - 1] || out_off[i] < out_off[i - 1] + out_cap[i - 1])) *monotone = false;
    }
    return SWC_OK;
}

int copy_back_regions(uint8_t *out_base, const u8 *d_out, const uint64_t *out_off, const uint64_t *out_cap, uint64_t b,
                      uint64_t e, cudaStream_t s) {
    for (uint64_t i = b; i < e;) {
        const uint64_t r0 = out_off[i];
        uint64_t r1 = r0 + out_cap[i++];
        while (i < e && out_off[i] == r1) r1 += out_cap[i++];
        if (r1 > r0) SWC_CUDA_TRY(cudaMemcpyAsync(out_base + r0, d_out + r0, r1 - r0, cudaMemcpyDeviceToHost, s));
    }
    return SWC_OK;
}

// ---- per-kernel timing (bench.py roofline leg): events recorded on the launch stream, read back after a sync ----
static bool g_timing = false;
static std::vector<cudaEvent_t> g_marks;
static size_t g_mark_used = 0;
void timing_mark(cudaStream_t stream) {
    if (!g_timing) return;
    if (g_mark_used == g_marks.size()) {
        cudaEvent_t e;
        if (cudaEventCreate(&e) != cudaSuccess) return;
        g_marks.push_back(e);
    }
    cudaEventRecord(g_marks[g_mark_used++], stream);
}

int ensure_device() {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
        g_err = "no CUDA device (libswcgpu has no CPU fallback)";
        cudaGetLastError();
        return SWC_ERR_NO_DEVICE;
    }
    return SWC_OK;
}

}  // namespace swc

extern "C" {

int32_t swc_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}
int32_t swc_set_device(int32_t device) {
    if (swc::ensure_device()) return SWC_ERR_NO_DEVICE;
    SWC_CUDA_TRY(cudaSetDevice(device));
    return SWC_OK;
}
const char *swc_last_error_string(void) { return swc::g_err.c_str(); }
void *swc_alloc(size_t bytes) { return malloc(bytes ? bytes : 1); }
void swc_free(void *p) { free(p); }
void *swc_alloc_pinned(size_t bytes) {
    void *p = nullptr;
    if (cudaMallocHost(&p, bytes ? bytes : 1) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    return p;
}
void swc_free_pinned(void *p) { if (p) cudaFreeHost(p); }
uint64_t swc_kernel_launches(void) { return swc::g_launches.load(); }
int32_t swc_release_scratch(void) {
    std::lock_guard<std::mutex> lk(swc::g_pool_mu);
    for (auto &dev : swc::g_pools)
        for (auto &pool : dev)
            if (pool.p) { cudaFree(pool.p); pool.p = nullptr; pool.bytes = 0; }
    std::lock_guard<std::mutex> lk2(swc::g_pin_mu);
    if (swc::g_pin) { cudaFreeHost(swc::g_pin); swc::g_pin = nullptr; swc::g_pin_bytes = 0; }
    return SWC_OK;
}

void swc_timing_enable(int32_t on) { swc::g_timing = on != 0; swc::g_mark_used = 0; }
// elapsed ms between consecutive marks since swc_timing_enable(1); returns the number of intervals written
int32_t swc_timing_collect(float *ms, int32_t max_n) {
    int32_t n = 0;
    for (size_t i = 1; i < swc::g_mark_used && n < max_n; i++) {
        float t = 0;
        if (cudaEventElapsedTime(&t, swc::g_marks[i - 1], swc::g_marks[i]) != cudaSuccess) { cudaGetLastError(); break; }
        ms[n++] = t;
    }
    swc::g_mark_used = 0;
    return n;
}

const char *swc_status_name(int32_t s) {
    switch (s) {
    case SWC_OK: return "ok";
    case SWC_ERR_OUTPUT_OVERFLOW: return "engine.outputOverflow";
    case SWC_ERR_REFERENCE_TRAP: return "engine.referenceTrap";
    case SWC_ERR_CUDA: return "engine.cuda";
    case SWC_ERR_INVALID_ARG: return "engine.invalidArgument";
    case SWC_ERR_NO_DEVICE: return "engine.noDevice";
    case SWC_ERR_UNSUPPORTED: return "engine.unsupported";
    case SWC_DEFLATE_WRONG_UNCOMPRESSED_BLOCK_LENGTHS: return "DeflateError.wrongUncompressedBlockLengths";
    case SWC_DEFLATE_WRONG_BLOCK_TYPE: return "DeflateError.wrongBlockType";
    case SWC_DEFLATE_WRONG_SYMBOL: return "DeflateError.wrongSymbol";
    case SWC_DEFLATE_SYMBOL_NOT_FOUND: return "DeflateError.symbolNotFound";
    case SWC_BZIP2_WRONG_MAGIC: return "BZip2Error.wrongMagic";
    case SWC_BZIP2_WRONG_VERSION: return "BZip2Error.wrongVersion";
    case SWC_BZIP2_WRONG_BLOCK_SIZE: return "BZip2Error.wrongBlockSize";
    case SWC_BZIP2_WRONG_BLOCK_TYPE: return "BZip2Error.wrongBlockType";
    case SWC_BZIP2_RANDOMIZED_BLOCK: return "BZip2Error.randomizedBlock";
    case SWC_BZIP2_WRONG_HUFFMAN_GROUPS: return "BZip2Error.wrongHuffmanGroups";
    case SWC_BZIP2_WRONG_SELECTOR: return "BZip2Error.wrongSelector";
    case SWC_BZIP2_WRONG_HUFFMAN_CODE_LENGTH: return "BZip2Error.wrongHuffmanCodeLength";
    case SWC_BZIP2_SYMBOL_NOT_FOUND: return "BZip2Error.symbolNotFound";
    case SWC_BZIP2_WRONG_CRC: return "BZip2Error.wrongCRC";
    case SWC_LZMA_WRONG_PROPERTIES: return "LZMAError.wrongProperties";
    case SWC_LZMA_RANGE_DECODER_INIT_ERROR: return "LZMAError.rangeDecoderInitError";
    case SWC_LZMA_EXCEEDED_UNCOMPRESSED_SIZE: return "LZMAError.exceededUncompressedSize";
    case SWC_LZMA_WINDOW_IS_EMPTY: return "LZMAError.windowIsEmpty";
    case SWC_LZMA_RANGE_DECODER_FINISH_ERROR: return "LZMAError.rangeDecoderFinishError";
    case SWC_LZMA_REPEAT_WILL_EXCEED: return "LZMAError.repeatWillExceed";
    case SWC_LZMA_NOT_ENOUGH_TO_REPEAT: return "LZMAError.notEnoughToRepeat";
    case SWC_LZMA2_WRONG_DICTIONARY_SIZE: return "LZMA2Error.wrongDictionarySize";
    case SWC_LZMA2_WRONG_CONTROL_BYTE: return "LZMA2Error.wrongControlByte";
    case SWC_LZMA2_WRONG_RESET: return "LZMA2Error.wrongReset";
    case SWC_LZMA2_WRONG_SIZES: return "LZMA2Error.wrongSizes";
    case SWC_DATA_TRUNCATED: return "DataError.truncated";
    case SWC_DATA_CORRUPTED: return "DataError.corrupted";
    case SWC_DATA_CHECKSUM_MISMATCH: return "DataError.checksumMismatch";
    case SWC_DATA_UNSUPPORTED_FEATURE: return "DataError.unsupportedFeature";
    case SWC_GZIP_WRONG_MAGIC: return "GzipError.wrongMagic";
    case SWC_GZIP_WRONG_COMPRESSION_METHOD: return "GzipError.wrongCompressionMethod";
    case SWC_GZIP_WRONG_FLAGS: return "GzipError.wrongFlags";
    case SWC_GZIP_WRONG_HEADER_CRC: return "GzipError.wrongHeaderCRC";
    case SWC_GZIP_WRONG_CRC: return "GzipError.wrongCRC";
    case SWC_GZIP_WRONG_ISIZE: return "GzipError.wrongISize";
    case SWC_GZIP_CANNOT_ENCODE_ISO_LATIN1: return "GzipError.cannotEncodeISOLatin1";
    case SWC_ZLIB_WRONG_COMPRESSION_METHOD: return "ZlibError.wrongCompressionMethod";
    case SWC_ZLIB_WRONG_COMPRESSION_INFO: return "ZlibError.wrongCompressionInfo";
    case SWC_ZLIB_WRONG_FCHECK: return "ZlibError.wrongFcheck";
    case SWC_ZLIB_WRONG_COMPRESSION_LEVEL: return "ZlibError.wrongCompressionLevel";
    case SWC_ZLIB_WRONG_ADLER32: return "ZlibError.wrongAdler32";
    case SWC_XZ_WRONG_MAGIC: return "XZError.wrongMagic";
    case SWC_XZ_WRONG_FIELD: return "XZError.wrongField";
    case SWC_XZ_WRONG_INFO_CRC: return "XZError.wrongInfoCRC";
    case SWC_XZ_WRONG_FILTER_ID: return "XZError.wrongFilterID";
    case SWC_XZ_CHECK_TYPE_SHA256: return "XZError.checkTypeSHA256";
    case SWC_XZ_WRONG_DATA_SIZE: return "XZError.wrongDataSize";
    case SWC_XZ_WRONG_CHECK: return "XZError.wrongCheck";
    case SWC_XZ_WRONG_PADDING: return "XZError.wrongPadding";
    case SWC_XZ_MULTI_BYTE_INTEGER_ERROR: return "XZError.multiByteIntegerError";
    case SWC_ZIP_NOT_FOUND_CENTRAL_DIRECTORY_END: return "ZipError.notFoundCentralDirectoryEnd";
    case SWC_ZIP_WRONG_SIGNATURE: return "ZipError.wrongSignature";
    case SWC_ZIP_WRONG_SIZE: return "ZipError.wrongSize";
    case SWC_ZIP_WRONG_VERSION: return "ZipError.wrongVersion";
    case SWC_ZIP_MULTI_VOLUMES_NOT_SUPPORTED: return "ZipError.multiVolumesNotSupported";
    case SWC_ZIP_ENCRYPTION_NOT_SUPPORTED: return "ZipError.encryptionNotSupported";
    case SWC_ZIP_PATCHING_NOT_SUPPORTED: return "ZipError.patchingNotSupported";
    case SWC_ZIP_COMPRESSION_NOT_SUPPORTED: return "ZipError.compressionNotSupported";
    case SWC_ZIP_WRONG_LOCAL_HEADER: return "ZipError.wrongLocalHeader";
    case SWC_ZIP_WRONG_CRC: return "ZipError.wrongCRC";
    case SWC_ZIP_WRONG_TEXT_FIELD: return "ZipError.wrongTextField";
    case SWC_TAR_TOO_SMALL_FILE_IS_PASSED: return "TarError.tooSmallFileIsPassed";
    case SWC_TAR_WRONG_FIELD: return "TarError.wrongField";
    case SWC_TAR_WRONG_HEADER_CHECKSUM: return "TarError.wrongHeaderChecksum";
    case SWC_TAR_WRONG_PAX_HEADER_ENTRY: return "TarError.wrongPaxHeaderEntry";
    default: return "unknown";
    }
}

}  // extern "C"
