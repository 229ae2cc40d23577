/* swcgpu.h — C ABI of libswcgpu.so: H100 (sm_90a) batched decompression engine that replaces the decode hot path of
 * tsolomko/SWCompression 4.9.0 (pure Swift).  The reference has no FFI layer; its "operator API" is the set of Swift
 * static functions cited next to each entry point below.  A Swift / ctypes shim keeps those names and signatures and
 * routes the bodies through this header (see INTEGRATION.md for the module map + Swift binding).
 *
 * Conventions
 *   - extern "C", no exceptions, no torch types.  Return value / status[] entries are `enum swc_status` codes
 *     (include/swc_status.h): 0 = OK, <base>+k = k-th case of the corresponding Swift error enum.
 *   - "payload-carrying" errors (wrongCRC(Data), checksumMismatch([Data]), wrongAdler32(Data), wrongCheck([Data]))
 *     return the status AND the decoded bytes, as the Swift errors do.
 *   - single-unit calls take HOST pointers, run on the current device and return a buffer allocated with swc_alloc
 *     (caller frees with swc_free).  *_batch calls take DEVICE pointers and are asynchronous on `cuda_stream`.
 *     *_batch_host calls take HOST pointers and include the host<->device copies (blocking).
 *   - every decode reports how much input it consumed, because the reference's wrappers keep parsing after the
 *     payload (GzipArchive.swift:88-94, ZlibArchive.swift:31-37, ZipContainer.swift:74-79, XZBlock.swift:78-82).
 *   - there is no CPU fallback: without a CUDA device every call returns SWC_ERR_NO_DEVICE.
 *   - threading: like the reference, the library may be called from any number of host threads.  Mutable state is one lazily
 *     created context per device (scratch arenas, staging streams, pinned result buffers) behind a per-device mutex: calls on
 *     the same device are serialised, calls on different devices run concurrently.  The asynchronous *_batch calls only hold
 *     the mutex while they enqueue; when several of them are in flight on one device at the same time each needs its own
 *     `scratch` (the NULL = library-pool form shares one arena).
 *   - multi-member / multi-stream / multi-block archives are discovered up front and decoded as one batch; the
 *     reference's in-order walk is kept as the validator, so results and errors are those of the sequential loop.
 *
 * Batch layout (all arrays have n entries, device memory):
 *   unit i reads  in_base[in_off[i] .. in_off[i]+in_len[i])           (any byte alignment; 16-B aligned is fastest)
 *   unit i writes out_base[out_off[i] .. out_off[i]+out_cap[i])       (out_off[i] must be a multiple of 16)
 *   results: out_len[i] (bytes produced), consumed[i], status[i].  On SWC_ERR_OUTPUT_OVERFLOW the Deflate and LZ4 batches
 *   report the size required in out_len[i]; the BZip2 and LZMA decoders need their output as the window and stop at the
 *   capacity, so theirs is only a lower bound of it.
 *   Output regions must not overlap.  Bytes between out_len[i] and out_cap[i] are scratch and may be clobbered; nothing
 *   outside the regions is written (this holds for the *_batch_host forms too: the caller's bytes between regions stay).
 */
#ifndef SWCGPU_H
#define SWCGPU_H

#include <stddef.h>
#include <stdint.h>
#include "swc_status.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---- library / memory ---- */
int32_t     swc_device_count(void);
int32_t     swc_set_device(int32_t device);
const char *swc_last_error_string(void);               /* thread-local text for the last SWC_ERR_CUDA */
const char *swc_status_name(int32_t status);           /* "DeflateError.wrongSymbol", ... */
void       *swc_alloc(size_t bytes);                   /* host memory for single-unit results */
void        swc_free(void *p);
void       *swc_alloc_pinned(size_t bytes);            /* page-locked host memory for *_batch_host callers */
void        swc_free_pinned(void *p);
uint64_t    swc_kernel_launches(void);                 /* number of CUDA kernels this library has launched so far */
int32_t     swc_release_scratch(void);                 /* free the per-device scratch pools */
/* measurement aid: while enabled, every batched call drops CUDA events on its stream before/between/after its kernels;
 * swc_timing_collect (after a stream sync) returns the elapsed ms of each interval in launch order */
void        swc_timing_enable(int32_t on);
int32_t     swc_timing_collect(float *ms, int32_t max_n);

/* ---- Deflate ------------------------------------------------------------------------------------------------
 * Deflate.decompress(data:)                Sources/Deflate/Deflate.swift:24-28
 * Deflate.decompress(_: LsbBitReader)      Sources/Deflate/Deflate.swift:30-249   (start_bit/consumed_bits form) */
int32_t swc_deflate_decompress(const uint8_t *in, size_t in_len, size_t start_bit,
                               uint8_t **out, size_t *out_len, size_t *consumed_bits);
/* scratch the batched call needs for `out_capacity_total` bytes of output buffer */
size_t  swc_deflate_batch_scratch_bytes(uint64_t n, uint64_t out_capacity_total);
int32_t swc_deflate_decompress_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                                     const uint8_t *start_bits /* n entries 0..7, or NULL */,
                                     uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                     uint64_t out_capacity_total,
                                     uint64_t *out_len, uint64_t *consumed_bits, int32_t *status,
                                     uint64_t n, void *scratch, size_t scratch_bytes /* NULL,0 = library pool */,
                                     void *cuda_stream);
/* Every Deflate decode (batched, single-stream, gzip / zlib / ZIP entries) produces at most 0xFFFFFFF0 bytes (4 GiB - 16)
 * per unit: a stream that decodes to more reports SWC_ERR_UNSUPPORTED whatever its capacity (0 included). */
int32_t swc_deflate_decompress_batch_host(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                                          uint64_t in_total,
                                          uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                          uint64_t out_capacity_total,
                                          uint64_t *out_len, uint64_t *consumed_bits, int32_t *status, uint64_t n);

/* ---- LZ4 ----------------------------------------------------------------------------------------------------
 * LZ4.decompress(data:)                                   Sources/LZ4/LZ4.swift:49-51
 * LZ4.decompress(data:dictionary:dictionaryID:)           Sources/LZ4/LZ4.swift:73-91
 * LZ4.multiDecompress(data:dictionary:dictionaryID:)      Sources/LZ4/LZ4.swift:116-146
 * LZ4.process(block:_:) (private raw-block decoder)       Sources/LZ4/LZ4.swift:332-413  -> *_block_batch
 * swc_lz4_decompress: *consumed_bytes is where the frame ended on SWC_OK and SWC_DATA_CHECKSUM_MISMATCH, and 0 on every
 * other status, as consumed_bytes[i] of swc_lz4_frame_decompress_batch below, whose one-unit case it is. */
int32_t swc_lz4_decompress(const uint8_t *in, size_t in_len, const uint8_t *dict /* NULL = nil */, size_t dict_len,
                           int32_t has_dict_id, uint32_t dict_id,
                           uint8_t **out, size_t *out_len, size_t *consumed_bytes);
/* frames are concatenated into *out; frame_ends[i] = end offset of frame i; returns the number of frames in *n_frames */
int32_t swc_lz4_multi_decompress(const uint8_t *in, size_t in_len, const uint8_t *dict, size_t dict_len,
                                 int32_t has_dict_id, uint32_t dict_id,
                                 uint8_t **out, size_t *out_len, size_t **frame_ends, size_t *n_frames);
/* raw blocks; dict (device pointer, may be NULL) is the prefix every block may reference (independent-block mode) */
int32_t swc_lz4_block_decompress_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                                       const uint8_t *dict, uint64_t dict_len,
                                       uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                       uint64_t *out_len, int32_t *status, uint64_t n, void *cuda_stream);
int32_t swc_lz4_block_decompress_batch_host(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                                            uint64_t in_total,
                                            uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                            uint64_t out_capacity_total,
                                            uint64_t *out_len, int32_t *status, uint64_t n);

/* Whole frames, device memory, one asynchronous enqueue on `cuda_stream`.  Unit i is in_base[in_off[i] ..+ in_len[i]), any
 * alignment ("Batch layout"), decoded as LZ4.decompress(data:dictionary:dictionaryID:) decodes it: leading skippable frames
 * are skipped, then the first frame or legacy frame is decoded and the bytes behind it are ignored; consumed_bytes[i] is
 * where it ended.  One dictionary (device pointer, NULL = nil; an empty dictionary is a non-NULL pointer with dict_len 0)
 * serves the whole batch.  A unit that starts with a skippable frame is decoded without the dictionary and the dictionary
 * ID, as the reference's recursion into decompress(data:) does.
 * status[i] is the first failure the reference's sequential loop meets (descriptor checks, then per block: mark, size,
 * room, block checksum, decode; then content size, content checksum); swc_lz4_decompress is this batch on one unit.
 * SWC_DATA_CHECKSUM_MISMATCH carries its data: the unit's output region holds the decoded bytes.
 * Capacity: a unit that would be SWC_OK or SWC_DATA_CHECKSUM_MISMATCH but decodes to more than out_cap[i] reports
 * SWC_ERR_OUTPUT_OVERFLOW with out_len[i] = the exact decoded size, so one rerun with that capacity gives the final
 * answer; every other failure is reported as with unlimited capacity.  out_len[i] is the decoded size on OK /
 * checksumMismatch, the required size on overflow and 0 otherwise; consumed_bytes[i] is set on OK / checksumMismatch and 0
 * otherwise.  Nothing is written outside [out_off[i], out_off[i] + out_cap[i]); no byte outside a unit affects its result.
 * max_blocks > 0 is the capacity of the batch's block table (at most 2^32 - 1): grids are sized from it and, with a
 * caller scratch of swc_lz4_frame_batch_scratch_bytes(n, sum of in_len, max_blocks) bytes, the call reads nothing back and
 * allocates nothing, so it can be captured in a CUDA graph.  Units are placed in order; a unit whose blocks do not fit in
 * what is left of the table (or of the scratch) reports SWC_ERR_UNSUPPORTED and writes nothing; units without blocks
 * always fit.  max_blocks == 0 lets the library count first (one walk, one synchronisation); a caller scratch too small for
 * the count is SWC_ERR_INVALID_ARG.  scratch == NULL takes the library pool (and, with max_blocks > 0, reads in_len back).
 * swc_lz4_frame_info_batch is the walk on its own, for sizing max_blocks and, when the frame declares it, out_cap. */
#define SWC_LZ4F_DICTIONARY_DROPPED 0x100u   /* flags: a skippable frame came first, the unit decodes without dictionary */
#define SWC_LZ4F_CHECKSUM_CUT       0x200u   /* flags: the EndMark was reached but the content checksum is cut short */
typedef struct swc_lz4_frame_info {
    int32_t  status;          /* the first framing failure (descriptor, block marks, end), or SWC_OK */
    uint32_t kind;            /* 0 no frame (status says why), 1 independent blocks, 2 dependent blocks, 3 legacy */
    uint64_t n_blocks;        /* blocks in front of the EndMark or of the framing failure */
    uint32_t flags;           /* the FLG byte (0 for a legacy frame) | SWC_LZ4F_* */
    uint32_t max_block_size;  /* from the BD byte; 0 for a legacy frame */
    uint64_t content_size;    /* UINT64_MAX when the frame does not declare it */
    uint64_t frame_start;     /* offset of the frame's magic in the unit (behind the skippable frames) */
    uint64_t frame_end;       /* offset behind the frame when the walk reached it (= consumed_bytes), else 0 */
} swc_lz4_frame_info;
size_t  swc_lz4_frame_batch_scratch_bytes(uint64_t n, uint64_t in_bytes_total, uint64_t max_blocks);
int32_t swc_lz4_frame_decompress_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                                       const uint8_t *dict /* device, NULL = nil */, uint64_t dict_len,
                                       int32_t has_dict_id, uint32_t dict_id,
                                       uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                       uint64_t *out_len, uint64_t *consumed_bytes, int32_t *status,
                                       uint64_t n, uint64_t max_blocks,
                                       void *scratch, size_t scratch_bytes, void *cuda_stream);
int32_t swc_lz4_frame_info_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                                 int32_t has_dict, int32_t has_dict_id, uint32_t dict_id,
                                 swc_lz4_frame_info *info /* device, n entries */,
                                 uint64_t n, void *cuda_stream);

/* ---- LZ4 compression ----------------------------------------------------------------------------------------
 * LZ4.compress(data:)                                                     Sources/LZ4/LZ4+Compress.swift:16-19
 * LZ4.compress(data:independentBlocks:blockChecksums:contentChecksum:contentSize:blockSize:dictionary:dictionaryID:)
 *                                                                          Sources/LZ4/LZ4+Compress.swift:47-154
 * LZ4.compress(block:_:) (private raw-block compressor)                   Sources/LZ4/LZ4+Compress.swift:156-298 -> *_batch
 * The output bytes equal the reference's for every option combination (its greedy parse, not liblz4's).  The reference
 * cannot fail; where it traps (block_size outside 1 ... 4 MiB, a 1-3 byte dictionary, a dependent frame of blocks of
 * 1-3 bytes) these calls return SWC_ERR_REFERENCE_TRAP.
 * swc_lz4_compress: one frame from host memory; dict == NULL is `dictionary: nil`, has_dict_id == 0 `dictionaryID: nil`.
 * It runs as the one-unit swc_lz4_frame_compress_batch below. */
int32_t swc_lz4_compress(const uint8_t *in, size_t in_len, int32_t independent_blocks, int32_t block_checksums,
                         int32_t content_checksum, int32_t content_size, int64_t block_size,
                         const uint8_t *dict, size_t dict_len, int32_t has_dict_id, uint32_t dict_id,
                         uint8_t **out, size_t *out_len);
/* Raw blocks, device memory, asynchronous on `cuda_stream` (the unit sizes are read back first, which synchronises).
 * Unit i compresses in_base[in_off[i] ..+ in_len[i]) with the dictionary window in_base[dict_off[i] ..+ dict_len[i])
 * (dict_off == dict_len == NULL: no dictionary).  The window expresses both frame modes: the user's dictionary, or the
 * last <= 64 KiB of the previous block.  Windows longer than 64 KiB act as their last 64 KiB, as in the reference.
 * out_len[i] is the exact size of the raw block compress(block:_:) returns, even when it is longer than the input; if it
 * exceeds out_cap[i] the unit reports SWC_ERR_OUTPUT_OVERFLOW and writes nothing.  Any input or output alignment; an empty
 * unit encodes to the single token 0x00 (the reference's release build; its assert at :261 is compiled out).  Units longer
 * than 4 MiB report SWC_ERR_UNSUPPORTED.  scratch may be NULL (library pool); a caller's scratch of
 * swc_lz4_compress_batch_scratch_bytes(n, sum of in_len[i] + min(dict_len[i], 65536)) bytes runs the batch in one
 * slice, a smaller one in several (it must hold the largest unit). */
size_t  swc_lz4_compress_batch_scratch_bytes(uint64_t n, uint64_t window_bytes_total);
int32_t swc_lz4_block_compress_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                                     const uint64_t *dict_off /* NULL = none */, const uint64_t *dict_len,
                                     uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                     uint64_t *out_len, int32_t *status, uint64_t n,
                                     void *scratch, size_t scratch_bytes, void *cuda_stream);
/* Whole frames, device memory, one asynchronous enqueue on `cuda_stream`.  Unit i is in_base[in_off[i] ..+ in_len[i]) and
 * its frame goes to out_base[out_off[i] ..+ out_cap[i]), both at any alignment; the frame equals LZ4.compress(data:...)'s
 * (swc_lz4_compress's) for the unit.  The options, the dictionary (device pointer, NULL = nil; an empty dictionary is a
 * non-NULL pointer with dict_len 0; only its last 64 KiB is used) and the dictionary ID apply to the whole batch.
 * block_size outside 1 ... 4 MiB returns SWC_ERR_REFERENCE_TRAP (:51) and enqueues nothing.  status[i]:
 *   SWC_OK;
 *   SWC_ERR_REFERENCE_TRAP from the unit's first failing block, as the reference traps in compress(block:_:): a non-empty
 *     unit with a 1-3 byte dictionary, or a dependent frame of 1-3 byte blocks with more than one block (an empty unit is
 *     header + EndMark (+ the content checksum of no bytes) and never traps);
 *   SWC_ERR_OUTPUT_OVERFLOW when the frame is longer than out_cap[i]: out_len[i] is then the exact frame size, so one rerun
 *     with that capacity gives the frame.  Bytes inside the region are unspecified (a unit's first blocks may be written
 *     before its total is known); nothing outside it is written;
 *   SWC_ERR_UNSUPPORTED when the unit's blocks do not fit in what is left of the block table; nothing is written.
 * out_len[i] is the frame size on OK, the required size on overflow and 0 otherwise.
 * swc_lz4_frame_compress_max_bytes is exact: 7 + 8 content_size + 4 has_dict_id + in_len + nb (4 + 4 block_checksums) + 4 +
 * 4 content_checksum with nb = ceil(in_len / block_size), the size of a frame whose blocks are all stored; a capacity of
 * that size never overflows (0 for an invalid block_size).
 * max_blocks > 0 is the capacity of the block table (at most 2^32 - 1), filled with the units' ceil(in_len / block_size)
 * blocks in unit order; with a caller scratch the call reads nothing back and allocates nothing, and its launches depend
 * only on (n, max_blocks, scratch_bytes), so it can be captured in a CUDA graph.  max_blocks == 0 reads in_len back (one
 * synchronisation) and counts the blocks.  scratch == NULL takes the library pool.  A scratch of
 * swc_lz4_frame_compress_batch_scratch_bytes(n, max_blocks, ...) runs the batch in one slice; a smaller one runs it in
 * slices of whole blocks with the same results; one that cannot hold the columns and one block is SWC_ERR_INVALID_ARG. */
size_t  swc_lz4_frame_compress_max_bytes(uint64_t in_len, int64_t block_size, int32_t block_checksums,
                                         int32_t content_checksum, int32_t content_size, int32_t has_dict_id);
size_t  swc_lz4_frame_compress_batch_scratch_bytes(uint64_t n, uint64_t max_blocks, int64_t block_size,
                                                   int32_t independent_blocks, uint64_t dict_len);
int32_t swc_lz4_frame_compress_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                                     int32_t independent_blocks, int32_t block_checksums, int32_t content_checksum,
                                     int32_t content_size, int64_t block_size,
                                     const uint8_t *dict /* device, NULL = nil */, uint64_t dict_len,
                                     int32_t has_dict_id, uint32_t dict_id,
                                     uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                     uint64_t *out_len, int32_t *status, uint64_t n, uint64_t max_blocks,
                                     void *scratch, size_t scratch_bytes, void *cuda_stream);

/* ---- Deflate compression ------------------------------------------------------------------------------------
 * Deflate.compress(data:)                                                 Sources/Deflate/Deflate+Compress.swift:22-42
 * ZlibArchive.archive(data:)                                              Sources/Zlib/ZlibArchive.swift:54-70
 * GzipArchive.archive(data:comment:fileName:writeHeaderCRC:isTextFile:osType:modificationTime:extraFields:)
 *                                                                          Sources/GZip/GzipArchive.swift:126-241
 * The output bytes equal the reference's: one block, stored or static Huffman, from its greedy parse (not zlib's).  The
 * single calls read host memory and return an swc_alloc'ed buffer; the CRC-32 / Adler-32 of the input run on the device.
 * Inputs of 4 GiB or more return SWC_ERR_UNSUPPORTED. */
int32_t swc_deflate_compress(const uint8_t *in, size_t in_len, uint8_t **out, size_t *out_len);
int32_t swc_zlib_archive(const uint8_t *in, size_t in_len, uint8_t **out, size_t *out_len);
/* GzipArchive.archive's options.  file_name / comment: NULL = nil, else ISO-Latin-1 bytes (the caller encodes; a NUL is
 * appended unless the last byte is one, so an empty string becomes a single NUL).  os_type: the OS byte (255 = nil or
 * .other).  mtime: Int(timeIntervalSince1970) when has_mtime, of which the low 32 bits are written.  Extra field i has
 * the ids extra_ids[2i], extra_ids[2i+1] and extra_lens[i] bytes; the fields' bytes follow each other in extra_bytes.
 * An XLEN (sum of 4 + length) over 65 535 returns SWC_GZIP_CANNOT_ENCODE_ISO_LATIN1, as the reference throws. */
typedef struct swc_gzip_options {
    const uint8_t *file_name; size_t file_name_len;
    const uint8_t *comment; size_t comment_len;
    int32_t write_header_crc, is_text_file;
    int32_t has_mtime; int64_t mtime;
    uint8_t os_type;
    size_t n_extra;
    const uint8_t *extra_ids;
    const uint64_t *extra_lens;
    const uint8_t *extra_bytes;
} swc_gzip_options;
int32_t swc_gzip_archive(const uint8_t *in, size_t in_len, const swc_gzip_options *options, uint8_t **out, size_t *out_len);
/* Raw Deflate streams, device memory, asynchronous on `cuda_stream` (the unit sizes are read back first, which
 * synchronises).  Unit i compresses in_base[in_off[i] ..+ in_len[i]) (any alignment) into out_base + out_off[i] (a
 * multiple of 16).  out_len[i] is the exact stream size, at most (9 in_len[i] + 17) / 8; if it exceeds out_cap[i] the
 * unit reports SWC_ERR_OUTPUT_OVERFLOW and writes nothing.  Nothing outside [out_off[i], out_off[i] + out_cap[i]) is
 * written, nor past out_len[i].  scratch may be NULL (library pool); a caller's scratch of
 * swc_deflate_compress_batch_scratch_bytes(n, sum of in_len[i]) bytes runs the batch in one slice, a smaller one in
 * several (it must hold the largest unit). */
size_t  swc_deflate_compress_batch_scratch_bytes(uint64_t n, uint64_t in_bytes_total);
int32_t swc_deflate_compress_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                                   uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                   uint64_t *out_len, int32_t *status, uint64_t n,
                                   void *scratch, size_t scratch_bytes, void *cuda_stream);
/* GzipArchive.archive's header for `options`: the bytes swc_gzip_archive writes before the Deflate stream (FHCRC
 * included).  Host only, needs no device.  *len = the header's size; if cap < *len nothing is written and
 * SWC_ERR_OUTPUT_OVERFLOW is returned (buf may be NULL with cap 0).  XLEN > 65 535 -> SWC_GZIP_CANNOT_ENCODE_ISO_LATIN1,
 * as swc_gzip_archive. */
int32_t swc_gzip_archive_header(const swc_gzip_options *options, uint8_t *buf, size_t cap, size_t *len);
/* the largest archive of in_len bytes: header_len + (9 in_len + 17) / 8 + 8 (gzip), 2 + (9 in_len + 17) / 8 + 4 (zlib) */
size_t  swc_gzip_archive_max_bytes(uint64_t in_len, uint64_t header_len);
size_t  swc_zlib_archive_max_bytes(uint64_t in_len);
/* Whole gzip members / zlib streams, device memory, asynchronous on `cuda_stream`.  Unit i compresses
 * in_base[in_off[i] ..+ in_len[i]) into out_base[out_off[i] ..+ out_cap[i]); input and output at any alignment.
 *   gzip: header i (hdr_base[hdr_off[i] ..+ hdr_len[i]), device memory, written as given), the Deflate.compress stream,
 *         then CRC-32 and ISIZE little-endian.  A batch that shares one header passes all-zero offsets.
 *   zlib: 78 DA, the stream, then the big-endian Adler-32 (1 for an empty unit).
 * With a header from swc_gzip_archive_header the result equals swc_gzip_archive / swc_zlib_archive's, byte for byte.
 * status[i] / out_len[i]: SWC_OK / the archive's size; SWC_ERR_OUTPUT_OVERFLOW / the exact archive size (nothing
 * written; one rerun with that capacity succeeds); SWC_ERR_UNSUPPORTED / 0 (in_len[i] >= 4 GiB, or the unit does not fit
 * in max_in_bytes; nothing written).  Nothing outside [out_off[i], out_off[i] + out_len[i]) is ever written.
 * max_in_bytes > 0: units are taken in order while the exclusive prefix sum of in_len plus the unit's own length is at
 * most max_in_bytes.  With a caller scratch of at least swc_archive_compress_batch_scratch_bytes(n, max_in_bytes) the
 * call reads nothing back and allocates nothing, and its launches and grids depend only on (n, max_in_bytes,
 * scratch_bytes): it can be captured in a CUDA graph.  A smaller caller scratch is SWC_ERR_INVALID_ARG.
 * max_in_bytes == 0: in_len is read back (one synchronisation) and the batch runs in slices of the scratch, which may be
 * NULL (library pool); a caller scratch must then hold the largest unit, else SWC_ERR_INVALID_ARG. */
size_t  swc_archive_compress_batch_scratch_bytes(uint64_t n, uint64_t max_in_bytes);
int32_t swc_gzip_archive_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                               const uint8_t *hdr_base, const uint64_t *hdr_off, const uint64_t *hdr_len,
                               uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                               uint64_t *out_len, int32_t *status, uint64_t n, uint64_t max_in_bytes,
                               void *scratch, size_t scratch_bytes, void *cuda_stream);
int32_t swc_zlib_archive_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                               uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                               uint64_t *out_len, int32_t *status, uint64_t n, uint64_t max_in_bytes,
                               void *scratch, size_t scratch_bytes, void *cuda_stream);

/* ---- BZip2 compression ---------------------------------------------------------------------------------------
 * BZip2.compress(data:) / compress(data:blockSize:)   Sources/BZip2/BZip2+Compress.swift:19-74
 * block_size is BlockSize.rawValue (1 = .one ... 9 = .nine); any other value returns SWC_ERR_INVALID_ARG.  The output
 * bytes equal the reference's: raw blocks of 80 000 x block_size bytes, its table choice and its code lengths (libbz2
 * and the engine's own decoder read them).  The reference cannot fail, so there are no other statuses; inputs of
 * 2^40 bytes or more return SWC_ERR_UNSUPPORTED.
 * swc_bzip2_compress_max_bytes is the proved largest stream for in_len bytes (DESIGN.md §4.11, lemma 4):
 *   14 + ceil(sum over raw blocks of r bytes, R = r + floor(r / 4), of
 *             (395 + 6 ceil((R + 1) / 50) + 6 x 283 + 11 (R + 1)) / 8)   (with the 4 header and 10 EOS bytes summed
 *   as bits: 112 + that sum, rounded up to bytes).
 * Device memory: a unit is never split across slices, so one unit of n bytes needs about 40 n bytes of device scratch
 * (swc_bzip2_compress_batch_scratch_bytes(1, n, k)) besides its input and output.  The single call takes it from the
 * library's grow-only pool, which keeps it for later calls (swc_release_scratch frees it).  On an 80 GB card that caps
 * one call at about 1.8 GB of input; a larger input returns SWC_ERR_CUDA (the allocation fails) rather than a stream. */
int32_t swc_bzip2_compress(const uint8_t *in, size_t in_len, int32_t block_size, uint8_t **out, size_t *out_len);
size_t  swc_bzip2_compress_max_bytes(uint64_t in_len, int32_t block_size);
/* .bz2 streams, device memory, asynchronous on `cuda_stream` (the unit sizes are read back first, which synchronises).
 * Unit i compresses in_base[in_off[i] ..+ in_len[i]) (any alignment) into one complete stream at out_base + out_off[i]
 * (any alignment).  out_len[i] is the exact stream size; if it exceeds out_cap[i] the unit reports
 * SWC_ERR_OUTPUT_OVERFLOW and writes nothing.  Nothing outside [out_off[i], out_off[i] + out_len[i]) is written.  The
 * result depends only on the unit's bytes and block_size.  scratch may be NULL (library pool); a caller's scratch of
 * swc_bzip2_compress_batch_scratch_bytes(n, sum of in_len[i], block_size) bytes runs the batch in one slice, a
 * smaller one in several (it must hold the largest unit, else SWC_ERR_INVALID_ARG). */
size_t  swc_bzip2_compress_batch_scratch_bytes(uint64_t n, uint64_t in_bytes_total, int32_t block_size);
int32_t swc_bzip2_compress_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, int32_t block_size,
                                 uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                 uint64_t *out_len, int32_t *status, uint64_t n,
                                 void *scratch, size_t scratch_bytes, void *cuda_stream);

/* ---- BZip2--------------------------------------------------------------------------------------------------
 * BZip2.decompress(data:)            Sources/BZip2/BZip2.swift:22-26
 * BZip2.multiDecompress(data:)       Sources/BZip2/BZip2.swift:40-48
 * BZip2.decompress(_: MsbBitReader)  Sources/BZip2/BZip2.swift:50-95 */
int32_t swc_bzip2_decompress(const uint8_t *in, size_t in_len, size_t start_bit,
                             uint8_t **out, size_t *out_len, size_t *consumed_bits);
int32_t swc_bzip2_multi_decompress(const uint8_t *in, size_t in_len,
                                   uint8_t **out, size_t *out_len, size_t **stream_ends, size_t *n_streams);
/* one .bz2 stream per unit */
int32_t swc_bzip2_decompress_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                                   uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                   uint64_t *out_len, uint64_t *consumed_bits, int32_t *status,
                                   uint64_t n, void *cuda_stream);
/* One .bz2 stream per unit with the blocks of every stream decoded side by side, device memory, one asynchronous enqueue on
 * `cuda_stream`.  Unit i is in_base[in_off[i] ..+ in_len[i]) in the layout above, decoded as BZip2.decompress(data:) decodes
 * it: the first stream, the bytes behind it ignored (multi-stream input: swc_bzip2_multi_decompress_batch).
 *   Equality: for every unit and capacity, status[i] is what swc_bzip2_decompress_batch returns for the same unit and
 *     capacity; on SWC_OK and SWC_BZIP2_WRONG_CRC the bytes [0, out_len[i]) and consumed_bits[i] are equal too.
 *   Overflow: the one exception is out_len[i] on SWC_ERR_OUTPUT_OVERFLOW.  When the stream validated block-parallel it is
 *     the exact decoded size, so one rerun with that capacity succeeds; otherwise it is the lower bound the stream kernel
 *     reports.  consumed_bits[i] is 0 on a validated overflow.
 *   Block table: max_blocks > 0 is its capacity (at most 2^32 - 1).  A stream whose block candidates (block magics at any
 *     bit from bit 32 up to its first end-of-stream magic) do not fit in what is left of the table, or whose header, first
 *     block or end magic is not where a valid stream has them, is decoded by the stream kernel: max_blocks changes the
 *     speed, never the results.  With a caller scratch the call reads nothing back and allocates nothing, and its launches
 *     depend only on (n, max_blocks, scratch_bytes), so it can be captured in a CUDA graph.  max_blocks == 0 lets the
 *     library count the candidates and the stream kernel's scratch first (one synchronisation).
 *   Scratch: scratch == NULL takes the library pool.  With a caller scratch of swc_bzip2_stream_batch_scratch_bytes(n,
 *     max_blocks, sum of out_cap) bytes every unit gets its exact status; with max_blocks == 0 the library then keeps the
 *     block table to what that scratch holds beside every unit's fallback.  A smaller scratch runs the block stage in
 *     several slices; it must hold the tables and one block slot (about 16 MB), else the call returns SWC_ERR_INVALID_ARG.
 *     Units are taken in order: a stream goes through the block stage only if the stream kernel's scratch (about 7.5 x
 *     out_cap[i]) would still fit for it and every unit in front of it; otherwise the stream kernel decodes it.  A unit whose
 *     stream-kernel scratch no longer fits reports SWC_ERR_UNSUPPORTED with out_len[i] = consumed_bits[i] = 0, and nothing
 *     is written in its region.
 *   Writes: nothing is written outside [out_off[i], out_off[i] + out_cap[i]). */
size_t  swc_bzip2_stream_batch_scratch_bytes(uint64_t n, uint64_t max_blocks, uint64_t out_capacity_total);
int32_t swc_bzip2_stream_decompress_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                                          uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                          uint64_t *out_len, uint64_t *consumed_bits, int32_t *status,
                                          uint64_t n, uint64_t max_blocks,
                                          void *scratch, size_t scratch_bytes, void *cuda_stream);
/* BZip2.multiDecompress(data:) (BZip2.swift:40-48) over n multi-stream .bz2 files (pbzip2 output, the multistream dumps,
 * `cat a.bz2 b.bz2`), device memory, on `cuda_stream`, with the blocks of every stream of every file decoded side by side.
 * The scan takes the block magics at every bit from bit 32 to the unit end into one block table; the blocks decode as in
 * swc_bzip2_stream_decompress_batch and are laid out back to back; a thread per unit walks the streams as the reference
 * does (header, each block the next table entry, combined CRC per stream, align) and the stream kernel decodes the rest of
 * a unit from its first stream not accepted, stream after stream.
 *   Equality: for every unit whose capacity suffices, status[i] is what swc_bzip2_multi_decompress returns for the same
 *     bytes.  On SWC_OK out_base[out_off[i] ..+ out_len[i]) holds the streams back to back; on SWC_BZIP2_WRONG_CRC every
 *     stream walked, up to and including the failing one, whose bytes [stream_end[k - 1], out_len[i]) are the reference's
 *     payload (the table's last entry is the failing stream).  A 0-byte unit is SWC_OK with 0 streams.  On every other
 *     status out_len[i] = n_streams[i] = 0, also for an error in a later stream (1-3 trailing bytes: wrongMagic; a trailing
 *     "BZh0": wrongBlockSize), except:
 *   Overflow: SWC_ERR_OUTPUT_OVERFLOW with out_len[i] > out_cap[i].  When every stream validated block-parallel out_len[i]
 *     is the exact size, so one rerun with that capacity is final; otherwise it is the stream kernel's lower bound.
 *   Stream table (n_streams, stream_off, stream_cap, stream_end, stream_in_off: device, n entries for the first three; the
 *     last four all or none; n_streams may be NULL on its own): n_streams[i] is the number of streams returned, also when
 *     it exceeds stream_cap[i]; at most stream_cap[i] entries are written at stream_off[i]: stream_end, each stream's
 *     output end relative to out_off[i] (swc_bzip2_multi_decompress's stream_ends), and stream_in_off, each stream's first
 *     byte inside the unit.  in_len[i] / 14 + 1 entries always suffice (an empty stream is 14 bytes).
 *   parallel_streams (device, n entries, or NULL): the leading streams of unit i accepted from the block stage and fitting
 *     out_cap[i]; the stream kernel decoded the rest.
 *   Block table, scratch and graph capture: as swc_bzip2_stream_decompress_batch, with swc_bzip2_stream_batch_scratch_bytes,
 *     except that a unit's candidates are its block magics in the whole unit and it is placed when its header is at byte 0
 *     and a block or end magic at bit 32.  max_blocks and the scratch size change the speed, never the results, apart from
 *     SWC_ERR_UNSUPPORTED when the stream kernel's scratch (about 7.5 x out_cap[i]) no longer fits for a unit.
 *   Writes: nothing is written outside [out_off[i], out_off[i] + out_cap[i]) and the unit's stream table entries, and no
 *     byte outside the unit's input range affects its result. */
int32_t swc_bzip2_multi_decompress_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                                         uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                         uint64_t *out_len, int32_t *status,
                                         uint64_t *n_streams, const uint64_t *stream_off, const uint64_t *stream_cap,
                                         uint64_t *stream_end, uint64_t *stream_in_off,   /* table: may be NULL */
                                         uint32_t *parallel_streams /* device, n, or NULL */,
                                         uint64_t n, uint64_t max_blocks,
                                         void *scratch, size_t scratch_bytes, void *cuda_stream);

/* ---- LZMA / LZMA2 -------------------------------------------------------------------------------------------
 * LZMA.decompress(data:)                                   Sources/LZMA/LZMA.swift:25-34
 * LZMA.decompress(data:properties:uncompressedSize:)       Sources/LZMA/LZMA.swift:56-61
 * LZMA2.decompress(data:)                                  Sources/LZMA2/LZMA2.swift:25-30
 * LZMA2.decompress(_:_:) (reader + dict byte, used by XZ)  Sources/LZMA2/LZMA2.swift:32-36 */
int32_t swc_lzma_decompress(const uint8_t *in, size_t in_len, uint8_t **out, size_t *out_len, size_t *consumed_bytes);
int32_t swc_lzma_decompress_raw(const uint8_t *in, size_t in_len, int32_t lc, int32_t lp, int32_t pb,
                                int64_t dictionary_size, int64_t uncompressed_size /* <0 = nil */,
                                uint8_t **out, size_t *out_len, size_t *consumed_bytes);
int32_t swc_lzma2_decompress(const uint8_t *in, size_t in_len, uint8_t **out, size_t *out_len, size_t *consumed_bytes);
/* one raw LZMA stream per unit (the ZIP / 7-Zip form, LZMA.decompress(data:properties:uncompressedSize:), LZMA.swift:56-61):
 * props[i] = lc | lp << 8 | pb << 16, dict_size[i] as in LZMAProperties, uncompressed_size[i] < 0 = nil (end marker).
 * lc + lp must be <= 4 in the batched form (the literal coders live in shared memory); other units report SWC_ERR_UNSUPPORTED,
 * as do lc > 8, lp > 4 or pb > 4 here and in swc_lzma_decompress_raw: no properties byte expresses them. */
int32_t swc_lzma_decompress_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                                  const uint32_t *props, const int64_t *dict_size, const int64_t *uncompressed_size,
                                  uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                  uint64_t *out_len, uint64_t *consumed_bytes, int32_t *status,
                                  uint64_t n, void *cuda_stream);
/* one raw LZMA2 stream per unit; dict_bytes[i] is the XZ filter property byte.  The reference accepts any properties byte
 * below 225 in a chunk (lc <= 8, lp <= 4), but here too the literal coders live in shared memory: a unit reaching an LZMA
 * chunk with lc + lp > 4 reports SWC_ERR_UNSUPPORTED.  swc_lzma2_decompress and swc_xz_unarchive take such streams. */
int32_t swc_lzma2_decompress_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                                   const uint8_t *dict_bytes,
                                   uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                   uint64_t *out_len, uint64_t *consumed_bytes, int32_t *status,
                                   uint64_t n, void *cuda_stream);

/* ---- wrappers -----------------------------------------------------------------------------------------------
 * GzipArchive.unarchive(archive:) / multiUnarchive   Sources/GZip/GzipArchive.swift:38-77
 * ZlibArchive.unarchive(archive:)                     Sources/Zlib/ZlibArchive.swift:25-42
 * XZArchive.unarchive(archive:) / splitUnarchive      Sources/XZ/XZArchive.swift:27-88 */
/* GzipHeader(archive:) / GzipHeader.init(_: LsbBitReader)   Sources/GZip/GzipHeader.swift:10-60, 63-199
 * ZlibHeader(archive:)                                       Sources/Zlib/ZlibHeader.swift:10-40, 42-93
 * Pure framing: these two calls need no device.  String / extra-field bytes are returned as offsets into `in`
 * (file name and comment are ISO-Latin-1, GzipHeader.swift:160,178; extra fields are the SI1 SI2 LEN data... records). */
typedef struct swc_gzip_header {
    int32_t  compression_method;     /* CompressionMethod.deflate = 8 */
    uint32_t modification_time;      /* MTIME; 0 = nil */
    uint8_t  os_type;                /* raw OS byte (FileSystemType(rawOsType)) */
    uint8_t  is_text_file;           /* FTEXT */
    uint8_t  has_file_name, has_comment;
    size_t   file_name_off, file_name_len;     /* without the terminating zero */
    size_t   comment_off, comment_len;
    size_t   extra_off, extra_len;             /* the XLEN bytes behind the XLEN field (0,0 without FEXTRA) */
    size_t   header_len;                       /* bytes from the member start to the first Deflate byte */
} swc_gzip_header;
typedef struct swc_zlib_header {
    int32_t compression_method;      /* always 8 */
    int32_t compression_level;       /* ZlibHeader.CompressionLevel raw value 0..3 */
    int32_t window_size;             /* 1 << (CINFO + 8) */
    size_t  header_len;              /* 2, or 6 with FDICT */
} swc_zlib_header;
int32_t swc_gzip_header_parse(const uint8_t *in, size_t in_len, size_t member_off, swc_gzip_header *hdr);
int32_t swc_zlib_header_parse(const uint8_t *in, size_t in_len, swc_zlib_header *hdr);
int32_t swc_gzip_unarchive(const uint8_t *in, size_t in_len, uint8_t **out, size_t *out_len, size_t *consumed_bytes);
/* GzipArchive.multiUnarchive -> [Member] (GzipArchive.swift:13-22, 52-77): as swc_gzip_multi_unarchive, plus the offset of
 * every member inside `in` (n_members + 1 entries, the last one = where the walk stopped) so the caller can rebuild
 * Member.header with swc_gzip_header_parse.  On SWC_GZIP_WRONG_CRC the failing member is the last one returned. */
int32_t swc_gzip_multi_unarchive_members(const uint8_t *in, size_t in_len,
                                         uint8_t **out, size_t *out_len, size_t **member_ends, size_t **member_in_off,
                                         size_t *n_members);
int32_t swc_gzip_multi_unarchive(const uint8_t *in, size_t in_len,
                                 uint8_t **out, size_t *out_len, size_t **member_ends, size_t *n_members);
int32_t swc_zlib_unarchive(const uint8_t *in, size_t in_len, uint8_t **out, size_t *out_len);
/* GzipArchive.unarchive(archive:) / ZlibArchive.unarchive(archive:) over n archives, device memory, asynchronous on
 * `cuda_stream` (no host read, no synchronisation, and no allocation when the caller passes scratch).  Unit i is one
 * archive in_base[in_off[i] ..+ in_len[i]) in the layout above; its first member is decoded and the bytes after it are
 * ignored, as the reference does (multi-member archives: swc_gzip_multi_unarchive).  status[i] follows the reference's
 * order of checks:
 *   gzip: in_len < 20 -> wrongMagic; a header error; any Deflate status (SWC_ERR_OUTPUT_OVERFLOW with the size required in
 *         out_len[i]); fewer than 8 bytes after the Deflate stream (after align()) -> wrongMagic; out_len mod 2^32 != ISIZE
 *         -> wrongISize; a CRC-32 mismatch -> wrongCRC, with the data in the unit's output region;
 *   zlib: a header error; any Deflate status; fewer than 4 bytes after the Deflate stream, or a big-endian Adler-32
 *         mismatch -> wrongAdler32, with the data in the unit's output region.
 * consumed_bytes[i] is how many bytes of the archive the reference read on OK and on the payload-carrying statuses (header
 * + whole Deflate bytes + the 8-byte gzip / 4-byte zlib trailer, or no trailer for a zlib unit whose trailer is missing),
 * and 0 on every other status.  A unit whose header fails reports out_len[i] = 0.
 * headers (gzip, device, n entries, or NULL) receives each unit's swc_gzip_header as swc_gzip_header_parse fills it, its
 * file name / comment / extra offsets relative to in_base (fields the header lacks stay 0); all zero when the header fails.
 * scratch == NULL uses the library pool; a caller's scratch must hold swc_unarchive_batch_scratch_bytes(n,
 * out_capacity_total) bytes, else the call returns SWC_ERR_INVALID_ARG. */
size_t  swc_unarchive_batch_scratch_bytes(uint64_t n, uint64_t out_capacity_total);
int32_t swc_gzip_unarchive_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                                 uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                 uint64_t out_capacity_total,
                                 uint64_t *out_len, uint64_t *consumed_bytes, int32_t *status,
                                 swc_gzip_header *headers /* device, n entries, or NULL */,
                                 uint64_t n, void *scratch, size_t scratch_bytes, void *cuda_stream);
int32_t swc_zlib_unarchive_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                                 uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                 uint64_t out_capacity_total,
                                 uint64_t *out_len, uint64_t *consumed_bytes, int32_t *status,
                                 uint64_t n, void *scratch, size_t scratch_bytes, void *cuda_stream);
/* GzipArchive.multiUnarchive(archive:) (GzipArchive.swift:52-100) over n multi-member gzip files (BGZF, `cat a.gz b.gz`),
 * device memory, on `cuda_stream`, with the members of every file decoded side by side.  Candidate member starts (the
 * signature 1f 8b 08 with the reserved flag bits clear and 20 bytes left in the unit, and always position 0) cut each unit
 * into spans: from a candidate whose FEXTRA holds a BGZF "BC" subfield the span ends at c + BSIZE + 1 when that is a
 * candidate or the unit end, else at the next candidate.  Each span decodes as one unit of the swc_gzip_unarchive_batch
 * stages straight into place (its capacity the ISIZE in its last 4 bytes, its output at the sum of the ISIZEs in front of
 * it), the reference's in-order walk accepts member k iff it is OK or wrongCRC, consumed exactly its span and starts where
 * member k - 1 ended, and a sequential walk on the device decodes the rest of a unit from its first member not accepted.
 *   Equality: for every unit whose capacity suffices, status[i] is what swc_gzip_multi_unarchive returns for the same
 *     bytes.  On SWC_OK and SWC_GZIP_WRONG_CRC, out_base[out_off[i] ..+ out_len[i]) holds the members concatenated (on
 *     wrongCRC up to and including the failing member), consumed_bytes[i] is the end of the last member returned, and the
 *     member table holds its ends and starts.  A 0-byte unit is SWC_OK with 0 members; 1-19 bytes behind valid members
 *     are wrongMagic.  On every other status consumed_bytes[i] = 0, n_members[i] = 0 and out_len[i] = 0, except:
 *   Overflow: SWC_ERR_OUTPUT_OVERFLOW when a member does not fit out_cap[i].  The walk then goes on counting: every later
 *     member is decoded without keeping its bytes, its header, Deflate stream and ISIZE checked but not its CRC-32, up to
 *     the unit end or the first error.  out_len[i] is the bytes counted: the exact size when the unit's members validate
 *     against their trailers, otherwise (a member past the capacity with a wrong CRC-32 or a later error) an upper bound
 *     of what the walk keeps.  Either way a rerun with out_cap[i] >= out_len[i] does not overflow and is final.
 *   Member table (n_members, member_off, member_cap, member_end, member_in_off: device, n entries for the first three; all
 *     four arrays or none of them; n_members may be NULL on its own): n_members[i] is the number of members returned,
 *     also when it exceeds member_cap[i]; at most member_cap[i] entries are written at member_off[i]: member_end, each
 *     member's output end relative to out_off[i] (swc_gzip_multi_unarchive's member_ends), and member_in_off, each
 *     member's start inside the unit.  One past the last member is consumed_bytes[i].  in_len[i] / 20 + 1 entries always
 *     suffice.
 *   parallel_members (device, n entries, or NULL): the members of unit i accepted from the parallel spans; the
 *     sequential walk decoded the rest.  It equals n_members[i] for BGZF files and clean concatenations whose members
 *     each decode to 0 or at least 16 bytes and fit out_cap[i]: a member whose output region would be 1-15 bytes (its
 *     size, or what out_cap[i] leaves of it), and every member behind it, takes the sequential walk (the Deflate stage's
 *     scratch for so small an output region cannot hold its literals).
 *   Member table capacity: max_members > 0 (at most 2^32 - 1) holds the candidates of the units in order; a unit whose
 *     candidates do not fit is decoded by the sequential walk alone: max_members changes the speed, never the results.
 *     With a caller scratch and max_members > 0 the call reads nothing back and allocates nothing, and its launches
 *     depend only on (n, max_members, scratch_bytes), so it can be captured in a CUDA graph.  max_members == 0 lets the
 *     library count the candidates first (one synchronisation), and read in_len, out_off and out_cap back; its table then
 *     holds at most in_len[i] / 20 + 1 entries per unit.
 *   Scratch: scratch == NULL takes the library pool (reading out_off / out_cap back).  A caller scratch must hold
 *     swc_gzip_member_batch_scratch_bytes(n, max_members, out_capacity_total) bytes, where out_capacity_total >=
 *     out_off[i] + out_cap[i] for every unit (as for swc_gzip_unarchive_batch); one smaller than that for
 *     out_capacity_total = 0 returns SWC_ERR_INVALID_ARG.  A member whose output region lies past the arena the scratch
 *     covers takes the sequential walk, so a smaller scratch changes the speed, never the results or the memory touched.
 *     With max_members == 0 the table is then the largest the scratch holds.
 *   Writes: nothing is written outside [out_off[i], out_off[i] + out_cap[i]), and no byte outside the unit's input range
 *     affects a result: the scan loads the aligned 16-byte lines that hold the unit's bytes and matches none outside it,
 *     and every span and the sequential walk are bounded by the unit's end. */
size_t  swc_gzip_member_batch_scratch_bytes(uint64_t n, uint64_t max_members, uint64_t out_capacity_total);
int32_t swc_gzip_multi_unarchive_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                                       uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                       uint64_t *out_len, uint64_t *consumed_bytes, int32_t *status,
                                       uint64_t *n_members, const uint64_t *member_off, const uint64_t *member_cap,
                                       uint64_t *member_end, uint64_t *member_in_off,   /* table: may be NULL */
                                       uint32_t *parallel_members /* device, n, or NULL */,
                                       uint64_t n, uint64_t max_members, void *scratch, size_t scratch_bytes, void *cuda_stream);
int32_t swc_xz_unarchive(const uint8_t *in, size_t in_len, uint8_t **out, size_t *out_len);
/* XZArchive.unarchive(archive:) over n whole .xz files, device memory, asynchronous on `cuda_stream`: one launch, no host
 * read, no allocation, no synchronisation and no scratch, so the call can be captured in a CUDA graph.  Unit i is the file
 * in_base[in_off[i] ..+ in_len[i]) in the layout above; every stream (with its stream padding) and every block is decoded and
 * the outputs are concatenated in out_base[out_off[i] ..+ out_cap[i]).  Nothing is written outside the output range, and no
 * byte outside the input range affects a result: the container walk reads byte by byte inside it, while the LZMA2 decoder,
 * like swc_lzma2_decompress_batch, loads the 4-byte words of the 128-byte-aligned lines that hold the unit's bytes and
 * discards the bytes of those words that lie outside it.  status[i] is what swc_xz_unarchive returns for the same bytes, in the reference's order of checks (a read past
 * in_len[i] is SWC_ERR_REFERENCE_TRAP where the single call reports it).  out_len[i] is:
 *   SWC_OK                   the decoded size;
 *   SWC_XZ_WRONG_CHECK       the data up to and including the failing block, which is in the unit's output region;
 *   SWC_ERR_OUTPUT_OVERFLOW  (the unit would write past out_cap[i] before any other status arises) the size the archive
 *                            declares: the sum of its indexes' uncompressed sizes, read backwards from the end of the unit
 *                            through footers, indexes and stream padding, when that walk reaches byte 0; else 0;
 *   any other status         0.
 * Two deviations (DESIGN §6), each reported where the reference would start running the block's filter chain, so every
 * earlier error still wins: a chain other than zero to three Delta filters followed by one LZMA2 filter, and an LZMA chunk
 * with lc + lp > 4, report SWC_ERR_UNSUPPORTED.  swc_xz_unarchive decodes both. */
int32_t swc_xz_unarchive_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                               uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                               uint64_t *out_len, int32_t *status, uint64_t n, void *cuda_stream);
/* XZArchive.unarchive(archive:) over n whole .xz files with the blocks of every file decoded side by side, device memory, on
 * `cuda_stream`.  Each stream's index, read backwards from the end of the unit, gives every block's start and the offset of
 * its output; the blocks decode in parallel straight into the unit's region, the reference's forward walk then checks them,
 * and a unit that does not come out SWC_OK that way is decoded by the kernel of swc_xz_unarchive_batch.
 *   Equality: for every unit and capacity, status[i] and out_len[i] are what swc_xz_unarchive_batch returns for the same unit
 *     and out_cap[i], and on SWC_OK and SWC_XZ_WRONG_CHECK so are the bytes [0, out_len[i]).  There are no exceptions (an
 *     overflow is decoded by the same kernel, with the same declared-size hint).  Bytes of the region past out_len[i] are
 *     unspecified.
 *   parallel_blocks (device, n entries, or NULL): the number of blocks of unit i that were decoded block-parallel and
 *     accepted, which is all of its blocks; 0 when the fallback kernel decoded the unit.
 *   Block table: max_blocks > 0 is its capacity (at most 2^32 - 1).  A unit qualifies when the backward walk through stream
 *     padding, footers, indexes and records reaches byte 0 and the declared total fits out_cap[i]; a qualifying unit is
 *     placed when its records end inside the table, in unit order.  Every other unit goes to the fallback: max_blocks
 *     changes the speed, never the results.  With a caller scratch and max_blocks > 0 the call reads nothing back and
 *     allocates nothing, and its launches depend only on (n, max_blocks, scratch_bytes), so it can be captured in a CUDA
 *     graph.  max_blocks == 0 lets the library count the records first (one synchronisation); with a caller scratch the
 *     table is then the largest the scratch holds.
 *   Scratch: scratch == NULL takes the library pool.  A caller scratch smaller than swc_xz_block_batch_scratch_bytes(n,
 *     max_blocks) returns SWC_ERR_INVALID_ARG; the size depends on n and max_blocks only, never on the output.
 *   Writes: nothing is written outside [out_off[i], out_off[i] + out_cap[i]), and no byte outside the unit's input range
 *     affects a result: the backward walk reads in_base[in_off[i] ..+ in_len[i]) only, and each block is decoded with its
 *     input bounded by the unit's end and its output bounded by its index record.
 * The deviations of swc_xz_unarchive_batch (DESIGN §6) apply unchanged. */
size_t  swc_xz_block_batch_scratch_bytes(uint64_t n, uint64_t max_blocks);
int32_t swc_xz_block_unarchive_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                                     uint8_t *out_base, const uint64_t *out_off, const uint64_t *out_cap,
                                     uint64_t *out_len, int32_t *status,
                                     uint32_t *parallel_blocks /* device, n entries, or NULL */,
                                     uint64_t n, uint64_t max_blocks,
                                     void *scratch, size_t scratch_bytes, void *cuda_stream);
/* resident warps per SM of the LZMA / LZMA2 batch kernel and of the XZ batch kernel on the current device (either pointer
 * may be NULL) */
int32_t swc_xz_occupancy(int32_t *lzma_warps_per_sm, int32_t *xz_warps_per_sm);
int32_t swc_xz_split_unarchive(const uint8_t *in, size_t in_len,
                               uint8_t **out, size_t *out_len, size_t **stream_ends, size_t *n_streams);

/* ---- ZIP container -------------------------------------------------------------------------------------------
 * ZipContainer.open(container:) -> [ZipEntry]     Sources/ZIP/ZipContainer.swift:43-58 (entry data: getEntryData :62-125)
 * ZipContainer.info(container:) -> [ZipEntryInfo] Sources/ZIP/ZipContainer.swift:132-134 (host only, no device needed)
 * One entry per central-directory record, in its order.  All Deflate / BZip2 / LZMA entries of a container are decoded as
 * one batch each; errors (and the entries returned with SWC_ZIP_WRONG_CRC: the failing one last) are those of the reference's
 * entry-by-entry loop.  `*out` holds every entry's data at [data_off, data_off + data_len); free both results with swc_free. */
typedef struct swc_zip_entry {
    uint64_t name_off, name_len;         /* ZipEntryInfo.name: bytes inside the container (central directory) */
    uint64_t comment_off, comment_len;   /* ZipEntryInfo.comment */
    uint64_t data_off, data_len;         /* ZipEntry.data inside *out (0, 0 for directories and for swc_zip_info) */
    uint64_t size;                       /* ZipEntryInfo.size */
    uint32_t crc;                        /* ZipEntryInfo.crc */
    uint32_t external_attrs;             /* externalFileAttributes: permissions = (attrs & 0x0FFF0000) >> 16, dosAttributes = attrs & 0xFF */
    uint16_t method;                     /* raw compression method: 0 copy, 8 deflate, 12 bzip2, 14 lzma, else .other */
    uint16_t version_made_by;            /* FileSystemType(versionMadeBy) */
    uint16_t internal_attrs;             /* isTextFile = internal_attrs & 1 */
    uint16_t dos_time, dos_date;         /* native modification time */
    uint8_t  is_directory;               /* ZipEntryInfo.type == .directory */
    uint8_t  utf8;                       /* general purpose bit 11: name / comment are UTF-8 (else CP437 unless the bytes need UTF-8) */
} swc_zip_entry;
int32_t swc_zip_open(const uint8_t *in, size_t in_len, uint8_t **out, size_t *out_len, swc_zip_entry **entries, size_t *n_entries);
int32_t swc_zip_info(const uint8_t *in, size_t in_len, swc_zip_entry **entries, size_t *n_entries);

/* ---- TAR container -------------------------------------------------------------------------------------------
 * TarContainer.open(container:) -> [TarEntry]         Sources/TAR/TarContainer.swift:187-224
 * TarContainer.info(container:) -> [TarEntryInfo]     Sources/TAR/TarContainer.swift:239-261
 * TarContainer.formatOf(container:) -> Format         Sources/TAR/TarContainer.swift:36-71
 * All three drive TarParser.next() (TarParser.swift:35-79).  One record per non-special header, in walk order, holding
 * what TarEntryInfo.init (TarEntryInfo.swift:184-242) resolves.  Offsets are relative to the unit's first byte; text
 * fields are byte ranges into the unit, already resolved to the winning source (local PAX, global PAX, GNU L / K entry,
 * header).  The host decodes text (String(cString:) repair), converts PAX times with Double(String) and splits the
 * extended-header payloads into the unknown records. */
enum {
    SWC_TAR_MODE = 1u << 0, SWC_TAR_UID = 1u << 1, SWC_TAR_GID = 1u << 2, SWC_TAR_DEV_MAJOR = 1u << 3,
    SWC_TAR_DEV_MINOR = 1u << 4, SWC_TAR_MTIME = 1u << 5, SWC_TAR_ATIME = 1u << 6, SWC_TAR_CTIME = 1u << 7,
    SWC_TAR_UNAME = 1u << 8, SWC_TAR_GNAME = 1u << 9, SWC_TAR_CHARSET = 1u << 10, SWC_TAR_COMMENT = 1u << 11,
    SWC_TAR_LOCAL = 1u << 12, SWC_TAR_GLOBAL = 1u << 13, SWC_TAR_PREFIX = 1u << 14,
    SWC_TAR_PAX_TIME0 = 1u << 16               /* << k for pax_time[k], k = 0..5 */
};
enum { SWC_TAR_PRE_POSIX = 0, SWC_TAR_USTAR = 1, SWC_TAR_GNU = 2, SWC_TAR_PAX = 3 };   /* TarContainer.Format */
typedef struct swc_tar_entry {
    uint64_t header_off, data_off;       /* the entry's header; its data starts 512 bytes later */
    int64_t  size;                       /* TarEntryInfo.size as info reports it: PAX size when given, else the header's */
    int64_t  open_size;                  /* as open reports it: 0 for directories (their data is nil) */
    int64_t  mode;                       /* permissions (& 0xFFF); SWC_TAR_MODE */
    int64_t  uid, gid;                   /* ownerID / groupID, resolved; SWC_TAR_UID / SWC_TAR_GID */
    int64_t  dev_major, dev_minor;       /* header only (ustar / GNU magic) */
    int64_t  mtime, atime, ctime;        /* the header's times as integers (atime / ctime: GNU only) */
    uint64_t name_off, name_len;         /* winning name; with SWC_TAR_PREFIX the header's prefix goes in front */
    uint64_t prefix_off, prefix_len;
    uint64_t link_off, link_len;         /* winning linkName */
    uint64_t uname_off, uname_len, gname_off, gname_len, charset_off, charset_len, comment_off, comment_len;
    uint64_t pax_time_off[6], pax_time_len[6];  /* last UTF-8 value of mtime, atime, ctime: local 0-2, global 3-5 */
    uint64_t local_off, local_len, global_off, global_len;  /* extended-header payloads in force (unknown records) */
    uint32_t present;                    /* SWC_TAR_* bits */
    uint8_t  typeflag;                   /* raw typeflag byte (ContainerEntryType+Tar.swift) */
    uint8_t  reserved[3];
} swc_tar_entry;
/* Walks units in_base[in_off[i] ..+ in_len[i]) (device memory, any alignment), one warp each, asynchronous on
 * `cuda_stream`; it reads nothing back and can be captured in a CUDA graph.  Two optional columns (NULL: absent) let the
 * units be another batch's outputs as that batch left them (out_off, out_len, out_cap, status):
 *   in_cap[i]     the unit is at most in_cap[i] bytes: the walk never reads past min(in_len[i], in_cap[i]), so an
 *                 out_len that reports a required size past the capacity (SWC_ERR_OUTPUT_OVERFLOW) stays in its region;
 *   in_status[i]  a unit whose status is not SWC_OK is not walked: it reports 0 records and that status in info_status,
 *                 open_status and format_status (the archive was never produced, so there is nothing to open).
 * Unit i writes up to entry_cap[i] records at entries[entry_off[i] ..) and reports:
 *   n_entries[i]      the records the walk produced (also when more than entry_cap[i]);
 *   info_status[i]    info's status: SWC_OK, a TarError, or SWC_ERR_REFERENCE_TRAP where the reference traps or never
 *                     returns (DESIGN §6); SWC_ERR_OUTPUT_OVERFLOW when it would be SWC_OK but the table is too small;
 *   open_status[i]    open's status: info's, unless an earlier entry fails open's data bound (tooSmallFileIsPassed) or
 *                     its data range is inverted or overflows (trap); overflow as for info;
 *   format[i], format_status[i]  formatOf's result (SWC_TAR_*) and status; formatOf returns early, so it never reports
 *                     an error behind the point where it returns.
 * in_len[i] / 512 + 1 records suffice for every archive without a negative size. */
int32_t swc_tar_walk_batch(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len,
                           const uint64_t *in_cap, const int32_t *in_status, swc_tar_entry *entries, const uint64_t *entry_off, const uint64_t *entry_cap,
                           uint64_t *n_entries, int32_t *info_status, int32_t *open_status, int32_t *format,
                           int32_t *format_status, uint64_t n, void *cuda_stream);
/* The one-unit batch on a host container.  *entries (swc_alloc'ed, free with swc_free) is filled on SWC_OK; open's
 * entry data is in[data_off ..+ open_size), nothing is copied.  swc_tar_format stores the format only on SWC_OK. */
int32_t swc_tar_info(const uint8_t *in, size_t in_len, swc_tar_entry **entries, size_t *n_entries);
int32_t swc_tar_open(const uint8_t *in, size_t in_len, swc_tar_entry **entries, size_t *n_entries);
int32_t swc_tar_format(const uint8_t *in, size_t in_len, int32_t *format);

/* ---- checks (device-side, used by the wrappers; exposed for the shim and the tests) ---------------------------
 * CheckSums.crc32 / bzip2crc32 / crc64 / adler32   Sources/Common/CheckSums.swift:12-57
 * XxHash32.hash                                     Sources/LZ4/XxHash32.swift:24-83
 * Sha256.hash                                       Sources/XZ/Sha256.swift */
int32_t swc_crc32(const uint8_t *in, size_t n, uint32_t *result);
int32_t swc_bzip2_crc32(const uint8_t *in, size_t n, uint32_t *result);
int32_t swc_crc64(const uint8_t *in, size_t n, uint64_t *result);
int32_t swc_adler32(const uint8_t *in, size_t n, uint32_t *result);
int32_t swc_xxh32(const uint8_t *in, size_t n, uint32_t *result);
int32_t swc_sha256(const uint8_t *in, size_t n, uint8_t digest[32]);
/* batched epilogues on DEVICE buffers (asynchronous on `cuda_stream`): one result per unit in_base[off[i] .. off[i]+len[i]).
 * `status` may be NULL; units whose status[i] != 0 are not read (their result is 0, for Adler-32 too). */
int32_t swc_crc32_batch(const uint8_t *in_base, const uint64_t *off, const uint64_t *len, const int32_t *status,
                        uint32_t *result, uint64_t n, void *cuda_stream);
int32_t swc_xxh32_batch(const uint8_t *in_base, const uint64_t *off, const uint64_t *len,
                        uint32_t *result, uint64_t n, void *cuda_stream);
int32_t swc_adler32_batch(const uint8_t *in_base, const uint64_t *off, const uint64_t *len, const int32_t *status,
                          uint32_t *result, uint64_t n, void *cuda_stream);
int32_t swc_crc64_batch(const uint8_t *in_base, const uint64_t *off, const uint64_t *len, const int32_t *status,
                        uint64_t *result, uint64_t n, void *cuda_stream);

#ifdef __cplusplus
}
#endif
#endif /* SWCGPU_H */
