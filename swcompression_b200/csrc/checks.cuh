// checks.cuh — device checksum entry points (all pointers are device pointers; results are 64-bit slots).
#pragma once
#include <vector>
#include "common.cuh"

namespace swc {
namespace checks {

size_t partial_bytes(u64 n);   // scratch for the per-chunk partials
int crc32(const u8 *d, u64 n, u64 *d_result, u64 *d_partial, cudaStream_t s);
int bzip2_crc32(const u8 *d, u64 n, u64 *d_result, u64 *d_partial, cudaStream_t s);
int crc64(const u8 *d, u64 n, u64 *d_result, u64 *d_partial, cudaStream_t s);
int adler32(const u8 *d, u64 n, u64 *d_result, u64 *d_partial, cudaStream_t s);
int xxh32_batch(const u8 *base, const u64 *off /* may be null */, const u64 *len, u32 *result, u64 n, cudaStream_t s);
int sha256(const u8 *d, u64 n, u8 *d_digest, cudaStream_t s);
int crc32_units(const u8 *base, const u64 *off, const u64 *len, const int32_t *status, u32 *result, u64 n, cudaStream_t s);   // warp per buffer; units with status != 0 are skipped (status may be null)
int crc64_units(const u8 *base, const u64 *off, const u64 *len, const int32_t *status, u64 *result, u64 n, cudaStream_t s);   // the same for CRC-64
int adler32_units(const u8 *base, const u64 *off, const u64 *len, const int32_t *status, u32 *result, u64 n, cudaStream_t s);  // the same for Adler-32 (skipped units: 0)
// gzip member candidates of n unit ranges base[off[u] ..+ len[u]) (device columns; the rule is above gzip_scan_kernel)
struct GzipScan {
    const u8 *base;
    const u64 *off, *len;
    u64 n;
    unsigned long long *count;   // per unit, added to
    const u64 *first;            // per unit: first list slot, ~0 = not scanned (or null)
    u64 *list;                   // candidate positions in the unit (or null: count only)
    u64 cap;                     // list capacity when `first` is null
    bool with_zero;              // position 0 is always a candidate
};
int gzip_scan(const GzipScan &s, cudaStream_t stream);
int find_gzip_members(const u8 *d_in, u64 n, std::vector<size_t> &pos);   // sorted candidate member starts (one-unit scan)
int find_bzip2_magics(const u8 *d_in, u64 begin, u64 n, std::vector<u64> &entries);   // sorted (bit position << 1 | is_end_magic), device scan
int gather_units(const u8 *src, const u64 *src_off, const u64 *len, u8 *dst, const u64 *dst_off, u64 n, cudaStream_t s);

// host convenience: run a 32/64-bit check over a device buffer and fetch the value (blocking)
enum Kind { CRC32 = 0, BZIP2_CRC32 = 1, CRC64 = 2, ADLER32 = 3, XXH32 = 4 };
int check_device(Kind k, const u8 *d, u64 n, u64 *value);
// CRC32 or ADLER32 of one unit of a decode batch, chunked like check_device, its offset, length and status read on the device:
// the grid covers `cap` >= length bytes, d_partial holds partial_bytes(cap); a unit whose status is not 0 gets 0
int unit_check(Kind k, const u8 *base, const u64 *off, const u64 *len, const int32_t *status, u64 cap, u32 *result, u64 *d_partial,
               cudaStream_t s);

}  // namespace checks
}  // namespace swc
