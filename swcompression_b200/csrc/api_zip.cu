// api_zip.cu — C ABI for ZIP containers: ZipContainer.open / info (reference Sources/ZIP/ZipContainer.swift:43-180).
// The central directory gives every entry's method, sizes and offset up front, so a container is a ready-made batch: the
// host walks End of Central Directory -> central directory -> local headers (ZipEndOfCentralDirectory.swift:22-110,
// ZipCentralDirectoryEntry.swift:45-141, ZipLocalHeader.swift:39-139) exactly once, then ALL Deflate entries go through one
// swc_deflate_decompress_batch call, all BZip2 entries through one swc_bzip2_decompress_batch call, all LZMA entries through
// one swc_lzma_decompress_batch call, stored entries are device-to-device copies, and one batched CRC-32 launch covers every
// entry.  The reference's per-entry loop (ZipContainer.swift:46-57, getEntryData :62-125) is kept as the in-order validator,
// so the error that is reported — and the entries returned with ZipError.wrongCRC — are those of the sequential walk.
#include <cstring>
#include <string>
#include <vector>
#include "../../include/swcgpu.h"
#include "host_util.h"

namespace swc {
namespace {

// ---- bounds-aware little-endian view: any access outside the container is a BitByteData precondition failure (trap) ----
struct View {
    const uint8_t *p; size_t n;
    bool trapped = false;
    uint64_t le(int64_t at, int bytes) {
        if (at < 0 || (uint64_t)at + (uint64_t)bytes > n) { trapped = true; return 0; }
        uint64_t v = 0;
        for (int i = bytes - 1; i >= 0; i--) v = (v << 8) | p[at + i];
        return v;
    }
};
struct Seq {                       // sequential reads on top of a View: `at` may be set anywhere, like reader.offset
    View &v; int64_t at;
    uint64_t take(int bytes) { const uint64_t x = v.le(at, bytes); at += bytes; return x; }
};

// String(data:encoding:.utf8) != nil
constexpr uint64_t kDeflateUnitMax = ((uint64_t)1 << 28) - 1;     // longest Deflate unit every batch kernel takes

bool utf8_ok(const uint8_t *s, size_t n) {
    for (size_t i = 0; i < n;) {
        const unsigned b = s[i];
        if (b < 0x80) { i++; continue; }
        int k = b >= 0xC2 && b <= 0xDF ? 1 : b >= 0xE0 && b <= 0xEF ? 2 : b >= 0xF0 && b <= 0xF4 ? 3 : -1;
        if (k < 0 || i + (size_t)k >= n) return false;
        uint32_t cp = k == 1 ? b & 0x1F : k == 2 ? b & 0x0F : b & 0x07;
        for (int j = 1; j <= k; j++) { if ((s[i + j] & 0xC0) != 0x80) return false; cp = cp << 6 | (s[i + j] & 0x3F); }
        if (k == 2 && (cp < 0x800 || (cp >= 0xD800 && cp <= 0xDFFF))) return false;
        if (k == 3 && (cp < 0x10000 || cp > 0x10FFFF)) return false;
        i += (size_t)k + 1;
    }
    return true;
}
// Data.needsUtf8(), LittleEndianByteReader+Zip.swift:44-98: BOM, or the FIRST non-ASCII byte starts a well-formed sequence
bool wants_utf8(const uint8_t *s, size_t n) {
    if (n >= 3 && s[0] == 0xEF && s[1] == 0xBB && s[2] == 0xBF) return true;
    size_t i = 0;
    while (i < n && s[i] < 0x80) i++;
    if (i == n) return false;
    const unsigned b = s[i];
    const int len = b >= 0xC2 && b <= 0xDF ? 2 : b >= 0xE0 && b <= 0xEF ? 3 : b >= 0xF0 && b <= 0xF4 ? 4 : 0;
    if (!len || i + len - 1 >= n) return false;
    for (int k = 1; k < len; k++) if ((s[i + k] & 0xC0) != 0x80) return false;
    if (len == 3) {
        const uint32_t ch = (uint32_t)(s[i] & 0x0F) << 12 | (uint32_t)(s[i + 1] & 0x3F) << 6 | (uint32_t)(s[i + 2] & 0x3F);
        return !(ch < 0x800 || (ch >> 11) == 0x1B);
    }
    if (len == 4) {
        const uint32_t ch = (uint32_t)(s[i] & 0x07) << 18 | (uint32_t)(s[i + 1] & 0x3F) << 12 | (uint32_t)(s[i + 2] & 0x3F) << 6 | (uint32_t)(s[i + 3] & 0x3F);
        return !(ch < 0x10000 || ch > 0x10FFFF);
    }
    return true;
}
// zipString (:11-24): false = nil -> ZipError.wrongTextField
bool text_field(Seq &q, int64_t len, bool utf8_flag, uint64_t *off, uint64_t *n) {
    *off = 0; *n = 0;
    if (len <= 0) return true;
    if (q.at < 0 || (uint64_t)q.at + (uint64_t)len > q.v.n) { q.v.trapped = true; q.at += len; return true; }
    const uint8_t *s = q.v.p + q.at;
    *off = (uint64_t)q.at; *n = (uint64_t)len;
    q.at += len;
    if (utf8_flag || wants_utf8(s, (size_t)len)) return utf8_ok(s, (size_t)len);
    return true;                                                    // CP437 decodes any byte string
}

struct Item {
    swc_zip_entry e;
    uint16_t flags = 0;
    bool has_dd = false, zip64_local = false;
    int64_t data_off = 0;
    uint64_t comp = 0, uncomp = 0;
};

// Extra fields only matter for how far they move the reader and for the Zip64 sizes (BuiltinExtraFields.swift:19-127).
struct Sizes { uint64_t comp, uncomp, local_off; uint32_t disk; bool zip64; };
void skip_extra(Seq &q, unsigned id, int64_t size, bool central, Sizes &z) {
    if (id == 0x0001) {
        if (central) {
            if (z.uncomp == 0xFFFFFFFFull) z.uncomp = q.take(8);
            if (z.comp == 0xFFFFFFFFull) z.comp = q.take(8);
            if (z.local_off == 0xFFFFFFFFull) z.local_off = q.take(8);
            if (z.disk == 0xFFFF) z.disk = (uint32_t)q.take(4);
        } else { z.uncomp = q.take(8); z.comp = q.take(8); z.zip64 = true; }
    } else if (id == 0x5455) {
        const int64_t end = q.at + size;
        const unsigned f = (unsigned)q.take(1);
        const int words = (f & 1) + (central ? 0 : ((f >> 1) & 1) + ((f >> 2) & 1));
        for (int i = 0; i < words; i++) q.take(4);
        q.at = end;
    } else if (id == 0x000a) {
        q.at += 4;
        const unsigned tag = (unsigned)q.take(2);
        q.at += 2;
        if (tag == 1) q.take(8), q.take(8), q.take(8);
    } else if (id == 0x7855) {
        if (central) q.at += size; else q.take(4);
    } else if (id == 0x7875) {
        if (q.take(1) == 1) {
            for (int k = 0; k < 2; k++) {
                const int64_t w = (int64_t)q.take(1);
                if (w > 8) q.at += w; else q.take((int)w);
            }
        }
    } else {
        q.at += size;
    }
}

// infoWithHelper (ZipContainer.swift:136-180): fills `items` in central-directory order
int read_directory(const uint8_t *in, size_t n, std::vector<Item> &items) {
    if (n < 22) return SWC_ZIP_NOT_FOUND_CENTRAL_DIRECTORY_END;
    View v{in, n};
    int64_t sig_at = (int64_t)n - 22;
    while (v.le(sig_at, 4) != 0x06054b50u) {                          // the reader steps back one byte per probe (:147-157)
        if (sig_at == 0) return SWC_ZIP_NOT_FOUND_CENTRAL_DIRECTORY_END;
        sig_at--;
    }
    Seq q{v, sig_at + 4};
    uint64_t disk = q.take(2), cd_disk = q.take(2);
    if (v.trapped) return SWC_ERR_REFERENCE_TRAP;
    if (disk != cd_disk) return SWC_ZIP_MULTI_VOLUMES_NOT_SUPPORTED;
    uint64_t here = q.take(2), total = q.take(2);
    if (v.trapped) return SWC_ERR_REFERENCE_TRAP;
    if (here != total) return SWC_ZIP_MULTI_VOLUMES_NOT_SUPPORTED;
    uint64_t cd_size = q.take(4), cd_off = q.take(4);
    if (v.trapped) return SWC_ERR_REFERENCE_TRAP;
    if (disk == 0xFFFF || here == 0xFFFF || cd_size == 0xFFFFFFFFull || cd_off == 0xFFFFFFFFull) {       // Zip64 records
        q.at -= 40;                                                       // locator: 20 bytes in front of the end record
        if (q.take(4) != 0x07064b50u) return v.trapped ? SWC_ERR_REFERENCE_TRAP : SWC_ZIP_WRONG_SIGNATURE;
        const uint64_t start_disk = q.take(4);
        if (v.trapped) return SWC_ERR_REFERENCE_TRAP;
        if (disk != start_disk) return SWC_ZIP_MULTI_VOLUMES_NOT_SUPPORTED;
        const int64_t end64 = (int64_t)q.take(8);
        const uint64_t disks = q.take(4);
        if (v.trapped) return SWC_ERR_REFERENCE_TRAP;
        if (disks != 1) return SWC_ZIP_MULTI_VOLUMES_NOT_SUPPORTED;
        q.at = end64;
        if (q.take(4) != 0x06064b50u) return v.trapped ? SWC_ERR_REFERENCE_TRAP : SWC_ZIP_WRONG_SIGNATURE;
        q.at += 10;                                                       // record size (8), version made by (2)
        const uint64_t needed = q.take(2);
        if (v.trapped) return SWC_ERR_REFERENCE_TRAP;
        if ((needed & 0xFF) > 63) return SWC_ZIP_WRONG_VERSION;
        disk = q.take(4); cd_disk = q.take(4);
        if (v.trapped) return SWC_ERR_REFERENCE_TRAP;
        if (disk != cd_disk) return SWC_ZIP_MULTI_VOLUMES_NOT_SUPPORTED;
        here = q.take(8); total = q.take(8);
        if (v.trapped) return SWC_ERR_REFERENCE_TRAP;
        if (here != total) return SWC_ZIP_MULTI_VOLUMES_NOT_SUPPORTED;
        cd_size = q.take(8); cd_off = q.take(8);
        if (v.trapped) return SWC_ERR_REFERENCE_TRAP;
    }
    q.at = (int64_t)cd_off;
    if (q.take(4) == 0x08064b50u) q.at += (int64_t)q.take(4); else q.at -= 4;      // archive extra data record
    if (v.trapped || total > n) return SWC_ERR_REFERENCE_TRAP;
    items.reserve((size_t)total);
    for (uint64_t k = 0; k < total; k++) {
        Item it;
        memset(&it.e, 0, sizeof(it.e));
        // ---- central directory entry ----
        if (q.take(4) != 0x02014b50u) return v.trapped ? SWC_ERR_REFERENCE_TRAP : SWC_ZIP_WRONG_SIGNATURE;
        it.e.version_made_by = (uint16_t)q.take(2);
        const unsigned cd_needed = (unsigned)q.take(2), cd_flags = (unsigned)q.take(2), cd_method = (unsigned)q.take(2);
        it.e.dos_time = (uint16_t)q.take(2); it.e.dos_date = (uint16_t)q.take(2);
        const uint32_t cd_crc = (uint32_t)q.take(4);
        Sizes cz{0, 0, 0, 0, false};
        cz.comp = q.take(4); cz.uncomp = q.take(4);
        const int64_t name_len = (int64_t)q.take(2), extra_len = (int64_t)q.take(2), comment_len = (int64_t)q.take(2);
        cz.disk = (uint32_t)q.take(2);
        it.e.internal_attrs = (uint16_t)q.take(2); it.e.external_attrs = (uint32_t)q.take(4);
        cz.local_off = q.take(4);
        if (v.trapped) return SWC_ERR_REFERENCE_TRAP;
        const bool utf8 = (cd_flags & 0x800) != 0;
        it.e.utf8 = utf8;
        if (!text_field(q, name_len, utf8, &it.e.name_off, &it.e.name_len)) return SWC_ZIP_WRONG_TEXT_FIELD;
        if (v.trapped) return SWC_ERR_REFERENCE_TRAP;
        for (const int64_t start = q.at; q.at - start < extra_len;) {
            const unsigned id = (unsigned)q.take(2);
            const int64_t size = (int64_t)q.take(2);
            if (v.trapped) return SWC_ERR_REFERENCE_TRAP;
            skip_extra(q, id, size, true, cz);
            if (v.trapped) return SWC_ERR_REFERENCE_TRAP;
        }
        if (!text_field(q, comment_len, utf8, &it.e.comment_off, &it.e.comment_len)) return v.trapped ? SWC_ERR_REFERENCE_TRAP : SWC_ZIP_WRONG_TEXT_FIELD;
        if (v.trapped) return SWC_ERR_REFERENCE_TRAP;
        const int64_t next_cd = q.at;
        // ---- local header ----
        q.at = (int64_t)cz.local_off;
        if (q.take(4) != 0x04034b50u) return v.trapped ? SWC_ERR_REFERENCE_TRAP : SWC_ZIP_WRONG_SIGNATURE;
        const unsigned lh_needed = (unsigned)q.take(2), lh_flags = (unsigned)q.take(2), lh_method = (unsigned)q.take(2);
        const unsigned lh_time = (unsigned)q.take(2), lh_date = (unsigned)q.take(2);
        const uint32_t lh_crc = (uint32_t)q.take(4);
        Sizes lz{0, 0, 0, 0, false};
        lz.comp = q.take(4); lz.uncomp = q.take(4);
        const int64_t lname = (int64_t)q.take(2), lextra = (int64_t)q.take(2);
        if (v.trapped) return SWC_ERR_REFERENCE_TRAP;
        uint64_t o_, n_;
        if (!text_field(q, lname, (lh_flags & 0x800) != 0, &o_, &n_)) return SWC_ZIP_WRONG_TEXT_FIELD;
        if (v.trapped) return SWC_ERR_REFERENCE_TRAP;
        for (const int64_t start = q.at; q.at - start < lextra;) {
            const unsigned id = (unsigned)q.take(2);
            const int64_t size = (int64_t)q.take(2);
            if (v.trapped) return SWC_ERR_REFERENCE_TRAP;
            skip_extra(q, id, size, false, lz);
            if (v.trapped) return SWC_ERR_REFERENCE_TRAP;
        }
        it.data_off = q.at;
        // ---- ZipLocalHeader.validate(with:) ----
        if ((lh_needed & 0xFF) > 63) return SWC_ZIP_WRONG_VERSION;
        if (lh_flags & (0x2000 | 0x40 | 0x01)) return SWC_ZIP_ENCRYPTION_NOT_SUPPORTED;
        if (lh_flags & 0x20) return SWC_ZIP_PATCHING_NOT_SUPPORTED;
        if ((cd_needed & 0xFF) > 63) return SWC_ZIP_WRONG_VERSION;
        if (cz.disk != (uint32_t)disk) return SWC_ZIP_MULTI_VOLUMES_NOT_SUPPORTED;
        if (lh_flags != cd_flags || lh_method != cd_method || lh_time != it.e.dos_time || lh_date != it.e.dos_date) return SWC_ZIP_WRONG_LOCAL_HEADER;
        // ---- ZipEntryInfoHelper / ZipEntryInfo ----
        it.flags = (uint16_t)lh_flags;
        it.has_dd = (lh_flags & 0x08) != 0;
        it.zip64_local = lz.zip64;
        it.comp = it.has_dd ? cz.comp : lz.comp;
        it.uncomp = it.has_dd ? cz.uncomp : lz.uncomp;
        it.e.size = it.uncomp;
        it.e.crc = it.has_dd ? cd_crc : lh_crc;
        it.e.method = (uint16_t)lh_method;
        const uint32_t unix_type = (it.e.external_attrs & 0xF0000000u) >> 16;
        switch (unix_type) {                                              // ContainerEntryType(unixType), else the DOS directory bit
        case 0040000: it.e.is_directory = 1; break;
        case 0010000: case 0020000: case 0060000: case 0100000: case 0120000: case 0140000: it.e.is_directory = 0; break;
        default: it.e.is_directory = (it.e.external_attrs & 0x10) != 0;
        }
        items.push_back(it);
        q.at = next_cd;
    }
    return SWC_OK;
}

}  // namespace
}  // namespace swc

using namespace swc;

extern "C" {

int32_t swc_zip_info(const uint8_t *in, size_t in_len, swc_zip_entry **entries, size_t *n_entries) {
    if (!in || !entries || !n_entries) return SWC_ERR_INVALID_ARG;
    *entries = nullptr; *n_entries = 0;
    std::vector<Item> items;
    const int st = read_directory(in, in_len, items);
    if (st) return st;
    *entries = (swc_zip_entry *)swc_alloc(sizeof(swc_zip_entry) * (items.size() + 1));
    if (!*entries) return SWC_ERR_OUTPUT_OVERFLOW;
    for (size_t i = 0; i < items.size(); i++) (*entries)[i] = items[i].e;
    *n_entries = items.size();
    return SWC_OK;
}

int32_t swc_zip_open(const uint8_t *in, size_t in_len, uint8_t **out, size_t *out_len, swc_zip_entry **entries, size_t *n_entries) {
    if (!in || !out || !out_len || !entries || !n_entries) return SWC_ERR_INVALID_ARG;
    *out = nullptr; *out_len = 0; *entries = nullptr; *n_entries = 0;
    std::vector<Item> items;
    int st = read_directory(in, in_len, items);
    if (st) return st;
    if (ensure_device()) return SWC_ERR_NO_DEVICE;
    ApiLock api_lock;
    const size_t n = items.size();
    // ---- lay the batch out: one output region per file entry (16-byte aligned), units grouped by method ----
    struct Unit { size_t item; uint64_t in_off, in_len, out_off, cap; };
    std::vector<Unit> grp[4];                                           // 0 stored, 1 deflate, 2 bzip2, 3 lzma
    std::vector<int> early(n, SWC_OK);                                  // errors known before any decoding (reported in entry order)
    std::vector<char> clipped(n, 0);                                    // Deflate units given less than the rest of the container
    uint64_t out_total = 0;
    for (size_t i = 0; i < n; i++) {
        Item &it = items[i];
        if (it.e.is_directory) continue;
        const int g = it.e.method == 0 ? 0 : it.e.method == 8 ? 1 : it.e.method == 12 ? 2 : it.e.method == 14 ? 3 : -1;
        if (it.data_off < 0 || (uint64_t)it.data_off > in_len) { early[i] = SWC_ERR_REFERENCE_TRAP; continue; }
        const uint64_t avail = in_len - (uint64_t)it.data_off;
        if (g < 0) { early[i] = SWC_ZIP_COMPRESSION_NOT_SUPPORTED; continue; }
        if (g == 0 && it.uncomp > avail) { early[i] = SWC_ERR_REFERENCE_TRAP; continue; }
        if (g == 3) {
            if (avail < 9) { early[i] = SWC_ERR_REFERENCE_TRAP; continue; }
            if (in[it.data_off + 4] >= 225) { early[i] = SWC_LZMA_WRONG_PROPERTIES; continue; }
        }
        // capacity = the declared size; a declared size no stream of this length can reach is clipped (it will end as wrongSize)
        uint64_t cap = g == 0 ? it.uncomp : it.uncomp + 16;              // slack: the LZMA kernel wants room behind the last byte,
                                                                          // and a stream slightly longer than declared ends as wrongSize without a second decode
        const uint64_t reach = g == 1 ? avail * 1032 + 64 : g == 2 ? avail * 65536 + 4096 : g == 3 ? avail * 8192 + 4096 : avail;
        if (cap > reach + 16) cap = reach + 16;
        if (cap > ((uint64_t)8 << 30)) cap = (uint64_t)8 << 30;
        // A Deflate stream has no length of its own: the reference reads it from the rest of the container.  The batch's
        // table-lookup kernel keeps 32-bit bit positions and refuses units of 2^28 bytes or more, so in a container past
        // 256 MiB a unit gets at most 2^28 - 1 bytes; a clipped unit that fails is decoded again on its own with everything.
        uint64_t in_len = avail - (g == 3 ? 9 : 0);
        if (g == 1 && in_len > kDeflateUnitMax) { in_len = kDeflateUnitMax; clipped[i] = 1; }
        Unit u{i, (uint64_t)it.data_off + (g == 3 ? 9 : 0), in_len, out_total, cap};
        out_total += round16((size_t)cap) + 16;
        grp[g].push_back(u);
    }
    DevBuf d_in, d_out;
    if ((st = upload_input(d_in, in, in_len))) return st;
    if ((st = d_out.alloc((size_t)out_total + 64))) return st;
    const size_t nu = grp[0].size() + grp[1].size() + grp[2].size() + grp[3].size();
    // stored units are copies: their length, consumed bytes and (zero) status are filled in here
    UnitTable t;
    const Col<u64> in_off = t.in<u64>(nu), in_len_c = t.in<u64>(nu), out_off = t.in<u64>(nu), cap = t.in<u64>(nu);
    const Col<u64> got_len = t.in<u64>(nu), consumed = t.in<u64>(nu);
    const Col<int32_t> status = t.in<int32_t>(nu);
    const Col<uint32_t> props = t.in<uint32_t>(nu);
    const Col<int64_t> dict = t.in<int64_t>(nu), usize = t.in<int64_t>(nu);
    const Col<uint32_t> crc = t.out<uint32_t>(nu);
    if ((st = t.alloc())) return st;
    int64_t *h_dict = t.host(dict);
    const u64 *h_out_off = t.host(out_off);
    std::vector<size_t> unit_of_item(n, (size_t)-1);
    size_t base[5] = {0, grp[0].size(), 0, 0, 0};
    base[2] = base[1] + grp[1].size(); base[3] = base[2] + grp[2].size(); base[4] = base[3] + grp[3].size();
    for (int g = 0; g < 4; g++)
        for (size_t k = 0; k < grp[g].size(); k++) {
            const Unit &u = grp[g][k];
            const size_t j = base[g] + k;
            unit_of_item[u.item] = j;
            t.host(in_off)[j] = u.in_off; t.host(in_len_c)[j] = u.in_len; t.host(out_off)[j] = u.out_off; t.host(cap)[j] = u.cap;
            if (g == 0) { t.host(got_len)[j] = u.cap; t.host(consumed)[j] = u.cap; }      // stored: length and consumed are the size
            if (g == 3) {
                const uint8_t *p = in + items[u.item].data_off;
                const unsigned b = p[4];
                t.host(props)[j] = (b % 9) | (((b / 9) % 5) << 8) | (((b / 9) / 5) << 16);    // LZMAProperties.swift:49-58
                h_dict[j] = (int64_t)p[5] | (int64_t)p[6] << 8 | (int64_t)p[7] << 16 | (int64_t)p[8] << 24;
                t.host(usize)[j] = (int64_t)items[u.item].uncomp;
            }
        }
    cudaStream_t s = 0;
    if (nu && (st = t.upload(s))) return st;
    for (const Unit &u : grp[0])
        if (u.cap) SWC_CUDA_TRY(cudaMemcpyAsync(d_out.as<u8>() + u.out_off, d_in.as<u8>() + u.in_off, (size_t)u.cap, cudaMemcpyDeviceToDevice, s));
    auto at = [&](auto c, int g) { return t.dev(c) + base[g]; };     // the columns of method group g
    if (!grp[1].empty() &&
        (st = swc_deflate_decompress_batch(d_in.as<u8>(), at(in_off, 1), at(in_len_c, 1), nullptr, d_out.as<u8>(), at(out_off, 1), at(cap, 1),
                                           out_total, at(got_len, 1), at(consumed, 1), at(status, 1), grp[1].size(), nullptr, 0, s))) return st;
    if (!grp[2].empty() &&
        (st = swc_bzip2_decompress_batch(d_in.as<u8>(), at(in_off, 2), at(in_len_c, 2), d_out.as<u8>(), at(out_off, 2), at(cap, 2),
                                         at(got_len, 2), at(consumed, 2), at(status, 2), grp[2].size(), s))) return st;
    if (!grp[3].empty() &&
        (st = swc_lzma_decompress_batch(d_in.as<u8>(), at(in_off, 3), at(in_len_c, 3), at(props, 3), at(dict, 3), at(usize, 3), d_out.as<u8>(),
                                        at(out_off, 3), at(cap, 3), at(got_len, 3), at(consumed, 3), at(status, 3), grp[3].size(), s))) return st;
    if (nu && (st = swc_crc32_batch(d_out.as<u8>(), t.dev(out_off), t.dev(got_len), t.dev(status), t.dev(crc), nu, s))) return st;
    std::vector<uint64_t> r_len, r_used;
    std::vector<int32_t> r_st;
    std::vector<uint32_t> r_crc;
    if ((st = t.fetch(got_len, r_len, s)) || (st = t.fetch(consumed, r_used, s)) || (st = t.fetch(status, r_st, s)) ||
        (st = t.fetch(crc, r_crc, s))) return st;
    // ---- the reference's loop over the entries (ZipContainer.swift:46-57), now only checking ----
    View v{in, in_len};
    int result = SWC_OK;
    size_t returned = n;
    std::vector<std::pair<uint8_t *, size_t>> redone(n, {nullptr, 0});       // entries that had to be decoded again on their own
    auto free_redone = [&] { for (auto &r : redone) if (r.first) swc_free(r.first); };
    for (size_t i = 0; i < n && result == SWC_OK; i++) {
        Item &it = items[i];
        if (it.e.is_directory) continue;
        if (early[i]) { result = early[i]; break; }
        const size_t j = unit_of_item[i];
        const int g = it.e.method == 0 ? 0 : it.e.method == 8 ? 1 : it.e.method == 12 ? 2 : 3;
        int ust = r_st[j];
        uint64_t got = r_len[j], used = r_used[j];
        uint32_t crc_got = r_crc[j];
        if (ust == SWC_ERR_OUTPUT_OVERFLOW || ust == SWC_ERR_UNSUPPORTED || (ust != SWC_OK && clipped[i])) {
            // more output than declared (-> wrongSize, unless the stream fails further on), an LZMA stream the batch kernel
            // does not take (lc + lp > 4), or a clipped Deflate unit that may have run out of input: decode this entry alone
            // through the single-unit path, which sizes itself and reads the whole rest of the container
            const uint8_t *p = in + it.data_off;
            const size_t avail = in_len - (size_t)it.data_off;
            uint8_t *o = nullptr; size_t ol = 0, c = 0;
            if (g == 1) { ust = swc_deflate_decompress(p, avail, 0, &o, &ol, &c); used = c; }
            else if (g == 2) { ust = swc_bzip2_decompress(p, avail, 0, &o, &ol, &c); used = c; }
            else {
                const unsigned b = p[4];
                ust = swc_lzma_decompress_raw(p + 9, avail - 9, b % 9, (b / 9) % 5, (b / 9) / 5, h_dict[j], (int64_t)it.uncomp, &o, &ol, &c);
                used = c;
            }
            got = ol;
            redone[i] = {o, ol};
            if (ust == SWC_OK && ol) { uint32_t c32 = 0; if ((st = swc_crc32(o, ol, &c32))) { free_redone(); return st; } crc_got = c32; }
            else crc_got = 0;
        }
        if (ust != SWC_OK) { result = ust; break; }
        const uint64_t real_comp = g == 0 ? it.uncomp : g == 3 ? used + 9 : (used + 7) / 8;     // align() after a bit reader (:78, :86)
        uint64_t comp = it.comp, uncomp = it.uncomp;
        uint32_t crc = it.e.crc;
        if (it.has_dd) {                                                  // data descriptor (:97-112)
            Seq d{v, it.data_off + (int64_t)real_comp};
            if (d.take(4) != 0x08074b50u) d.at -= 4;
            crc = (uint32_t)d.take(4);
            const int w = it.zip64_local ? 8 : 4;
            comp = d.take(w); uncomp = d.take(w);
            if (v.trapped) { result = SWC_ERR_REFERENCE_TRAP; break; }
        }
        if (!(comp == real_comp && uncomp == got)) { result = SWC_ZIP_WRONG_SIZE; break; }
        it.e.data_len = got;
        if (crc != crc_got) { result = SWC_ZIP_WRONG_CRC; returned = i + 1; }        // the entry is still part of the payload
    }
    if (result != SWC_OK && result != SWC_ZIP_WRONG_CRC) { free_redone(); return result; }
    // ---- hand the data back: one device->host copy, entries point into it ----
    bool any_redone = false;
    for (size_t i = 0; i < returned; i++) any_redone = any_redone || redone[i].first;
    size_t extra = 0;
    for (size_t i = 0; i < returned; i++) if (redone[i].first) extra += round16(redone[i].second);
    uint8_t *h = (uint8_t *)swc_alloc((size_t)out_total + extra + 16);
    if (!h) { free_redone(); return SWC_ERR_OUTPUT_OVERFLOW; }
    if (out_total && (st = copy_pageable(h, d_out.p, (size_t)out_total, false))) { swc_free(h); free_redone(); return st; }
    size_t tail = (size_t)out_total;
    swc_zip_entry *es = (swc_zip_entry *)swc_alloc(sizeof(swc_zip_entry) * (returned + 1));
    if (!es) { swc_free(h); free_redone(); return SWC_ERR_OUTPUT_OVERFLOW; }
    for (size_t i = 0; i < returned; i++) {
        es[i] = items[i].e;
        if (items[i].e.is_directory) { es[i].data_off = 0; es[i].data_len = 0; continue; }
        if (redone[i].first) {
            memcpy(h + tail, redone[i].first, redone[i].second);
            es[i].data_off = tail; es[i].data_len = redone[i].second;
            tail += round16(redone[i].second);
        } else {
            es[i].data_off = h_out_off[unit_of_item[i]];
        }
    }
    free_redone();
    *out = h; *out_len = tail; *entries = es; *n_entries = returned;
    return result;
}

}  // extern "C"
