// Public decode API of the reference, bodies routed through libswcgpu (include/swcgpu.h).
//   DecompressionAlgorithm  Sources/Common/DecompressionAlgorithm.swift:9-14
//   Archive                 Sources/Common/Archive.swift:9-14
//   CompressionAlgorithm    Sources/Common/CompressionAlgorithm.swift (LZ4 is its only GPU-backed conformer here)
import CSWCGPU
import Foundation

public protocol DecompressionAlgorithm { static func decompress(data: Data) throws -> Data }
public protocol Archive { static func unarchive(archive: Data) throws -> Data }
public protocol CompressionAlgorithm { static func compress(data: Data) -> Data }

private let payloadCodes: Set<Int32> = [210, 503, 605, 705, 807]

/// Calls a single-unit entry point `(in, len, &out, &outLen) -> status` and wraps the swc_alloc'ed result.
@inline(__always)
private func single(_ data: Data, _ body: (UnsafePointer<UInt8>?, Int, UnsafeMutablePointer<UnsafeMutablePointer<UInt8>?>,
                                         UnsafeMutablePointer<Int>) -> Int32) throws -> Data {
    var out: UnsafeMutablePointer<UInt8>? = nil
    var outLen = 0
    let status: Int32 = data.withUnsafeBytes { raw in
        body(raw.bindMemory(to: UInt8.self).baseAddress, raw.count, &out, &outLen)
    }
    let result = out.map { Data(bytes: $0, count: outLen) } ?? Data()
    swc_free(out)
    guard status == 0 else { throw swcError(status, payload: payloadCodes.contains(status) ? [result] : []) }
    return result
}

/// Same for the multi-* entry points that also return end offsets.
private func multi(_ data: Data, _ body: (UnsafePointer<UInt8>?, Int, UnsafeMutablePointer<UnsafeMutablePointer<UInt8>?>,
                                         UnsafeMutablePointer<Int>, UnsafeMutablePointer<UnsafeMutablePointer<Int>?>,
                                         UnsafeMutablePointer<Int>) -> Int32) throws -> [Data] {
    var out: UnsafeMutablePointer<UInt8>? = nil
    var outLen = 0, count = 0
    var ends: UnsafeMutablePointer<Int>? = nil
    let status: Int32 = data.withUnsafeBytes { raw in
        body(raw.bindMemory(to: UInt8.self).baseAddress, raw.count, &out, &outLen, &ends, &count)
    }
    var parts = [Data]()
    var prev = 0
    for i in 0..<count { let e = ends![i]; parts.append(Data(bytes: out! + prev, count: e - prev)); prev = e }
    swc_free(out); swc_free(ends)
    guard status == 0 else { throw swcError(status, payload: payloadCodes.contains(status) ? parts : []) }
    return parts
}

public class Deflate: DecompressionAlgorithm {                       // Sources/Deflate/Deflate.swift:10-28
    public static func decompress(data: Data) throws -> Data {
        try single(data) { p, n, o, ol in var used = 0; return swc_deflate_decompress(p, n, 0, o, ol, &used) }
    }
}

public class BZip2: DecompressionAlgorithm {                         // Sources/BZip2/BZip2.swift:10-48
    public static func decompress(data: Data) throws -> Data {
        try single(data) { p, n, o, ol in var used = 0; return swc_bzip2_decompress(p, n, 0, o, ol, &used) }
    }
    public static func multiDecompress(data: Data) throws -> [Data] {
        try multi(data) { p, n, o, ol, e, c in swc_bzip2_multi_decompress(p, n, o, ol, e, c) }
    }
}

public struct LZMAProperties {                                       // Sources/LZMA/LZMAProperties.swift:9-47
    public var lc = 3, lp = 0, pb = 2
    public var dictionarySize = 1 << 24 { didSet { if dictionarySize < 1 << 12 { dictionarySize = 1 << 12 } } }
    public init() {}
    public init(lc: Int, lp: Int, pb: Int, dictionarySize: Int) { self.lc = lc; self.lp = lp; self.pb = pb; self.dictionarySize = dictionarySize }
}

public class LZMA: DecompressionAlgorithm {                          // Sources/LZMA/LZMA.swift:10-61
    public static func decompress(data: Data) throws -> Data {
        try single(data) { p, n, o, ol in var used = 0; return swc_lzma_decompress(p, n, o, ol, &used) }
    }
    public static func decompress(data: Data, properties: LZMAProperties, uncompressedSize: Int? = nil) throws -> Data {
        try single(data) { p, n, o, ol in
            var used = 0
            return swc_lzma_decompress_raw(p, n, Int32(properties.lc), Int32(properties.lp), Int32(properties.pb),
                                           Int64(properties.dictionarySize), Int64(uncompressedSize ?? -1), o, ol, &used)
        }
    }
}

public class LZMA2: DecompressionAlgorithm {                         // Sources/LZMA2/LZMA2.swift:10-30
    public static func decompress(data: Data) throws -> Data {
        try single(data) { p, n, o, ol in var used = 0; return swc_lzma2_decompress(p, n, o, ol, &used) }
    }
}

public enum LZ4: DecompressionAlgorithm {                            // Sources/LZ4/LZ4.swift:33-146
    public static func decompress(data: Data) throws -> Data { try decompress(data: data, dictionary: nil) }
    public static func decompress(data: Data, dictionary: Data?, dictionaryID: UInt32? = nil) throws -> Data {
        try withDictionary(dictionary) { dp, dn in
            try single(data) { p, n, o, ol in var used = 0; return swc_lz4_decompress(p, n, dp, dn, dictionaryID == nil ? 0 : 1, dictionaryID ?? 0, o, ol, &used) }
        }
    }
    public static func multiDecompress(data: Data, dictionary: Data? = nil, dictionaryID: UInt32? = nil) throws -> [Data] {
        try withDictionary(dictionary) { dp, dn in
            try multi(data) { p, n, o, ol, e, c in swc_lz4_multi_decompress(p, n, dp, dn, dictionaryID == nil ? 0 : 1, dictionaryID ?? 0, o, ol, e, c) }
        }
    }
}

extension LZ4: CompressionAlgorithm {                                // Sources/LZ4/LZ4+Compress.swift:8-154
    public static func compress(data: Data) -> Data {
        compress(data: data, independentBlocks: true, blockChecksums: false, contentChecksum: true, contentSize: false,
                 blockSize: 4 * 1024 * 1024, dictionary: nil, dictionaryID: nil)
    }
    /// Non-throwing as in the reference: an engine status (a trap of the reference, no device, CUDA failure) stops the program.
    public static func compress(data: Data, independentBlocks: Bool, blockChecksums: Bool, contentChecksum: Bool,
                                contentSize: Bool, blockSize: Int = 4 * 1024 * 1024, dictionary: Data? = nil,
                                dictionaryID: UInt32? = nil) -> Data {
        var out: UnsafeMutablePointer<UInt8>? = nil
        var outLen = 0
        let status: Int32 = withDictionary(dictionary) { dp, dn in
            data.withUnsafeBytes { raw in
                swc_lz4_compress(raw.bindMemory(to: UInt8.self).baseAddress, raw.count, independentBlocks ? 1 : 0,
                                 blockChecksums ? 1 : 0, contentChecksum ? 1 : 0, contentSize ? 1 : 0, Int64(blockSize),
                                 dp, dn, dictionaryID == nil ? 0 : 1, dictionaryID ?? 0, &out, &outLen)
            }
        }
        defer { swc_free(out) }
        guard status == 0 else { fatalError("LZ4.compress: \(String(cString: swc_status_name(status)))") }
        return out.map { Data(bytes: $0, count: outLen) } ?? Data()
    }
}

extension LZ4 {
    fileprivate static func withDictionary<T>(_ d: Data?, _ body: (UnsafePointer<UInt8>?, Int) throws -> T) rethrows -> T {
        guard let d = d else { return try body(nil, 0) }
        var one: UInt8 = 0     // a non-nil pointer distinguishes an EMPTY dictionary from `nil`
        return try d.withUnsafeBytes { raw in
            try withUnsafePointer(to: &one) { try body(raw.count > 0 ? raw.bindMemory(to: UInt8.self).baseAddress : $0, raw.count) }
        }
    }
}

public class GzipArchive: Archive {                                  // Sources/GZip/GzipArchive.swift:10-77
    public static func unarchive(archive data: Data) throws -> Data {
        try single(data) { p, n, o, ol in var used = 0; return swc_gzip_unarchive(p, n, o, ol, &used) }
    }
    /// Represents the member of a multi-member GZip archive (GzipArchive.swift:13-22).
    public struct Member: Sendable {
        public let header: GzipHeader
        public let data: Data
        let crcError: Bool
    }
    /// GzipArchive.swift:52-77.  The engine returns the decoded bytes, the end of every member inside them and the offset of
    /// every member inside `archive`; each Member.header is parsed at its offset with swc_gzip_header_parse.
    public static func multiUnarchive(archive data: Data) throws -> [Member] {
        var out: UnsafeMutablePointer<UInt8>? = nil, outLen = 0
        var ends: UnsafeMutablePointer<Int>? = nil, offs: UnsafeMutablePointer<Int>? = nil, count = 0
        let st = data.withUnsafeBytes { raw in
            swc_gzip_multi_unarchive_members(raw.bindMemory(to: UInt8.self).baseAddress, raw.count, &out, &outLen, &ends, &offs, &count)
        }
        defer { swc_free(out); swc_free(ends); swc_free(offs) }
        var members = [Member](), prev = 0
        for i in 0..<count {
            let header = try GzipHeader(archive: data, memberOffset: offs![i])
            let failing = st == 605 && i == count - 1
            members.append(Member(header: header, data: Data(bytes: out! + prev, count: ends![i] - prev), crcError: failing))
            prev = ends![i]
        }
        if st == 605 { throw GzipError.wrongCRC(members) }                              // SWC_GZIP_WRONG_CRC; GzipArchive.swift:73-75
        guard st == 0 else { throw swcError(st) }
        return members
    }
}

/// Sources/GZip/GzipHeader.swift:10-60 — same stored properties; `init(archive:)` goes through swc_gzip_header_parse.
public struct GzipHeader: Sendable {
    public var compressionMethod: CompressionMethod
    public var modificationTime: Date?
    public var osType: FileSystemType
    public var fileName: String?
    public var comment: String?
    public var isTextFile: Bool
    public var extraFields: [ExtraField]

    public init(archive data: Data) throws { try self.init(archive: data, memberOffset: 0) }

    init(archive data: Data, memberOffset: Int) throws {
        var h = swc_gzip_header()
        let st = data.withUnsafeBytes { raw in
            swc_gzip_header_parse(raw.bindMemory(to: UInt8.self).baseAddress, raw.count, memberOffset, &h)
        }
        guard st == 0 else { throw swcError(st) }
        let base = data.startIndex
        func field(_ off: Int, _ len: Int) -> Data { data[(base + off)..<(base + off + len)] }
        compressionMethod = .deflate
        modificationTime = h.modification_time == 0 ? nil : Date(timeIntervalSince1970: TimeInterval(h.modification_time))
        osType = FileSystemType(h.os_type)
        fileName = h.has_file_name != 0 ? String(data: field(h.file_name_off, h.file_name_len), encoding: .isoLatin1) : nil
        comment = h.has_comment != 0 ? String(data: field(h.comment_off, h.comment_len), encoding: .isoLatin1) : nil
        isTextFile = h.is_text_file != 0
        extraFields = []
        var p = h.extra_off
        let end = h.extra_off + h.extra_len
        while p < end {
            let len = Int(data[base + p + 2]) | Int(data[base + p + 3]) << 8
            extraFields.append(ExtraField(data[base + p], data[base + p + 1], [UInt8](field(p + 4, len))))
            p += 4 + len
        }
    }
}

/// Sources/Zlib/ZlibHeader.swift:10-45
public struct ZlibHeader: Sendable {
    public enum CompressionLevel: Int, Sendable { case fastestAlgorithm = 0, fastAlgorithm, defaultAlgorithm, slowAlgorithm }
    public let compressionMethod: CompressionMethod = .deflate
    public let compressionLevel: CompressionLevel
    public let windowSize: Int

    public init(archive data: Data) throws {
        var h = swc_zlib_header()
        let st = data.withUnsafeBytes { raw in swc_zlib_header_parse(raw.bindMemory(to: UInt8.self).baseAddress, raw.count, &h) }
        guard st == 0 else { throw swcError(st) }
        compressionLevel = CompressionLevel(rawValue: Int(h.compression_level))!
        windowSize = Int(h.window_size)
    }
}

public class ZlibArchive: Archive {                                  // Sources/Zlib/ZlibArchive.swift:10-42
    public static func unarchive(archive data: Data) throws -> Data {
        try single(data) { p, n, o, ol in swc_zlib_unarchive(p, n, o, ol) }
    }
}

public class XZArchive: Archive {                                    // Sources/XZ/XZArchive.swift:10-88
    public static func unarchive(archive data: Data) throws -> Data {
        try single(data) { p, n, o, ol in swc_xz_unarchive(p, n, o, ol) }
    }
    public static func splitUnarchive(archive data: Data) throws -> [Data] {
        try multi(data) { p, n, o, ol, e, c in swc_xz_split_unarchive(p, n, o, ol, e, c) }
    }
}

// ---- ZIP container (Sources/ZIP/ZipContainer.swift:10-180) -------------------------------------------------------------
/// `ZipContainer.open(container:)`: the engine walks the central directory once, decodes every entry of a method as one batch
/// and returns the entries in central-directory order.  ZipEntryInfo's remaining metadata (timestamps from extra fields,
/// owner ids, custom extra fields) stays in Swift: ZipEntryInfo.swift / BuiltinExtraFields.swift are unchanged and read the
/// same bytes; the engine supplies name, comment, size, crc, method, attributes and the entry data.
public class ZipContainer: Container {
    public static func open(container data: Data) throws -> [ZipEntry] {
        var out: UnsafeMutablePointer<UInt8>? = nil, outLen = 0
        var es: UnsafeMutablePointer<swc_zip_entry>? = nil, count = 0
        let st = data.withUnsafeBytes { raw in
            swc_zip_open(raw.bindMemory(to: UInt8.self).baseAddress, raw.count, &out, &outLen, &es, &count)
        }
        defer { swc_free(out); swc_free(es) }
        var entries = [ZipEntry]()
        for i in 0..<count {
            let e = es![i]
            let info = ZipEntryInfo(container: data, engineEntry: e)                 // thin init added next to the reference's
            let payload = e.is_directory != 0 ? nil : Data(bytes: out! + Int(e.data_off), count: Int(e.data_len))
            entries.append(ZipEntry(info, payload))
        }
        if st == 910 { throw ZipError.wrongCRC(entries) }                            // SWC_ZIP_WRONG_CRC; ZipContainer.swift:53-55
        guard st == 0 else { throw swcError(st) }
        return entries
    }
    public static func info(container data: Data) throws -> [ZipEntryInfo] {
        var es: UnsafeMutablePointer<swc_zip_entry>? = nil, count = 0
        let st = data.withUnsafeBytes { raw in swc_zip_info(raw.bindMemory(to: UInt8.self).baseAddress, raw.count, &es, &count) }
        defer { swc_free(es) }
        guard st == 0 else { throw swcError(st) }
        return (0..<count).map { ZipEntryInfo(container: data, engineEntry: es![$0]) }
    }
}
