"""Host-side mirror of the reference's Swift API for the decode hot path (same type and method names, same argument
meaning, same error cases), routed through the C ABI of libswcgpu.so.

    Swift (reference)                                   here
    Deflate.decompress(data:)                           Deflate.decompress(data)
    BZip2.decompress(data:) / multiDecompress(data:)    BZip2.decompress(data) / BZip2.multiDecompress(data)
    LZMA.decompress(data:[properties:uncompressedSize:]) LZMA.decompress(data[, properties, uncompressedSize])
    LZMA2.decompress(data:)                             LZMA2.decompress(data)
    LZ4.decompress(data:[dictionary:dictionaryID:])     LZ4.decompress(data[, dictionary, dictionaryID])
    LZ4.multiDecompress(data:dictionary:dictionaryID:)  LZ4.multiDecompress(...)
    LZ4.compress(data:[independentBlocks:...])          LZ4.compress(data[, independentBlocks, ...])
    Deflate.compress(data:)                             Deflate.compress(data)
    GzipArchive.archive(data:comment:...)               GzipArchive.archive(data, comment=None, fileName=None, ...)
    ZlibArchive.archive(data:)                          ZlibArchive.archive(data)
    GzipArchive.unarchive / multiUnarchive -> [Member]  GzipArchive.unarchive / multiUnarchive -> [GzipArchive.Member]
    GzipHeader(archive:) / ZlibHeader(archive:)         GzipHeader(archive) / ZlibHeader(archive)
    ZlibArchive.unarchive                               ZlibArchive.unarchive
    XZArchive.unarchive / splitUnarchive                XZArchive.unarchive / splitUnarchive
"""
import ctypes as C
import datetime
from dataclasses import dataclass, field

from . import _lib
from .errors import check, error_for

_PAYLOAD_CODES = {210, 503, 605, 705, 807, 910}


def _single(fn, data, *extra, consumed=True):
    L = _lib.lib()
    buf, n = _lib.inbuf(data)
    out, out_len, used = C.c_void_p(), C.c_size_t(0), C.c_size_t(0)
    args = [buf, n, *extra, C.byref(out), C.byref(out_len)] + ([C.byref(used)] if consumed else [])
    st = getattr(L, fn)(*args)
    payload = _lib.take(out, out_len)
    if st != 0:
        raise error_for(st, payload if st in _PAYLOAD_CODES else None)
    return payload, used.value


def _multi(fn, data, *extra):
    L = _lib.lib()
    buf, n = _lib.inbuf(data)
    out, out_len, ends, cnt = C.c_void_p(), C.c_size_t(0), C.c_void_p(), C.c_size_t(0)
    st = getattr(L, fn)(buf, n, *extra, C.byref(out), C.byref(out_len), C.byref(ends), C.byref(cnt))
    whole = _lib.take(out, out_len)
    e = _lib.take_sizes(ends, cnt)
    parts, prev = [], 0
    for x in e:
        parts.append(whole[prev:x])
        prev = x
    if st != 0:
        raise error_for(st, parts if st in _PAYLOAD_CODES else None)
    return parts


def _compressed(fn, data, *extra):
    L = _lib.lib()
    buf, n = _lib.inbuf(data)
    out, out_len = C.c_void_p(), C.c_size_t(0)
    st = getattr(L, fn)(buf, n, *extra, C.byref(out), C.byref(out_len))
    payload = _lib.take(out, out_len)
    if st != 0:
        raise error_for(st, None)
    return payload


class Deflate:
    """Sources/Deflate/Deflate.swift:10-28, Sources/Deflate/Deflate+Compress.swift:22-42"""

    @staticmethod
    def compress(data):
        """Deflate.compress(data:): one stored or static-Huffman block, equal to the reference's byte for byte."""
        return _compressed("swc_deflate_compress", data)

    @staticmethod
    def decompress(data):
        return _single("swc_deflate_decompress", data, C.c_size_t(0))[0]

    @staticmethod
    def decompress_from(data, start_bit):
        """reader-based overload (Deflate.swift:30): returns (bytes, consumed_bits)"""
        return _single("swc_deflate_decompress", data, C.c_size_t(start_bit))


class BZip2:
    """Sources/BZip2/BZip2.swift:10-48"""

    @staticmethod
    def decompress(data):
        return _single("swc_bzip2_decompress", data, C.c_size_t(0))[0]

    @staticmethod
    def multiDecompress(data):
        return _multi("swc_bzip2_multi_decompress", data)


@dataclass
class LZMAProperties:
    """Sources/LZMA/LZMAProperties.swift:9-47"""
    lc: int = 3
    lp: int = 0
    pb: int = 2
    dictionarySize: int = 1 << 24

    def __setattr__(self, name, value):
        # the reference's didSet (LZMAProperties.swift:26-32) raises a dictionarySize below 4096 to 4096 when the property is
        # assigned; Swift does not call didSet from the type's own initializers, so the constructor keeps any value
        if name == "dictionarySize" and "dictionarySize" in self.__dict__ and value < (1 << 12):
            value = 1 << 12
        object.__setattr__(self, name, value)


class LZMA:
    """Sources/LZMA/LZMA.swift:10-73"""

    @staticmethod
    def decompress(data, properties=None, uncompressedSize=None):
        if properties is None:
            return _single("swc_lzma_decompress", data)[0]
        us = -1 if uncompressedSize is None else int(uncompressedSize)
        return _single("swc_lzma_decompress_raw", data, C.c_int32(properties.lc), C.c_int32(properties.lp), C.c_int32(properties.pb),
                       C.c_int64(properties.dictionarySize), C.c_int64(us))[0]


class LZMA2:
    """Sources/LZMA2/LZMA2.swift:10-36"""

    @staticmethod
    def decompress(data):
        return _single("swc_lzma2_decompress", data)[0]


def _dict_args(dictionary, dictionaryID):
    if dictionary is None:
        return [None, C.c_size_t(0), C.c_int32(0 if dictionaryID is None else 1), C.c_uint32(dictionaryID or 0)], None
    buf, n = _lib.inbuf(dictionary)
    return [buf, C.c_size_t(n), C.c_int32(0 if dictionaryID is None else 1), C.c_uint32(dictionaryID or 0)], buf


class LZ4:
    """Sources/LZ4/LZ4.swift:33-146, Sources/LZ4/LZ4+Compress.swift:16-154"""

    @staticmethod
    def compress(data, independentBlocks=True, blockChecksums=False, contentChecksum=True, contentSize=False,
                 blockSize=4 * 1024 * 1024, dictionary=None, dictionaryID=None):
        """LZ4.compress(data:) with the defaults, or the overload with every option; the frame equals the reference's byte
        for byte.  The reference cannot throw; where it traps (blockSize outside 1 ... 4 MiB, a 1-3 byte dictionary) this
        raises the engine's referenceTrap error."""
        L = _lib.lib()
        buf, n = _lib.inbuf(data)
        if dictionary is None:
            dp, dn = None, 0
        else:
            dp, dn = _lib.inbuf(dictionary)
        out, out_len = C.c_void_p(), C.c_size_t(0)
        st = L.swc_lz4_compress(buf, n, int(bool(independentBlocks)), int(bool(blockChecksums)), int(bool(contentChecksum)),
                                int(bool(contentSize)), int(blockSize), dp, dn, 0 if dictionaryID is None else 1,
                                int(dictionaryID or 0), C.byref(out), C.byref(out_len))
        payload = _lib.take(out, out_len)
        if st != 0:
            raise error_for(st, None)
        return payload

    @staticmethod
    def decompress(data, dictionary=None, dictionaryID=None):
        args, _keep = _dict_args(dictionary, dictionaryID)
        return _single("swc_lz4_decompress", data, *args)[0]

    @staticmethod
    def multiDecompress(data, dictionary=None, dictionaryID=None):
        args, _keep = _dict_args(dictionary, dictionaryID)
        return _multi("swc_lz4_multi_decompress", data, *args)


class _CGzipHeader(C.Structure):
    _fields_ = [("compression_method", C.c_int32), ("modification_time", C.c_uint32), ("os_type", C.c_uint8),
                ("is_text_file", C.c_uint8), ("has_file_name", C.c_uint8), ("has_comment", C.c_uint8),
                ("file_name_off", C.c_size_t), ("file_name_len", C.c_size_t), ("comment_off", C.c_size_t),
                ("comment_len", C.c_size_t), ("extra_off", C.c_size_t), ("extra_len", C.c_size_t), ("header_len", C.c_size_t)]


class _CZlibHeader(C.Structure):
    _fields_ = [("compression_method", C.c_int32), ("compression_level", C.c_int32), ("window_size", C.c_int32),
                ("header_len", C.c_size_t)]


@dataclass
class ExtraField:
    """GzipHeader.ExtraField (Sources/GZip/GzipHeader+ExtraField.swift)"""
    si1: int
    si2: int
    bytes: bytes


# FileSystemType(rawOsType), Sources/Common/FileSystemType.swift (gzip OS byte)
_OS_TYPES = {0: "fat", 3: "unix", 7: "macintosh", 11: "ntfs"}
_OS_BYTES = {v: k for k, v in _OS_TYPES.items()}      # osTypeByte (FileSystemType+Gzip.swift:23-36); others are 255


class _CGzipOptions(C.Structure):
    _fields_ = [("file_name", C.c_void_p), ("file_name_len", C.c_size_t), ("comment", C.c_void_p), ("comment_len", C.c_size_t),
                ("write_header_crc", C.c_int32), ("is_text_file", C.c_int32), ("has_mtime", C.c_int32), ("mtime", C.c_int64),
                ("os_type", C.c_uint8), ("n_extra", C.c_size_t), ("extra_ids", C.c_void_p), ("extra_lens", C.c_void_p),
                ("extra_bytes", C.c_void_p)]


def _latin1(text):
    """String.data(using: .isoLatin1) of the text with a NUL appended unless it ends with one (GzipArchive.swift:132-161)"""
    if not text or text[-1] != "\0":
        text = text + "\0"
    try:
        return text.encode("latin-1")
    except UnicodeEncodeError:
        raise error_for(607, None) from None


class GzipHeader:
    """Sources/GZip/GzipHeader.swift:10-60 — init(archive:) parses the header of the first member (:63-66)."""

    def __init__(self, archive, _member_off=0):
        data = bytes(archive)
        buf, n = _lib.inbuf(data)
        h = _CGzipHeader()
        check(_lib.lib().swc_gzip_header_parse(buf, n, C.c_size_t(_member_off), C.byref(h)))
        self.compressionMethod = "deflate"
        self.modificationTime = (None if h.modification_time == 0 else
                                 datetime.datetime.fromtimestamp(h.modification_time, datetime.timezone.utc))
        self.osType = _OS_TYPES.get(h.os_type, "other")
        self.fileName = data[h.file_name_off:h.file_name_off + h.file_name_len].decode("latin-1") if h.has_file_name else None
        self.comment = data[h.comment_off:h.comment_off + h.comment_len].decode("latin-1") if h.has_comment else None
        self.isTextFile = bool(h.is_text_file)
        self.extraFields = []
        p, end = h.extra_off, h.extra_off + h.extra_len
        while p < end:
            ln = data[p + 2] | data[p + 3] << 8
            self.extraFields.append(ExtraField(data[p], data[p + 1], data[p + 4:p + 4 + ln]))
            p += 4 + ln
        self.headerLength = h.header_len


class ZlibHeader:
    """Sources/Zlib/ZlibHeader.swift:10-45"""
    LEVELS = ("fastestAlgorithm", "fastAlgorithm", "defaultAlgorithm", "slowAlgorithm")

    def __init__(self, archive):
        buf, n = _lib.inbuf(archive)
        h = _CZlibHeader()
        check(_lib.lib().swc_zlib_header_parse(buf, n, C.byref(h)))
        self.compressionMethod = "deflate"
        self.compressionLevel = self.LEVELS[h.compression_level]
        self.windowSize = h.window_size


class GzipArchive:
    """Sources/GZip/GzipArchive.swift:10-241"""

    @staticmethod
    def archive(data, comment=None, fileName=None, writeHeaderCRC=False, isTextFile=False, osType=None,
                modificationTime=None, extraFields=()):
        """GzipArchive.archive(data:comment:fileName:writeHeaderCRC:isTextFile:osType:modificationTime:extraFields:).
        osType is a FileSystemType name ("fat", "unix", "macintosh", "ntfs", "other") or None; modificationTime a
        datetime or seconds since 1970.  Text that is not ISO-Latin-1, and extra fields whose XLEN exceeds 65 535, raise
        GzipError.cannotEncodeISOLatin1 as the reference throws."""
        # the reference encodes the comment first, then the file name (:130-157); both fail the same way
        c = None if comment is None else _latin1(comment)
        f = None if fileName is None else _latin1(fileName)
        o = _CGzipOptions()
        keep = []
        for text, ptr, ln in ((f, "file_name", "file_name_len"), (c, "comment", "comment_len")):
            if text is not None:
                b = C.create_string_buffer(text, len(text))
                keep.append(b)
                setattr(o, ptr, C.cast(b, C.c_void_p))
                setattr(o, ln, len(text))
        o.write_header_crc, o.is_text_file = int(bool(writeHeaderCRC)), int(bool(isTextFile))
        if modificationTime is not None:
            t = modificationTime.timestamp() if isinstance(modificationTime, datetime.datetime) else modificationTime
            o.has_mtime, o.mtime = 1, int(t)                 # Int(timeIntervalSince1970) truncates toward zero
        o.os_type = 255 if osType is None else _OS_BYTES.get(osType, 255)
        fields = list(extraFields)
        if fields:
            ids = (C.c_uint8 * (2 * len(fields)))(*[v for e in fields for v in (e.si1, e.si2)])
            lens = (C.c_uint64 * len(fields))(*[len(e.bytes) for e in fields])
            blob = b"".join(bytes(e.bytes) for e in fields)
            bb = C.create_string_buffer(blob, max(len(blob), 1))
            keep += [ids, lens, bb]
            o.n_extra, o.extra_ids, o.extra_lens = len(fields), C.cast(ids, C.c_void_p), C.cast(lens, C.c_void_p)
            o.extra_bytes = C.cast(bb, C.c_void_p)
        return _compressed("swc_gzip_archive", data, C.byref(o))

    @dataclass
    class Member:
        """GzipArchive.Member (GzipArchive.swift:13-22)"""
        header: GzipHeader
        data: bytes

    @staticmethod
    def unarchive(archive):
        return _single("swc_gzip_unarchive", archive)[0]

    @staticmethod
    def multiUnarchive(archive):
        """-> [Member]; GzipError.wrongCRC carries the members decoded so far, the failing one last (GzipArchive.swift:62-76)."""
        L = _lib.lib()
        data = bytes(archive)
        buf, n = _lib.inbuf(data)
        out, out_len, ends, offs, cnt = C.c_void_p(), C.c_size_t(0), C.c_void_p(), C.c_void_p(), C.c_size_t(0)
        st = L.swc_gzip_multi_unarchive_members(buf, n, C.byref(out), C.byref(out_len), C.byref(ends), C.byref(offs), C.byref(cnt))
        whole = _lib.take(out, out_len)
        e = _lib.take_sizes(ends, cnt)
        o = _lib.take_sizes(offs, C.c_size_t(cnt.value + 1)) if offs.value else []
        members, prev = [], 0
        for i, x in enumerate(e):
            members.append(GzipArchive.Member(GzipHeader(data, _member_off=o[i]), whole[prev:x]))
            prev = x
        if st != 0:
            raise error_for(st, members if st in _PAYLOAD_CODES else None)
        return members


class ZlibArchive:
    """Sources/Zlib/ZlibArchive.swift:10-70"""

    @staticmethod
    def archive(data):
        """ZlibArchive.archive(data:): 78 DA, the Deflate.compress stream, the big-endian Adler-32."""
        return _compressed("swc_zlib_archive", data)

    @staticmethod
    def unarchive(archive):
        return _single("swc_zlib_unarchive", archive, consumed=False)[0]


class XZArchive:
    """Sources/XZ/XZArchive.swift:10-88"""

    @staticmethod
    def unarchive(archive):
        return _single("swc_xz_unarchive", archive, consumed=False)[0]

    @staticmethod
    def splitUnarchive(archive):
        return _multi("swc_xz_split_unarchive", archive)


class _CZipEntry(C.Structure):
    _fields_ = [("name_off", C.c_uint64), ("name_len", C.c_uint64), ("comment_off", C.c_uint64), ("comment_len", C.c_uint64),
                ("data_off", C.c_uint64), ("data_len", C.c_uint64), ("size", C.c_uint64), ("crc", C.c_uint32),
                ("external_attrs", C.c_uint32), ("method", C.c_uint16), ("version_made_by", C.c_uint16),
                ("internal_attrs", C.c_uint16), ("dos_time", C.c_uint16), ("dos_date", C.c_uint16), ("is_directory", C.c_uint8),
                ("utf8", C.c_uint8)]


_ZIP_METHODS = {0: "copy", 8: "deflate", 12: "bzip2", 14: "lzma"}


def _zip_text(raw, utf8):
    """zipString (LittleEndianByteReader+Zip.swift:11-24): UTF-8 when flagged, or when the bytes only make sense as UTF-8;
    CP437 otherwise.  The library has already rejected what String(data:encoding:) would."""
    if utf8:
        return raw.decode("utf-8")
    try:
        if any(b >= 0x80 for b in raw):
            return raw.decode("utf-8")
    except UnicodeDecodeError:
        pass
    return raw.decode("cp437")


@dataclass
class ZipEntryInfo:
    """Sources/ZIP/ZipEntryInfo.swift:9-95 (the fields the container walk itself produces)"""
    name: str
    size: int
    type: str                       # "directory" | "regular" (other Unix types are reported as "regular" here)
    compressionMethod: str
    crc: int
    comment: str
    isTextFile: bool
    externalFileAttributes: int
    permissions: int
    dosAttributes: int
    versionMadeBy: int
    modificationTime: datetime.datetime = None


@dataclass
class ZipEntry:
    """Sources/ZIP/ZipEntry.swift:9-20"""
    info: ZipEntryInfo
    data: bytes = None


def _zip_infos(container, es, count):
    arr = C.cast(es, C.POINTER(_CZipEntry))
    out = []
    for i in range(count):
        e = arr[i]
        d, t = e.dos_date, e.dos_time
        try:
            mt = datetime.datetime(1980 + ((d & 0xFE00) >> 9), (d & 0x1E0) >> 5, d & 0x1F, (t & 0xF800) >> 11, (t & 0x7E0) >> 5, 2 * (t & 0x1F))
        except ValueError:
            mt = None
        info = ZipEntryInfo(name=_zip_text(container[e.name_off:e.name_off + e.name_len], e.utf8), size=e.size,
                            type="directory" if e.is_directory else "regular",
                            compressionMethod=_ZIP_METHODS.get(e.method, "other"), crc=e.crc,
                            comment=_zip_text(container[e.comment_off:e.comment_off + e.comment_len], e.utf8),
                            isTextFile=bool(e.internal_attrs & 1), externalFileAttributes=e.external_attrs,
                            permissions=(e.external_attrs & 0x0FFF0000) >> 16, dosAttributes=e.external_attrs & 0xFF,
                            versionMadeBy=e.version_made_by, modificationTime=mt)
        out.append((info, e.data_off, e.data_len, bool(e.is_directory)))
    return out


class ZipContainer:
    """Sources/ZIP/ZipContainer.swift:10-180"""

    @staticmethod
    def info(container):
        data = bytes(container)
        buf, n = _lib.inbuf(data)
        es, cnt = C.c_void_p(), C.c_size_t(0)
        st = _lib.lib().swc_zip_info(buf, n, C.byref(es), C.byref(cnt))
        try:
            check(st)
            return [x[0] for x in _zip_infos(data, es, cnt.value)]
        finally:
            if es.value:
                _lib.lib().swc_free(es)

    @staticmethod
    def open(container):
        """-> [ZipEntry]; ZipError.wrongCRC carries the entries processed so far, the failing one last (ZipContainer.swift:53-55)."""
        data = bytes(container)
        buf, n = _lib.inbuf(data)
        out, out_len, es, cnt = C.c_void_p(), C.c_size_t(0), C.c_void_p(), C.c_size_t(0)
        st = _lib.lib().swc_zip_open(buf, n, C.byref(out), C.byref(out_len), C.byref(es), C.byref(cnt))
        try:
            whole = _lib.take(out, out_len)
            entries = [ZipEntry(info, None if is_dir else whole[off:off + ln]) for info, off, ln, is_dir in _zip_infos(data, es, cnt.value)]
        finally:
            if es.value:
                _lib.lib().swc_free(es)
        if st != 0:
            raise error_for(st, entries if st in _PAYLOAD_CODES else None)
        return entries


# ---- checks (CheckSums.swift / XxHash32.swift / Sha256.swift) ----
def _check32(fn, data):
    buf, n = _lib.inbuf(data)
    v = C.c_uint32(0)
    check(getattr(_lib.lib(), fn)(buf, n, C.byref(v)))
    return v.value


def crc32(data):
    return _check32("swc_crc32", data)


def bzip2_crc32(data):
    return _check32("swc_bzip2_crc32", data)


def adler32(data):
    return _check32("swc_adler32", data)


def xxh32(data):
    return _check32("swc_xxh32", data)


def crc64(data):
    buf, n = _lib.inbuf(data)
    v = C.c_uint64(0)
    check(_lib.lib().swc_crc64(buf, n, C.byref(v)))
    return v.value


def sha256(data):
    buf, n = _lib.inbuf(data)
    dg = (C.c_uint8 * 32)()
    check(_lib.lib().swc_sha256(buf, n, dg))
    return bytes(dg)
