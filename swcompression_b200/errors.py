"""Error types mirroring the reference's Swift error enums (one exception class per enum, one `case` per code).

DeflateError (Sources/Deflate/DeflateError.swift:10-19), BZip2Error (Sources/BZip2/BZip2Error.swift:12-44),
LZMAError (Sources/LZMA/LZMAError.swift:10-25), LZMA2Error (Sources/LZMA2/LZMA2Error.swift:10-22),
DataError (Sources/Common/DataError.swift:9-25), GzipError (Sources/GZip/GzipError.swift:10-35),
ZlibError (Sources/Zlib/ZlibError.swift:12-26), XZError (Sources/XZ/XZError.swift:12-48), ZipError (Sources/ZIP/ZipError.swift:12-36),
TarError (Sources/TAR/TarError.swift:10-18).
Payload-carrying cases (`wrongCRC(Data)`, `checksumMismatch([Data])`, ...) expose the decoded bytes as `.payload`.
"""


class SWCompressionError(Exception):
    cases = {}

    def __init__(self, code, payload=None):
        self.code = code
        self.case = self.cases.get(code, f"status{code}")
        self.payload = payload
        super().__init__(f"{type(self).__name__}.{self.case}")

    def __eq__(self, other):
        if isinstance(other, str):
            return self.case == other
        return isinstance(other, SWCompressionError) and type(self) is type(other) and self.code == other.code

    __hash__ = Exception.__hash__


class EngineError(SWCompressionError):
    cases = {1: "outputOverflow", 2: "referenceTrap", 3: "cuda", 4: "invalidArgument", 5: "noDevice", 6: "unsupported"}


class DeflateError(SWCompressionError):
    cases = {101: "wrongUncompressedBlockLengths", 102: "wrongBlockType", 103: "wrongSymbol", 104: "symbolNotFound"}


class BZip2Error(SWCompressionError):
    cases = {201: "wrongMagic", 202: "wrongVersion", 203: "wrongBlockSize", 204: "wrongBlockType", 205: "randomizedBlock",
             206: "wrongHuffmanGroups", 207: "wrongSelector", 208: "wrongHuffmanCodeLength", 209: "symbolNotFound", 210: "wrongCRC"}


class LZMAError(SWCompressionError):
    cases = {301: "wrongProperties", 302: "rangeDecoderInitError", 303: "exceededUncompressedSize", 304: "windowIsEmpty",
             305: "rangeDecoderFinishError", 306: "repeatWillExceed", 307: "notEnoughToRepeat"}


class LZMA2Error(SWCompressionError):
    cases = {401: "wrongDictionarySize", 402: "wrongControlByte", 403: "wrongReset", 404: "wrongSizes"}


class DataError(SWCompressionError):
    cases = {501: "truncated", 502: "corrupted", 503: "checksumMismatch", 504: "unsupportedFeature"}


class GzipError(SWCompressionError):
    cases = {601: "wrongMagic", 602: "wrongCompressionMethod", 603: "wrongFlags", 604: "wrongHeaderCRC", 605: "wrongCRC",
             606: "wrongISize", 607: "cannotEncodeISOLatin1"}


class ZlibError(SWCompressionError):
    cases = {701: "wrongCompressionMethod", 702: "wrongCompressionInfo", 703: "wrongFcheck", 704: "wrongCompressionLevel",
             705: "wrongAdler32"}


class XZError(SWCompressionError):
    cases = {801: "wrongMagic", 802: "wrongField", 803: "wrongInfoCRC", 804: "wrongFilterID", 805: "checkTypeSHA256",
             806: "wrongDataSize", 807: "wrongCheck", 808: "wrongPadding", 809: "multiByteIntegerError"}


class ZipError(SWCompressionError):
    """Sources/ZIP/ZipError.swift:12-36; wrongCRC carries the entries processed so far (the failing one last)"""
    cases = {901: "notFoundCentralDirectoryEnd", 902: "wrongSignature", 903: "wrongSize", 904: "wrongVersion",
             905: "multiVolumesNotSupported", 906: "encryptionNotSupported", 907: "patchingNotSupported",
             908: "compressionNotSupported", 909: "wrongLocalHeader", 910: "wrongCRC", 911: "wrongTextField"}


class TarError(SWCompressionError):
    """Sources/TAR/TarError.swift:10-18"""
    cases = {1001: "tooSmallFileIsPassed", 1002: "wrongField", 1003: "wrongHeaderChecksum", 1004: "wrongPaxHeaderEntry"}


_BY_RANGE = [(1, 99, EngineError), (101, 199, DeflateError), (201, 299, BZip2Error), (301, 399, LZMAError),
             (401, 499, LZMA2Error), (501, 599, DataError), (601, 699, GzipError), (701, 799, ZlibError), (801, 899, XZError), (901, 999, ZipError),
             (1001, 1099, TarError)]


def error_for(code, payload=None):
    for lo, hi, cls in _BY_RANGE:
        if lo <= code <= hi:
            return cls(code, payload)
    return EngineError(code, payload)


def check(code, payload=None):
    if code != 0:
        raise error_for(code, payload)
