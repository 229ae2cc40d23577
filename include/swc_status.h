/* swc_status.h — status codes shared by libswcgpu (the product) and the CPU oracle (test infrastructure).
 *
 * One namespace per Swift error enum of the reference, 0 = OK.  The numeric value of each code is
 * <namespace base> + <1-based case index in the reference enum>, so a Swift/ctypes shim can map it back
 * with a table lookup.
 *
 *   DeflateError  Sources/Deflate/DeflateError.swift:10-19
 *   BZip2Error    Sources/BZip2/BZip2Error.swift:12-44
 *   LZMAError     Sources/LZMA/LZMAError.swift:10-25
 *   LZMA2Error    Sources/LZMA2/LZMA2Error.swift:10-22
 *   DataError     Sources/Common/DataError.swift:9-25   (used by LZ4)
 *   GzipError     Sources/GZip/GzipError.swift:10-35
 *   ZlibError     Sources/Zlib/ZlibError.swift:12-26
 *   XZError       Sources/XZ/XZError.swift:12-48
 *   TarError      Sources/TAR/TarError.swift:10-18
 */
#ifndef SWC_STATUS_H
#define SWC_STATUS_H

enum swc_status {
    SWC_OK = 0,

    /* engine-level conditions that have no Swift enum case */
    SWC_ERR_OUTPUT_OVERFLOW = 1,   /* out capacity fence too small; out_len holds the required size when known */
    SWC_ERR_REFERENCE_TRAP  = 2,   /* input on which the Swift reference hits a precondition/array-bounds trap
                                      (SURVEY.md Appendix A "Traps"); we return instead of crashing */
    SWC_ERR_CUDA            = 3,   /* CUDA runtime failure; see swc_last_error_string() */
    SWC_ERR_INVALID_ARG     = 4,
    SWC_ERR_NO_DEVICE       = 5,   /* no CUDA device: there is no CPU fallback by design */
    SWC_ERR_UNSUPPORTED     = 6,   /* valid input the engine cannot take (e.g. unit > 4 GiB) */

    SWC_DEFLATE_WRONG_UNCOMPRESSED_BLOCK_LENGTHS = 101,
    SWC_DEFLATE_WRONG_BLOCK_TYPE                 = 102,
    SWC_DEFLATE_WRONG_SYMBOL                     = 103,
    SWC_DEFLATE_SYMBOL_NOT_FOUND                 = 104,

    SWC_BZIP2_WRONG_MAGIC               = 201,
    SWC_BZIP2_WRONG_VERSION             = 202,
    SWC_BZIP2_WRONG_BLOCK_SIZE          = 203,
    SWC_BZIP2_WRONG_BLOCK_TYPE          = 204,
    SWC_BZIP2_RANDOMIZED_BLOCK          = 205,
    SWC_BZIP2_WRONG_HUFFMAN_GROUPS      = 206,
    SWC_BZIP2_WRONG_SELECTOR            = 207,
    SWC_BZIP2_WRONG_HUFFMAN_CODE_LENGTH = 208,
    SWC_BZIP2_SYMBOL_NOT_FOUND          = 209,
    SWC_BZIP2_WRONG_CRC                 = 210,  /* payload-carrying: output is still returned */

    SWC_LZMA_WRONG_PROPERTIES           = 301,
    SWC_LZMA_RANGE_DECODER_INIT_ERROR   = 302,
    SWC_LZMA_EXCEEDED_UNCOMPRESSED_SIZE = 303,
    SWC_LZMA_WINDOW_IS_EMPTY            = 304,
    SWC_LZMA_RANGE_DECODER_FINISH_ERROR = 305,
    SWC_LZMA_REPEAT_WILL_EXCEED         = 306,
    SWC_LZMA_NOT_ENOUGH_TO_REPEAT       = 307,

    SWC_LZMA2_WRONG_DICTIONARY_SIZE = 401,
    SWC_LZMA2_WRONG_CONTROL_BYTE    = 402,
    SWC_LZMA2_WRONG_RESET           = 403,
    SWC_LZMA2_WRONG_SIZES           = 404,

    SWC_DATA_TRUNCATED           = 501,
    SWC_DATA_CORRUPTED           = 502,
    SWC_DATA_CHECKSUM_MISMATCH   = 503,  /* payload-carrying */
    SWC_DATA_UNSUPPORTED_FEATURE = 504,

    SWC_GZIP_WRONG_MAGIC              = 601,
    SWC_GZIP_WRONG_COMPRESSION_METHOD = 602,
    SWC_GZIP_WRONG_FLAGS              = 603,
    SWC_GZIP_WRONG_HEADER_CRC         = 604,
    SWC_GZIP_WRONG_CRC                = 605,  /* payload-carrying */
    SWC_GZIP_WRONG_ISIZE              = 606,
    SWC_GZIP_CANNOT_ENCODE_ISO_LATIN1 = 607,  /* swc_gzip_archive: extra fields longer than 65 535 bytes */

    SWC_ZLIB_WRONG_COMPRESSION_METHOD = 701,
    SWC_ZLIB_WRONG_COMPRESSION_INFO   = 702,
    SWC_ZLIB_WRONG_FCHECK             = 703,
    SWC_ZLIB_WRONG_COMPRESSION_LEVEL  = 704,
    SWC_ZLIB_WRONG_ADLER32            = 705,  /* payload-carrying */

    SWC_XZ_WRONG_MAGIC              = 801,
    SWC_XZ_WRONG_FIELD              = 802,
    SWC_XZ_WRONG_INFO_CRC           = 803,
    SWC_XZ_WRONG_FILTER_ID          = 804,
    SWC_XZ_CHECK_TYPE_SHA256        = 805,
    SWC_XZ_WRONG_DATA_SIZE          = 806,
    SWC_XZ_WRONG_CHECK              = 807,  /* payload-carrying */
    SWC_XZ_WRONG_PADDING            = 808,
    SWC_XZ_MULTI_BYTE_INTEGER_ERROR = 809,

    /* ZipError, Sources/ZIP/ZipError.swift:12-36 */
    SWC_ZIP_NOT_FOUND_CENTRAL_DIRECTORY_END = 901,
    SWC_ZIP_WRONG_SIGNATURE            = 902,
    SWC_ZIP_WRONG_SIZE                 = 903,
    SWC_ZIP_WRONG_VERSION              = 904,
    SWC_ZIP_MULTI_VOLUMES_NOT_SUPPORTED = 905,
    SWC_ZIP_ENCRYPTION_NOT_SUPPORTED   = 906,
    SWC_ZIP_PATCHING_NOT_SUPPORTED     = 907,
    SWC_ZIP_COMPRESSION_NOT_SUPPORTED  = 908,
    SWC_ZIP_WRONG_LOCAL_HEADER         = 909,
    SWC_ZIP_WRONG_CRC                  = 910,  /* payload-carrying: the entries processed so far, the failing one last */
    SWC_ZIP_WRONG_TEXT_FIELD           = 911,

    /* TarError, Sources/TAR/TarError.swift:10-18 */
    SWC_TAR_TOO_SMALL_FILE_IS_PASSED = 1001,
    SWC_TAR_WRONG_FIELD              = 1002,
    SWC_TAR_WRONG_HEADER_CHECKSUM    = 1003,
    SWC_TAR_WRONG_PAX_HEADER_ENTRY   = 1004
};

#endif /* SWC_STATUS_H */
