"""ctypes binding of the C ABI in include/zstdb200.h (libzstdb200.so).

The library holds the sm_90a kernels; there is deliberately no fallback: if the
shared object is missing or no CUDA device is usable, loading / context creation
raises, it never routes through a CPU implementation.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

_PKG = Path(__file__).resolve().parent
LIB_PATH = _PKG / "lib" / "libzstdb200.so"

c_size_p = C.POINTER(C.c_size_t)
c_u64_p = C.POINTER(C.c_uint64)


class FrameHeader(C.Structure):          # ZSTD_FrameHeader, N/zstd.h:1512-1522
    _fields_ = [("frameContentSize", C.c_ulonglong), ("windowSize", C.c_ulonglong), ("blockSizeMax", C.c_uint), ("frameType", C.c_int),
                ("headerSize", C.c_uint), ("dictID", C.c_uint), ("checksumFlag", C.c_uint), ("_reserved1", C.c_uint), ("_reserved2", C.c_uint)]


class FrameProgression(C.Structure):     # ZSTD_frameProgression, N/zstd.h:2736-2743
    _fields_ = [("ingested", C.c_ulonglong), ("consumed", C.c_ulonglong), ("produced", C.c_ulonglong), ("flushed", C.c_ulonglong),
                ("currentJobID", C.c_uint), ("nbActiveWorkers", C.c_uint)]


class NativeLibraryMissing(RuntimeError):
    pass


_lib = None


def lib() -> C.CDLL:
    """Load (once) and return libzstdb200.so with argtypes declared."""
    global _lib
    if _lib is not None:
        return _lib
    path = Path(os.environ.get("ZSTDB200_LIBRARY", LIB_PATH))
    if not path.exists():
        raise NativeLibraryMissing(
            f"{path} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). There is no CPU fallback.")
    L = C.CDLL(str(path))
    sz, vp, i, u64 = C.c_size_t, C.c_void_p, C.c_int, C.c_uint64

    def sig(name, res, *args):
        f = getattr(L, name)
        f.restype = res
        f.argtypes = list(args)

    sig("ZSTD_isError", C.c_uint, sz)
    sig("ZSTD_getErrorName", C.c_char_p, sz)
    sig("ZSTD_getErrorCode", i, sz)
    sig("ZSTD_versionNumber", C.c_uint)
    sig("ZSTD_versionString", C.c_char_p)
    sig("ZSTD_minCLevel", i)
    sig("ZSTD_maxCLevel", i)
    sig("ZSTD_defaultCLevel", i)
    sig("ZSTD_compressBound", sz, sz)
    sig("ZSTD_createCCtx", vp)
    sig("ZSTD_freeCCtx", sz, vp)
    sig("ZSTD_createDCtx", vp)
    sig("ZSTD_freeDCtx", sz, vp)
    sig("ZSTD_CCtx_setParameter", sz, vp, i, i)
    sig("ZSTD_CCtx_reset", sz, vp, i)
    sig("ZSTD_DCtx_reset", sz, vp, i)
    sig("ZSTD_CCtx_setPledgedSrcSize", sz, vp, C.c_ulonglong)
    sig("ZSTD_compress2", sz, vp, vp, sz, vp, sz)
    sig("ZSTD_compress", sz, vp, sz, vp, sz, i)
    sig("ZSTD_compressCCtx", sz, vp, vp, sz, vp, sz, i)
    sig("ZSTD_decompressDCtx", sz, vp, vp, sz, vp, sz)
    sig("ZSTD_decompress", sz, vp, sz, vp, sz)
    sig("ZSTD_DCtx_setParameter", sz, vp, i, i)
    sig("ZSTD_getFrameProgression", FrameProgression, vp)
    sig("ZSTD_getFrameHeader", sz, C.POINTER(FrameHeader), vp, sz)
    sig("ZSTD_getFrameHeader_advanced", sz, C.POINTER(FrameHeader), vp, sz, i)
    sig("ZSTD_frameHeaderSize", sz, vp, sz)
    sig("ZSTD_isFrame", C.c_uint, vp, sz)
    sig("ZSTD_isSkippableFrame", C.c_uint, vp, sz)
    sig("ZSTD_getDictID_fromFrame", C.c_uint, vp, sz)
    sig("ZSTD_getFrameContentSize", C.c_ulonglong, vp, sz)
    sig("ZSTD_findFrameCompressedSize", sz, vp, sz)
    sig("ZSTD_decompressBound", C.c_ulonglong, vp, sz)
    sig("ZSTD_createCStream", vp)
    sig("ZSTD_freeCStream", sz, vp)
    sig("ZSTD_initCStream", sz, vp, i)
    sig("ZSTD_compressStream2", sz, vp, vp, vp, i)
    sig("ZSTD_compressStream", sz, vp, vp, vp)
    sig("ZSTD_flushStream", sz, vp, vp)
    sig("ZSTD_endStream", sz, vp, vp)
    sig("ZSTD_CStreamInSize", sz)
    sig("ZSTD_CStreamOutSize", sz)
    sig("ZSTD_createDStream", vp)
    sig("ZSTD_freeDStream", sz, vp)
    sig("ZSTD_initDStream", sz, vp)
    sig("ZSTD_decompressStream", sz, vp, vp, vp)
    sig("ZSTD_DStreamInSize", sz)
    sig("ZSTD_DStreamOutSize", sz)

    sig("zstdb200_create", vp, i)
    sig("zstdb200_free", None, vp)
    sig("zstdb200_last_error", C.c_char_p)
    sig("zstdb200_device_count", i)
    sig("zstdb200_set_option", i, vp, C.c_char_p, C.c_longlong)
    sig("zstdb200_kernel_launches", C.c_ulonglong, vp)
    sig("zstdb200_kernel_times", sz, vp, C.c_char_p, sz)
    sig("zstdb200_compress_chunks", sz, vp, i, vp, sz, sz, vp, sz, c_size_p, c_size_p)
    sig("zstdb200_decompress_frames", sz, vp, vp, c_size_p, sz, vp, sz, c_size_p)
    sig("zstdb200_compress_chunks_begin", sz, vp, i, i, vp, sz, sz)
    sig("zstdb200_compress_chunks_end", sz, vp, i, vp, sz, c_size_p, c_size_p)
    sig("zstdb200_decompress_frames_begin", sz, vp, i, vp, c_size_p, sz, vp, sz, c_size_p)
    sig("zstdb200_decompress_frames_end", sz, vp, i, c_size_p)
    sig("zstdb200_host_register", sz, vp, sz)
    sig("zstdb200_host_unregister", sz, vp)
    sig("zstdb200_compress_batch", sz, vp, i, sz, C.POINTER(vp), c_size_p, C.POINTER(vp), c_size_p, c_size_p)
    sig("zstdb200_decompress_batch", sz, vp, sz, C.POINTER(vp), c_size_p, C.POINTER(vp), c_size_p, c_size_p)
    sig("zstdb200_generate_sequences", sz, vp, i, sz, C.POINTER(vp), c_size_p, C.POINTER(vp), c_size_p, c_size_p)
    sig("zstdb200_createSequenceProducerState", vp, i)
    sig("zstdb200_freeSequenceProducerState", None, vp)
    sig("zstdb200_sequenceProducer", sz, vp, vp, sz, vp, sz, vp, sz, i, sz)
    sig("zstdb200_compress_device", sz, vp, i, sz, vp, vp, vp, sz, vp, vp)
    sig("zstdb200_compact_device", sz, vp, sz, vp, sz, vp, vp, vp, vp)
    sig("zstdb200_decompress_device", sz, vp, sz, vp, vp, vp, vp, vp, vp)
    sig("zstdb200_sync", sz, vp, vp)
    _lib = L
    return L


class InBuffer(C.Structure):
    _fields_ = [("src", C.c_void_p), ("size", C.c_size_t), ("pos", C.c_size_t)]


class OutBuffer(C.Structure):
    _fields_ = [("dst", C.c_void_p), ("size", C.c_size_t), ("pos", C.c_size_t)]


ERROR_MAX = (1 << 64) - 120


def is_error(code: int) -> bool:
    return code > ERROR_MAX


def error_code(code: int) -> int:
    return (1 << 64) - code if is_error(code) else 0
