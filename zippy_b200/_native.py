"""ctypes binding of libzippy_b200.so (include/zippy_b200.h).  No fallback: a missing
library or a machine without a CUDA device raises."""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libzippy_b200.so")

c_u8p = ctypes.c_void_p
c_u64p = ctypes.c_void_p
c_intp = ctypes.c_void_p
c_size_t = ctypes.c_size_t
c_int = ctypes.c_int


class Timing(ctypes.Structure):
    _fields_ = [("lz_ms", ctypes.c_float), ("huff_ms", ctypes.c_float), ("scan_ms", ctypes.c_float),
                ("pack_ms", ctypes.c_float), ("inflate_ms", ctypes.c_float), ("verify_ms", ctypes.c_float),
                ("checksum_ms", ctypes.c_float), ("h2d_ms", ctypes.c_float), ("d2h_ms", ctypes.c_float),
                ("h2d_bytes", ctypes.c_uint64), ("d2h_bytes", ctypes.c_uint64),
                ("kernel_launches", ctypes.c_uint32), ("n_chunks", ctypes.c_uint32), ("plan_ms", ctypes.c_float)]


# name -> (restype, argtypes); every symbol include/zippy_b200.h declares
SYMBOLS = {
    "zb200_init": (c_int, [c_int, ctypes.POINTER(ctypes.c_void_p)]),
    "zb200_shutdown": (None, [ctypes.c_void_p]),
    "zb200_strerror": (ctypes.c_char_p, [c_int]),
    "zb200_last_cuda_error": (ctypes.c_char_p, [ctypes.c_void_p]),
    "zb200_device_count": (c_int, []),
    "zb200_set_stream": (c_int, [ctypes.c_void_p, ctypes.c_void_p]),
    "zb200_deflate_bound": (c_size_t, [c_size_t]),
    "zb200_compress_bound": (c_size_t, [c_size_t, c_int]),
    "zb200_deflate": (c_int, [ctypes.c_void_p, c_u8p, c_size_t, c_int, c_u8p, c_size_t, ctypes.POINTER(c_size_t)]),
    "zb200_inflate": (c_int, [ctypes.c_void_p, c_u8p, c_size_t, c_size_t, c_u8p, c_size_t, ctypes.POINTER(c_size_t)]),
    "zb200_inflate_size": (c_int, [ctypes.c_void_p, c_u8p, c_size_t, c_size_t, ctypes.POINTER(c_size_t)]),
    "zb200_decode_begin": (c_int, [ctypes.c_void_p, c_u8p, c_size_t, c_int, c_size_t, ctypes.POINTER(c_size_t)]),
    "zb200_decode_finish": (c_int, [ctypes.c_void_p, c_u8p, c_size_t, ctypes.POINTER(c_size_t)]),
    "zb200_crc32": (c_int, [ctypes.c_void_p, c_u8p, c_size_t, ctypes.POINTER(ctypes.c_uint32)]),
    "zb200_adler32": (c_int, [ctypes.c_void_p, c_u8p, c_size_t, ctypes.POINTER(ctypes.c_uint32)]),
    "zb200_compress_batch": (c_int, [ctypes.c_void_p, c_u8p, c_u64p, c_size_t, c_int, c_int, c_u8p, c_u8p, c_size_t,
                                     c_u64p, c_intp]),
    "zb200_compress_batch_strategy": (c_int, [ctypes.c_void_p, c_u8p, c_u64p, c_size_t, c_int, c_int, c_int, c_u8p, c_u8p,
                                              c_size_t, c_u64p, c_intp]),
    "zb200_compress_batch_device_strategy": (c_int, [ctypes.c_void_p, c_u8p, c_u64p, c_size_t, c_int, c_int, c_int, c_u8p,
                                                     c_u8p, c_size_t, c_u64p, c_intp]),
    "zb200_compress_batch_window": (c_int, [ctypes.c_void_p, c_u8p, c_u64p, c_size_t, c_int, c_int, c_int, c_int, c_u8p,
                                            c_u8p, c_size_t, c_u64p, c_intp]),
    "zb200_compress_batch_device_window": (c_int, [ctypes.c_void_p, c_u8p, c_u64p, c_size_t, c_int, c_int, c_int, c_int,
                                                   c_u8p, c_u8p, c_size_t, c_u64p, c_intp]),
    "zb200_compress_batch_optimal": (c_int, [ctypes.c_void_p, c_u8p, c_u64p, c_size_t, c_int, c_int, c_u8p, c_u8p,
                                             c_size_t, c_u64p, c_intp]),
    "zb200_compress_batch_device_optimal": (c_int, [ctypes.c_void_p, c_u8p, c_u64p, c_size_t, c_int, c_int, c_u8p,
                                                    c_u8p, c_size_t, c_u64p, c_intp]),
    "zb200_compress_batch_rsyncable": (c_int, [ctypes.c_void_p, c_u8p, c_u64p, c_size_t, c_int, c_int, c_u8p, c_u8p,
                                               c_size_t, c_u64p, c_intp]),
    "zb200_compress_batch_device_rsyncable": (c_int, [ctypes.c_void_p, c_u8p, c_u64p, c_size_t, c_int, c_int, c_u8p,
                                                      c_u8p, c_size_t, c_u64p, c_intp]),
    "zb200_compress_bound_rsyncable": (c_size_t, [c_size_t, c_int]),
    "zb200_rsyncable_chunks_bound": (c_size_t, [c_size_t]),
    "zb200_rsyncable_chunks": (c_int, [ctypes.c_void_p, c_u8p, c_u64p, c_size_t, c_u64p, c_u64p, c_size_t]),
    "zb200_compress_batch_h2d": (c_int, [ctypes.c_void_p, c_u8p, c_u64p, c_size_t, c_int, c_int, c_u8p, c_u8p, c_size_t,
                                         c_u64p, c_intp]),
    "zb200_download": (c_int, [ctypes.c_void_p, c_u8p, c_u8p, c_size_t]),
    "zb200_host_register": (c_int, [ctypes.c_void_p, c_size_t]),
    "zb200_host_unregister": (c_int, [ctypes.c_void_p]),
    "zb200_uncompress_sizes": (c_int, [ctypes.c_void_p, c_u8p, c_u64p, c_size_t, c_int, c_u64p, c_intp]),
    "zb200_uncompress_batch": (c_int, [ctypes.c_void_p, c_u8p, c_u64p, c_size_t, c_int, c_u8p, c_u64p, c_u64p, c_intp]),
    "zb200_inflate_batch_crc32": (c_int, [ctypes.c_void_p, c_u8p, c_u64p, c_size_t, c_u8p, c_u64p, c_u64p,
                                          ctypes.c_void_p, c_intp]),
    "zb200_checksum_batch": (c_int, [ctypes.c_void_p, c_u8p, c_u64p, c_size_t, c_int, ctypes.c_void_p]),
    "zb200_compress_batch_dict": (c_int, [ctypes.c_void_p, c_u8p, c_u64p, c_size_t, c_int, c_int, c_u8p, c_size_t, c_u8p,
                                          c_size_t, c_u64p, c_intp]),
    "zb200_uncompress_sizes_dict": (c_int, [ctypes.c_void_p, c_u8p, c_u64p, c_size_t, c_int, c_u8p, c_size_t, c_u64p,
                                            c_intp]),
    "zb200_uncompress_batch_dict": (c_int, [ctypes.c_void_p, c_u8p, c_u64p, c_size_t, c_int, c_u8p, c_size_t, c_u8p,
                                            c_u64p, c_u64p, c_intp]),
    "zb200_compress_batch_dicts": (c_int, [ctypes.c_void_p, c_u8p, c_u64p, c_size_t, c_int, c_int, c_int, c_u8p, c_u64p,
                                           c_size_t, c_intp, c_u8p, c_size_t, c_u64p, c_intp]),
    "zb200_uncompress_sizes_dicts": (c_int, [ctypes.c_void_p, c_u8p, c_u64p, c_size_t, c_int, c_u8p, c_u64p, c_size_t,
                                             c_intp, c_u64p, c_intp]),
    "zb200_uncompress_batch_dicts": (c_int, [ctypes.c_void_p, c_u8p, c_u64p, c_size_t, c_int, c_u8p, c_u64p, c_size_t,
                                             c_intp, c_u8p, c_u64p, c_u64p, c_intp]),
    "zb200_decode_begin_dict": (c_int, [ctypes.c_void_p, c_u8p, c_size_t, c_int, c_u8p, c_size_t,
                                        ctypes.POINTER(c_size_t)]),
    "zb200_compress_batch_device": (c_int, [ctypes.c_void_p, c_u8p, c_u64p, c_size_t, c_int, c_int, c_u8p, c_u8p,
                                            c_size_t, c_u64p, c_intp]),
    "zb200_uncompress_batch_device": (c_int, [ctypes.c_void_p, c_u8p, c_u64p, c_size_t, c_int, c_u8p, c_u64p, c_u64p,
                                              c_intp]),
    "zb200_uncompress_sizes_device": (c_int, [ctypes.c_void_p, c_u8p, c_u64p, c_size_t, c_int, c_u64p, c_intp]),
    "zb200_checksum_batch_device": (c_int, [ctypes.c_void_p, c_u8p, c_u64p, c_size_t, c_int, ctypes.c_void_p]),
    "zb200_compress_stream_begin": (c_int, [ctypes.c_void_p, c_int, c_int, c_int, ctypes.POINTER(ctypes.c_void_p)]),
    "zb200_compress_stream_begin_strategy": (c_int, [ctypes.c_void_p, c_int, c_int, c_int, c_int,
                                                     ctypes.POINTER(ctypes.c_void_p)]),
    "zb200_compress_stream_begin_window": (c_int, [ctypes.c_void_p, c_int, c_int, c_int, c_int, c_int,
                                                   ctypes.POINTER(ctypes.c_void_p)]),
    "zb200_compress_stream_begin_optimal": (c_int, [ctypes.c_void_p, c_int, c_int, c_int,
                                                    ctypes.POINTER(ctypes.c_void_p)]),
    "zb200_compress_stream_begin_dict": (c_int, [ctypes.c_void_p, c_int, c_int, c_u8p, c_size_t,
                                                 ctypes.POINTER(ctypes.c_void_p)]),
    "zb200_compress_stream_bound": (c_size_t, [ctypes.c_void_p, c_size_t]),
    "zb200_compress_stream_write": (c_int, [ctypes.c_void_p, c_u8p, c_size_t, c_u8p, c_size_t, ctypes.POINTER(c_size_t)]),
    "zb200_compress_stream_flush": (c_int, [ctypes.c_void_p, c_int, c_u8p, c_size_t, ctypes.POINTER(c_size_t)]),
    "zb200_compress_stream_finish": (c_int, [ctypes.c_void_p, c_u8p, c_size_t, ctypes.POINTER(c_size_t)]),
    "zb200_compress_stream_free": (None, [ctypes.c_void_p]),
    "zb200_decompress_stream_begin": (c_int, [ctypes.c_void_p, c_int, ctypes.POINTER(ctypes.c_void_p)]),
    "zb200_decompress_stream_begin_dict": (c_int, [ctypes.c_void_p, c_int, c_u8p, c_size_t,
                                                   ctypes.POINTER(ctypes.c_void_p)]),
    "zb200_decompress_stream_write": (c_int, [ctypes.c_void_p, c_u8p, c_size_t, ctypes.POINTER(c_size_t)]),
    "zb200_decompress_stream_drain": (c_int, [ctypes.c_void_p, ctypes.POINTER(c_size_t)]),
    "zb200_decompress_stream_finish": (c_int, [ctypes.c_void_p, ctypes.POINTER(c_size_t)]),
    "zb200_decompress_stream_read": (c_int, [ctypes.c_void_p, c_u8p, c_size_t, ctypes.POINTER(c_size_t)]),
    "zb200_decompress_stream_free": (None, [ctypes.c_void_p]),
    "zb200_index_build": (c_int, [ctypes.c_void_p, c_u8p, c_size_t, c_int, ctypes.c_uint64,
                                  ctypes.POINTER(ctypes.c_void_p)]),
    "zb200_index_extract_batch": (c_int, [ctypes.c_void_p, ctypes.c_void_p, c_u8p, c_size_t, c_u64p, c_u64p, c_size_t,
                                          c_u8p, c_u64p, c_intp]),
    "zb200_index_size": (ctypes.c_uint64, [ctypes.c_void_p]),
    "zb200_index_points": (c_size_t, [ctypes.c_void_p, c_u64p, c_u64p, ctypes.c_void_p, c_u8p, c_size_t]),
    "zb200_index_free": (None, [ctypes.c_void_p]),
    "zb200_index_export": (c_int, [ctypes.c_void_p, ctypes.c_void_p, c_u8p, c_size_t, ctypes.POINTER(c_size_t)]),
    "zb200_index_import": (c_int, [ctypes.c_void_p, c_u8p, c_size_t, ctypes.POINTER(ctypes.c_void_p)]),
    "zb200_compress_batch_index": (c_int, [ctypes.c_void_p, c_u8p, c_u64p, c_size_t, c_int, c_int, c_u8p, c_u8p,
                                           c_size_t, c_u64p, c_intp, ctypes.c_uint64, ctypes.c_void_p]),
    "zb200_compress_batch_device_index": (c_int, [ctypes.c_void_p, c_u8p, c_u64p, c_size_t, c_int, c_int, c_u8p, c_u8p,
                                                  c_size_t, c_u64p, c_intp, ctypes.c_uint64, ctypes.c_void_p]),
    "zb200_compress_stream_begin_index": (c_int, [ctypes.c_void_p, c_int, c_int, c_int, ctypes.c_uint64,
                                                  ctypes.POINTER(ctypes.c_void_p)]),
    "zb200_compress_stream_index": (c_int, [ctypes.c_void_p, ctypes.POINTER(ctypes.c_void_p)]),
    "zb200_mgpu_init": (c_int, [ctypes.c_void_p, c_int, ctypes.POINTER(ctypes.c_void_p)]),
    "zb200_mgpu_shutdown": (None, [ctypes.c_void_p]),
    "zb200_mgpu_device_count": (c_int, [ctypes.c_void_p]),
    "zb200_mgpu_compress_batch": (c_int, [ctypes.c_void_p, c_u8p, c_u64p, c_size_t, c_int, c_int, c_u8p, c_u8p, c_size_t,
                                          c_u64p, c_intp]),
    "zb200_mgpu_uncompress_batch": (c_int, [ctypes.c_void_p, c_u8p, c_u64p, c_size_t, c_int, c_u8p, c_u64p, c_u64p, c_intp]),
    "zb200_mgpu_checksum_batch": (c_int, [ctypes.c_void_p, c_u8p, c_u64p, c_size_t, c_int, ctypes.c_void_p]),
    "zb200_last_timing": (c_int, [ctypes.c_void_p, ctypes.POINTER(Timing)]),
}

_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                "zippy_b200: %s is missing -- build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc, sm_90a).  There is no CPU fallback." % LIB_PATH)
        L = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SYMBOLS.items():
            f = getattr(L, name)  # AttributeError if the ABI and the header drift apart
            f.restype = res
            f.argtypes = args
        _lib = L
    return _lib
