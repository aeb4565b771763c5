"""zippy_b200 -- host-side mirror of guzba/zippy's public API over the H100 C ABI.

Same names, argument meaning and error behaviour as the reference module
(src/zippy.nim:11-177, src/zippy/common.nim:1-12, crc.nim:53-75, adler32.nim:6-66):

    compress(src, level=DefaultCompression, dataFormat=dfGzip) -> bytes
    uncompress(src, dataFormat=dfDetect) -> bytes
    crc32(src) / adler32(src) -> int
    ZippyError, dfDetect/dfZlib/dfGzip/dfDeflate, NoCompression/BestSpeed/...

plus the batch forms that make a GPU worthwhile, CompressStream, one member compressed from input
that arrives in pieces, and DecompressStream, one member decoded from compressed input that arrives in pieces
(no reference counterparts).  All codec
work happens in libzippy_b200.so's CUDA kernels; this module only owns buffers, draws the
reference's random gzip FNAME length (zippy.nim:28-42) and maps status codes to ZippyError.
There is no CPU fallback: without the library or a CUDA device every call raises.
"""
import ctypes
import os
import threading

import numpy as np

from . import _native

dfDetect, dfZlib, dfGzip, dfDeflate = 0, 1, 2, 3                       # common.nim:4-5
NoCompression, BestSpeed, BestCompression = 0, 1, 9                    # common.nim:7-12
DefaultCompression, HuffmanOnly = -1, -2
SyncFlush, FullFlush = 2, 3                                            # zlib's Z_SYNC_FLUSH / Z_FULL_FLUSH
# zlib's Z_DEFAULT_STRATEGY, Z_FILTERED, Z_HUFFMAN_ONLY, Z_RLE, Z_FIXED (zippy_b200.h, "compression strategies")
StrategyDefault, StrategyFiltered, StrategyHuffmanOnly, StrategyRle, StrategyFixed = 0, 1, 2, 3, 4

__all__ = ["compress", "uncompress", "crc32", "adler32", "deflate", "inflate", "compress_batch", "uncompress_batch",
           "uncompressed_sizes", "checksum_batch", "ZippyError", "Context", "CompressStream", "DecompressStream",
           "compress_with_index", "compress_batch_with_index", "rsyncable_chunks",
           "MultiGpu", "Index", "dfDetect",
           "dfZlib", "dfGzip",
           "dfDeflate", "NoCompression", "BestSpeed", "BestCompression", "DefaultCompression", "HuffmanOnly",
           "SyncFlush", "FullFlush", "StrategyDefault", "StrategyFiltered", "StrategyHuffmanOnly", "StrategyRle",
           "StrategyFixed"]


class ZippyError(Exception):
    """Raised if an operation fails (common.nim:2).  .code is the ZB200_* status."""

    def __init__(self, code, msg=None):
        self.code = code
        super().__init__(msg or _native.lib().zb200_strerror(code).decode())


def _check(ctx, rc):
    if rc != 0:
        extra = ""
        if rc in (20, 21) and ctx is not None:
            extra = " [" + _native.lib().zb200_last_cuda_error(ctx).decode() + "]"
        raise ZippyError(rc, _native.lib().zb200_strerror(rc).decode() + extra)


def _as_u8(buf):
    if isinstance(buf, np.ndarray):
        return np.ascontiguousarray(buf, dtype=np.uint8).reshape(-1)
    return np.frombuffer(bytes(buf) if not isinstance(buf, (bytes, bytearray, memoryview)) else buf, dtype=np.uint8)


def _dict(dictionary):
    """A preset dictionary (zlib's zdict) as a uint8 array; None and an empty dictionary give None: the calls
    without a dictionary, as zlib writes no FDICT for an empty zdict."""
    d = None if dictionary is None else _as_u8(dictionary)
    return d if d is not None and d.size else None


def _dict_table(dictionaries, n):
    """`dictionaries=`: n bytes-like or None, one per item -> (base uint8, offsets uint64[k + 1], dict_of int32[n]),
    the table of the *_dicts calls.  Items that pass the same object share one entry; None and an empty dictionary
    name none (-1)."""
    if len(dictionaries) != n:
        raise ZippyError(22, "dictionaries= needs one entry (bytes-like or None) per item")
    entry, parts = {}, []
    dict_of = np.full(max(n, 1), -1, dtype=np.int32)
    for i, d in enumerate(dictionaries):
        if d is None:
            continue
        j = entry.get(id(d))
        if j is None:
            a = _as_u8(d)
            j = entry[id(d)] = len(parts) if a.size else -1
            if a.size:
                parts.append(a)
        dict_of[i] = j
    offs = np.zeros(len(parts) + 1, dtype=np.uint64)
    np.cumsum([p.size for p in parts], out=offs[1:])
    base = np.concatenate(parts) if parts else np.zeros(1, np.uint8)
    return base, offs, dict_of


def _one_table(dictionary, dictionaries):
    """dictionary= and dictionaries= exclude each other."""
    if dictionary is not None and dictionaries is not None:
        raise ZippyError(22, "dictionary= and dictionaries= are not combined")


def _params_alone(strategy, window_bits=15, dictionary=None, index_span=None):
    """True for a strategy other than the default or a window other than 15 (the _window calls); either takes no
    dictionary and no compress-time index."""
    what = "a compression strategy" if strategy != StrategyDefault else "a window size other than 15" \
        if window_bits != 15 else None
    if what is None:
        return False
    if _dict(dictionary) is not None:
        raise ZippyError(22, what + " is not combined with a dictionary")
    if index_span is not None:
        raise ZippyError(22, what + " is not combined with a compress-time index")
    return True


def _check_optimal(level, strategy=StrategyDefault, dictionary=None, index_span=None, dictionaries=None):
    """optimal=True (the optimal parse, zb200_compress_batch_optimal): its members do not depend on the level, which
    must be an LZ level (-1, 1..9); a strategy, a dictionary or a compress-time index is not combined with it."""
    if level < -2 or level > 9:
        raise ZippyError(1, "Invalid compression level %d" % level)
    if level in (NoCompression, HuffmanOnly):
        raise ZippyError(22, "the optimal parse is not combined with level %d" % level)
    if strategy != StrategyDefault:
        raise ZippyError(22, "the optimal parse is not combined with a compression strategy")
    if dictionary is not None or dictionaries is not None:
        raise ZippyError(22, "the optimal parse is not combined with a dictionary")
    if index_span is not None:
        raise ZippyError(22, "the optimal parse is not combined with a compress-time index")


def _check_rsyncable(strategy=StrategyDefault, window_bits=15, dictionary=None, index_span=None, dictionaries=None,
                     optimal=False):
    """rsyncable=True (content-defined chunk starts, zb200_compress_batch_rsyncable) is combined with every level and
    format, and with none of these."""
    for bad, what in ((dictionary is not None or dictionaries is not None, "a dictionary"),
                      (index_span is not None, "a compress-time index"),
                      (strategy != StrategyDefault, "a compression strategy"),
                      (window_bits != 15, "a window size other than 15"),
                      (optimal, "the optimal parse")):
        if bad:
            raise ZippyError(22, "rsyncable compression is not combined with " + what)


def _pack(items):
    """list of bytes-like -> (base uint8 array, offsets uint64[n+1])"""
    lens = np.fromiter((len(x) for x in items), dtype=np.uint64, count=len(items))
    offs = np.zeros(len(items) + 1, dtype=np.uint64)
    np.cumsum(lens, out=offs[1:])
    base = np.frombuffer(b"".join(bytes(x) for x in items), dtype=np.uint8) if len(items) else np.zeros(0, np.uint8)
    return base, offs


class Context:
    """One zb200_ctx: a CUDA device + stream + cached device scratch."""

    def __init__(self, device=-1):
        self._h = ctypes.c_void_p()
        L = _native.lib()
        rc = L.zb200_init(device, ctypes.byref(self._h))
        if rc != 0:
            raise ZippyError(rc, "zb200_init failed: %s (zippy_b200 needs a CUDA device; there is no CPU fallback)"
                             % L.zb200_strerror(rc).decode())

    LEGACY_DEFAULT_STREAM = 1   # cudaStreamLegacy: the handle that names the default stream explicitly

    def set_stream(self, cuda_stream):
        """Run on a caller-owned cudaStream_t (int handle).  0 / None restores the ctx's own (non-blocking)
        stream, which is NOT ordered against work the caller queued elsewhere: a caller that fills device
        buffers on its default stream and wants ordering without synchronising passes LEGACY_DEFAULT_STREAM
        (torch: `ctx.set_stream(torch.cuda.current_stream().cuda_stream or ctx.LEGACY_DEFAULT_STREAM)`)."""
        _check(self._h, _native.lib().zb200_set_stream(self._h, ctypes.c_void_p(cuda_stream or 0)))

    def close(self):
        if self._h:
            _native.lib().zb200_shutdown(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- batches over host buffers -------------------------------------------------
    def compress_batch(self, base, offsets, level=DefaultCompression, dataFormat=dfGzip, fname_lens=None,
                       dictionary=None, index_span=None, strategy=StrategyDefault, window_bits=15, dictionaries=None,
                       optimal=False, rsyncable=False):
        """-> (out uint8 array, out_offsets uint64[n+1]).  fname_lens: per-input gzip FNAME letters (0..25).
        rsyncable: content-defined chunk starts, so an edit changes only the compressed bytes near it
        (zb200_compress_batch_rsyncable; any level and format; no strategy, window size, dictionary, index or
        optimal parse).
        optimal: the optimal parse, smaller than level 9 (zb200_compress_batch_optimal): any LZ level (-1, 1..9)
        gives the same bytes; no strategy, dictionary or index.
        strategy: zlib's compression strategy (Strategy*; zb200_compress_batch_window; no dictionary or index).
        window_bits: zlib's window size, 9..15 (8 for zlib: 9); no match reaches more than 2^window_bits back
        (zb200_compress_batch_window; no dictionary or index).
        dictionary: a preset dictionary shared by every input (zlib / raw only; zb200_compress_batch_dict).
        dictionaries: one preset dictionary (bytes-like or None) per input, with any window_bits (zlib / raw only;
        zb200_compress_batch_dicts; no strategy or index); inputs that pass the same object share it.
        index_span: also write each member's Index with this span (zb200_compress_batch_index; no dictionary):
        -> (out, out_offsets, list of Index)."""
        L = _native.lib()
        base = _as_u8(base)
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        n = len(offsets) - 1
        if rsyncable:
            _check_rsyncable(strategy, window_bits, dictionary, index_span, dictionaries, optimal)
        fbound = L.zb200_compress_bound_rsyncable if rsyncable else L.zb200_compress_bound
        bound = sum(fbound(int(offsets[i + 1] - offsets[i]), dataFormat) for i in range(n)) \
            if n <= 4096 else int(fbound(int(offsets[-1] - offsets[0]), dataFormat)) + 64 * n
        _one_table(dictionary, dictionaries)
        with_dicts = _dict(dictionary) is not None or dictionaries is not None
        out = np.empty(int(bound) + (4 * n if with_dicts else 0) + 64, dtype=np.uint8)
        out_offs = np.zeros(n + 1, dtype=np.uint64)
        st = np.zeros(max(n, 1), dtype=np.int32)
        if rsyncable:
            fl = np.ascontiguousarray(fname_lens, dtype=np.uint8) if fname_lens is not None else None
            _check(self._h, L.zb200_compress_batch_rsyncable(self._h, base.ctypes.data, offsets.ctypes.data, n, level,
                                                              dataFormat, fl.ctypes.data if fl is not None else None,
                                                              out.ctypes.data, out.size, out_offs.ctypes.data,
                                                              st.ctypes.data))
            return out[:int(out_offs[n])], out_offs
        if optimal:
            _check_optimal(level, strategy, dictionary, index_span, dictionaries)
            fl = np.ascontiguousarray(fname_lens, dtype=np.uint8) if fname_lens is not None else None
            _check(self._h, L.zb200_compress_batch_optimal(self._h, base.ctypes.data, offsets.ctypes.data, n,
                                                            window_bits, dataFormat,
                                                            fl.ctypes.data if fl is not None else None,
                                                            out.ctypes.data, out.size, out_offs.ctypes.data,
                                                            st.ctypes.data))
            return out[:int(out_offs[n])], out_offs
        if dictionaries is not None:
            if strategy != StrategyDefault:
                raise ZippyError(22, "a compression strategy is not combined with a dictionary")
            if index_span is not None:
                raise ZippyError(22, "a compress-time index is not written with a dictionary")
            if fname_lens is not None:
                raise ZippyError(22, "fname_lens is not combined with dictionaries")
            db, do, dof = _dict_table(dictionaries, n)
            _check(self._h, L.zb200_compress_batch_dicts(self._h, base.ctypes.data, offsets.ctypes.data, n, level,
                                                          dataFormat, window_bits, db.ctypes.data, do.ctypes.data,
                                                          do.size - 1, dof.ctypes.data, out.ctypes.data, out.size,
                                                          out_offs.ctypes.data, st.ctypes.data))
            return out[:int(out_offs[n])], out_offs
        d = _dict(dictionary)
        if _params_alone(strategy, window_bits, d, index_span):
            fl = np.ascontiguousarray(fname_lens, dtype=np.uint8) if fname_lens is not None else None
            _check(self._h, L.zb200_compress_batch_window(self._h, base.ctypes.data, offsets.ctypes.data, n, level,
                                                           strategy, window_bits, dataFormat,
                                                           fl.ctypes.data if fl is not None else None,
                                                           out.ctypes.data, out.size, out_offs.ctypes.data,
                                                           st.ctypes.data))
            return out[:int(out_offs[n])], out_offs
        if index_span is not None:
            if d is not None:
                raise ZippyError(22, "a compress-time index is not written with a dictionary")
            fl = np.ascontiguousarray(fname_lens, dtype=np.uint8) if fname_lens is not None else None
            hs = (ctypes.c_void_p * max(n, 1))()
            _check(self._h, L.zb200_compress_batch_index(self._h, base.ctypes.data, offsets.ctypes.data, n, level,
                                                          dataFormat, fl.ctypes.data if fl is not None else None,
                                                          out.ctypes.data, out.size, out_offs.ctypes.data,
                                                          st.ctypes.data, index_span, hs))
            return out[:int(out_offs[n])], out_offs, [Index(h, self) for h in hs[:n]]
        if d is not None:
            _check(self._h, L.zb200_compress_batch_dict(self._h, base.ctypes.data, offsets.ctypes.data, n, level,
                                                         dataFormat, d.ctypes.data, d.size, out.ctypes.data, out.size,
                                                         out_offs.ctypes.data, st.ctypes.data))
            return out[:int(out_offs[n])], out_offs
        fl = None
        if fname_lens is not None:
            fl = np.ascontiguousarray(fname_lens, dtype=np.uint8)
        rc = L.zb200_compress_batch(self._h, base.ctypes.data, offsets.ctypes.data, n, level, dataFormat,
                                    fl.ctypes.data if fl is not None else None, out.ctypes.data, out.size,
                                    out_offs.ctypes.data, st.ctypes.data)
        _check(self._h, rc)
        return out[:int(out_offs[n])], out_offs

    def uncompressed_sizes(self, base, offsets, dataFormat=dfDetect, dictionary=None, dictionaries=None):
        """dictionaries: one preset dictionary (bytes-like or None) per member (zb200_uncompress_sizes_dicts)."""
        _one_table(dictionary, dictionaries)
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        table = _dict_table(dictionaries, len(offsets) - 1) if dictionaries is not None else None
        return self._sizes(base, offsets, dataFormat, dictionary, table)

    def _sizes(self, base, offsets, dataFormat, dictionary, table):
        """uncompressed_sizes with the dictionary table (_dict_table) already built, or None."""
        L = _native.lib()
        base = _as_u8(base)
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        n = len(offsets) - 1
        sizes = np.zeros(max(n, 1), dtype=np.uint64)
        st = np.zeros(max(n, 1), dtype=np.int32)
        if table is not None:
            db, do, dof = table
            _check(self._h, L.zb200_uncompress_sizes_dicts(self._h, base.ctypes.data, offsets.ctypes.data, n,
                                                            dataFormat, db.ctypes.data, do.ctypes.data, do.size - 1,
                                                            dof.ctypes.data, sizes.ctypes.data, st.ctypes.data))
            return sizes[:n], st[:n]
        d = _dict(dictionary)
        if d is not None:
            _check(self._h, L.zb200_uncompress_sizes_dict(self._h, base.ctypes.data, offsets.ctypes.data, n, dataFormat,
                                                           d.ctypes.data, d.size, sizes.ctypes.data, st.ctypes.data))
            return sizes[:n], st[:n]
        _check(self._h, L.zb200_uncompress_sizes(self._h, base.ctypes.data, offsets.ctypes.data, n, dataFormat,
                                                  sizes.ctypes.data, st.ctypes.data))
        return sizes[:n], st[:n]

    def uncompress_batch(self, base, offsets, dataFormat=dfDetect, max_total=None, sizes=None, dictionary=None,
                         dictionaries=None):
        """-> (out uint8 array, out_offsets uint64[n+1], out_lens uint64[n], statuses int32[n]).
        `sizes`: uncompressed sizes known to the caller (a container's directory); skips the sizing pass.
        `dictionary`: a preset dictionary for every raw member and every zlib member with FDICT.
        `dictionaries`: one such dictionary (bytes-like or None) per member (zb200_uncompress_batch_dicts)."""
        L = _native.lib()
        base = _as_u8(base)
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        n = len(offsets) - 1
        _one_table(dictionary, dictionaries)
        d = _dict(dictionary)
        table = _dict_table(dictionaries, n) if dictionaries is not None else None   # built once for both calls
        if sizes is None:
            sizes, st0 = self._sizes(base, offsets, dataFormat, d, table)
        else:
            sizes, st0 = np.ascontiguousarray(sizes, dtype=np.uint64), np.zeros(n, dtype=np.int32)
        sizes = np.where(st0 == 0, sizes, 0).astype(np.uint64)
        # a gzip ISIZE is a claim, not a fact: DEFLATE cannot expand more than 1032:1, so a
        # larger claim can only end in a size/checksum failure -- never allocate for it.
        comp_lens = offsets[1:] - offsets[:-1]
        sizes = np.minimum(sizes, comp_lens * np.uint64(1032) + np.uint64(1024))
        if max_total is not None and int(sizes.sum()) > max_total:
            raise ZippyError(19)
        dst_offs = np.zeros(n + 1, dtype=np.uint64)
        np.cumsum(sizes, out=dst_offs[1:])
        out = np.empty(int(dst_offs[n]) + 64, dtype=np.uint8)
        lens = np.zeros(max(n, 1), dtype=np.uint64)
        st = np.zeros(max(n, 1), dtype=np.int32)
        if table is not None:
            db, do, dof = table
            _check(self._h, L.zb200_uncompress_batch_dicts(self._h, base.ctypes.data, offsets.ctypes.data, n,
                                                            dataFormat, db.ctypes.data, do.ctypes.data, do.size - 1,
                                                            dof.ctypes.data, out.ctypes.data, dst_offs.ctypes.data,
                                                            lens.ctypes.data, st.ctypes.data))
        elif d is None:
            _check(self._h, L.zb200_uncompress_batch(self._h, base.ctypes.data, offsets.ctypes.data, n, dataFormat,
                                                      out.ctypes.data, dst_offs.ctypes.data, lens.ctypes.data,
                                                      st.ctypes.data))
        else:
            _check(self._h, L.zb200_uncompress_batch_dict(self._h, base.ctypes.data, offsets.ctypes.data, n, dataFormat,
                                                           d.ctypes.data, d.size, out.ctypes.data, dst_offs.ctypes.data,
                                                           lens.ctypes.data, st.ctypes.data))
        st = np.where(st0 != 0, st0, st[:n]).astype(np.int32)
        out, dst_offs = self._redo_too_small(base, offsets, dataFormat, out[:int(dst_offs[n])], dst_offs, lens[:n], st,
                                             dictionary=d, dictionaries=dictionaries)
        return out, dst_offs, lens[:n], st

    def _redo_too_small(self, base, offsets, dataFormat, out, dst_offs, lens, st, crcs=None, dictionary=None,
                        dictionaries=None):
        """A size claim (gzip ISIZE, a container's directory) understated the content (status 19): the reference
        inflates anyway and lets its checksum / size checks decide (gzip.nim:80-88) -- redo those members one by
        one.  lens / st / crcs are updated in place; -> (out, dst_offs) with the redone outputs appended."""
        small = np.nonzero(st == 19)[0]
        if not len(small):
            return out, dst_offs
        extra = []
        end = int(dst_offs[-1])
        dst_offs = dst_offs.copy()
        for i in small:
            try:
                b = self.decode_one(base[int(offsets[i]):int(offsets[i + 1])], dataFormat,
                                    dictionary=dictionary if dictionaries is None else dictionaries[i])
                st[i] = 0
                dst_offs[i] = end          # appended behind the slots; callers use out[off : off + len]
                lens[i] = len(b)
                if crcs is not None:
                    crcs[i] = self.crc32(b)
                end += len(b)
                extra.append(np.frombuffer(b, dtype=np.uint8))
            except ZippyError as e:
                st[i] = e.code
        if extra:
            out = np.concatenate([out] + extra)
        return out, dst_offs

    def inflate_batch_crc32(self, base, offsets, sizes):
        """Raw deflate members into slots of `sizes` bytes (a ZIP directory's uncompressed sizes)
        -> (out uint8 array, out_offsets uint64[n+1], out_lens uint64[n], crcs uint32[n], statuses int32[n]):
        uncompress_batch(..., dfDeflate, sizes=sizes), plus the CRC-32 of every output that inflated, computed on
        the device in the decode call (zb200_inflate_batch_crc32).  crcs[i] is 0 where statuses[i] != 0."""
        L = _native.lib()
        base = _as_u8(base)
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        n = len(offsets) - 1
        comp_lens = offsets[1:] - offsets[:-1]
        sizes = np.minimum(np.ascontiguousarray(sizes, dtype=np.uint64), comp_lens * np.uint64(1032) + np.uint64(1024))
        dst_offs = np.zeros(n + 1, dtype=np.uint64)
        np.cumsum(sizes, out=dst_offs[1:])
        out = np.empty(int(dst_offs[n]) + 64, dtype=np.uint8)
        lens = np.zeros(max(n, 1), dtype=np.uint64)
        crcs = np.zeros(max(n, 1), dtype=np.uint32)
        st = np.zeros(max(n, 1), dtype=np.int32)
        _check(self._h, L.zb200_inflate_batch_crc32(self._h, base.ctypes.data, offsets.ctypes.data, n, out.ctypes.data,
                                                     dst_offs.ctypes.data, lens.ctypes.data, crcs.ctypes.data,
                                                     st.ctypes.data))
        lens, crcs, st = lens[:n], crcs[:n], st[:n]
        out, dst_offs = self._redo_too_small(base, offsets, dfDeflate, out[:int(dst_offs[n])], dst_offs, lens, st, crcs)
        return out, dst_offs, lens, crcs, st

    def checksum_batch(self, base, offsets, kind="crc32"):
        L = _native.lib()
        base = _as_u8(base)
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        n = len(offsets) - 1
        out = np.zeros(max(n, 1), dtype=np.uint32)
        _check(self._h, L.zb200_checksum_batch(self._h, base.ctypes.data, offsets.ctypes.data, n,
                                                0 if kind == "crc32" else 1, out.ctypes.data))
        return out[:n]

    # ---- device-resident batches (raw device pointers; e.g. torch tensor .data_ptr()) ----
    def compress_batch_device(self, d_src, offsets, level, dataFormat, d_dst, dst_cap, fname_lens=None,
                              index_span=None, strategy=StrategyDefault, window_bits=15, optimal=False,
                              rsyncable=False):
        """-> out_offsets; with index_span also each member's Index (zb200_compress_batch_device_index):
        -> (out_offsets, list of Index).  strategy, window_bits: zlib's compression strategy and window size
        (zb200_compress_batch_device_window; no index).  optimal: the optimal parse
        (zb200_compress_batch_device_optimal; no strategy or index).  rsyncable: content-defined chunk starts
        (zb200_compress_batch_device_rsyncable; size d_dst by zb200_compress_bound_rsyncable; no strategy, window
        size, index or optimal parse)."""
        L = _native.lib()
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        n = len(offsets) - 1
        out_offs = np.zeros(n + 1, dtype=np.uint64)
        fl = np.ascontiguousarray(fname_lens, dtype=np.uint8) if fname_lens is not None else None
        if rsyncable:
            _check_rsyncable(strategy, window_bits, None, index_span, None, optimal)
            _check(self._h, L.zb200_compress_batch_device_rsyncable(self._h, d_src, offsets.ctypes.data, n, level,
                                                                     dataFormat,
                                                                     fl.ctypes.data if fl is not None else None,
                                                                     d_dst, dst_cap, out_offs.ctypes.data, None))
            return out_offs
        if optimal:
            _check_optimal(level, strategy, None, index_span)
            _check(self._h, L.zb200_compress_batch_device_optimal(self._h, d_src, offsets.ctypes.data, n, window_bits,
                                                                   dataFormat, fl.ctypes.data if fl is not None else None,
                                                                   d_dst, dst_cap, out_offs.ctypes.data, None))
            return out_offs
        if _params_alone(strategy, window_bits, None, index_span):
            _check(self._h, L.zb200_compress_batch_device_window(self._h, d_src, offsets.ctypes.data, n, level,
                                                                  strategy, window_bits, dataFormat,
                                                                  fl.ctypes.data if fl is not None else None, d_dst,
                                                                  dst_cap, out_offs.ctypes.data, None))
            return out_offs
        if index_span is not None:
            hs = (ctypes.c_void_p * max(n, 1))()
            _check(self._h, L.zb200_compress_batch_device_index(self._h, d_src, offsets.ctypes.data, n, level,
                                                                 dataFormat, fl.ctypes.data if fl is not None else None,
                                                                 d_dst, dst_cap, out_offs.ctypes.data, None,
                                                                 index_span, hs))
            return out_offs, [Index(h, self) for h in hs[:n]]
        _check(self._h, L.zb200_compress_batch_device(self._h, d_src, offsets.ctypes.data, n, level, dataFormat,
                                                       fl.ctypes.data if fl is not None else None, d_dst, dst_cap,
                                                       out_offs.ctypes.data, None))
        return out_offs

    def compress_batch_h2d(self, h_src, offsets, level, dataFormat, d_dst, dst_cap, fname_lens=None):
        """Host inputs (raw pointer; page-locked memory lets the copies overlap the kernels) -> members left
        in device memory at d_dst.  Returns the member offsets (uint64[n+1])."""
        L = _native.lib()
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        n = len(offsets) - 1
        out_offs = np.zeros(n + 1, dtype=np.uint64)
        fl = np.ascontiguousarray(fname_lens, dtype=np.uint8) if fname_lens is not None else None
        _check(self._h, L.zb200_compress_batch_h2d(self._h, h_src, offsets.ctypes.data, n, level, dataFormat,
                                                    fl.ctypes.data if fl is not None else None, d_dst, dst_cap,
                                                    out_offs.ctypes.data, None))
        return out_offs

    def download(self, d_src, h_dst, nbytes):
        """Device -> host copy on the ctx stream; returns when the bytes have landed."""
        _check(self._h, _native.lib().zb200_download(self._h, d_src, h_dst, nbytes))

    def uncompress_batch_device(self, d_src, offsets, dataFormat, d_dst, dst_offsets):
        L = _native.lib()
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        dst_offsets = np.ascontiguousarray(dst_offsets, dtype=np.uint64)
        n = len(offsets) - 1
        lens = np.zeros(max(n, 1), dtype=np.uint64)
        st = np.zeros(max(n, 1), dtype=np.int32)
        _check(self._h, L.zb200_uncompress_batch_device(self._h, d_src, offsets.ctypes.data, n, dataFormat, d_dst,
                                                         dst_offsets.ctypes.data, lens.ctypes.data, st.ctypes.data))
        return lens[:n], st[:n]

    def uncompressed_sizes_device(self, d_src, offsets, dataFormat):
        L = _native.lib()
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        n = len(offsets) - 1
        sizes = np.zeros(max(n, 1), dtype=np.uint64)
        st = np.zeros(max(n, 1), dtype=np.int32)
        _check(self._h, L.zb200_uncompress_sizes_device(self._h, d_src, offsets.ctypes.data, n, dataFormat,
                                                         sizes.ctypes.data, st.ctypes.data))
        return sizes[:n], st[:n]

    def checksum_batch_device(self, d_src, offsets, kind="crc32"):
        L = _native.lib()
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        n = len(offsets) - 1
        out = np.zeros(max(n, 1), dtype=np.uint32)
        _check(self._h, L.zb200_checksum_batch_device(self._h, d_src, offsets.ctypes.data, n,
                                                       0 if kind == "crc32" else 1, out.ctypes.data))
        return out[:n]

    def timing(self):
        t = _native.Timing()
        _check(self._h, _native.lib().zb200_last_timing(self._h, ctypes.byref(t)))
        return {f: getattr(t, f) for f, _ in t._fields_}

    def rsyncable_chunks(self, base, offsets):
        """The chunk starts the rsyncable compress calls cut each member base[offsets[i], offsets[i + 1]) at
        (zb200_rsyncable_chunks): -> list of uint64 arrays, positions in the member, ascending, the first 0."""
        L = _native.lib()
        base = _as_u8(base)
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        n = len(offsets) - 1
        cap = sum(L.zb200_rsyncable_chunks_bound(int(offsets[i + 1] - offsets[i])) for i in range(n))
        counts = np.zeros(max(n, 1), dtype=np.uint64)
        starts = np.zeros(max(cap, 1), dtype=np.uint64)
        _check(self._h, L.zb200_rsyncable_chunks(self._h, base.ctypes.data, offsets.ctypes.data, n, counts.ctypes.data,
                                                  starts.ctypes.data, cap))
        at = np.zeros(n + 1, dtype=np.uint64)
        np.cumsum(counts[:n], out=at[1:])
        return [starts[int(at[i]):int(at[i + 1])].copy() for i in range(n)]

    # ---- the single-input seam (deflate.nim:207, inflate.nim:268, crc.nim:53, adler32.nim:6) ----
    def deflate(self, src, level=DefaultCompression, strategy=StrategyDefault, window_bits=15, optimal=False,
                rsyncable=False):
        L = _native.lib()
        src = _as_u8(src)
        if strategy != StrategyDefault or window_bits != 15 or optimal or rsyncable:   # one raw DEFLATE member of the batch call
            out, _ = self.compress_batch(src, [0, src.size], level, dfDeflate, strategy=strategy,
                                         window_bits=window_bits, optimal=optimal, rsyncable=rsyncable)
            return out.tobytes()
        cap = L.zb200_deflate_bound(src.size)
        out = np.empty(cap + 8, dtype=np.uint8)
        n = ctypes.c_size_t(0)
        _check(self._h, L.zb200_deflate(self._h, src.ctypes.data, src.size, level, out.ctypes.data, out.size,
                                        ctypes.byref(n)))
        return out[:n.value].tobytes()

    def decode_one(self, src, dataFormat=dfDetect, pos=0, dictionary=None):
        """One input of unknown size, decoded once: zb200_decode_begin (inflate + trailer check into device
        memory, size reported) then zb200_decode_finish (copy out).  With a dictionary: zb200_decode_begin_dict
        (raw members start at byte 0, so pos must be 0)."""
        L = _native.lib()
        src = _as_u8(src)
        n = ctypes.c_size_t(0)
        d = _dict(dictionary)
        if d is None:
            _check(self._h, L.zb200_decode_begin(self._h, src.ctypes.data, src.size, dataFormat, pos, ctypes.byref(n)))
        elif pos:
            raise ZippyError(22, "a dictionary decode starts at byte 0")
        else:
            _check(self._h, L.zb200_decode_begin_dict(self._h, src.ctypes.data, src.size, dataFormat, d.ctypes.data,
                                                       d.size, ctypes.byref(n)))
        out = np.empty(n.value + 8, dtype=np.uint8)
        m = ctypes.c_size_t(0)
        _check(self._h, L.zb200_decode_finish(self._h, out.ctypes.data, n.value, ctypes.byref(m)))
        return out[:m.value].tobytes()

    def inflate(self, src, pos=0):
        return self.decode_one(src, dfDeflate, pos)

    def crc32(self, src):
        src = _as_u8(src)
        v = ctypes.c_uint32(0)
        _check(self._h, _native.lib().zb200_crc32(self._h, src.ctypes.data, src.size, ctypes.byref(v)))
        return v.value

    def adler32(self, src):
        src = _as_u8(src)
        v = ctypes.c_uint32(0)
        _check(self._h, _native.lib().zb200_adler32(self._h, src.ctypes.data, src.size, ctypes.byref(v)))
        return v.value


class CompressStream:
    """One gzip / zlib / raw member written piece by piece (zb200_compress_stream_*): the concatenation of what
    write() and finish() return is exactly compress_batch([whole input]) with the same FNAME length.  Input is
    gathered until a batch is pending, so most small writes return b"".  With gzip and fname_len=None the FNAME
    length is drawn at random, as compress() does (zippy.nim:28-42)."""

    def __init__(self, level=DefaultCompression, dataFormat=dfGzip, fname_len=None, ctx=None, dictionary=None,
                 index_span=None, strategy=StrategyDefault, window_bits=15, optimal=False):
        """index_span: also write the member's Index with this span (zb200_compress_stream_begin_index; no
        dictionary), returned by index() after finish().  strategy, window_bits: zlib's compression strategy and
        window size, kept for the stream's whole life (zb200_compress_stream_begin_window; no dictionary or index).
        optimal: the optimal parse (zb200_compress_stream_begin_optimal; no strategy, dictionary or index)."""
        self._ctx = ctx if ctx is not None else default_context()
        self._h = ctypes.c_void_p()
        d = _dict(dictionary)
        if optimal:
            _check_optimal(level, strategy, d, index_span)
            if fname_len is None:
                fname_len = os.urandom(1)[0] % 26 if dataFormat == dfGzip else 0
            _check(self._ctx._h, _native.lib().zb200_compress_stream_begin_optimal(
                self._ctx._h, window_bits, dataFormat, fname_len, ctypes.byref(self._h)))
            return
        if _params_alone(strategy, window_bits, d, index_span):
            if fname_len is None:
                fname_len = os.urandom(1)[0] % 26 if dataFormat == dfGzip else 0
            _check(self._ctx._h, _native.lib().zb200_compress_stream_begin_window(
                self._ctx._h, level, strategy, window_bits, dataFormat, fname_len, ctypes.byref(self._h)))
            return
        if index_span is not None:
            if d is not None:
                raise ZippyError(22, "a compress-time index is not written with a dictionary")
            if fname_len is None:
                fname_len = os.urandom(1)[0] % 26 if dataFormat == dfGzip else 0
            _check(self._ctx._h, _native.lib().zb200_compress_stream_begin_index(
                self._ctx._h, level, dataFormat, fname_len, index_span, ctypes.byref(self._h)))
            return
        if d is not None:   # zb200_compress_stream_begin_dict: zlib / raw only, no FNAME
            _check(self._ctx._h, _native.lib().zb200_compress_stream_begin_dict(self._ctx._h, level, dataFormat,
                                                                                d.ctypes.data, d.size,
                                                                                ctypes.byref(self._h)))
            return
        if fname_len is None:
            fname_len = os.urandom(1)[0] % 26 if dataFormat == dfGzip else 0
        _check(self._ctx._h, _native.lib().zb200_compress_stream_begin(self._ctx._h, level, dataFormat, fname_len,
                                                                       ctypes.byref(self._h)))

    def _out(self, n):
        """-> (a destination for the next call that takes n input bytes, its length word)"""
        if not self._h:
            raise ZippyError(22, "the stream is closed")
        return np.empty(int(_native.lib().zb200_compress_stream_bound(self._h, n)) + 8, dtype=np.uint8), ctypes.c_size_t(0)

    def write(self, data):
        src = _as_u8(data)
        out, m = self._out(src.size)
        _check(self._ctx._h, _native.lib().zb200_compress_stream_write(self._h, src.ctypes.data, src.size, out.ctypes.data,
                                                                       out.size, ctypes.byref(m)))
        return out[:m.value].tobytes()

    def flush(self, mode=SyncFlush):
        """Emit everything written so far: what the stream has returned decodes to everything written.  SyncFlush
        keeps the compression history, FullFlush drops it so a raw inflater can start right after.  Returns b""
        when nothing was written since the last flush (zlib's Z_SYNC_FLUSH / Z_FULL_FLUSH)."""
        out, m = self._out(0)
        _check(self._ctx._h, _native.lib().zb200_compress_stream_flush(self._h, mode, out.ctypes.data, out.size,
                                                                       ctypes.byref(m)))
        return out[:m.value].tobytes()

    def finish(self):
        out, m = self._out(0)
        _check(self._ctx._h, _native.lib().zb200_compress_stream_finish(self._h, out.ctypes.data, out.size,
                                                                        ctypes.byref(m)))
        return out[:m.value].tobytes()

    def index(self):
        """The member's Index, after finish() on a stream begun with index_span."""
        if not self._h:
            raise ZippyError(22, "the stream is closed")
        h = ctypes.c_void_p()
        _check(self._ctx._h, _native.lib().zb200_compress_stream_index(self._h, ctypes.byref(h)))
        return Index(h, self._ctx)

    def close(self):
        if self._h:
            _native.lib().zb200_compress_stream_free(self._h)
            self._h = ctypes.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class DecompressStream:
    """One gzip / zlib / raw member decoded from compressed input that arrives in pieces (zb200_decompress_stream_*):
    the concatenation of what write() and finish() return is exactly uncompress(whole input, dataFormat), and a bad
    input raises the ZippyError uncompress raises (at the latest from finish()).  Input is gathered until a batch is
    pending, so most small writes return b""."""

    def __init__(self, dataFormat=dfDetect, ctx=None, dictionary=None):
        """dictionary: a preset dictionary for a raw stream or a zlib member with FDICT
        (zb200_decompress_stream_begin_dict)."""
        self._ctx = ctx if ctx is not None else default_context()
        self._h = ctypes.c_void_p()
        d = _dict(dictionary)
        if d is not None:
            _check(self._ctx._h, _native.lib().zb200_decompress_stream_begin_dict(self._ctx._h, dataFormat, d.ctypes.data,
                                                                                  d.size, ctypes.byref(self._h)))
            return
        _check(self._ctx._h, _native.lib().zb200_decompress_stream_begin(self._ctx._h, dataFormat, ctypes.byref(self._h)))

    def _handle(self):
        if not self._h:
            raise ZippyError(22, "the stream is closed")
        return self._h

    def _take(self, avail):
        out = np.empty(avail, dtype=np.uint8)
        m = ctypes.c_size_t(0)
        _check(self._ctx._h, _native.lib().zb200_decompress_stream_read(self._handle(), out.ctypes.data, avail,
                                                                        ctypes.byref(m)))
        return out[:m.value].tobytes()

    def write(self, data):
        src = _as_u8(data)
        avail = ctypes.c_size_t(0)
        _check(self._ctx._h, _native.lib().zb200_decompress_stream_write(self._handle(), src.ctypes.data, src.size,
                                                                         ctypes.byref(avail)))
        return self._take(avail.value)

    def drain(self):
        """Decode every block that is complete in the input so far, whatever the batching threshold: after a
        sender's flush, everything it wrote up to the flush -- once the header is decided: raw streams at once,
        otherwise after 19 member bytes and, for gzip, the whole header and 9 bytes more."""
        avail = ctypes.c_size_t(0)
        _check(self._ctx._h, _native.lib().zb200_decompress_stream_drain(self._handle(), ctypes.byref(avail)))
        return self._take(avail.value)

    def finish(self):
        avail = ctypes.c_size_t(0)
        _check(self._ctx._h, _native.lib().zb200_decompress_stream_finish(self._handle(), ctypes.byref(avail)))
        return self._take(avail.value)

    def close(self):
        if self._h:
            _native.lib().zb200_decompress_stream_free(self._h)
            self._h = ctypes.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class MultiGpu:
    """zb200_mgpu: several devices behind one call (one host thread and one ctx per device)."""

    def __init__(self, devices=None):
        self._h = ctypes.c_void_p()
        L = _native.lib()
        arr = (ctypes.c_int * len(devices))(*devices) if devices else None
        rc = L.zb200_mgpu_init(arr, len(devices) if devices else 0, ctypes.byref(self._h))
        if rc != 0:
            raise ZippyError(rc, "zb200_mgpu_init failed: %s" % L.zb200_strerror(rc).decode())

    def close(self):
        if self._h:
            _native.lib().zb200_mgpu_shutdown(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def device_count(self):
        return _native.lib().zb200_mgpu_device_count(self._h)

    def compress_batch(self, base, offsets, level=DefaultCompression, dataFormat=dfGzip):
        """-> (one concatenated uint8 stream, global member offsets uint64[n+1])"""
        L = _native.lib()
        base = _as_u8(base)
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        n = len(offsets) - 1
        bound = int(L.zb200_compress_bound(int(offsets[-1] - offsets[0]), dataFormat)) + 128 * n + 4096
        out = np.empty(bound, dtype=np.uint8)
        oo = np.zeros(n + 1, dtype=np.uint64)
        _check(None, L.zb200_mgpu_compress_batch(self._h, base.ctypes.data, offsets.ctypes.data, n, level, dataFormat, None,
                                                  out.ctypes.data, out.size, oo.ctypes.data, None))
        return out[:int(oo[n])], oo

    def uncompress_batch(self, base, offsets, sizes, dataFormat=dfDetect):
        """sizes: output slot sizes (uint64[n]).  -> (out, dst_offsets, lens, statuses)"""
        L = _native.lib()
        base = _as_u8(base)
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        n = len(offsets) - 1
        do = np.zeros(n + 1, dtype=np.uint64)
        np.cumsum(np.asarray(sizes, dtype=np.uint64), out=do[1:])
        out = np.empty(int(do[n]) + 64, dtype=np.uint8)
        lens = np.zeros(max(n, 1), dtype=np.uint64)
        st = np.zeros(max(n, 1), dtype=np.int32)
        _check(None, L.zb200_mgpu_uncompress_batch(self._h, base.ctypes.data, offsets.ctypes.data, n, dataFormat,
                                                    out.ctypes.data, do.ctypes.data, lens.ctypes.data, st.ctypes.data))
        return out[:int(do[n])], do, lens[:n], st[:n]

    def checksum_batch(self, base, offsets, kind="crc32"):
        L = _native.lib()
        base = _as_u8(base)
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        n = len(offsets) - 1
        out = np.zeros(max(n, 1), dtype=np.uint32)
        _check(None, L.zb200_mgpu_checksum_batch(self._h, base.ctypes.data, offsets.ctypes.data, n,
                                                  0 if kind == "crc32" else 1, out.ctypes.data))
        return out[:n]


class Index:
    """Random access into one gzip / zlib / raw member (zb200_index_*): access points found by one decode on the
    GPU, then batches of ranges decoded from the nearest window point.  The index lives in host memory; `ctx` is
    only the context its calls run on."""

    def __init__(self, handle, ctx):
        self._h = handle
        self._ctx = ctx

    @classmethod
    def build(cls, data, dataFormat=dfDetect, span=1 << 20, ctx=None):
        ctx = ctx or default_context()
        src = _as_u8(data)
        h = ctypes.c_void_p()
        _check(ctx._h, _native.lib().zb200_index_build(ctx._h, src.ctypes.data, src.size, dataFormat, span,
                                                       ctypes.byref(h)))
        return cls(h, ctx)

    def _handle(self):
        if not self._h:
            raise ZippyError(22, "the index is closed")
        return self._h

    @property
    def size(self):
        """The member's output size."""
        return int(_native.lib().zb200_index_size(self._handle()))

    @property
    def points(self):
        """dict of numpy arrays, one entry per segment point: bit (position in the member), out (output offset),
        crc (CRC-32 of the interval up to the next point) and window (1 at window points)."""
        L, h = _native.lib(), self._handle()
        n = int(L.zb200_index_points(h, None, None, None, None, 0))
        bits, outs = np.zeros(n, np.uint64), np.zeros(n, np.uint64)
        crcs, win = np.zeros(n, np.uint32), np.zeros(n, np.uint8)
        L.zb200_index_points(h, bits.ctypes.data, outs.ctypes.data, crcs.ctypes.data, win.ctypes.data, n)
        return {"bit": bits, "out": outs, "crc": crcs, "window": win}

    def extract_batch(self, data, offsets, lengths):
        """-> (out uint8 array, out_offsets uint64[n+1], statuses int32[n]): range i is
        out[out_offsets[i]:out_offsets[i+1]] where statuses[i] == 0."""
        src = _as_u8(data)
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64).reshape(-1)
        lengths = np.ascontiguousarray(lengths, dtype=np.uint64).reshape(-1)
        if offsets.size != lengths.size:
            raise ZippyError(22, "offsets and lengths differ in length")
        n = offsets.size
        out_offs = np.zeros(n + 1, dtype=np.uint64)
        np.cumsum(lengths, out=out_offs[1:])
        out = np.empty(int(out_offs[n]) + 1, dtype=np.uint8)
        st = np.zeros(max(n, 1), dtype=np.int32)
        _check(self._ctx._h, _native.lib().zb200_index_extract_batch(
            self._ctx._h, self._handle(), src.ctypes.data, src.size, offsets.ctypes.data, lengths.ctypes.data, n,
            out.ctypes.data, out_offs.ctypes.data, st.ctypes.data))
        return out[:int(out_offs[n])], out_offs, st[:n]

    def extract(self, data, offset, length):
        """The output bytes [offset, offset + length) of the member; raises ZippyError on a bad range or member."""
        out, _, st = self.extract_batch(data, [offset], [length])
        if st[0] != 0:
            raise ZippyError(int(st[0]))
        return out.tobytes()

    def to_bytes(self):
        """The index serialised (include/zippy_b200.h documents the format); Index.from_bytes reads it back."""
        L, h = _native.lib(), self._handle()
        n = ctypes.c_size_t(0)
        _check(self._ctx._h, L.zb200_index_export(self._ctx._h, h, None, 0, ctypes.byref(n)))
        out = np.empty(n.value, dtype=np.uint8)
        _check(self._ctx._h, L.zb200_index_export(self._ctx._h, h, out.ctypes.data, out.size, ctypes.byref(n)))
        return out[:n.value].tobytes()

    @classmethod
    def from_bytes(cls, buf, ctx=None):
        ctx = ctx or default_context()
        src = _as_u8(buf)
        h = ctypes.c_void_p()
        _check(ctx._h, _native.lib().zb200_index_import(ctx._h, src.ctypes.data, src.size, ctypes.byref(h)))
        return cls(h, ctx)

    def close(self):
        if self._h:
            _native.lib().zb200_index_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def host_register(ptr, nbytes):
    """Page-lock a caller-owned host range (cudaHostRegister) so host-buffer calls overlap their copies."""
    _check(None, _native.lib().zb200_host_register(ptr, nbytes))


def host_unregister(ptr):
    _check(None, _native.lib().zb200_host_unregister(ptr))


_default = None
_default_lock = threading.Lock()


def default_context():
    global _default
    with _default_lock:
        if _default is None:
            _default = Context(-1)
        return _default


# ---- the reference's public procs ------------------------------------------------------
def compress(src, level=DefaultCompression, dataFormat=dfGzip, dictionary=None, strategy=StrategyDefault,
             window_bits=15, optimal=False, rsyncable=False):
    """zippy.compress (zippy.nim:11-98).  dictionary: a preset dictionary (zlib / raw only; zlib's zdict).
    strategy: zlib's compression strategy (Strategy*), not with a dictionary.  window_bits: zlib's window size
    (9..15; 8 for zlib means 9): no match reaches more than 2^window_bits back; other than 15 not with a dictionary.
    optimal: the optimal parse, smaller than level 9 (any LZ level gives the same bytes; no strategy or dictionary).
    rsyncable: content-defined chunk starts (as gzip --rsyncable), so an edit to src changes only the compressed bytes
    near it; any level and format, no dictionary, strategy, window size or optimal parse.  A gzip member's FNAME length
    is still drawn at random: byte-stable gzip output needs compress_batch(..., fname_lens=...), or dfZlib / dfDeflate."""
    if level < -2 or level > 9:
        raise ZippyError(1, "Invalid compression level %d" % level)          # deflate.nim:208-209
    if dataFormat not in (dfGzip, dfZlib, dfDeflate):
        raise ZippyError(2, "Invalid data format dfDetect")                  # zippy.nim:83-84
    fl = None
    if dataFormat == dfGzip and _dict(dictionary) is None:
        fl = [os.urandom(1)[0] % 26]                                         # zippy.nim:28-42
    base, offs = _pack([src])
    out, _ = default_context().compress_batch(base, offs, level, dataFormat, fl, dictionary=dictionary,
                                              strategy=strategy, window_bits=window_bits, optimal=optimal,
                                              rsyncable=rsyncable)
    return out.tobytes()


def compress_with_index(src, level=DefaultCompression, dataFormat=dfGzip, span=1 << 20):
    """compress() that also returns the member's Index (the one Index.build(member, dataFormat, span) gives),
    written while compressing: -> (bytes, Index)."""
    return compress_batch_with_index([src], level, dataFormat, span=span)[0]


def compress_batch_with_index(items, level=DefaultCompression, dataFormat=dfGzip, fname_lens=None, span=1 << 20):
    """compress_batch() that also returns each member's Index: -> list of (bytes, Index)."""
    if fname_lens is None and dataFormat == dfGzip:
        fname_lens = [b % 26 for b in os.urandom(len(items))]                # zippy.nim:28-42
    base, offs = _pack(items)
    out, oo, idx = default_context().compress_batch(base, offs, level, dataFormat, fname_lens, index_span=span)
    return [(out[int(oo[i]):int(oo[i + 1])].tobytes(), idx[i]) for i in range(len(items))]


def uncompress(src, dataFormat=dfDetect, dictionary=None):
    """zippy.uncompress (zippy.nim:100-177).  dictionary: for raw members and zlib members with FDICT."""
    if dataFormat not in (dfDetect, dfZlib, dfGzip, dfDeflate):
        raise ZippyError(2)
    return default_context().decode_one(src, dataFormat, dictionary=dictionary)


def crc32(src):
    return default_context().crc32(src)


def adler32(src):
    return default_context().adler32(src)


def deflate(src, level=DefaultCompression, strategy=StrategyDefault, window_bits=15, optimal=False, rsyncable=False):
    return default_context().deflate(src, level, strategy, window_bits, optimal, rsyncable)


def inflate(src, pos=0):
    return default_context().inflate(src, pos)


def compress_batch(items, level=DefaultCompression, dataFormat=dfGzip, fname_lens=None, dictionary=None,
                   strategy=StrategyDefault, window_bits=15, dictionaries=None, optimal=False, rsyncable=False):
    """list of bytes -> list of bytes (one zippy.compress per item, one GPU launch sequence).  dictionaries: one
    preset dictionary (bytes-like or None) per item, with any window_bits (zb200_compress_batch_dicts).  optimal:
    the optimal parse (zb200_compress_batch_optimal).  rsyncable: content-defined chunk starts
    (zb200_compress_batch_rsyncable)."""
    base, offs = _pack(items)
    out, oo = default_context().compress_batch(base, offs, level, dataFormat, fname_lens, dictionary=dictionary,
                                               strategy=strategy, window_bits=window_bits, dictionaries=dictionaries,
                                               optimal=optimal, rsyncable=rsyncable)
    return [out[int(oo[i]):int(oo[i + 1])].tobytes() for i in range(len(items))]


def rsyncable_chunks(items):
    """list of bytes -> one uint64 array per item: the chunk starts compress(..., rsyncable=True) cuts it at."""
    base, offs = _pack(items)
    return default_context().rsyncable_chunks(base, offs)


def uncompress_batch(items, dataFormat=dfDetect, dictionary=None, dictionaries=None):
    """list of bytes -> list of (bytes | ZippyError).  dictionaries: one preset dictionary (bytes-like or None) per
    item (zb200_uncompress_batch_dicts)."""
    base, offs = _pack(items)
    out, do, lens, st = default_context().uncompress_batch(base, offs, dataFormat, dictionary=dictionary,
                                                           dictionaries=dictionaries)
    res = []
    for i in range(len(items)):
        res.append(ZippyError(int(st[i])) if st[i] != 0 else out[int(do[i]):int(do[i]) + int(lens[i])].tobytes())
    return res


def uncompressed_sizes(items, dataFormat=dfDetect, dictionary=None, dictionaries=None):
    base, offs = _pack(items)
    return default_context().uncompressed_sizes(base, offs, dataFormat, dictionary=dictionary,
                                                dictionaries=dictionaries)


def checksum_batch(items, kind="crc32"):
    base, offs = _pack(items)
    return default_context().checksum_batch(base, offs, kind)
