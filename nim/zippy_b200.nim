## zippy_b200.nim -- drop-in replacement for `import zippy` that routes the codec core
## through libzippy_b200.so (include/zippy_b200.h).  Mirrors src/zippy.nim:11-177 of the
## reference: same procs, defaults and ZippyError behaviour; framing stays here on the host
## for the single-input procs, exactly where zippy.nim has it.
##
## NOT COMPILED in this repository's environment (no Nim toolchain on either box); it is
## the binding a maintainer adds.  The ABI it binds is exercised by tests/ through ctypes.
## Complete for the reference's public surface: compress / uncompress (pointer, string and
## seq[uint8] overloads), uncompressGzip, crc32, adler32, plus the batch forms.

import std/sysrand

type
  ZippyError* = object of CatchableError
  CompressedDataFormat* = enum
    dfDetect, dfZlib, dfGzip, dfDeflate
  Zb200Ctx = pointer

const
  NoCompression* = 0
  BestSpeed* = 1
  BestCompression* = 9
  DefaultCompression* = -1
  HuffmanOnly* = -2
  lib = "libzippy_b200.so"

proc zb200_init(device: cint, ctx: ptr Zb200Ctx): cint {.importc, cdecl, dynlib: lib.}
proc zb200_strerror(status: cint): cstring {.importc, cdecl, dynlib: lib.}
proc zb200_deflate_bound(len: csize_t): csize_t {.importc, cdecl, dynlib: lib.}
proc zb200_deflate(ctx: Zb200Ctx, src: pointer, len: csize_t, level: cint,
                   dst: pointer, dstCap: csize_t, dstLen: ptr csize_t): cint {.importc, cdecl, dynlib: lib.}
proc zb200_inflate_size(ctx: Zb200Ctx, src: pointer, len, pos: csize_t,
                        outLen: ptr csize_t): cint {.importc, cdecl, dynlib: lib.}
proc zb200_inflate(ctx: Zb200Ctx, src: pointer, len, pos: csize_t,
                   dst: pointer, dstCap: csize_t, dstLen: ptr csize_t): cint {.importc, cdecl, dynlib: lib.}
proc zb200_decode_begin(ctx: Zb200Ctx, src: pointer, len: csize_t, dataFormat: cint, pos: csize_t,
                        outLen: ptr csize_t): cint {.importc, cdecl, dynlib: lib.}
proc zb200_decode_finish(ctx: Zb200Ctx, dst: pointer, dstCap: csize_t,
                         dstLen: ptr csize_t): cint {.importc, cdecl, dynlib: lib.}
proc zb200_crc32(ctx: Zb200Ctx, src: pointer, len: csize_t, res: ptr uint32): cint {.importc, cdecl, dynlib: lib.}
proc zb200_adler32(ctx: Zb200Ctx, src: pointer, len: csize_t, res: ptr uint32): cint {.importc, cdecl, dynlib: lib.}

var ctx {.threadvar.}: Zb200Ctx

template check(rc: cint) =
  if rc != 0:
    raise newException(ZippyError, $zb200_strerror(rc))

template failUncompress() =
  raise newException(ZippyError, "Invalid buffer, unable to uncompress")   # internal.nim:191-192

proc read32(s: ptr UncheckedArray[uint8], pos: int): uint32 {.inline.} =
  s[pos].uint32 or (s[pos + 1].uint32 shl 8) or (s[pos + 2].uint32 shl 16) or (s[pos + 3].uint32 shl 24)

proc getCtx(): Zb200Ctx =
  if ctx == nil:
    check zb200_init(-1, ctx.addr)
  ctx

proc crc32*(src: pointer, len: int): uint32 =          # crc.nim:53
  check zb200_crc32(getCtx(), src, len.csize_t, result.addr)
proc crc32*(src: string): uint32 = crc32(src.cstring, src.len)
proc adler32*(src: pointer, len: int): uint32 =        # adler32.nim:6
  check zb200_adler32(getCtx(), src, len.csize_t, result.addr)
proc adler32*(src: string): uint32 = adler32(src.cstring, src.len)

proc deflate(dst: var string, src: pointer, len, level: int) =   # deflate.nim:207 (appends)
  let start = dst.len
  dst.setLen(start + zb200_deflate_bound(len.csize_t).int)
  var n: csize_t
  check zb200_deflate(getCtx(), src, len.csize_t, level.cint, dst[start].addr,
                      (dst.len - start).csize_t, n.addr)
  dst.setLen(start + n.int)

proc inflate(dst: var string, src: pointer, len, pos: int) =     # inflate.nim:268
  ## one decode: the library inflates into its own device memory and reports the size
  ## (zb200_decode_begin), then copies the bytes into the string (zb200_decode_finish)
  var n: csize_t
  check zb200_decode_begin(getCtx(), src, len.csize_t, dfDeflate.cint, pos.csize_t, n.addr)
  dst.setLen(n.int)
  var dummy: char
  check zb200_decode_finish(getCtx(), (if n > 0: dst[0].addr else: dummy.addr), n, n.addr)

proc compress*(src: pointer, len: int, level = DefaultCompression,
               dataFormat = dfGzip): string {.raises: [ZippyError].} =
  ## zippy.nim:11-84, framing unchanged
  case dataFormat
  of dfGzip:
    result.setLen(10)
    result[0] = 31.char; result[1] = 139.char; result[2] = 8.char; result[3] = (1 shl 3).char
    var urand: array[1, uint8]
    if not urandom(urand):
      raise newException(ZippyError, "Failed to generate random number")
    for i in 0 ..< (urand[0] mod 26).int: result.add (97 + i).char
    result.add '\0'
    deflate(result, src, len, level)
    let checksum = crc32(src, len)
    for s in [0, 8, 16, 24]: result.add(((checksum shr s) and 255).char)
    for s in [0, 8, 16, 24]: result.add(((len shr s) and 255).char)
  of dfZlib:
    result.setLen(2)
    result[0] = 0x78.char; result[1] = 0x01.char
    deflate(result, src, len, level)
    let checksum = adler32(src, len)
    for s in [24, 16, 8, 0]: result.add(((checksum shr s) and 255).char)
  of dfDeflate:
    deflate(result, src, len, level)
  else:
    raise newException(ZippyError, "Invalid data format " & $dfDetect)

proc compress*(src: string, level = DefaultCompression, dataFormat = dfGzip): string =
  compress(src.cstring, src.len, level, dataFormat)

proc compress*(src: seq[uint8], level = DefaultCompression,
               dataFormat = dfGzip): seq[uint8] {.inline, raises: [ZippyError].} =
  ## zippy.nim:93-98: the seq overload shares the string's buffer
  cast[seq[uint8]](compress(cast[string](src), level, dataFormat))

proc uncompressGzip*(dst: var string, src: pointer, len: int, trustSize = false) {.raises: [ZippyError].} =
  ## gzip.nim:3-88: header checks, inflate, then CRC-32 and ISIZE from the LAST 8 bytes of the buffer
  ## (`trustSize` only pre-sizes `dst` in the reference, gzip.nim:72-76; here the library sizes it).
  if len < 18: failUncompress()
  let src = cast[ptr UncheckedArray[uint8]](src)
  let
    id1 = src[0]; id2 = src[1]; cm = src[2]; flg = src[3]
  if id1 != 31 or id2 != 139:
    raise newException(ZippyError, "Failed gzip identification values check")
  if cm != 8: raise newException(ZippyError, "Unsupported compression method")
  if (flg and 0b11100000) > 0.uint8: raise newException(ZippyError, "Reserved flag bits set")
  let
    fhcrc = (flg and (1.uint8 shl 1)) != 0
    fextra = (flg and (1.uint8 shl 2)) != 0
    fname = (flg and (1.uint8 shl 3)) != 0
    fcomment = (flg and (1.uint8 shl 4)) != 0
  var pos = 10
  if fextra: raise newException(ZippyError, "Currently unsupported flags are set")
  proc nextZeroByte(src: ptr UncheckedArray[uint8], len, start: int): int =
    for i in start ..< len:
      if src[i] == 0: return i
    failUncompress()
  if fname: pos = nextZeroByte(src, len, pos) + 1
  if fcomment: pos = nextZeroByte(src, len, pos) + 1
  if fhcrc:
    if pos + 2 >= len: failUncompress()
    pos += 2                               # not verified (gzip.nim:55-59)
  if pos + 8 >= len: failUncompress()
  let
    checksum = read32(src, len - 8)
    isize = read32(src, len - 4)
  inflate(dst, src, len, pos)
  if checksum != crc32(dst): raise newException(ZippyError, "Checksum verification failed")
  if isize != (dst.len mod (1 shl 32)).uint32: raise newException(ZippyError, "Size verification failed")

proc uncompress*(src: pointer, len: int, dataFormat = dfDetect): string {.raises: [ZippyError].} =
  ## zippy.nim:100-165, framing unchanged: detect, header checks, inflate, trailer verification
  let src = cast[ptr UncheckedArray[uint8]](src)
  case dataFormat
  of dfDetect:
    if len > 18 and src[0] == 31 and src[1] == 139 and src[2] == 8 and (src[3] and 0b11100000) == 0:
      return uncompress(src, len, dfGzip)
    if len > 6 and (src[0] and 0b00001111) == 8 and (src[0] shr 4) <= 7 and
        ((src[0].uint16 * 256) + src[1].uint16) mod 31 == 0:
      return uncompress(src, len, dfZlib)
    raise newException(ZippyError, "Unable to detect compressed data format")
  of dfGzip:
    uncompressGzip(result, src, len)
  of dfZlib:
    if len < 6: failUncompress()
    let
      cmf = src[0]; flg = src[1]
      cm = cmf and 0b00001111
      cinfo = cmf shr 4
    if cm != 8: raise newException(ZippyError, "Unsupported compression method")
    if cinfo > 7.uint8: raise newException(ZippyError, "Invalid compression info")
    if ((cmf.uint16 * 256) + flg.uint16) mod 31 != 0: raise newException(ZippyError, "Invalid header")
    if (flg and 0b00100000) != 0: raise newException(ZippyError, "Preset dictionary is not yet supported")
    inflate(result, src, len, 2)
    let checksum = (src[len - 4].uint32 shl 24) or (src[len - 3].uint32 shl 16) or
                   (src[len - 2].uint32 shl 8) or src[len - 1].uint32
    if checksum != adler32(result): raise newException(ZippyError, "Checksum verification failed")
  of dfDeflate:
    inflate(result, src, len, 0)

proc uncompress*(src: string, dataFormat = dfDetect): string {.inline, raises: [ZippyError].} =
  uncompress(src.cstring, src.len, dataFormat)          # zippy.nim:167-171

proc uncompress*(src: seq[uint8], dataFormat = dfDetect): seq[uint8] {.inline, raises: [ZippyError].} =
  cast[seq[uint8]](uncompress(cast[string](src), dataFormat))   # zippy.nim:173-177

# ---- preset dictionaries (zlib's zdict; include/zippy_b200.h "preset dictionaries"): zlib members start 78 20 and
# the DICTID (the Adler-32 of the whole dictionary), raw members carry nothing, gzip is refused; an empty
# dictionary is the call without one ----
proc zb200_compress_batch_dict(ctx: Zb200Ctx, srcBase: pointer, srcOffsets: ptr uint64, n: csize_t,
                               level, dataFormat: cint, dict: pointer, dictLen: csize_t, dstBase: pointer,
                               dstCap: csize_t, dstOffsets: ptr uint64, statuses: ptr cint): cint {.importc, cdecl, dynlib: lib.}
proc zb200_decode_begin_dict(ctx: Zb200Ctx, src: pointer, len: csize_t, dataFormat: cint, dict: pointer,
                             dictLen: csize_t, outLen: ptr csize_t): cint {.importc, cdecl, dynlib: lib.}

proc deflateDict(dst: var string, src: pointer, len, level: int, dictionary: string) =
  ## appends the raw stream of src against the dictionary (zb200_compress_batch_dict on one input)
  var offs = [0'u64, len.uint64]
  var outOffs = [0'u64, 0'u64]
  var st: cint
  var dummy: char
  let start = dst.len
  dst.setLen(start + zb200_deflate_bound(len.csize_t).int + 64)
  check zb200_compress_batch_dict(getCtx(), (if len > 0: src else: dummy.addr), offs[0].addr, 1, level.cint,
                                  dfDeflate.cint, dictionary.cstring, dictionary.len.csize_t, dst[start].addr,
                                  (dst.len - start).csize_t, outOffs[0].addr, st.addr)
  dst.setLen(start + outOffs[1].int)

proc inflateDict(dst: var string, src: pointer, len: int, dictionary: string) =
  ## a raw stream decoded against the dictionary (zb200_decode_begin_dict, then zb200_decode_finish)
  var n: csize_t
  var dummy: char
  check zb200_decode_begin_dict(getCtx(), (if len > 0: src else: dummy.addr), len.csize_t, dfDeflate.cint,
                                dictionary.cstring, dictionary.len.csize_t, n.addr)
  dst.setLen(n.int)
  check zb200_decode_finish(getCtx(), (if n > 0: dst[0].addr else: dummy.addr), n, n.addr)

proc compress*(src: pointer, len: int, level: int, dataFormat: CompressedDataFormat,
               dictionary: string): string {.raises: [ZippyError].} =
  if dictionary.len == 0: return compress(src, len, level, dataFormat)
  if level < -2 or level > 9: raise newException(ZippyError, "Invalid compression level")
  if dataFormat notin {dfZlib, dfDeflate}: raise newException(ZippyError, "Invalid data format")
  if dataFormat == dfZlib:
    result.setLen(2)
    result[0] = 0x78.char; result[1] = 0x20.char
    let id = adler32(dictionary)
    for s in [24, 16, 8, 0]: result.add(((id shr s) and 255).char)
  deflateDict(result, src, len, level, dictionary)
  if dataFormat == dfZlib:
    let checksum = adler32(src, len)
    for s in [24, 16, 8, 0]: result.add(((checksum shr s) and 255).char)

proc compress*(src: string, level: int, dataFormat: CompressedDataFormat, dictionary: string): string =
  compress(src.cstring, src.len, level, dataFormat, dictionary)

proc uncompress*(src: pointer, len: int, dataFormat: CompressedDataFormat,
                 dictionary: string): string {.raises: [ZippyError].} =
  ## raw members, and zlib members with FDICT, decode against the dictionary; gzip members and zlib members
  ## without FDICT ignore it
  if dictionary.len == 0: return uncompress(src, len, dataFormat)
  let s = cast[ptr UncheckedArray[uint8]](src)
  case dataFormat
  of dfDetect:
    if len > 18 and s[0] == 31 and s[1] == 139 and s[2] == 8 and (s[3] and 0b11100000) == 0:
      return uncompress(src, len, dfGzip)
    if len > 6 and (s[0] and 0b00001111) == 8 and (s[0] shr 4) <= 7 and
        ((s[0].uint16 * 256) + s[1].uint16) mod 31 == 0:
      return uncompress(src, len, dfZlib, dictionary)
    raise newException(ZippyError, "Unable to detect compressed data format")
  of dfGzip:
    return uncompress(src, len, dfGzip)
  of dfZlib:
    if len < 6 or (s[1] and 0b00100000) == 0: return uncompress(src, len, dfZlib)
    let cmf = s[0]; let flg = s[1]
    if (cmf and 0b00001111) != 8: raise newException(ZippyError, "Unsupported compression method")
    if (cmf shr 4) > 7.uint8: raise newException(ZippyError, "Invalid compression info")
    if ((cmf.uint16 * 256) + flg.uint16) mod 31 != 0: raise newException(ZippyError, "Invalid header")
    if len < 10: failUncompress()
    let id = (s[2].uint32 shl 24) or (s[3].uint32 shl 16) or (s[4].uint32 shl 8) or s[5].uint32
    if id != adler32(dictionary): raise newException(ZippyError, $zb200_strerror(23))
    inflateDict(result, s[6].addr, len - 6, dictionary)
    let checksum = (s[len - 4].uint32 shl 24) or (s[len - 3].uint32 shl 16) or
                   (s[len - 2].uint32 shl 8) or s[len - 1].uint32
    if checksum != adler32(result): raise newException(ZippyError, "Checksum verification failed")
  of dfDeflate:
    inflateDict(result, src, len, dictionary)

proc uncompress*(src: string, dataFormat: CompressedDataFormat, dictionary: string): string {.raises: [ZippyError].} =
  uncompress(src.cstring, src.len, dataFormat, dictionary)

# ---- batch (no counterpart in zippy.nim; what ziparchives.nim:505-540 should call instead of a
# per-entry loop of crc32 + compress): N independent inputs, one GPU launch sequence ----
proc zb200_compress_bound(len: csize_t, dataFormat: cint): csize_t {.importc, cdecl, dynlib: lib.}
proc zb200_compress_batch(ctx: Zb200Ctx, srcBase: pointer, srcOffsets: ptr uint64, n: csize_t,
                          level, dataFormat: cint, fnameLens: pointer,
                          dstBase: pointer, dstCap: csize_t, dstOffsets: ptr uint64,
                          statuses: ptr cint): cint {.importc, cdecl, dynlib: lib.}

proc compressBatch*(items: openArray[string], level = DefaultCompression,
                    dataFormat = dfGzip): seq[string] {.raises: [ZippyError].} =
  var
    base: string
    offs = newSeq[uint64](items.len + 1)
    outOffs = newSeq[uint64](items.len + 1)
    bound = 64
  for i, item in items:
    base.add item
    offs[i + 1] = base.len.uint64
    bound += zb200_compress_bound(item.len.csize_t, dataFormat.cint).int + 64
  var dst = newString(bound)
  if base.len == 0: base.add '\0'
  check zb200_compress_batch(getCtx(), base[0].addr, offs[0].addr, items.len.csize_t,
                             level.cint, dataFormat.cint, nil, dst[0].addr, dst.len.csize_t,
                             outOffs[0].addr, nil)
  for i in 0 ..< items.len:
    result.add dst[outOffs[i].int ..< outOffs[i + 1].int]

# ---- per-member preset dictionaries (include/zippy_b200.h): item i against dicts[dictOf[i]], -1 for none ----
proc zb200_compress_batch_dicts(ctx: Zb200Ctx, srcBase: pointer, srcOffsets: ptr uint64, n: csize_t,
                                level, dataFormat, windowBits: cint, dictBase: pointer, dictOffsets: ptr uint64,
                                k: csize_t, dictOf: ptr int32, dstBase: pointer, dstCap: csize_t,
                                dstOffsets: ptr uint64, statuses: ptr cint): cint {.importc, cdecl, dynlib: lib.}
proc zb200_uncompress_sizes_dicts(ctx: Zb200Ctx, srcBase: pointer, srcOffsets: ptr uint64, n: csize_t,
                                  dataFormat: cint, dictBase: pointer, dictOffsets: ptr uint64, k: csize_t,
                                  dictOf: ptr int32, sizes: ptr uint64, statuses: ptr cint): cint {.importc, cdecl, dynlib: lib.}
proc zb200_uncompress_batch_dicts(ctx: Zb200Ctx, srcBase: pointer, srcOffsets: ptr uint64, n: csize_t,
                                  dataFormat: cint, dictBase: pointer, dictOffsets: ptr uint64, k: csize_t,
                                  dictOf: ptr int32, dstBase: pointer, dstOffsets: ptr uint64, dstLens: ptr uint64,
                                  statuses: ptr cint): cint {.importc, cdecl, dynlib: lib.}

proc packBatch(items: openArray[string], base: var string, offs: var seq[uint64]) =
  offs = newSeq[uint64](items.len + 1)
  for i, item in items:
    base.add item
    offs[i + 1] = base.len.uint64
  if base.len == 0: base.add '\0'

proc compressBatch*(items: openArray[string], level: int, dataFormat: CompressedDataFormat, windowBits: int,
                    dicts: openArray[string], dictOf: openArray[int32]): seq[string] {.raises: [ZippyError].} =
  if dictOf.len != items.len: raise newException(ZippyError, "dictOf needs one entry per item")
  var
    base, dbase: string
    offs, doffs: seq[uint64]
    outOffs = newSeq[uint64](items.len + 1)
    dof = @dictOf
    bound = 64
  packBatch(items, base, offs)
  packBatch(dicts, dbase, doffs)
  for item in items:
    bound += zb200_compress_bound(item.len.csize_t, dataFormat.cint).int + 4 + 64
  if dof.len == 0: dof.add -1
  var dst = newString(bound)
  check zb200_compress_batch_dicts(getCtx(), base[0].addr, offs[0].addr, items.len.csize_t, level.cint,
                                   dataFormat.cint, windowBits.cint, dbase[0].addr, doffs[0].addr,
                                   dicts.len.csize_t, dof[0].addr, dst[0].addr, dst.len.csize_t, outOffs[0].addr, nil)
  for i in 0 ..< items.len:
    result.add dst[outOffs[i].int ..< outOffs[i + 1].int]

proc uncompressBatch*(members: openArray[string], dataFormat: CompressedDataFormat, dicts: openArray[string],
                      dictOf: openArray[int32]): seq[string] {.raises: [ZippyError].} =
  ## a member that does not decode raises its status
  if dictOf.len != members.len: raise newException(ZippyError, "dictOf needs one entry per member")
  var
    base, dbase: string
    offs, doffs: seq[uint64]
    dof = @dictOf
    sizes = newSeq[uint64](members.len + 1)
    dofs = newSeq[uint64](members.len + 1)
    lens = newSeq[uint64](members.len + 1)
    st = newSeq[cint](members.len + 1)
  packBatch(members, base, offs)
  packBatch(dicts, dbase, doffs)
  if dof.len == 0: dof.add -1
  check zb200_uncompress_sizes_dicts(getCtx(), base[0].addr, offs[0].addr, members.len.csize_t, dataFormat.cint,
                                     dbase[0].addr, doffs[0].addr, dicts.len.csize_t, dof[0].addr, sizes[0].addr,
                                     st[0].addr)
  for i in 0 ..< members.len:
    check st[i]
    dofs[i + 1] = dofs[i] + sizes[i]
  var dst = newString(dofs[members.len].int + 64)
  check zb200_uncompress_batch_dicts(getCtx(), base[0].addr, offs[0].addr, members.len.csize_t, dataFormat.cint,
                                     dbase[0].addr, doffs[0].addr, dicts.len.csize_t, dof[0].addr, dst[0].addr,
                                     dofs[0].addr, lens[0].addr, st[0].addr)
  for i in 0 ..< members.len:
    check st[i]
    result.add dst[dofs[i].int ..< (dofs[i] + lens[i]).int]

proc zb200_inflate_batch_crc32(ctx: Zb200Ctx, srcBase: pointer, srcOffsets: ptr uint64, n: csize_t,
                               dstBase: pointer, dstOffsets: ptr uint64, dstLens: ptr uint64,
                               crcs: ptr uint32, statuses: ptr cint): cint {.importc, cdecl, dynlib: lib.}

proc inflateBatchCrc32*(items: openArray[string], sizes: openArray[int]): seq[(string, uint32)] {.raises: [ZippyError].} =
  ## raw deflate members (a ZIP archive's entries) into slots of `sizes` bytes (its directory's uncompressed sizes)
  ## -> every output with its CRC-32, computed on the device in the decode call (what ziparchives_v1.nim:202-212
  ## does per entry with uncompress + crc32).  A member whose output does not fit its slot raises.
  var
    base: string
    offs = newSeq[uint64](items.len + 1)
    dofs = newSeq[uint64](items.len + 1)
    lens = newSeq[uint64](max(items.len, 1))
    crcs = newSeq[uint32](max(items.len, 1))
    st = newSeq[cint](max(items.len, 1))
  for i, item in items:
    base.add item
    offs[i + 1] = base.len.uint64
    dofs[i + 1] = dofs[i] + sizes[i].uint64
  var dst = newString(dofs[items.len].int + 64)
  if base.len == 0: base.add '\0'
  check zb200_inflate_batch_crc32(getCtx(), base[0].addr, offs[0].addr, items.len.csize_t, dst[0].addr,
                                  dofs[0].addr, lens[0].addr, crcs[0].addr, st[0].addr)
  for i in 0 ..< items.len:
    check st[i]
    result.add (dst[dofs[i].int ..< (dofs[i] + lens[i]).int], crcs[i])

# ---- streaming compression (no counterpart in zippy.nim): one member from input that arrives piece by
# piece; what write and finish return, concatenated, is compressBatch(@[whole input]) with the same FNAME ----
type Zb200CompressStream = pointer
proc zb200_compress_stream_begin(ctx: Zb200Ctx, level, dataFormat, fnameLen: cint,
                                 st: ptr Zb200CompressStream): cint {.importc, cdecl, dynlib: lib.}
proc zb200_compress_stream_bound(st: Zb200CompressStream, len: csize_t): csize_t {.importc, cdecl, dynlib: lib.}
proc zb200_compress_stream_write(st: Zb200CompressStream, src: pointer, len: csize_t, dst: pointer, dstCap: csize_t,
                                 dstLen: ptr csize_t): cint {.importc, cdecl, dynlib: lib.}
proc zb200_compress_stream_flush(st: Zb200CompressStream, mode: cint, dst: pointer, dstCap: csize_t,
                                 dstLen: ptr csize_t): cint {.importc, cdecl, dynlib: lib.}
proc zb200_compress_stream_finish(st: Zb200CompressStream, dst: pointer, dstCap: csize_t,
                                  dstLen: ptr csize_t): cint {.importc, cdecl, dynlib: lib.}
proc zb200_compress_stream_free(st: Zb200CompressStream) {.importc, cdecl, dynlib: lib.}

const
  SyncFlush* = 2   ## zlib's Z_SYNC_FLUSH: emit everything written, keep the history
  FullFlush* = 3   ## zlib's Z_FULL_FLUSH: emit everything written, drop the history

type CompressStream* = object
  st: Zb200CompressStream

proc newCompressStream*(level = DefaultCompression, dataFormat = dfGzip,
                        fnameLen = -1): CompressStream {.raises: [ZippyError].} =
  ## fnameLen < 0 with dfGzip draws the FNAME length at random, as compress does (zippy.nim:28-42)
  var k = fnameLen
  if k < 0:
    k = 0
    if dataFormat == dfGzip:
      var urand: array[1, uint8]
      if not urandom(urand):
        raise newException(ZippyError, "Failed to generate random number")
      k = (urand[0] mod 26).int
  check zb200_compress_stream_begin(getCtx(), level.cint, dataFormat.cint, k.cint, result.st.addr)

proc zb200_compress_stream_begin_dict(ctx: Zb200Ctx, level, dataFormat: cint, dict: pointer, dictLen: csize_t,
                                      st: ptr Zb200CompressStream): cint {.importc, cdecl, dynlib: lib.}

proc newCompressStream*(level: int, dataFormat: CompressedDataFormat,
                        dictionary: string): CompressStream {.raises: [ZippyError].} =
  ## with a preset dictionary (zlib / raw; no FNAME): zb200_compress_stream_begin_dict
  check zb200_compress_stream_begin_dict(getCtx(), level.cint, dataFormat.cint, dictionary.cstring,
                                         dictionary.len.csize_t, result.st.addr)

proc write*(s: var CompressStream, data: string): string {.raises: [ZippyError].} =
  ## small writes are gathered on the host and return ""
  result = newString(zb200_compress_stream_bound(s.st, data.len.csize_t).int + 1)
  var n: csize_t
  check zb200_compress_stream_write(s.st, data.cstring, data.len.csize_t, result[0].addr, result.len.csize_t, n.addr)
  result.setLen(n.int)

proc flush*(s: var CompressStream, mode = SyncFlush): string {.raises: [ZippyError].} =
  ## everything written so far; "" when nothing was written since the last flush
  result = newString(zb200_compress_stream_bound(s.st, 0).int + 1)
  var n: csize_t
  check zb200_compress_stream_flush(s.st, mode.cint, result[0].addr, result.len.csize_t, n.addr)
  result.setLen(n.int)

proc finish*(s: var CompressStream): string {.raises: [ZippyError].} =
  result = newString(zb200_compress_stream_bound(s.st, 0).int + 1)
  var n: csize_t
  check zb200_compress_stream_finish(s.st, result[0].addr, result.len.csize_t, n.addr)
  result.setLen(n.int)

proc close*(s: var CompressStream) =
  if s.st != nil:
    zb200_compress_stream_free(s.st)
    s.st = nil

# ---- streaming decompression (no counterpart in zippy.nim): one member from compressed input that arrives piece
# by piece; what write and finish return, concatenated, is uncompress(whole input, dataFormat), and a bad input
# raises uncompress's ZippyError message (strerror of the same status) ----
type Zb200DecompressStream = pointer
proc zb200_decompress_stream_begin(ctx: Zb200Ctx, dataFormat: cint,
                                   st: ptr Zb200DecompressStream): cint {.importc, cdecl, dynlib: lib.}
proc zb200_decompress_stream_write(st: Zb200DecompressStream, src: pointer, len: csize_t,
                                   avail: ptr csize_t): cint {.importc, cdecl, dynlib: lib.}
proc zb200_decompress_stream_drain(st: Zb200DecompressStream, avail: ptr csize_t): cint {.importc, cdecl, dynlib: lib.}
proc zb200_decompress_stream_finish(st: Zb200DecompressStream, avail: ptr csize_t): cint {.importc, cdecl, dynlib: lib.}
proc zb200_decompress_stream_read(st: Zb200DecompressStream, dst: pointer, dstCap: csize_t,
                                  dstLen: ptr csize_t): cint {.importc, cdecl, dynlib: lib.}
proc zb200_decompress_stream_free(st: Zb200DecompressStream) {.importc, cdecl, dynlib: lib.}

type DecompressStream* = object
  st: Zb200DecompressStream

proc newDecompressStream*(dataFormat = dfDetect): DecompressStream {.raises: [ZippyError].} =
  check zb200_decompress_stream_begin(getCtx(), dataFormat.cint, result.st.addr)

proc zb200_decompress_stream_begin_dict(ctx: Zb200Ctx, dataFormat: cint, dict: pointer, dictLen: csize_t,
                                        st: ptr Zb200DecompressStream): cint {.importc, cdecl, dynlib: lib.}

proc newDecompressStream*(dataFormat: CompressedDataFormat, dictionary: string): DecompressStream {.raises: [ZippyError].} =
  ## with a preset dictionary: zb200_decompress_stream_begin_dict
  check zb200_decompress_stream_begin_dict(getCtx(), dataFormat.cint, dictionary.cstring, dictionary.len.csize_t,
                                           result.st.addr)

proc take(s: var DecompressStream, avail: csize_t): string {.raises: [ZippyError].} =
  result = newString(avail.int + 1)
  var n: csize_t
  check zb200_decompress_stream_read(s.st, result[0].addr, avail, n.addr)
  result.setLen(n.int)

proc write*(s: var DecompressStream, data: string): string {.raises: [ZippyError].} =
  ## small writes are gathered on the host and return ""
  var avail: csize_t
  check zb200_decompress_stream_write(s.st, data.cstring, data.len.csize_t, avail.addr)
  s.take(avail)

proc drain*(s: var DecompressStream): string {.raises: [ZippyError].} =
  ## every block complete in the input so far: after a sender's flush, everything written up to it
  var avail: csize_t
  check zb200_decompress_stream_drain(s.st, avail.addr)
  s.take(avail)

proc finish*(s: var DecompressStream): string {.raises: [ZippyError].} =
  var avail: csize_t
  check zb200_decompress_stream_finish(s.st, avail.addr)
  s.take(avail)

proc close*(s: var DecompressStream) =
  if s.st != nil:
    zb200_decompress_stream_free(s.st)
    s.st = nil

# ---- random access into one member (zb200_index_*): build once, then read ranges of its output ----
type
  Zb200Index = pointer
  Index* = object
    idx: Zb200Index
  IndexPoint* = object
    bit*, output*: uint64
    crc*: uint32
    window*: bool

proc zb200_index_build(ctx: Zb200Ctx, src: pointer, len: csize_t, dataFormat: cint, span: uint64,
                       res: ptr Zb200Index): cint {.importc, cdecl, dynlib: lib.}
proc zb200_index_extract_batch(ctx: Zb200Ctx, idx: Zb200Index, src: pointer, len: csize_t, offsets, lens: ptr uint64,
                               n: csize_t, dst: pointer, dstOffsets: ptr uint64,
                               statuses: ptr cint): cint {.importc, cdecl, dynlib: lib.}
proc zb200_index_size(idx: Zb200Index): uint64 {.importc, cdecl, dynlib: lib.}
proc zb200_index_points(idx: Zb200Index, bits, outs: ptr uint64, crcs: ptr uint32, window: ptr uint8,
                        cap: csize_t): csize_t {.importc, cdecl, dynlib: lib.}
proc zb200_index_export(ctx: Zb200Ctx, idx: Zb200Index, dst: pointer, cap: csize_t,
                        len: ptr csize_t): cint {.importc, cdecl, dynlib: lib.}
proc zb200_index_import(ctx: Zb200Ctx, src: pointer, len: csize_t, res: ptr Zb200Index): cint {.importc, cdecl, dynlib: lib.}
proc zb200_index_free(idx: Zb200Index) {.importc, cdecl, dynlib: lib.}

proc buildIndex*(data: string, dataFormat = dfDetect, span = 1'u64 shl 20): Index {.raises: [ZippyError].} =
  check zb200_index_build(getCtx(), data.cstring, data.len.csize_t, dataFormat.cint, span, result.idx.addr)

proc indexFromBytes*(buf: string): Index {.raises: [ZippyError].} =
  check zb200_index_import(getCtx(), buf.cstring, buf.len.csize_t, result.idx.addr)

proc size*(ix: Index): uint64 = zb200_index_size(ix.idx)

proc points*(ix: Index): seq[IndexPoint] =
  let n = zb200_index_points(ix.idx, nil, nil, nil, nil, 0).int
  var bits, outs = newSeq[uint64](n + 1)
  var crcs = newSeq[uint32](n + 1)
  var win = newSeq[uint8](n + 1)
  discard zb200_index_points(ix.idx, bits[0].addr, outs[0].addr, crcs[0].addr, win[0].addr, n.csize_t)
  for i in 0 ..< n:
    result.add IndexPoint(bit: bits[i], output: outs[i], crc: crcs[i], window: win[i] != 0)

proc extractBatch*(ix: Index, data: string, offsets, lengths: seq[uint64],
                   statuses: var seq[cint]): seq[string] {.raises: [ZippyError].} =
  ## range i is [offsets[i], offsets[i] + lengths[i]); result[i] holds it where statuses[i] == 0
  if offsets.len != lengths.len: check 22
  let n = offsets.len
  var doff = newSeq[uint64](n + 1)
  for i in 0 ..< n: doff[i + 1] = doff[i] + lengths[i]
  var buf = newString(doff[n].int + 1)
  statuses = newSeq[cint](n + 1)
  var o = offsets & @[0'u64]
  var l = lengths & @[0'u64]
  check zb200_index_extract_batch(getCtx(), ix.idx, data.cstring, data.len.csize_t, o[0].addr, l[0].addr, n.csize_t,
                                  buf[0].addr, doff[0].addr, statuses[0].addr)
  statuses.setLen(n)
  for i in 0 ..< n:
    result.add(if statuses[i] == 0: buf[doff[i].int ..< doff[i + 1].int] else: "")

proc extract*(ix: Index, data: string, offset, length: uint64): string {.raises: [ZippyError].} =
  var st: seq[cint]
  let r = ix.extractBatch(data, @[offset], @[length], st)
  check st[0]
  r[0]

proc toBytes*(ix: Index): string {.raises: [ZippyError].} =
  var n: csize_t
  check zb200_index_export(getCtx(), ix.idx, nil, 0, n.addr)
  result = newString(n.int + 1)
  check zb200_index_export(getCtx(), ix.idx, result[0].addr, n + 1, n.addr)
  result.setLen(n.int)

proc close*(ix: var Index) =
  if ix.idx != nil:
    zb200_index_free(ix.idx)
    ix.idx = nil

# ---- an index written while compressing (zb200_compress_batch_index, zb200_compress_stream_begin_index): the
# index buildIndex(member, dataFormat, span) gives, without a decode pass ----
proc zb200_compress_batch_index(ctx: Zb200Ctx, srcBase: pointer, srcOffsets: ptr uint64, n: csize_t,
                                level, dataFormat: cint, fnameLens: pointer, dstBase: pointer, dstCap: csize_t,
                                dstOffsets: ptr uint64, statuses: ptr cint, span: uint64,
                                indexes: ptr Zb200Index): cint {.importc, cdecl, dynlib: lib.}
proc zb200_compress_stream_begin_index(ctx: Zb200Ctx, level, dataFormat, fnameLen: cint, span: uint64,
                                       st: ptr Zb200CompressStream): cint {.importc, cdecl, dynlib: lib.}
proc zb200_compress_stream_index(st: Zb200CompressStream, res: ptr Zb200Index): cint {.importc, cdecl, dynlib: lib.}

proc randomFnameLen(dataFormat: CompressedDataFormat): int {.raises: [ZippyError].} =
  if dataFormat != dfGzip: return 0
  var urand: array[1, uint8]
  if not urandom(urand):
    raise newException(ZippyError, "Failed to generate random number")
  (urand[0] mod 26).int

proc compressWithIndex*(src: string, level = DefaultCompression, dataFormat = dfGzip,
                        span = 1'u64 shl 20): (string, Index) {.raises: [ZippyError].} =
  ## compress that also returns the member's index
  let fl = [randomFnameLen(dataFormat).uint8]
  var offs = [0'u64, src.len.uint64]
  var dofs: array[2, uint64]
  var st: cint
  var dst = newString(zb200_compress_bound(src.len.csize_t, dataFormat.cint).int + 64)
  check zb200_compress_batch_index(getCtx(), src.cstring, offs[0].addr, 1, level.cint, dataFormat.cint, fl[0].unsafeAddr,
                                   dst[0].addr, dst.len.csize_t, dofs[0].addr, st.addr, span, result[1].idx.addr)
  dst.setLen(dofs[1].int)
  result[0] = dst

proc newCompressStream*(level: int, dataFormat: CompressedDataFormat, fnameLen: int,
                        span: uint64): CompressStream {.raises: [ZippyError].} =
  ## a stream that also writes the member's index: index() after finish
  let k = if fnameLen < 0: randomFnameLen(dataFormat) else: fnameLen
  check zb200_compress_stream_begin_index(getCtx(), level.cint, dataFormat.cint, k.cint, span, result.st.addr)

proc index*(s: CompressStream): Index {.raises: [ZippyError].} =
  check zb200_compress_stream_index(s.st, result.idx.addr)

# ---- compression strategies (zlib's `strategy`, with zlib's values; include/zippy_b200.h "compression
# strategies"): a strategy changes the compressed size, never what a member decodes to ----
type Strategy* = enum
  StrategyDefault = 0, StrategyFiltered = 1, StrategyHuffmanOnly = 2, StrategyRle = 3, StrategyFixed = 4

proc zb200_compress_batch_strategy(ctx: Zb200Ctx, srcBase: pointer, srcOffsets: ptr uint64, n: csize_t,
                                   level, strategy, dataFormat: cint, fnameLens: pointer, dstBase: pointer,
                                   dstCap: csize_t, dstOffsets: ptr uint64,
                                   statuses: ptr cint): cint {.importc, cdecl, dynlib: lib.}
proc zb200_compress_stream_begin_strategy(ctx: Zb200Ctx, level, strategy, dataFormat, fnameLen: cint,
                                          st: ptr Zb200CompressStream): cint {.importc, cdecl, dynlib: lib.}

proc compress*(src: string, level: int, dataFormat: CompressedDataFormat,
               strategy: Strategy): string {.raises: [ZippyError].} =
  ## one member of zb200_compress_batch_strategy; gzip draws its FNAME length at random, as compress does
  var
    offs = [0'u64, src.len.uint64]
    outOffs = [0'u64, 0'u64]
    fl = randomFnameLen(dataFormat).uint8
    dummy: uint8
  result = newString(zb200_compress_bound(src.len.csize_t, dataFormat.cint).int + 64)
  check zb200_compress_batch_strategy(getCtx(), (if src.len > 0: src[0].unsafeAddr else: dummy.addr),
                                      offs[0].addr, 1, level.cint, strategy.cint, dataFormat.cint, fl.addr,
                                      result[0].addr, result.len.csize_t, outOffs[0].addr, nil)
  result.setLen(outOffs[1].int)

proc newCompressStream*(level: int, dataFormat: CompressedDataFormat, strategy: Strategy,
                        fnameLen = -1): CompressStream {.raises: [ZippyError].} =
  ## a stream under a compression strategy: zb200_compress_stream_begin_strategy
  let k = if fnameLen < 0: randomFnameLen(dataFormat) else: fnameLen
  check zb200_compress_stream_begin_strategy(getCtx(), level.cint, strategy.cint, dataFormat.cint, k.cint,
                                             result.st.addr)

# ---- window size (zlib's `windowBits`, 9..15; 8 for dfZlib means 9; include/zippy_b200.h "window size"): no
# match reaches more than 2^windowBits back; not combined with dictionaries or compress-time indexes ----
proc zb200_compress_batch_window(ctx: Zb200Ctx, srcBase: pointer, srcOffsets: ptr uint64, n: csize_t,
                                 level, strategy, windowBits, dataFormat: cint, fnameLens: pointer, dstBase: pointer,
                                 dstCap: csize_t, dstOffsets: ptr uint64,
                                 statuses: ptr cint): cint {.importc, cdecl, dynlib: lib.}
proc zb200_compress_stream_begin_window(ctx: Zb200Ctx, level, strategy, windowBits, dataFormat, fnameLen: cint,
                                        st: ptr Zb200CompressStream): cint {.importc, cdecl, dynlib: lib.}

proc compress*(src: string, level: int, dataFormat: CompressedDataFormat, strategy: Strategy,
               windowBits: int): string {.raises: [ZippyError].} =
  ## one member of zb200_compress_batch_window; gzip draws its FNAME length at random, as compress does
  var
    offs = [0'u64, src.len.uint64]
    outOffs = [0'u64, 0'u64]
    fl = randomFnameLen(dataFormat).uint8
    dummy: uint8
  result = newString(zb200_compress_bound(src.len.csize_t, dataFormat.cint).int + 64)
  check zb200_compress_batch_window(getCtx(), (if src.len > 0: src[0].unsafeAddr else: dummy.addr),
                                    offs[0].addr, 1, level.cint, strategy.cint, windowBits.cint, dataFormat.cint,
                                    fl.addr, result[0].addr, result.len.csize_t, outOffs[0].addr, nil)
  result.setLen(outOffs[1].int)

proc newCompressStream*(level: int, dataFormat: CompressedDataFormat, strategy: Strategy, windowBits: int,
                        fnameLen = -1): CompressStream {.raises: [ZippyError].} =
  ## a stream with a window size (and a strategy): zb200_compress_stream_begin_window
  let k = if fnameLen < 0: randomFnameLen(dataFormat) else: fnameLen
  check zb200_compress_stream_begin_window(getCtx(), level.cint, strategy.cint, windowBits.cint, dataFormat.cint,
                                           k.cint, result.st.addr)

# ---- optimal parse (include/zippy_b200.h "optimal parse"): smaller members than level 9; windowBits as above; not
# combined with strategies, dictionaries or compress-time indexes ----
proc zb200_compress_batch_optimal(ctx: Zb200Ctx, srcBase: pointer, srcOffsets: ptr uint64, n: csize_t,
                                  windowBits, dataFormat: cint, fnameLens: pointer, dstBase: pointer,
                                  dstCap: csize_t, dstOffsets: ptr uint64,
                                  statuses: ptr cint): cint {.importc, cdecl, dynlib: lib.}
proc zb200_compress_stream_begin_optimal(ctx: Zb200Ctx, windowBits, dataFormat, fnameLen: cint,
                                         st: ptr Zb200CompressStream): cint {.importc, cdecl, dynlib: lib.}

proc compressOptimal*(src: string, dataFormat: CompressedDataFormat, windowBits = 15): string {.raises: [ZippyError].} =
  ## one member of zb200_compress_batch_optimal; gzip draws its FNAME length at random, as compress does
  var
    offs = [0'u64, src.len.uint64]
    outOffs = [0'u64, 0'u64]
    fl = randomFnameLen(dataFormat).uint8
    dummy: uint8
  result = newString(zb200_compress_bound(src.len.csize_t, dataFormat.cint).int + 64)
  check zb200_compress_batch_optimal(getCtx(), (if src.len > 0: src[0].unsafeAddr else: dummy.addr),
                                     offs[0].addr, 1, windowBits.cint, dataFormat.cint,
                                     fl.addr, result[0].addr, result.len.csize_t, outOffs[0].addr, nil)
  result.setLen(outOffs[1].int)

proc newOptimalCompressStream*(dataFormat: CompressedDataFormat, windowBits = 15,
                               fnameLen = -1): CompressStream {.raises: [ZippyError].} =
  ## a stream under the optimal parse: zb200_compress_stream_begin_optimal
  let k = if fnameLen < 0: randomFnameLen(dataFormat) else: fnameLen
  check zb200_compress_stream_begin_optimal(getCtx(), windowBits.cint, dataFormat.cint, k.cint, result.st.addr)

# ---- rsyncable compression (include/zippy_b200.h "rsyncable compression"): chunk starts taken from the content, so
# an edit changes only the compressed bytes near it; any level and format ----
proc zb200_compress_batch_rsyncable(ctx: Zb200Ctx, srcBase: pointer, srcOffsets: ptr uint64, n: csize_t,
                                    level, dataFormat: cint, fnameLens: pointer, dstBase: pointer,
                                    dstCap: csize_t, dstOffsets: ptr uint64,
                                    statuses: ptr cint): cint {.importc, cdecl, dynlib: lib.}
proc zb200_compress_bound_rsyncable(len: csize_t, dataFormat: cint): csize_t {.importc, cdecl, dynlib: lib.}

proc compressRsyncable*(src: string, level = DefaultCompression, dataFormat = dfGzip,
                        fnameLen = -1): string {.raises: [ZippyError].} =
  ## one member of zb200_compress_batch_rsyncable; gzip draws its FNAME length at random unless fnameLen >= 0
  var
    offs = [0'u64, src.len.uint64]
    outOffs = [0'u64, 0'u64]
    fl = (if fnameLen >= 0: fnameLen else: randomFnameLen(dataFormat)).uint8
    dummy: uint8
  result = newString(zb200_compress_bound_rsyncable(src.len.csize_t, dataFormat.cint).int + 64)
  check zb200_compress_batch_rsyncable(getCtx(), (if src.len > 0: src[0].unsafeAddr else: dummy.addr),
                                       offs[0].addr, 1, level.cint, dataFormat.cint,
                                       fl.addr, result[0].addr, result.len.csize_t, outOffs[0].addr, nil)
  result.setLen(outOffs[1].int)
