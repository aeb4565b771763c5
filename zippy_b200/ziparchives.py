"""ZIP archives over the batch entry points (SURVEY.md 8(f-2), a "next" row).

Host-side mirror of the reference's src/zippy/ziparchives.nim: `createZipArchive` (:458-634) is a
loop of crc32 + compress(BestSpeed, dfDeflate) over the entries and `extractFile` / `extractAll`
(:37-93, :398-452) a loop of uncompress(dfDeflate) + crc32 -- here each loop is ONE batched GPU
call (zb200_compress_batch / zb200_uncompress_batch / zb200_checksum_batch).  The container
format itself (local headers, central directory, ZIP64 records, CP437 names) stays on the host,
as in the reference.  Same checks and error messages as the reference; names follow its API:

    open_zip_archive(path | bytes) -> ZipArchiveReader   (openZipArchive, :183)
    reader.walk_files()                                   (walkFiles, :31)
    reader.extract_file(name) -> bytes                    (extractFile, :37)
    reader.extract_files(names=None) -> {name: bytes}     (batched; no reference counterpart)
    extract_all(zip_path, dest)                           (extractAll, :398)
    create_zip_archive({name: bytes}) -> bytes            (createZipArchive, :622-634)

and the object API of ziparchives_v1.nim, which ziparchives.nim re-exports:

    ZipArchive(), ArchiveEntry                            (ZipArchive, ArchiveEntry, v1 :11-22)
    archive.add_dir(dir) / add_file(path) / clear()       (addDir, addFile, clear, v1 :43-77)
    archive.open(path | bytes)                            (open, v1 :105-349)
    archive.write_zip_archive(path)                       (writeZipArchive, v1 :371-486)
    archive.extract_all(dest)                             (extractAll, v1 :488-546)
    create_zip_archive(source, dest)                      (createZipArchive, v1 :548-555)
"""
import os
import shutil
import stat
import struct
import time
from dataclasses import dataclass

import numpy as np

from . import BestSpeed, DefaultCompression, ZippyError, default_context, dfDeflate
from .tarballs import _ext, _split_path

_LOCAL = 0x04034B50
_CENTRAL = 0x02014B50
_EOCD = 0x06054B50
_EOCD64 = 0x06064B50
_LOC64 = 0x07064B50
_ERR_ARCHIVE = 3  # ZB200_ERR_UNCOMPRESS: the generic "invalid buffer" class


def _fail(msg):
    raise ZippyError(_ERR_ARCHIVE, msg)


def _eof():
    _fail("Attempted to read past end of file, corrupted archive?")


def _safe_path(path):
    """internal.nim verifyPathIsSafeToExtract: no absolute paths, no drive letters, no '..' parts."""
    if path.startswith("/") or path.startswith("\\") or (len(path) > 1 and path[1] == ":"):
        _fail("Absolute path not allowed " + path)
    if ".." in path.replace("\\", "/").split("/"):
        _fail("Path ../ not allowed " + path)


def _dos_time(t=None):
    lt = time.localtime(t)
    return ((lt.tm_hour << 11) | (lt.tm_min << 5) | (lt.tm_sec // 2),
            ((max(0, lt.tm_year - 1980)) << 9) | (lt.tm_mon << 5) | lt.tm_mday)


def _from_dos_time(tm, dt):
    sec, mi, ho = (tm & 31) * 2, (tm >> 5) & 63, (tm >> 11) & 31
    day, mon, yr = dt & 31, (dt >> 5) & 15, ((dt >> 9) & 127) + 1980
    if sec <= 59 and mi <= 59 and ho <= 23 and 1 <= mon <= 12 and 1 <= day <= 31:
        try:
            return time.mktime((yr, mon, day, ho, mi, sec, 0, 0, -1))
        except (OverflowError, ValueError):
            return None
    return None


class _Record:
    __slots__ = ("is_dir", "header_offset", "path", "crc", "csize", "usize", "mode")


class ZipArchiveReader:
    """ziparchives.nim:27-29 (records keep the central directory's order)."""

    def __init__(self, data, ctx=None):
        self._d = data if isinstance(data, (bytes, bytearray, memoryview)) else bytes(data)
        self._ctx = ctx
        self.records = {}
        self._parse()

    # ---- central directory (ziparchives.nim:183-395) ----
    def _u16(self, p):
        return struct.unpack_from("<H", self._d, p)[0]

    def _u32(self, p):
        return struct.unpack_from("<I", self._d, p)[0]

    def _u64(self, p):
        return struct.unpack_from("<Q", self._d, p)[0]

    def _parse(self):
        d, size = self._d, len(self._d)
        eocd = bytes(d).rfind(struct.pack("<I", _EOCD), 0, max(0, size - 22) + 4)
        if eocd < 0 or eocd + 22 > size:
            _eof()
        zip64 = eocd - 20 >= 0 and self._u32(eocd - 20) == _LOC64
        if zip64:
            if self._u32(eocd - 16) != 0:
                _fail("Unsupported archive, disk number")
            pos = self._u64(eocd - 12)
            if self._u32(eocd - 4) != 1:
                _fail("Unsupported archive, num disks")
            if pos + 64 > size:
                _eof()
            if self._u32(pos) != _EOCD64:
                _fail("Invalid central directory file header")
            disk, start_disk = self._u32(pos + 16), self._u32(pos + 20)
            n_disk, n_total = self._u64(pos + 24), self._u64(pos + 32)
            cd_size, cd_start = self._u64(pos + 40), self._u64(pos + 48)
        else:
            disk, start_disk, n_disk, n_total = (self._u16(eocd + 4), self._u16(eocd + 6), self._u16(eocd + 8),
                                                 self._u16(eocd + 10))
            cd_size, cd_start = self._u32(eocd + 12), self._u32(eocd + 16)
        if disk != 0:
            _fail("Unsupported archive, disk number")
        if start_disk != 0:
            _fail("Unsupported archive, start disk")
        if n_disk != n_total:
            _fail("Unsupported archive, record number")
        # an archive may be appended to another file (an .exe, a .jpg): locate the directory from
        # the end by counting its records backwards, fall back to the recorded offset
        socd, p = cd_start, eocd
        sig = struct.pack("<I", _CENTRAL)
        raw = bytes(d)
        for k in range(n_total):
            p = raw.rfind(sig, 0, p + 3)   # the last record header that starts before p
            if p < 0:
                break
            if k == n_total - 1:
                socd = p
        shift = socd - cd_start
        pos = socd
        for _ in range(n_total):
            if pos + 46 > size:
                _eof()
            if self._u32(pos) != _CENTRAL:
                _fail("Invalid central directory file header")
            flags, method = self._u16(pos + 8), self._u16(pos + 10)
            crc, csize, usize = self._u32(pos + 16), self._u32(pos + 20), self._u32(pos + 24)
            nlen, xlen, clen = self._u16(pos + 28), self._u16(pos + 30), self._u16(pos + 32)
            fdisk, xattr, hoff = self._u16(pos + 34), self._u32(pos + 38), self._u32(pos + 42)
            if method not in (0, 8):
                _fail("Unsupported archive, compression method")
            if fdisk != 0:
                _fail("Invalid file disk number")
            pos += 46
            if pos + nlen > size:
                _eof()
            name_b = bytes(d[pos:pos + nlen])
            pos += nlen
            q, end = pos, pos + xlen
            while q + 4 <= end:  # ZIP64 extended information (id 1): only the saturated fields are present
                fid, flen = self._u16(q), self._u16(q + 2)
                q += 4
                if fid == 1:
                    z, zend = q, q + flen
                    for field in ("usize", "csize", "hoff"):
                        cur = {"usize": usize, "csize": csize, "hoff": hoff}[field]
                        if cur == 0xFFFFFFFF:
                            if z + 8 > zend or z + 8 > size:
                                _eof()
                            v = self._u64(z)
                            z += 8
                            if field == "usize":
                                usize = v
                            elif field == "csize":
                                csize = v
                            else:
                                hoff = v
                    break
                q += flen
            pos += xlen + clen
            if pos > socd + cd_size:
                _fail("Invalid central directory size")
            if flags & 0x800:  # language encoding flag: UTF-8
                name = name_b.decode("utf-8", "replace")
            else:
                try:
                    name = name_b.decode("utf-8")
                except UnicodeDecodeError:
                    name = name_b.decode("cp437")  # DOS / OEM names
            if name in self.records:
                _fail("Unsupported archive, duplicate entry")
            r = _Record()
            r.is_dir = bool(xattr & 0x10) or bool((xattr >> 16) & stat.S_IFDIR) or name.endswith("/")
            r.header_offset = hoff + shift
            r.path, r.crc, r.csize, r.usize = name, crc, csize, usize
            r.mode = (xattr >> 16) & 0o777
            self.records[name] = r

    # ---- access ----
    def walk_files(self):
        for r in self.records.values():
            if not r.is_dir:
                yield r.path

    def _payload(self, r):
        """(method, start) of an entry's data; checks of extractFile (ziparchives.nim:52-78)."""
        pos, size = r.header_offset, len(self._d)
        if pos + 30 > size:
            _eof()
        if self._u32(pos) != _LOCAL:
            _fail("Invalid file header")
        method = self._u16(pos + 8)
        pos += 30 + self._u16(pos + 26) + self._u16(pos + 28)
        if pos + r.csize > size:
            _eof()
        if method not in (0, 8):
            _fail("Unsupported archive, compression method")
        return method, pos

    def extract_files(self, names=None):
        """All requested entries in one batched inflate + one batched CRC-32 on the GPU."""
        ctx = self._ctx or default_context()
        names = list(self.walk_files()) if names is None else list(names)
        recs = []
        for nme in names:
            r = self.records.get(nme)
            if r is None or r.is_dir:
                _fail("No file record found for " + nme)
            recs.append(r)
        out = {}
        packed, offs, sizes, which = [], [0], [], []
        for r in recs:
            method, pos = self._payload(r)
            if method == 0:
                out[r.path] = bytes(self._d[pos:pos + r.csize])
            else:
                packed.append(bytes(self._d[pos:pos + r.csize]))
                offs.append(offs[-1] + r.csize)
                sizes.append(r.usize)
                which.append(r)
        if which:
            base = np.frombuffer(b"".join(packed), dtype=np.uint8) if offs[-1] else np.zeros(1, dtype=np.uint8)
            data, do, lens, st = ctx.uncompress_batch(base, np.array(offs, dtype=np.uint64), dfDeflate,
                                                      sizes=np.array(sizes, dtype=np.uint64))
            for i, r in enumerate(which):
                if st[i] != 0:
                    raise ZippyError(int(st[i]))
                out[r.path] = data[int(do[i]):int(do[i]) + int(lens[i])].tobytes()
        # crc32 of every extracted file against the directory (ziparchives.nim:92-93), one batch
        blobs = [out[r.path] for r in recs]
        if blobs:
            o2 = np.zeros(len(blobs) + 1, dtype=np.uint64)
            o2[1:] = np.cumsum([len(b) for b in blobs])
            joined = np.frombuffer(b"".join(blobs), dtype=np.uint8) if o2[-1] else np.zeros(1, dtype=np.uint8)
            crcs = ctx.checksum_batch(joined, o2, "crc32")
            for r, c in zip(recs, crcs):
                if int(c) != r.crc:
                    _fail("Verifying crc32 failed")
        return out

    def extract_file(self, path):
        return self.extract_files([path])[path]

    def close(self):
        self._d = b""


def open_zip_archive(src, ctx=None):
    if isinstance(src, (bytes, bytearray, memoryview)):
        return ZipArchiveReader(src, ctx)
    with open(src, "rb") as f:
        return ZipArchiveReader(f.read(), ctx)


def extract_all(zip_path, dest, ctx=None):
    """ziparchives.nim:398-452: dest must not exist, its parent must; nothing is left behind on failure."""
    if dest == "" or os.path.isdir(dest):
        _fail("Destination " + dest + " already exists")
    head = os.path.dirname(dest.rstrip("/\\"))
    if head and not os.path.isdir(head):
        _fail("Path to " + dest + " does not exist")
    reader = open_zip_archive(zip_path, ctx)
    for r in reader.records.values():
        _safe_path(r.path)
    try:
        files = reader.extract_files()
        for r in reader.records.values():
            target = os.path.join(dest, r.path)
            if r.is_dir:
                os.makedirs(target, exist_ok=True)
            else:
                os.makedirs(os.path.dirname(target), exist_ok=True)
                with open(target, "wb") as f:
                    f.write(files[r.path])
                if r.mode:
                    os.chmod(target, r.mode)
        for r in reader.records.values():  # second pass: directories would be touched by their files
            tm, dt = struct.unpack_from("<HH", reader._d, r.header_offset + 10)
            t = _from_dos_time(tm, dt)
            if t is not None:
                os.utime(os.path.join(dest, r.path), (t, t))
    except Exception:
        shutil.rmtree(dest, ignore_errors=True)
        raise
    finally:
        reader.close()


def create_zip_archive(entries, *args, ctx=None):
    """Two forms, as in the reference.

    create_zip_archive({name: bytes}, ctx=None) -> archive bytes.  Layout of ziparchives.nim:458-620: version 45,
    UTF-8 flag, ZIP64 extra fields everywhere, entries written from the LAST key to the first (the reference pops
    keys off the end), empty files stored, everything else deflated at BestSpeed -- in one batch.

    create_zip_archive(source, dest, ctx=None) with a path as `source`: ziparchives_v1.nim:548-555, every
    directory and file inside source (ZipArchive.add_dir) written to the file dest (ZipArchive.write_zip_archive)."""
    if isinstance(entries, (str, os.PathLike)):
        dest, = args
        archive = ZipArchive(ctx)
        archive.add_dir(os.fspath(entries))
        archive.write_zip_archive(dest)
        return None
    if args:
        ctx, = args
    ctx = ctx or default_context()
    names = list(entries.keys())[::-1]
    for nme in names:
        if nme == "":
            _fail("Invalid empty file name")
        if nme[0] == "/":
            _fail("File paths must be relative")
        if len(nme.encode("utf-8")) > 0xFFFF:
            _fail("File name len > uint16.high")
    blobs = [bytes(entries[nme]) for nme in names]
    n = len(blobs)
    offs = np.zeros(n + 1, dtype=np.uint64)
    if n:
        offs[1:] = np.cumsum([len(b) for b in blobs])
    joined = np.frombuffer(b"".join(blobs), dtype=np.uint8) if n and offs[-1] else np.zeros(1, dtype=np.uint8)
    crcs = ctx.checksum_batch(joined, offs, "crc32") if n else []
    comp, co = (ctx.compress_batch(joined, offs, BestSpeed, dfDeflate) if n else (np.zeros(0, np.uint8), offs))
    tm, dt = _dos_time()
    out = bytearray()
    recs = []
    for i, nme in enumerate(names):
        nb = nme.encode("utf-8")
        ulen = len(blobs[i])
        data = b"" if ulen == 0 else comp[int(co[i]):int(co[i + 1])].tobytes()
        method = 0 if ulen == 0 else 8
        recs.append((nb, len(out), ulen, len(data), method, int(crcs[i])))
        out += struct.pack("<IHHHHHIIIHH", _LOCAL, 45, 1 << 11, method, tm, dt, int(crcs[i]), 0xFFFFFFFF, 0xFFFFFFFF,
                           len(nb), 20)
        out += nb + struct.pack("<HHQQ", 1, 16, ulen, len(data)) + data
    cd_start = len(out)
    for nb, hoff, ulen, clen, method, crc in recs:
        out += struct.pack("<IHHHHHHIIIHHHHHII", _CENTRAL, 45, 45, 1 << 11, method, tm, dt, crc, 0xFFFFFFFF, 0xFFFFFFFF,
                           len(nb), 28, 0, 0, 0, 0, 0xFFFFFFFF)
        out += nb + struct.pack("<HHQQQ", 1, 24, ulen, clen, hoff)
    cd_end = len(out)
    out += struct.pack("<IQHHIIQQQQ", _EOCD64, 44, 45, 45, 0, 0, len(recs), len(recs), cd_end - cd_start, cd_start)
    out += struct.pack("<IIQI", _LOC64, 0, cd_end, 1)
    out += struct.pack("<IHHHHIIH", _EOCD, 0, 0, 0xFFFF, 0xFFFF, 0xFFFFFFFF, 0xFFFFFFFF, 0)
    return bytes(out)


# ---- the ZipArchive object (ziparchives_v1.nim) ----
# An in-memory archive: add_dir / add_file / open fill `contents`, write_zip_archive / extract_all write it out.
# Reading walks the local headers in order as v1 does, but decodes every deflated entry in ONE
# inflate_batch_crc32 call (the CRC-32 of each output comes back from the decode on the GPU), and writing
# compresses every entry in ONE compress_batch and checksums them in ONE checksum_batch.  DESIGN.md lists where
# this differs from the reference.

@dataclass
class ArchiveEntry:
    """ziparchives_v1.nim:15-19.  kind: "file" or "dir"; last_modified: Unix seconds; permissions: mode bits."""
    kind: str = "file"
    contents: bytes = b""
    last_modified: int = 0
    permissions: int = 0


def _name_bytes(path):
    return path.encode("utf-8", "surrogateescape")


def _name_str(raw):
    return bytes(raw).decode("utf-8", "surrogateescape")


def _to_ms_dos(t):
    """toMsDos (ziparchives_v1.nim:351-369): local time, seconds / 2, years since 1980 (at least 0)."""
    lt = time.localtime(t)
    return (((lt.tm_hour << 11) | (lt.tm_min << 5) | (lt.tm_sec // 2)) & 0xFFFF,
            ((max(0, lt.tm_year - 1980) << 9) | (lt.tm_mon << 5) | lt.tm_mday) & 0xFFFF)


def _days_in_month(year, month):
    if month == 2:
        return 29 if year % 4 == 0 and (year % 100 != 0 or year % 400 == 0) else 28
    return 30 if month in (4, 6, 9, 11) else 31


def _from_ms_dos(tm, dt):
    """ziparchives_v1.nim:161-179: the local time of a DOS time and date, 0 when the time fields are out of range.
    A date that initDateTime rejects (day or month 0, a day past the month's end) raises a Defect in the
    reference; here it is 0 as well."""
    sec, mi, ho = (tm & 31) * 2, (tm >> 5) & 63, (tm >> 11) & 31
    day, mon, yr = dt & 31, (dt >> 5) & 15, ((dt >> 9) & 127) + 1980
    if sec > 59 or mi > 59 or ho > 23 or not 1 <= mon <= 12 or not 1 <= day <= _days_in_month(yr, mon):
        return 0
    return int(time.mktime((yr, mon, day, ho, mi, sec, 0, 0, -1)))


def _extract_permissions(xattr):
    """extractPermissions (ziparchives_v1.nim:84-103): the mode bits of the high half, 0o664 when there are none."""
    perms = xattr >> 16
    return 0o664 if perms == 0 else perms & 0o777


def _fail_eof():
    _fail("Attempted to read past end of file, corrupted zip archive?")


def _fail_open():
    _fail("Unexpected error opening zip archive")


class ZipArchive:
    """ziparchives_v1.nim:21-22: `contents` maps path -> ArchiveEntry in insertion order.  Directory keys end
    in '/'.  ctx: the codec context (default_context() when None)."""

    def __init__(self, ctx=None):
        self.contents = {}
        self._ctx = ctx

    def _context(self):
        return self._ctx or default_context()

    def add_dir(self, dir):
        """ziparchives_v1.nim:24-54: dir itself as "tail/", then every directory and regular file under it in
        directory order; symlinks and other kinds are skipped.  A directory that does not exist adds only its
        own entry."""
        if _ext(dir):
            _fail("Error adding dir " + dir + " to archive, appears to be a file?")
        head, tail = _split_path(dir)
        self._add_dir(head, tail)

    def _add_dir(self, base, relative):
        if relative and relative not in self.contents:
            self.contents[relative + "/"] = ArchiveEntry("dir")
        full = os.path.join(base, relative)
        try:
            it = os.scandir(full)
        except OSError:  # walkDir yields nothing for a path it cannot open
            return
        with it:
            for e in it:
                rel = os.path.join(relative, e.name)
                if e.is_file(follow_symlinks=False):
                    st = e.stat(follow_symlinks=False)
                    with open(e.path, "rb") as f:
                        data = f.read()
                    self.contents[rel] = ArchiveEntry("file", data, st.st_mtime_ns // 10 ** 9, st.st_mode & 0o777)
                elif e.is_dir(follow_symlinks=False):
                    self._add_dir(base, rel)

    def add_file(self, path):
        """ziparchives_v1.nim:56-74: one file (a symlink is followed), keyed by its file name."""
        st = os.stat(path)
        if not stat.S_ISREG(st.st_mode):
            _fail("Error adding file " + path + " to archive, appears to be a directory?")
        with open(path, "rb") as f:
            data = f.read()
        self.contents[_split_path(path)[1]] = ArchiveEntry("file", data, st.st_mtime_ns // 10 ** 9,
                                                            st.st_mode & 0o777)

    def clear(self):
        self.contents.clear()

    def zip_image(self):
        """The bytes write_zip_archive writes (ziparchives_v1.nim:371-481): per entry a local header (version 20,
        UTF-8 flag, no extra field) and the data, then the central directory and the end record.  Counts, sizes
        and offsets are cut to the 16 / 32 bits of their fields, as the reference's casts do."""
        if not self.contents:
            _fail("Zip archive has no contents")
        ctx = self._context()
        paths = list(self.contents)
        blobs = [bytes(self.contents[p].contents) for p in paths]
        n = len(paths)
        offs = np.zeros(n + 1, dtype=np.uint64)
        offs[1:] = np.cumsum([len(b) for b in blobs])
        joined = np.frombuffer(b"".join(blobs), dtype=np.uint8) if offs[-1] else np.zeros(1, dtype=np.uint8)
        crcs = ctx.checksum_batch(joined, offs, "crc32")
        # every entry with contents is deflated, even one stored under method 0 (a "dir/" key with contents):
        # the reference writes its deflate stream there (ziparchives_v1.nim:397-413)
        full = [i for i in range(n) if blobs[i]]
        comp = {}
        if full:
            fo = np.zeros(len(full) + 1, dtype=np.uint64)
            fo[1:] = np.cumsum([len(blobs[i]) for i in full])
            cdata, co = ctx.compress_batch(np.frombuffer(b"".join(blobs[i] for i in full), dtype=np.uint8), fo,
                                           DefaultCompression, dfDeflate)
            for k, i in enumerate(full):
                comp[i] = cdata[int(co[k]):int(co[k + 1])].tobytes()
        out = bytearray()
        recs = []
        for i, p in enumerate(paths):
            e = self.contents[p]
            nb = _name_bytes(p)
            data = comp.get(i, b"")
            method = 0 if p[p.rfind("/") + 1:] == "" or not blobs[i] else 8  # splitFile(path).name is empty
            tm, dt = _to_ms_dos(e.last_modified)
            rec = (method, tm, dt, int(crcs[i]), len(data) & 0xFFFFFFFF, len(blobs[i]) & 0xFFFFFFFF, len(nb) & 0xFFFF)
            recs.append((rec, len(out) & 0xFFFFFFFF, 0x10 if e.kind == "dir" else 0x20, nb))
            out += struct.pack("<IHHHHHIIIHH", _LOCAL, 20, 0x800, *rec, 0) + nb + data
        cd_start, cd_size = len(out), 0
        for rec, hoff, xattr, nb in recs:
            out += struct.pack("<IHHHHHHIIIHHHHHII", _CENTRAL, 63, 20, 0x800, *rec, 0, 0, 0, 0, xattr, hoff) + nb
            cd_size += 46 + len(nb)
        out += struct.pack("<IHHHHIIH", _EOCD, 0, 0, n & 0xFFFF, n & 0xFFFF, cd_size & 0xFFFFFFFF,
                           cd_start & 0xFFFFFFFF, 0)
        return bytes(out)

    def write_zip_archive(self, path):
        """ziparchives_v1.nim:371-486: zip_image() to path; nothing is written on error."""
        data = self.zip_image()
        with open(path, "wb") as f:
            f.write(data)

    def open(self, src):
        """ziparchives_v1.nim:105-349: read an archive (a path or the bytes) into `contents`, replacing what was
        there.  The local headers are walked in order up to the end record; every entry is decoded and checked
        against its header's CRC-32 and size.  Errors are raised in archive order, as the reference's walk
        raises them: a bad entry before a header error wins."""
        if isinstance(src, (bytes, bytearray, memoryview)):
            d = bytes(src)
        else:
            with open(src, "rb") as f:
                d = f.read()
        self.clear()
        size = len(d)
        u16 = lambda p: struct.unpack_from("<H", d, p)[0]  # noqa: E731
        u32 = lambda p: struct.unpack_from("<I", d, p)[0]  # noqa: E731
        entries = []   # local entries: [raw name, method, crc, usize, last_modified, payload]
        steps = []     # ("local", index) / ("central", raw name, external attributes), in archive order
        header_error = None
        pos = 0
        try:
            while True:
                if pos + 4 > size:
                    _fail_eof()
                sig = u32(pos)
                if sig == _LOCAL:
                    if pos + 30 > size:
                        _fail_eof()
                    flag, method, tm, dt, crc, csize, usize, nlen, xlen = struct.unpack_from("<HHHHIIIHH", d, pos + 6)
                    pos += 30
                    if flag & 0b100:
                        _fail("Unsupported zip archive, data descriptor bit set")
                    if flag & 0b1000:
                        _fail("Unsupported zip archive, uses deflate64")
                    if method not in (0, 8):
                        _fail("Unsupported zip archive compression method %d" % method)
                    if pos + nlen + xlen > size:
                        _fail_eof()
                    name = d[pos:pos + nlen]
                    pos += nlen + xlen
                    if pos + csize > size:
                        _fail_eof()
                    steps.append(("local", len(entries)))
                    entries.append([name, method, crc, usize, _from_ms_dos(tm, dt), d[pos:pos + csize]])
                    pos += csize
                elif sig == _CENTRAL:
                    if pos + 46 > size:
                        _fail_eof()
                    nlen, xlen, clen = struct.unpack_from("<HHH", d, pos + 28)
                    xattr = u32(pos + 38)
                    pos += 46
                    if pos + nlen + xlen + clen > size:
                        _fail_eof()
                    steps.append(("central", d[pos:pos + nlen], xattr))
                    pos += nlen + xlen + clen
                elif sig == _EOCD:
                    if pos + 22 > size:
                        _fail_eof()
                    if pos + 22 + u16(pos + 20) > size:
                        _fail_eof()
                    break
                else:
                    _fail_open()
        except ZippyError as e:
            header_error = e
        outputs = self._decode(entries)
        for step in steps:
            if step[0] == "local":
                name, method, crc, usize, mtime, _ = entries[step[1]]
                if isinstance(outputs[step[1]], int):
                    raise ZippyError(outputs[step[1]])
                data, got_crc = outputs[step[1]]
                if got_crc != crc:
                    _fail("Verifying archive entry " + _name_str(name) + " CRC-32 failed")
                if len(data) != usize:
                    _fail("Unexpected error verifying " + _name_str(name) + " uncompressed size")
                self.contents[_name_str(name).replace("\\", "/")] = ArchiveEntry("file", data, mtime)
            else:
                key = _name_str(step[1])   # looked up as written, not unix-pathed (ziparchives_v1.nim:282-293)
                if key not in self.contents:
                    _fail_open()
                if step[2] & 0x10:
                    self.contents[key].kind = "dir"
                self.contents[key].permissions = _extract_permissions(step[2])
        if header_error is not None:
            raise header_error

    def _decode(self, entries):
        """-> per entry (bytes, crc32), or the status code of a failed decode: every deflated entry in ONE
        inflate_batch_crc32 (slots sized by the headers), every stored one through ONE checksum_batch."""
        ctx = self._context() if entries else None
        res = [None] * len(entries)
        for method in (8, 0):
            idx = [i for i, e in enumerate(entries) if e[1] == method]
            if not idx:
                continue
            offs = np.zeros(len(idx) + 1, dtype=np.uint64)
            offs[1:] = np.cumsum([len(entries[i][5]) for i in idx])
            joined = b"".join(entries[i][5] for i in idx)
            base = np.frombuffer(joined, dtype=np.uint8) if joined else np.zeros(1, dtype=np.uint8)
            if method == 8:
                out, do, lens, crcs, st = ctx.inflate_batch_crc32(base, offs, [entries[i][3] for i in idx])
                for k, i in enumerate(idx):
                    res[i] = (int(st[k]) if st[k] != 0 else
                              (out[int(do[k]):int(do[k]) + int(lens[k])].tobytes(), int(crcs[k])))
            else:
                crcs = ctx.checksum_batch(base, offs, "crc32")
                for k, i in enumerate(idx):
                    res[i] = (entries[i][5], int(crcs[k]))
        return res

    def extract_all(self, dest):
        """ziparchives_v1.nim:488-546: dest must not exist and its parent must (Nim's splitPath: a bare relative
        name has no parent and is refused).  Files get their mtime when it is after 1970 and their permissions as
        stored.  dest is removed again on failure."""
        if os.path.isdir(dest):
            _fail("Destination " + dest + " already exists")
        head, tail = _split_path(dest)
        if tail != "" and not os.path.isdir(head):
            _fail("Path to destination " + dest + " does not exist")
        try:
            for path, e in self.contents.items():
                if path.startswith("/"):
                    _fail("Extracting absolute paths is not supported (" + path + ")")
                if path.startswith("../") or path.startswith("..\\"):
                    _fail("Extracting paths starting with `..` is not supported (" + path + ")")
                if "/../" in path or "\\..\\" in path:
                    _fail("Extracting paths containing `/../` is not supported (" + path + ")")
                target = os.path.join(dest, path)
                if e.kind == "dir":
                    os.makedirs(target, exist_ok=True)
                else:
                    os.makedirs(os.path.join(dest, _split_path(path)[0]), exist_ok=True)
                    with open(target, "wb") as f:
                        f.write(e.contents)
                    if e.last_modified > 0:
                        os.utime(target, (e.last_modified, e.last_modified))
                    os.chmod(target, e.permissions)
        except (OSError, ZippyError):
            shutil.rmtree(dest, ignore_errors=True)
            raise

