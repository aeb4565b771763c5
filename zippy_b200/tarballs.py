"""Tarballs (SURVEY.md 8(f-3), a "next" row): host-side mirror of src/zippy/tarballs.nim:25-141
(reading) and tarballs_v1.nim (the `Tarball` object and the writer).

`extract_all(tar_path, dest)` reads a .tar or .tar.gz: a gzip tarball is ONE gzip member, inflated
by the GPU path (uncompressGzip, tarballs.nim:50; a single member is decoded by one 8-lane group,
so this is a convenience, not a fast path), then the 512-byte header walk stays on the host exactly
as in the reference: ustar prefix, GNU 'L' long names, files / directories / symlinks, pax and
vendor records skipped, anything else is an error; paths are checked before anything is written
and nothing is left behind on failure.

`create_tarball(source, dest)` / `Tarball.write_tarball(path)` write the byte layout of
tarballs_v1.nim:210-261 (built on the host by `tar_image`); a .tar.gz is the whole image compressed
as ONE gzip member at DefaultCompression by the GPU path (zippy_b200.compress)."""
import os
import shutil
from dataclasses import dataclass

from . import DefaultCompression, ZippyError, compress, dfGzip, uncompress

_ERR = 3


def _fail(msg):
    raise ZippyError(_ERR, msg)


def _oct(field):
    """tarballs.nim:5-23: the first run of ASCII digits in the field, base 8 (0 if none)."""
    i = 0
    while i < len(field) and not (48 <= field[i] <= 57):
        i += 1
    j = i
    while j < len(field) and 48 <= field[j] <= 57:
        j += 1
    if j == i:
        return 0
    try:
        return int(bytes(field[i:j]), 8)
    except ValueError as e:
        _fail(str(e))


def _cstr(field):
    k = bytes(field).find(b"\0")
    return bytes(field if k < 0 else field[:k]).decode("utf-8", "surrogateescape")


def _safe(path):
    if path.startswith("/") or path.startswith("\\") or (len(path) > 1 and path[1] == ":"):
        _fail("Absolute path not allowed " + path)
    if ".." in path.replace("\\", "/").split("/"):
        _fail("Path ../ not allowed " + path)


def read_tarball(data, gunzip=None):
    """-> list of (kind, path, payload | linkname, mode, mtime); kind in 'file', 'dir', 'symlink'."""
    data = bytes(data)
    if len(data) < 2:
        _fail("Invalid buffer, unable to uncompress")
    if data[0] == 31 and data[1] == 139:
        data = (gunzip or (lambda b: uncompress(b, dfGzip)))(data)
    out, pos, long_name = [], 0, ""
    while pos < len(data):
        if pos + 512 > len(data):
            _fail("Attempted to read past end of file, corrupted tarball?")
        h = data[pos:pos + 512]
        name, mode, size, mtime = _cstr(h[0:100]), _oct(h[100:107]), _oct(h[124:135]), _oct(h[136:147])
        typeflag, linkname = chr(h[156]), _cstr(h[157:257])
        prefix = _cstr(h[345:500]) if _cstr(h[257:263]) == "ustar" else ""
        pos += 512
        if pos + size > len(data):
            _fail("Attempted to read past end of file, corrupted tarball?")
        if name or long_name:
            if long_name:
                path, long_name = long_name, ""
            else:
                path = os.path.join(prefix, name) if prefix else name
            _safe(path)
            if typeflag in ("0", "\0"):
                out.append(("file", path, data[pos:pos + size], mode, mtime))
            elif typeflag == "5":
                out.append(("dir", path, b"", mode, mtime))
            elif typeflag == "2":
                out.append(("symlink", path, linkname, mode, mtime))
            elif typeflag == "L":
                long_name = _cstr(data[pos:pos + size])
            elif typeflag in ("g", "x") or "A" <= typeflag <= "Z":
                pass
            else:
                _fail("Unsupported header type " + typeflag)
        pos += (size + 511) & ~511
    return out


def _check_dest(dest):
    if dest == "" or os.path.isdir(dest):
        _fail("Destination " + dest + " already exists")
    head = os.path.dirname(dest.rstrip("/\\"))
    if head and not os.path.isdir(head):
        _fail("Path to " + dest + " does not exist")


def extract_all(tar_path, dest, gunzip=None):
    _check_dest(dest)
    with open(tar_path, "rb") as f:
        entries = read_tarball(f.read(), gunzip)
    _write_entries(entries, dest)


def _write_entries(entries, dest):
    """Entries as read_tarball returns them -> files under dest (removed again on failure)."""
    try:
        times = []
        for kind, path, payload, mode, mtime in entries:
            target = os.path.join(dest, path)
            if kind == "file":
                os.makedirs(os.path.dirname(target) or dest, exist_ok=True)
                with open(target, "wb") as f:
                    f.write(payload)
                if mode:
                    os.chmod(target, mode & 0o777)
                times.append((target, mtime))
            elif kind == "dir":
                os.makedirs(target, exist_ok=True)
                times.append((target, mtime))
            else:
                os.makedirs(os.path.dirname(target) or dest, exist_ok=True)
                os.symlink(payload, target)
        for target, mtime in times:  # second pass: directories would be touched by their files
            if mtime > 0:
                os.utime(target, (mtime, mtime))
    except Exception:
        shutil.rmtree(dest, ignore_errors=True)
        raise


# ---- the Tarball object and the writer (tarballs_v1.nim) ----
_EXTENSIONS = (".tar", ".gz", ".taz", ".tgz")
_TYPEFLAG = {"file": ord("0"), "dir": ord("5")}  # ekNormalFile, ekDirectory (tarballs_v1.nim:5-7)


@dataclass
class TarballEntry:
    """tarballs_v1.nim:9-13.  kind: "file" or "dir"; last_modified: Unix seconds; permissions: mode bits."""
    kind: str = "file"
    contents: bytes = b""
    last_modified: int = 0
    permissions: int = 0


def _bytes(s):
    return s.encode("utf-8", "surrogateescape")


def _split_path(path):
    """Nim's os.splitPath: (head, tail) around the last '/'."""
    i = path.rfind("/")
    if i < 0:
        return "", path
    return path[:i] if i > 0 else "/", path[i + 1:]


def _ext(path):
    """Nim's os.splitFile(path).ext: the last '.' suffix of the last path component ('' for a dotfile)."""
    name = path[path.rfind("/") + 1:]
    for j in range(len(name) - 2, 0, -1):
        if name[j] == "." and name[j + 1] != ".":
            return name[j:]
    return ""


def _to_oct(x, n):
    """strutils.toOct(x, n): the low n octal digits of x, zero-padded."""
    return b"%0*o" % (n, x & ((1 << (3 * n)) - 1))


def _header(path, entry):
    head_s, tail_s = _split_path(path)
    head, tail = _bytes(head_s), _bytes(tail_s)
    if len(head) >= 155:
        _fail("File path " + head_s + " too long, must be < 155 characters")
    if len(tail) >= 100:
        _fail("File name " + tail_s + " too long, must be < 100 characters")
    if entry.kind not in _TYPEFLAG:
        _fail("Unsupported tarball entry kind " + str(entry.kind))
    h = bytearray(512)
    h[0:len(tail)] = tail
    h[100:156] = (b"000777 \0" + b"000000 \0" * 2 + _to_oct(len(entry.contents), 11) + b" "
                  + _to_oct(int(entry.last_modified), 11) + b" " + b" " * 8)
    h[156] = _TYPEFLAG[entry.kind]
    h[257:265] = b"ustar\0" + b"00"
    h[329:345] = b"000000\0 " * 2
    h[345:345 + len(head)] = head
    h[148:155] = _to_oct(sum(h), 6) + b"\0"  # summed with the field as 8 spaces; byte 155 stays a space
    return h


def tar_image(contents):
    """{path: TarballEntry} -> the uncompressed tarball of tarballs_v1.nim:210-261: per entry, in order, one
    512-byte ustar header and the contents zero-padded to 512 bytes; then two zero records."""
    if not contents:
        _fail("Tarball has no contents")
    parts = []
    for path, entry in contents.items():
        parts.append(_header(path, entry))
        parts.append(entry.contents)
        parts.append(bytes(-len(entry.contents) % 512))
    parts.append(bytes(1024))
    return b"".join(parts)


class Tarball:
    """tarballs_v1.nim:15-16: `contents` maps path -> TarballEntry in insertion order."""

    def __init__(self):
        self.contents = {}

    def add_dir(self, dir):
        """tarballs_v1.nim:21-56: dir itself, every directory and every regular file under it; symlinks and
        other kinds are skipped.  Keys are relative to dir's parent and use '/'."""
        if _ext(dir):
            _fail("Error adding dir " + dir + " to tarball, appears to be a file?")
        head, tail = _split_path(dir)
        self._add_dir(head, tail)

    def _add_dir(self, base, relative):
        full = os.path.join(base, relative)
        if not os.path.exists(full):
            _fail("Path " + full + " does not exist")
        if relative and relative not in self.contents:
            self.contents[relative] = TarballEntry("dir")
        if not os.path.isdir(full):
            return
        with os.scandir(full) as it:
            for e in it:
                rel = relative + "/" + e.name if relative else e.name
                if e.is_file(follow_symlinks=False):
                    st = e.stat(follow_symlinks=False)
                    with open(e.path, "rb") as f:
                        data = f.read()
                    self.contents[rel] = TarballEntry("file", data, st.st_mtime_ns // 1000000000, st.st_mode & 0o777)
                elif e.is_dir(follow_symlinks=False):
                    self._add_dir(base, rel)

    def clear(self):
        self.contents.clear()

    def write_tarball(self, path, gzip=None):
        """tarballs_v1.nim:203-271.  .tar writes the image; .gz / .taz / .tgz write it as one gzip member at
        DefaultCompression (the GPU path unless a `gzip` callable is given).  Nothing is written on error."""
        data = tar_image(self.contents)
        ext = _ext(path)
        if ext not in _EXTENSIONS:
            _fail("Unsupported tarball extension " + ext)
        if ext != ".tar":
            data = (gzip or (lambda b: compress(b, DefaultCompression, dfGzip)))(data)
        with open(path, "wb") as f:
            f.write(data)

    def open(self, path, gunzip=None):
        """tarballs_v1.nim:174-201 over read_tarball (see DESIGN.md §8 f-3 for how the two walks differ).
        Symlinks have no TarballEntry kind and are left out."""
        with open(path, "rb") as f:
            data = f.read()
        ext = _ext(path)
        if ext not in _EXTENSIONS:
            _fail("Unsupported tarball extension " + ext)
        self.clear()
        for kind, p, payload, mode, mtime in read_tarball(data, gunzip):
            if kind == "file":
                self.contents[p] = TarballEntry("file", payload, mtime, mode & 0o777)
            elif kind == "dir":
                self.contents[p] = TarballEntry("dir")

    def extract_all(self, dest):
        """tarballs_v1.nim:273-331: dest must not exist, its parent must; nothing is left behind on failure."""
        _check_dest(dest)
        for p in self.contents:
            _safe(p)
        _write_entries([(e.kind, p, e.contents, e.permissions, e.last_modified) for p, e in self.contents.items()],
                       dest)


def create_tarball(source, dest, gzip=None):
    """tarballs_v1.nim:333-342: every directory and file inside source, written to dest."""
    t = Tarball()
    t.add_dir(source)
    t.write_tarball(dest, gzip)
