"""The ZipArchive object API of ziparchives_v1.nim (zippy_b200/ziparchives.py, include/zippy_b200_zip.hpp) and the
decode call behind its reader, Context.inflate_batch_crc32 / zb200_inflate_batch_crc32.

not-gpu: the writer's bytes rebuilt field by field with struct, zipfile reading them, every error of `open` on
hand-built archives in the reference's order, add_dir / add_file / extract_all on real directories, and the C++
form against the Python one -- all with a zlib stand-in for the codec context.  gpu: inflate_batch_crc32 against
zlib.crc32 and uncompress_batch on members from every encoder and every decode path, a 64 MiB tree written and
read on the GPU, and the C++ program on libzippy_b200.so."""
import io
import os
import stat
import struct
import subprocess
import time
import zipfile
import zlib

import numpy as np
import pytest

from zippy_b200 import ZippyError

HERE = os.path.dirname(os.path.abspath(__file__))
ZDIR = os.path.join(HERE, "golden", "ziparchives")


class ZlibCtx:
    """Stand-in for the Context methods ZipArchive calls (CPU tests only).  It compresses at zlib level 1 whatever
    the level, as tests/native/mock_abi_zlib.cpp does, so Python and C++ write the same bytes."""

    def checksum_batch(self, base, offsets, kind="crc32"):
        b = bytes(base)
        return np.array([zlib.crc32(b[int(offsets[i]):int(offsets[i + 1])]) for i in range(len(offsets) - 1)],
                        dtype=np.uint32)

    def compress_batch(self, base, offsets, level, fmt, fname_lens=None):
        b = bytes(base)
        outs = [_deflate(b[int(offsets[i]):int(offsets[i + 1])]) for i in range(len(offsets) - 1)]
        oo = np.zeros(len(outs) + 1, dtype=np.uint64)
        oo[1:] = np.cumsum([len(x) for x in outs])
        return np.frombuffer(b"".join(outs), dtype=np.uint8), oo

    def inflate_batch_crc32(self, base, offsets, sizes):
        b = bytes(base)
        outs, st = [], []
        for i in range(len(offsets) - 1):
            d = zlib.decompressobj(-15)
            try:
                out = d.decompress(b[int(offsets[i]):int(offsets[i + 1])])
                ok = d.eof
            except zlib.error:
                ok = False
            outs.append(out if ok else b"")
            st.append(0 if ok else 3)
        do = np.zeros(len(outs) + 1, dtype=np.uint64)
        do[1:] = np.cumsum([len(x) for x in outs])
        return (np.frombuffer(b"".join(outs) or b"\0", dtype=np.uint8), do,
                np.array([len(x) for x in outs], dtype=np.uint64),
                np.array([zlib.crc32(x) for x in outs], dtype=np.uint32), np.array(st, dtype=np.int32))


def _deflate(data):
    c = zlib.compressobj(1, zlib.DEFLATED, -15)
    return c.compress(data) + c.flush()


def _za():
    import zippy_b200.ziparchives as za
    return za


class _TZ:
    """A fixed local time zone for the duration of a test (restored afterwards)."""

    def __init__(self, tz):
        self.tz = tz

    def __enter__(self):
        self.old = os.environ.get("TZ")
        os.environ["TZ"] = self.tz
        time.tzset()

    def __exit__(self, *exc):
        if self.old is None:
            del os.environ["TZ"]
        else:
            os.environ["TZ"] = self.old
        time.tzset()


TZ = "EST+5"        # UTC-5, no DST: local DOS times differ from UTC ones
T1 = 1700000000     # 2023-11-14 22:13:20 UTC = 17:13:20 EST
T2 = 1234567891     # an odd second: the DOS time keeps seconds / 2


def _dos(t):
    lt = time.gmtime(t - 5 * 3600)   # EST+5 by hand
    return ((lt.tm_hour << 11) | (lt.tm_min << 5) | (lt.tm_sec // 2),
            (max(0, lt.tm_year - 1980) << 9) | (lt.tm_mon << 5) | lt.tm_mday)


def _layout_contents():
    E = _za().ArchiveEntry
    return {
        "a.txt": E("file", b"alpha\n" * 1000, T1, 0o640),
        "empty": E("file", b"", T2, 0o600),
        "dir/": E("dir"),
        "dir/b.bin": E("file", bytes(range(256)) * 3, T2, 0o755),
        "café.txt": E("file", "naïve".encode(), T1, 0o644),
    }


def _expected_zip(contents):
    """The archive of ziparchives_v1.nim:371-481, field by field."""
    out, cd = b"", b""
    for path, e in contents.items():
        nb = path.encode()
        data = _deflate(e.contents) if e.contents else b""
        method = 0 if path.endswith("/") or not e.contents else 8
        tm, dt = _dos(e.last_modified)  # time 0 is 1969-12-31 19:00 EST: year field 0
        crc = zlib.crc32(e.contents)
        fixed = struct.pack("<HHHHIII", 0x800, method, tm, dt, crc, len(data), len(e.contents))
        cd += (struct.pack("<IHH", 0x02014B50, 63, 20) + fixed + struct.pack("<HHHHHI", len(nb), 0, 0, 0, 0,
               0x10 if e.kind == "dir" else 0x20) + struct.pack("<I", len(out)) + nb)
        out += struct.pack("<IH", 0x04034B50, 20) + fixed + struct.pack("<HH", len(nb), 0) + nb + data
    n = len(contents)
    return out + cd + struct.pack("<IHHHHIIH", 0x06054B50, 0, 0, n, n, len(cd), len(out), 0)


def _archive(contents, ctx=None):
    a = _za().ZipArchive(ctx or ZlibCtx())
    a.contents.update(contents)
    return a


def test_writer_layout_cpu(tmp_path):
    with _TZ(TZ):
        contents = _layout_contents()
        contents["dir2/"] = _za().ArchiveEntry("dir", b"stored, but written deflated", T1)  # the reference's quirk
        p = tmp_path / "x.zip"
        _archive(contents).write_zip_archive(str(p))
        assert p.read_bytes() == _expected_zip(contents)
        data = p.read_bytes()
        # the dir2/ entry: method 0, sizes of the deflate stream and of the contents
        k = data.index(b"dir2/") - 30
        method, clen, ulen = struct.unpack_from("<H", data, k + 8)[0], *struct.unpack_from("<II", data, k + 18)
        assert method == 0 and clen == len(_deflate(b"stored, but written deflated")) and ulen == 28


def test_writer_read_by_zipfile_cpu(tmp_path):
    with _TZ(TZ):
        contents = _layout_contents()
        p = tmp_path / "x.zip"
        _archive(contents).write_zip_archive(str(p))
        with zipfile.ZipFile(p) as zf:
            assert zf.testzip() is None
            assert [i.filename for i in zf.infolist()] == list(contents)
            for path, e in contents.items():
                i = zf.getinfo(path)
                assert zf.read(path) == e.contents
                assert i.external_attr == (0x10 if e.kind == "dir" else 0x20) and i.create_version == 63
                if e.last_modified:
                    lt = time.localtime(e.last_modified)
                    assert i.date_time == (lt.tm_year, lt.tm_mon, lt.tm_mday, lt.tm_hour, lt.tm_min, lt.tm_sec // 2 * 2)


def test_writer_count_wraps_at_16_bits_cpu():
    E = _za().ArchiveEntry
    contents = {"e%05d" % i: E() for i in range(65537)}
    data = _archive(contents).zip_image()
    local = sum(30 + len(k) for k in contents)
    cd = sum(46 + len(k) for k in contents)
    assert len(data) == local + cd + 22
    assert data[-22:] == struct.pack("<IHHHHIIH", 0x06054B50, 0, 0, 1, 1, cd, local, 0)


def test_writer_errors_cpu(tmp_path):
    p = tmp_path / "x.zip"
    with pytest.raises(ZippyError) as ei:
        _archive({}).write_zip_archive(str(p))
    assert str(ei.value) == "Zip archive has no contents" and not p.exists()


def test_open_reads_writer_output_cpu(tmp_path):
    with _TZ(TZ):
        contents = _layout_contents()
        p = tmp_path / "x.zip"
        _archive(contents).write_zip_archive(str(p))
        za = _za()
        for src in (str(p), p.read_bytes()):
            a = za.ZipArchive(ZlibCtx())
            a.contents["stale"] = za.ArchiveEntry()
            a.open(src)
            assert list(a.contents) == list(contents)
            for path, e in contents.items():
                got = a.contents[path]
                # a DOS time has 2-second steps; permissions come from the high half of the attributes, which the
                # writer leaves 0 (-> rw-rw-r--)
                assert (got.kind, got.contents, got.permissions) == (e.kind, e.contents, 0o664)
                # time 0 went out as 1969-12-31 19:00 with the year clamped to 1980: it comes back as 1980-12-31
                assert got.last_modified == (e.last_modified // 2 * 2 if e.last_modified else 347155200)


# ---- hand-built archives for `open` ----
def _local(name, data, method=8, flag=0x800, crc=None, usize=None, csize=None, raw=None, tm=0, dt=0x21):
    payload = raw if raw is not None else (_deflate(data) if method == 8 else data)
    return (struct.pack("<IHHHHHIIIHH", 0x04034B50, 20, flag, method, tm, dt,
                        zlib.crc32(data) if crc is None else crc, len(payload) if csize is None else csize,
                        len(data) if usize is None else usize, len(name), 0) + name + payload)


def _central(name, xattr=0x20):
    return struct.pack("<IHHHHHHIIIHHHHHII", 0x02014B50, 63, 20, 0x800, 8, 0, 0, 0, 0, 0, len(name), 0, 0, 0, 0,
                       xattr, 0) + name


def _eocd(comment=b"", clen=None):
    return struct.pack("<IHHHHIIH", 0x06054B50, 0, 0, 0, 0, 0, 0, len(comment) if clen is None else clen) + comment


def _open_error(data, ctx=None):
    a = _za().ZipArchive(ctx or ZlibCtx())
    with pytest.raises(ZippyError) as ei:
        a.open(data)
    return str(ei.value)


EOF_MSG = "Attempted to read past end of file, corrupted zip archive?"
OPEN_MSG = "Unexpected error opening zip archive"


def test_open_eof_checks_cpu():
    good = _local(b"a", b"hello")
    cases = {
        "empty input": b"",
        "short signature": b"PK\x03",
        "no end record": good,
        "short local header": good + b"PK\x03\x04" + bytes(20),
        "name past the end": _local(b"a", b"")[:-1] + b"",
        "data past the end": good[:-1],
        "short central header": good + _central(b"a")[:45],
        "central name past the end": good + _central(b"abc")[:-1],
        "short end record": good + _eocd()[:21],
        "comment past the end": good + _eocd(b"xyz", clen=4),
    }
    cases["name past the end"] = struct.pack("<IHHHHHIIIHH", 0x04034B50, 20, 0, 0, 0, 0, 0, 0, 0, 5, 0) + b"abcd"
    for what, data in cases.items():
        assert _open_error(data) == EOF_MSG, what
    a = _za().ZipArchive(ZlibCtx())
    a.open(good + _central(b"a") + _eocd(b"xyz") + b"trailing bytes are never read")
    assert a.contents["a"].contents == b"hello"


def test_open_header_errors_cpu():
    assert _open_error(_local(b"a", b"x", flag=0x804) + _eocd()) == "Unsupported zip archive, data descriptor bit set"
    assert _open_error(_local(b"a", b"x", flag=0x808) + _eocd()) == "Unsupported zip archive, uses deflate64"
    assert _open_error(_local(b"a", b"x", flag=0x80C) + _eocd()) == "Unsupported zip archive, data descriptor bit set"
    assert _open_error(_local(b"a", b"x", method=12, raw=b"") + _eocd()) == \
        "Unsupported zip archive compression method 12"
    assert _open_error(_local(b"a", b"x") + b"PK\x05\x05" + bytes(40)) == OPEN_MSG
    assert _open_error(_local(b"a", b"x") + _central(b"b") + _eocd()) == OPEN_MSG
    # the directory names are looked up as written; the local names were unix-pathed
    assert _open_error(_local(b"d\\a", b"x") + _central(b"d\\a") + _eocd()) == OPEN_MSG
    a = _za().ZipArchive(ZlibCtx())
    a.open(_local(b"d\\a", b"x") + _central(b"d/a", 0x10 | (0o751 << 16)) + _eocd())
    assert list(a.contents) == ["d/a"] and a.contents["d/a"].kind == "dir" and a.contents["d/a"].permissions == 0o751


def test_open_entry_errors_and_their_order_cpu():
    crc_bad = _local(b"c.txt", b"data", crc=1)
    size_bad = _local(b"s.txt", b"data", usize=5)
    both_bad = _local(b"b.txt", b"data", crc=1, usize=5)
    stored_bad = _local(b"t.txt", b"data", method=0, crc=2)
    corrupt = _local(b"z.txt", b"data", raw=b"\xff\xff\xff")
    truncated = _local(b"z.txt", b"data" * 100, raw=_deflate(b"data" * 100)[:-3])
    crc_msg = "Verifying archive entry %s CRC-32 failed"
    assert _open_error(crc_bad + _eocd()) == crc_msg % "c.txt"
    assert _open_error(stored_bad + _eocd()) == crc_msg % "t.txt"
    assert _open_error(size_bad + _eocd()) == "Unexpected error verifying s.txt uncompressed size"
    assert _open_error(both_bad + _eocd()) == crc_msg % "b.txt"
    za = _za()
    for data in (corrupt, truncated):
        with pytest.raises(ZippyError) as ei:
            za.ZipArchive(ZlibCtx()).open(data + _eocd())
        assert ei.value.code == 3
    # archive order: the first bad entry wins, and a bad entry before a header error wins over it
    assert _open_error(_local(b"ok", b"1") + size_bad + crc_bad + _eocd()) == \
        "Unexpected error verifying s.txt uncompressed size"
    assert _open_error(crc_bad + _local(b"a", b"x", flag=0x804) + _eocd()) == crc_msg % "c.txt"
    assert _open_error(crc_bad + b"JUNK") == crc_msg % "c.txt"
    assert _open_error(crc_bad + _local(b"a", b"x")[:20]) == crc_msg % "c.txt"
    assert _open_error(_local(b"a", b"x", flag=0x808) + crc_bad + _eocd()) == "Unsupported zip archive, uses deflate64"
    assert _open_error(_local(b"a", b"x") + _central(b"b") + crc_bad + _eocd()) == OPEN_MSG


def test_open_duplicates_and_dates_cpu():
    za = _za()
    a = za.ZipArchive(ZlibCtx())
    a.open(_local(b"a", b"first") + _local(b"b", b"other") + _local(b"a", b"second") + _central(b"a")
           + _central(b"a", 0x10) + _eocd())
    assert list(a.contents) == ["a", "b"] and a.contents["a"].contents == b"second"
    assert a.contents["a"].kind == "dir" and a.contents["b"].permissions == 0
    with _TZ(TZ):
        for tm, dt, want in [((17 << 11) | (13 << 5) | 10, (43 << 9) | (11 << 5) | 14, T1),  # 17:13:20 EST
                             (0, (43 << 9) | (0 << 5) | 14, 0),      # month 0: initDateTime refuses it
                             (0, (43 << 9) | (2 << 5) | 0, 0),       # day 0
                             (0, (44 << 9) | (2 << 5) | 30, 0),      # 30 February
                             (30, (43 << 9) | (11 << 5) | 14, 0),    # 60 seconds
                             ((24 << 11), (43 << 9) | (11 << 5) | 14, 0)]:
            a.open(_local(b"a", b"x", tm=tm, dt=dt) + _eocd())
            assert a.contents["a"].last_modified == want, (tm, dt)


def test_open_fixtures_cpu():
    za = _za()
    assert _open_error(os.path.join(ZDIR, "Bagnon-10.2.31.zip")) == "Unsupported zip archive, uses deflate64"
    assert _open_error(os.path.join(ZDIR, "cat.jpg")) == OPEN_MSG
    v2 = za.create_zip_archive({"a.txt": b"some text", "empty": b""}, ZlibCtx())
    assert _open_error(v2) == EOF_MSG   # ZIP64: its 0xFFFFFFFF sizes run past the end
    for name in sorted(os.listdir(ZDIR)):
        if name.endswith(".zip") and name != "Bagnon-10.2.31.zip":
            try:
                za.ZipArchive(ZlibCtx()).open(os.path.join(ZDIR, name))
            except ZippyError:
                pass   # only the messages above are pinned; nothing else may escape


# ---- directories ----
def _make_tree(root):
    src = root / "src"
    (src / "nested" / "deeper").mkdir(parents=True)
    (src / "a.txt").write_bytes(b"alpha\n" * 1000)
    (src / "empty").write_bytes(b"")
    (src / "nested" / "b.bin").write_bytes(bytes(range(256)) * 41)
    (src / "nested" / "deeper" / "c").write_bytes(b"c" * 70000)
    os.symlink("a.txt", src / "link")          # skipped, as walkDir's pcLinkToFile is
    os.symlink("nested", src / "dirlink")      # and pcLinkToDir
    for i, (f, mode) in enumerate([("a.txt", 0o640), ("empty", 0o600), ("nested/b.bin", 0o755),
                                   ("nested/deeper/c", 0o444)]):
        os.chmod(src / f, mode)
        os.utime(src / f, (1600000000 + i, 1600000000 + 1001 * i))
    return src


TREE_KEYS = ["src/", "src/a.txt", "src/empty", "src/nested/", "src/nested/b.bin", "src/nested/deeper/",
             "src/nested/deeper/c"]


def test_add_dir_add_file_clear_cpu(tmp_path):
    za = _za()
    src = _make_tree(tmp_path)
    a = za.ZipArchive(ZlibCtx())
    a.add_dir(str(src))
    assert sorted(a.contents) == TREE_KEYS and list(a.contents)[0] == "src/"
    e = a.contents["src/nested/b.bin"]
    assert (e.kind, e.contents, e.last_modified, e.permissions) == ("file", bytes(range(256)) * 41, 1600002002, 0o755)
    assert a.contents["src/nested/"] == za.ArchiveEntry("dir")
    a.clear()
    assert a.contents == {}
    a.add_dir(str(src) + "/")    # a trailing '/': keys relative to the directory itself, no entry for it
    assert "src/" not in a.contents and "a.txt" in a.contents and "nested/deeper/c" in a.contents
    a.clear()
    a.add_dir(str(tmp_path / "missing"))
    assert list(a.contents) == ["missing/"]
    a.add_file(str(src / "nested" / "deeper" / "c"))
    a.add_file(str(src / "link"))    # followed
    assert list(a.contents) == ["missing/", "c", "link"] and a.contents["link"].contents == b"alpha\n" * 1000
    assert a.contents["c"].permissions == 0o444
    with pytest.raises(ZippyError) as ei:
        a.add_file(str(src / "nested"))
    assert str(ei.value) == "Error adding file %s to archive, appears to be a directory?" % (src / "nested")
    with pytest.raises(ZippyError) as ei:
        a.add_dir(str(src / "a.txt"))
    assert str(ei.value) == "Error adding dir %s to archive, appears to be a file?" % (src / "a.txt")
    with pytest.raises(OSError):
        a.add_file(str(src / "nope"))


def _compare_tree(src, out):
    want, got = set(), set()
    for root, dirs, files in os.walk(src):
        for nme in dirs + files:
            p = os.path.join(root, nme)
            if not os.path.islink(p):
                want.add(os.path.relpath(p, src))
    for root, dirs, files in os.walk(out):
        got.update(os.path.relpath(os.path.join(root, nme), out) for nme in dirs + files)
    assert got == want
    for rel in want:
        a, b = os.path.join(src, rel), os.path.join(out, rel)
        if os.path.isfile(a):
            assert open(a, "rb").read() == open(b, "rb").read(), rel
            assert os.stat(b).st_mode & 0o777 == os.stat(a).st_mode & 0o777, rel
            assert int(os.stat(b).st_mtime) == os.stat(a).st_mtime_ns // 10 ** 9, rel


def test_extract_all_cpu(tmp_path):
    za = _za()
    src = _make_tree(tmp_path)
    a = za.ZipArchive(ZlibCtx())
    a.add_dir(str(src))
    a.extract_all(str(tmp_path / "out"))
    _compare_tree(str(src), str(tmp_path / "out" / "src"))
    msgs = []
    for dest in [str(tmp_path / "out"), "out_rel", str(tmp_path / "missing" / "x")]:
        with pytest.raises(ZippyError) as ei:
            a.extract_all(dest)
        msgs.append(str(ei.value))
    assert msgs == ["Destination %s already exists" % (tmp_path / "out"),
                    "Path to destination out_rel does not exist",   # splitPath gives no parent to check
                    "Path to destination %s does not exist" % (tmp_path / "missing" / "x")]
    assert not os.path.exists("out_rel")
    E = za.ArchiveEntry
    for bad, msg in [("/abs", "Extracting absolute paths is not supported (/abs)"),
                     ("../up", "Extracting paths starting with `..` is not supported (../up)"),
                     ("..\\up", "Extracting paths starting with `..` is not supported (..\\up)"),
                     ("a/../b", "Extracting paths containing `/../` is not supported (a/../b)"),
                     ("a\\..\\b", "Extracting paths containing `/../` is not supported (a\\..\\b)")]:
        b = za.ZipArchive(ZlibCtx())
        b.contents.update({"ok.txt": E("file", b"1", 0, 0o644), bad: E("file", b"x")})
        with pytest.raises(ZippyError) as ei:
            b.extract_all(str(tmp_path / "bad"))
        assert str(ei.value) == msg
        assert not (tmp_path / "bad").exists()   # ok.txt was written, then everything removed
    # permissions as stored (none: mode 0), the mtime only when after 1970, directories made on the way
    c = za.ZipArchive(ZlibCtx())
    c.contents.update({"d/e/f.txt": E("file", b"f", 0, 0), "g/": E("dir"), "h.txt": E("file", b"h", 1500000001, 0o600)})
    c.extract_all(str(tmp_path / "c") + "/")
    f = tmp_path / "c" / "d" / "e" / "f.txt"
    assert stat.S_IMODE(os.stat(f).st_mode) == 0 and (tmp_path / "c" / "g").is_dir()
    assert os.stat(tmp_path / "c" / "h.txt").st_mtime == 1500000001
    os.chmod(f, 0o644)


def test_create_zip_archive_round_trip_cpu(tmp_path):
    za = _za()
    src = _make_tree(tmp_path)
    dest = tmp_path / "x.zip"
    with _TZ(TZ):
        za.create_zip_archive(str(src), str(dest), ctx=ZlibCtx())
        ref = za.ZipArchive(ZlibCtx())
        ref.add_dir(str(src))
        assert dest.read_bytes() == ref.zip_image()
        with zipfile.ZipFile(dest) as zf:
            assert zf.testzip() is None and sorted(zf.namelist()) == TREE_KEYS
        a = za.ZipArchive(ZlibCtx())
        a.open(str(dest))
        assert list(a.contents) == list(ref.contents)
        for k, e in ref.contents.items():
            assert (a.contents[k].kind, a.contents[k].contents) == (e.kind, e.contents)
    za.create_zip_archive(src, tmp_path / "y.zip", ctx=ZlibCtx())   # a PathLike source
    assert (tmp_path / "y.zip").exists()
    # the mapping form keeps its meaning, with the context positional or by keyword
    blob = za.create_zip_archive({"a": b"x"}, ZlibCtx())
    assert blob == za.create_zip_archive({"a": b"x"}, ctx=ZlibCtx()) and blob[4:6] == b"\x2d\x00"
    with pytest.raises(ZippyError) as ei:
        za.create_zip_archive(str(src / "a.txt"), str(tmp_path / "z.zip"), ctx=ZlibCtx())
    assert "appears to be a file?" in str(ei.value) and not (tmp_path / "z.zip").exists()


# ---- C++ ----
def _cpp_manifest(tmp_path):
    lines = []
    for i, (path, e) in enumerate(_layout_contents().items()):
        data = str(tmp_path / ("data%d" % i))
        with open(data, "wb") as f:
            f.write(e.contents)
        lines.append("%s\t%d\t%o\t%s\t%s" % (e.kind, e.last_modified, e.permissions, path, data))
    (tmp_path / "manifest").write_text("\n".join(lines) + "\n")


def _run_cpp_v1(tmp_path, link_args, ctx):
    """tests/native/cpp_zip_v1_test.cpp: the ZipArchive of include/zippy_b200_zip.hpp must write the bytes
    zippy_b200/ziparchives.py writes for the same entries and times, and read them back."""
    za = _za()
    exe = str(tmp_path / "cpp_zip_v1_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-o", exe, os.path.join(HERE, "native", "cpp_zip_v1_test.cpp")]
                          + link_args)
    _cpp_manifest(tmp_path)
    out = tmp_path / "cppout"
    out.mkdir()
    src = _make_tree(tmp_path)
    with _TZ(TZ):
        r = subprocess.run([exe, str(tmp_path / "manifest"), str(out), str(src)], capture_output=True, text=True,
                           timeout=600)
        assert r.returncode == 0 and r.stdout.strip().split("\n")[-1] == "OK", (r.stdout, r.stderr)
        assert (out / "cpp.zip").read_bytes() == _archive(_layout_contents(), ctx).zip_image()
        za.create_zip_archive(str(src), str(tmp_path / "py.zip"), ctx=ctx)
        assert (out / "create.zip").read_bytes() == (tmp_path / "py.zip").read_bytes()
    _compare_tree(str(src), str(out / "extracted" / "src"))


def test_cpp_zip_v1_cpu(tmp_path):
    native = os.path.join(HERE, "native")
    _run_cpp_v1(tmp_path, [os.path.join(native, "mock_abi_zlib.cpp"), os.path.join(native, "mock_abi_deflate.cpp"),
                           os.path.join(native, "mock_abi_inflate_crc32.cpp"), "-lz"], ZlibCtx())


# ---- the GPU path ----
def _crc_members(z, o, big):
    """(members, raw contents, slot sizes, names): raw deflate from the reference's encoder at 1 / 6 / 9, zlib and
    this library at 1 and Default, plus empty, corrupted and truncated members and a slot that is too small.  With
    `big`, members of 512 KiB and more that take the large-member paths: this library's level-1 chunks (sync
    markers), a foreign zlib stream (speculative segments) and Default-level chunks (whatever decodes them)."""
    from tests import util
    corpus = util.load_corpus()
    T = util.text_corpus(corpus)
    rng = np.random.default_rng(11)
    raws = [corpus["alice29.txt"], corpus["html"], b"", b"a" * 1000, rng.integers(0, 256, 70000, np.uint8).tobytes(),
            corpus["geo.protodata"][:5000]]
    if big:
        raws = [(T + T[::-1])[:2300000], T[:1500000] + rng.integers(0, 256, 200000, np.uint8).tobytes()]
    members, want, names = [], [], []
    for k, r in enumerate(raws):
        for name, enc in [("ref1", lambda b: o.compress(b, 1, o.dfDeflate)), ("ref6", lambda b: o.compress(b, 6, o.dfDeflate)),
                          ("ref9", lambda b: o.compress(b, 9, o.dfDeflate)),
                          ("zlib", lambda b: zlib.compress(b, 6, -15)),
                          ("gpu1", lambda b: z.compress(b, z.BestSpeed, z.dfDeflate)),
                          ("gpuD", lambda b: z.compress(b, z.DefaultCompression, z.dfDeflate))]:
            members.append(enc(r))
            want.append(r)
            names.append("%s/%d" % (name, k))
    sizes = [len(r) for r in want]
    r = want[0]
    c = z.compress(r, z.BestSpeed, z.dfDeflate)
    members += [b"", c[:len(c) // 2], c[:40] + bytes([c[40] ^ 0xA5]) + c[41:], c]
    want += [None, None, None, r]
    sizes += [0, len(r), len(r), len(r) // 3]    # the last: a size claim that is too small
    names += ["empty", "truncated", "corrupted", "small slot"]
    return members, want, sizes, names


def _check_crc_batch(ctx, members, want, sizes, names, pin):
    import zippy_b200 as z
    lens0 = np.array([len(m) for m in members], dtype=np.uint64)
    offs = np.zeros(len(members) + 1, dtype=np.uint64)
    offs[1:] = np.cumsum(lens0)
    base = np.frombuffer(b"".join(members), dtype=np.uint8).copy()
    if pin:
        z.host_register(base.ctypes.data, base.nbytes)
    try:
        out, do, lens, crcs, st = ctx.inflate_batch_crc32(base, offs, sizes)
        out2, do2, lens2, st2 = ctx.uncompress_batch(base, offs, z.dfDeflate, sizes=np.array(sizes, dtype=np.uint64))
    finally:
        if pin:
            z.host_unregister(base.ctypes.data)
    assert list(st) == list(st2)
    assert list(lens) == list(lens2)
    for i, nme in enumerate(names):
        a = out[int(do[i]):int(do[i]) + int(lens[i])].tobytes()
        assert a == out2[int(do2[i]):int(do2[i]) + int(lens2[i])].tobytes(), nme
        if st[i] == 0:
            assert int(crcs[i]) == zlib.crc32(a), nme
            if want[i] is not None:
                assert a == want[i], nme
        else:
            assert int(crcs[i]) == 0, nme
    return st


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["pageable", "pinned", "ungated"])
def test_inflate_batch_crc32_gpu(mode, monkeypatch):
    import zippy_b200 as z
    from oracle import oracle as o
    if mode == "ungated":
        monkeypatch.setenv("ZB200_UNC_GATED", "0")
        monkeypatch.setenv("ZB200_UNC_GROUP_BYTES", "150000")   # several groups
    ctx = z.Context()
    monkeypatch.delenv("ZB200_UNC_GATED", raising=False)
    monkeypatch.delenv("ZB200_UNC_GROUP_BYTES", raising=False)
    try:
        for big in (False, True):
            members, want, sizes, names = _crc_members(z, o, big)
            if big:
                assert sum(len(m) >= 512 << 10 for m in members) >= 6
            st = _check_crc_batch(ctx, members, want, sizes, names, mode == "pinned")
            assert st[names.index("empty")] != 0 and st[names.index("truncated")] != 0
            assert st[names.index("corrupted")] != 0 and st[names.index("small slot")] == 0
    finally:
        ctx.close()


@pytest.mark.gpu
def test_zip_archive_round_trip_gpu(tmp_path):
    from oracle import oracle as o
    from tests.test_tarball_write import _big_tree
    za = _za()
    src = _big_tree(tmp_path, total=64 << 20, seed=20261016)
    dest = tmp_path / "big.zip"
    za.create_zip_archive(str(src), str(dest))
    data = dest.read_bytes()
    with zipfile.ZipFile(dest) as zf:
        assert zf.testzip() is None
        for info in zf.infolist():
            if info.file_size:
                p = info.header_offset + 30 + len(info.filename.encode())
                raw = o.uncompress(data[p:p + info.compress_size], o.dfDeflate)
                assert zlib.crc32(raw) == info.CRC and raw == zf.read(info), info.filename
    a = za.ZipArchive()
    a.open(str(dest))
    ref = za.ZipArchive(ZlibCtx())
    ref.add_dir(str(src))
    assert list(a.contents) == list(ref.contents)
    for k, e in ref.contents.items():
        assert (a.contents[k].kind, a.contents[k].contents) == (e.kind, e.contents), k
    a.extract_all(str(tmp_path / "out"))
    got = {}
    for root, dirs, files in os.walk(tmp_path / "out"):
        for nme in dirs:
            got[os.path.relpath(os.path.join(root, nme), tmp_path / "out") + "/"] = b""
        for nme in files:
            p = os.path.join(root, nme)
            assert stat.S_IMODE(os.stat(p).st_mode) == 0o664   # extractPermissions of an attribute without mode bits
            got[os.path.relpath(p, tmp_path / "out")] = open(p, "rb").read()
    assert got == {k: e.contents for k, e in ref.contents.items()}


@pytest.mark.gpu
def test_cpp_zip_v1_gpu(tmp_path):
    import zippy_b200 as z
    libdir = os.path.join(os.path.dirname(HERE), "zippy_b200")
    _run_cpp_v1(tmp_path, ["-L" + libdir, "-l:libzippy_b200.so", "-Wl,-rpath," + libdir], z.default_context())
