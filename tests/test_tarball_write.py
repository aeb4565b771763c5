"""SURVEY.md 8(f-3), the writer: `Tarball` / `create_tarball` (zippy_b200/tarballs.py) and `writeTarball` /
`createTarball` (include/zippy_b200_tar.hpp) against the byte layout of tarballs_v1.nim:210-261.

not-gpu: headers rebuilt field by field from that layout, Python's tarfile, `tar` where present and
read_tarball agree on the image; round trips and the C++ writer run with zlib as the gzip.  gpu: the
.tar.gz member comes from the GPU compressor (zlib and the oracle inflate it), a tarball of 64 MiB and
more is one multi-chunk member that reads back through the GPU path, and the C++ writer runs on
libzippy_b200.so."""
import datetime
import os
import shutil
import subprocess
import tarfile
import zlib

import numpy as np
import pytest

from zippy_b200 import ZippyError

HERE = os.path.dirname(os.path.abspath(__file__))
ZLIB_GZ = lambda b: zlib.compress(b, 6, 31)  # noqa: E731
ZLIB_GUNZIP = lambda b: zlib.decompress(b, 31)  # noqa: E731
TAIL99 = "t" * 99   # the longest name the reference accepts
HEAD154 = "h" * 154  # the longest prefix it accepts


def _field_header(tail, head, size, mtime, typeflag):
    """One header written field by field from the layout of tarballs_v1.nim:229-255."""
    h = bytearray(512)
    h[0:100] = tail.ljust(100, b"\0")
    h[100:108] = b"000777 \0"
    h[108:116] = b"000000 \0"
    h[116:124] = b"000000 \0"
    h[124:136] = b"%011o " % size
    h[136:148] = b"%011o " % mtime
    h[148:156] = b" " * 8
    h[156:157] = typeflag
    h[257:263] = b"ustar\0"
    h[263:265] = b"00"
    h[329:337] = b"000000\0 "
    h[337:345] = b"000000\0 "
    h[345:345 + len(head)] = head
    h[148:155] = b"%06o\0" % sum(h)
    return bytes(h)


def _layout_contents():
    import zippy_b200.tarballs as tb
    E = tb.TarballEntry
    return {
        "src": E("dir"),
        "src/a.txt": E("file", b"alpha\n" * 1000, 1700000000, 0o640),
        "src/empty": E("file", b"", 1600000000, 0o600),
        "src/nested": E("dir"),
        "src/nested/deeper": E("dir"),
        "src/nested/deeper/b.bin": E("file", bytes(range(256)) * 3 + b"x", 1234567890, 0o755),
        TAIL99: E("file", b"long name", 1500000000, 0o644),
        HEAD154 + "/" + TAIL99: E("file", b"long path" * 100, 1400000000, 0o644),
    }


def _expected_image(contents):
    out = b""
    for path, e in contents.items():
        head, _, tail = path.rpartition("/")
        out += _field_header(tail.encode(), head.encode(), len(e.contents), e.last_modified,
                             b"5" if e.kind == "dir" else b"0")
        out += e.contents + bytes(-len(e.contents) % 512)
    return out + bytes(1024)


def test_tar_image_layout_cpu():
    import zippy_b200.tarballs as tb
    contents = _layout_contents()
    image = tb.tar_image(contents)
    assert image == _expected_image(contents)
    assert len(image) % 512 == 0 and image[-1024:] == bytes(1024)
    pos = 0
    for path, e in contents.items():
        h = image[pos:pos + 512]
        assert h[100:108] == b"000777 \0"  # 0777 whatever the entry's permissions
        # the checksum of POSIX: every byte, the checksum field counted as 8 spaces; byte 155 stays a space
        assert int(h[148:154], 8) == sum(h[:148]) + 8 * 32 + sum(h[156:])
        assert h[154:156] == b"\0 "
        if e.kind == "dir":
            assert h[124:136] == b"00000000000 " and h[136:148] == b"00000000000 "
        pos += 512 + len(e.contents) + (-len(e.contents) % 512)
    longest = h  # the last header: 154-byte prefix, 99-byte name
    assert longest[:99] == TAIL99.encode() and longest[99] == 0 and longest[345:499] == HEAD154.encode()


def test_tar_image_readers_agree_cpu(tmp_path):
    import zippy_b200.tarballs as tb
    contents = _layout_contents()
    p = tmp_path / "x.tar"
    t = tb.Tarball()
    t.contents.update(contents)
    t.write_tarball(str(p))
    assert p.read_bytes() == tb.tar_image(contents)
    with tarfile.open(p) as tf:
        members = tf.getmembers()
        assert [m.name for m in members] == list(contents)
        for m, e in zip(members, contents.values()):
            assert m.isdir() == (e.kind == "dir") and m.isfile() == (e.kind == "file")
            assert (m.size, m.mtime, m.mode, m.uid, m.gid) == (len(e.contents), e.last_modified, 0o777, 0, 0)
            if m.isfile():
                assert tf.extractfile(m).read() == e.contents
    got = tb.read_tarball(p.read_bytes())
    assert [(k, path, payload if k == "file" else b"", mode, mtime) for k, path, payload, mode, mtime in got] == \
        [(e.kind, path, e.contents, 0o777, e.last_modified) for path, e in contents.items()]
    t2 = tb.Tarball()
    t2.open(str(p))
    assert list(t2.contents) == list(contents)
    for path, e in contents.items():
        if e.kind == "file":
            assert t2.contents[path] == tb.TarballEntry("file", e.contents, e.last_modified, 0o777)
        else:
            assert t2.contents[path] == tb.TarballEntry("dir")


def test_tar_image_gnu_tar_agrees_cpu(tmp_path):
    import zippy_b200.tarballs as tb
    if shutil.which("tar") is None:
        pytest.skip("no tar binary")
    contents = _layout_contents()
    p = tmp_path / "x.tar"
    p.write_bytes(tb.tar_image(contents))
    env = dict(os.environ, TZ="UTC0", LC_ALL="C")
    lines = subprocess.run(["tar", "--full-time", "-tvf", str(p)], capture_output=True, text=True, env=env,
                           check=True).stdout.splitlines()
    assert len(lines) == len(contents)
    for line, (path, e) in zip(lines, contents.items()):
        perms, owner, size, day, clock, name = line.split(None, 5)
        when = datetime.datetime.fromtimestamp(e.last_modified, datetime.timezone.utc)
        assert perms == ("d" if e.kind == "dir" else "-") + "rwxrwxrwx"
        assert owner == "0/0" and int(size) == len(e.contents)
        assert (day, clock) == (when.strftime("%Y-%m-%d"), when.strftime("%H:%M:%S"))
        assert name == path  # directories are written without a trailing '/', as the reference does
        if e.kind == "file":
            assert subprocess.run(["tar", "-xOf", str(p), path], capture_output=True, check=True).stdout == e.contents


def _make_tree(root):
    src = root / "src"
    (src / "nested" / "deeper").mkdir(parents=True)
    (src / "a.txt").write_bytes(b"alpha\n" * 1000)
    (src / "empty").write_bytes(b"")
    (src / "nested" / "b.bin").write_bytes(bytes(range(256)) * 41)
    (src / "nested" / "deeper" / "c").write_bytes(b"c" * 70000)
    os.symlink("a.txt", src / "link")          # skipped, as walkDir's pcLinkToFile is
    os.symlink("nested", src / "dirlink")      # and pcLinkToDir
    os.chmod(src / "a.txt", 0o640)
    for i, f in enumerate(["a.txt", "empty", "nested/b.bin", "nested/deeper/c"]):
        os.utime(src / f, (1600000000 + i, 1600000000 + 1000 * i))
    return src


def _compare_tree(src, out):
    """Every directory and regular file of src is in out with its bytes and whole-second mtime, at mode
    0777; symlinks are left out."""
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
            assert os.stat(b).st_mode & 0o777 == 0o777, rel
            assert int(os.stat(b).st_mtime) == os.stat(a).st_mtime_ns // 10 ** 9, rel


def test_add_dir_cpu(tmp_path):
    import zippy_b200.tarballs as tb
    src = _make_tree(tmp_path)
    t = tb.Tarball()
    t.add_dir(str(src))
    assert sorted(t.contents) == ["src", "src/a.txt", "src/empty", "src/nested", "src/nested/b.bin",
                                  "src/nested/deeper", "src/nested/deeper/c"]
    assert list(t.contents)[0] == "src"
    a = t.contents["src/a.txt"]
    assert (a.kind, a.contents, a.last_modified, a.permissions) == ("file", b"alpha\n" * 1000, 1600000000, 0o640)
    assert t.contents["src/nested"] == tb.TarballEntry("dir")
    t.clear()
    assert t.contents == {}
    t.add_dir(str(src) + "/")  # a trailing '/': the entries are relative to the directory itself
    assert "src" not in t.contents and "a.txt" in t.contents and "nested/deeper/c" in t.contents


@pytest.mark.parametrize("name", ["x.tar", "x.tar.gz", "x.taz", "x.tgz"])
def test_create_tarball_round_trip_cpu(tmp_path, name):
    import zippy_b200.tarballs as tb
    src = _make_tree(tmp_path)
    dest = tmp_path / name
    tb.create_tarball(str(src), str(dest), gzip=ZLIB_GZ)
    data = dest.read_bytes()
    t = tb.Tarball()
    t.add_dir(str(src))
    image = tb.tar_image(t.contents)
    assert (data if name == "x.tar" else zlib.decompress(data, 31)) == image
    tb.extract_all(str(dest), str(tmp_path / "out"), ZLIB_GUNZIP)
    _compare_tree(str(src), str(tmp_path / "out" / "src"))
    t2 = tb.Tarball()
    t2.open(str(dest), ZLIB_GUNZIP)
    t2.extract_all(str(tmp_path / "out2"))
    _compare_tree(str(src), str(tmp_path / "out2" / "src"))
    with pytest.raises(ZippyError, match="already exists"):
        t2.extract_all(str(tmp_path / "out2"))


def test_write_errors_cpu(tmp_path):
    import zippy_b200.tarballs as tb
    src = _make_tree(tmp_path)
    E = tb.TarballEntry

    def check(msg, fn, dest):
        with pytest.raises(ZippyError) as ei:
            fn(str(dest))
        assert str(ei.value) == msg
        assert not os.path.exists(dest)

    def write(contents):
        def fn(dest):
            t = tb.Tarball()
            t.contents.update(contents)
            t.write_tarball(dest, gzip=ZLIB_GZ)
        return fn

    check("Tarball has no contents", write({}), tmp_path / "a.tar")
    check("File name %st too long, must be < 100 characters" % TAIL99, write({TAIL99 + "t": E()}), tmp_path / "b.tar")
    check("File path %sh too long, must be < 155 characters" % HEAD154, write({HEAD154 + "h/x": E()}),
          tmp_path / "c.tgz")
    check("Unsupported tarball extension .zip", lambda d: tb.create_tarball(str(src), d, gzip=ZLIB_GZ),
          tmp_path / "d.zip")
    check("Unsupported tarball extension ", lambda d: tb.create_tarball(str(src), d, gzip=ZLIB_GZ), tmp_path / "e")
    missing = str(tmp_path / "missing")
    check("Path %s does not exist" % missing, lambda d: tb.create_tarball(missing, d), tmp_path / "f.tar")
    check("Error adding dir %s to tarball, appears to be a file?" % (src / "a.txt"),
          lambda d: tb.create_tarball(str(src / "a.txt"), d), tmp_path / "g.tar")
    (tmp_path / "h.zip").write_bytes(b"x")
    with pytest.raises(ZippyError, match="Unsupported tarball extension .zip"):
        tb.Tarball().open(str(tmp_path / "h.zip"))
    with pytest.raises(ZippyError, match="Path ../ not allowed"):
        t = tb.Tarball()
        t.contents["../evil"] = E("file", b"x")
        t.extract_all(str(tmp_path / "out"))
    assert not (tmp_path / "out").exists()


def _run_cpp_writer(tmp_path, link_args, gunzip):
    """tests/native/cpp_tar_write_test.cpp: writeTarball / createTarball of include/zippy_b200_tar.hpp must
    write what zippy_b200/tarballs.py writes for the same entries and the same tree."""
    import zippy_b200.tarballs as tb
    exe = str(tmp_path / "cpp_tar_write_test")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-o", exe, os.path.join(HERE, "native", "cpp_tar_write_test.cpp")]
                          + link_args)
    contents = _layout_contents()
    lines = []
    for i, (path, e) in enumerate(contents.items()):
        data = "-"
        if e.kind == "file":
            data = str(tmp_path / ("data%d" % i))
            with open(data, "wb") as f:
                f.write(e.contents)
        lines.append("%s\t%d\t%s\t%s" % (e.kind, e.last_modified, path, data))
    (tmp_path / "manifest").write_text("\n".join(lines) + "\n")
    out = tmp_path / "cppout"
    out.mkdir()
    src = _make_tree(tmp_path)
    r = subprocess.run([exe, str(tmp_path / "manifest"), str(out), str(src)], capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0 and r.stdout.strip().split("\n")[-1] == "OK", (r.stdout, r.stderr)
    image = tb.tar_image(contents)
    assert (out / "cpp.tar").read_bytes() == image
    gz = (out / "cpp.tar.gz").read_bytes()
    assert gz[:4] == b"\x1f\x8b\x08\x08" and zlib.decompress(gz, 31) == image and gunzip(gz) == image
    tb.create_tarball(str(src), str(tmp_path / "py.tar"))
    want = (tmp_path / "py.tar").read_bytes()
    assert (out / "create.tar").read_bytes() == want
    assert zlib.decompress((out / "create.tgz").read_bytes(), 31) == want


def test_cpp_tar_writer_cpu(tmp_path):
    native = os.path.join(HERE, "native")
    _run_cpp_writer(tmp_path, [os.path.join(native, "mock_abi_zlib.cpp"), os.path.join(native, "mock_abi_deflate.cpp"),
                               "-lz"], ZLIB_GUNZIP)


# ---- the GPU path ----
def _fname_ok(member):
    """gzip header of zippy.nim:21-42: FNAME set, 0..25 letters 'a', 'b', ... then NUL."""
    assert member[:4] == b"\x1f\x8b\x08\x08"
    k = member.index(b"\0", 10) - 10
    assert k <= 25 and member[10:10 + k] == bytes(range(97, 97 + k))


@pytest.mark.gpu
def test_tar_gz_written_by_gpu(tmp_path):
    import zippy_b200.tarballs as tb
    from oracle import oracle as o
    src = _make_tree(tmp_path)
    dest = tmp_path / "x.tar.gz"
    tb.create_tarball(str(src), str(dest))
    t = tb.Tarball()
    t.add_dir(str(src))
    image = tb.tar_image(t.contents)
    member = dest.read_bytes()
    _fname_ok(member)
    assert zlib.decompress(member, 31) == image
    assert o.uncompress(member) == image
    tb.extract_all(str(dest), str(tmp_path / "out"))
    _compare_tree(str(src), str(tmp_path / "out" / "src"))
    t2 = tb.Tarball()
    t2.open(str(dest))
    assert list(t2.contents) == list(t.contents)


def _big_tree(root, total=68 << 20, seed=20261015):
    """A seeded tree of `total` bytes: text windows of the test corpus, runs and random bytes, in files of
    0..4 MiB across nested directories."""
    from tests import util
    T = util.text_corpus(util.load_corpus())
    rng = np.random.default_rng(seed)
    src = root / "big"
    done, i = 0, 0
    while done < total:
        d = src / ("d%d" % (i % 5)) / ("e%d" % (i % 3))
        d.mkdir(parents=True, exist_ok=True)
        n = int(min(rng.integers(0, 4 << 20), total - done))
        kind = i % 3
        if kind == 0:
            o = int(rng.integers(0, len(T)))
            data = (T * (2 + n // len(T)))[o:o + n]
        elif kind == 1:
            runs = rng.integers(1, 256, n // 64 + 1)
            data = np.repeat(rng.integers(0, 256, len(runs), dtype=np.uint8), runs)[:n].tobytes()
        else:
            data = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        (d / ("f%d.bin" % i)).write_bytes(data)
        os.utime(d / ("f%d.bin" % i), (1700000000 + i, 1700000000 + i))
        done += len(data)
        i += 1
    return src


@pytest.mark.gpu
def test_large_tarball_is_one_multichunk_member_gpu(tmp_path):
    import zippy_b200.tarballs as tb
    from zippy_b200 import default_context
    src = _big_tree(tmp_path)
    dest = tmp_path / "big.tar.gz"
    t = tb.Tarball()
    t.add_dir(str(src))
    image = tb.tar_image(t.contents)
    assert len(image) >= 64 << 20
    t.write_tarball(str(dest))
    assert default_context().timing()["n_chunks"] > 1
    member = dest.read_bytes()
    _fname_ok(member)
    d = zlib.decompressobj(31)
    assert d.decompress(member) == image and d.eof and d.unused_data == b""  # exactly one gzip member
    tb.extract_all(str(dest), str(tmp_path / "out"))
    _compare_tree(str(src), str(tmp_path / "out" / "big"))


@pytest.mark.gpu
def test_cpp_tar_writer_gpu(tmp_path):
    from oracle import oracle as o
    libdir = os.path.join(os.path.dirname(HERE), "zippy_b200")
    _run_cpp_writer(tmp_path, ["-L" + libdir, "-l:libzippy_b200.so", "-Wl,-rpath," + libdir], o.uncompress)
