// zippy_b200_tar.hpp -- header-only C++ form of the reference's tarball reader
// (src/zippy/tarballs.nim:25-141) and writer (tarballs_v1.nim:203-342) over include/zippy_b200.hpp
// (SURVEY.md 8(f-3)).
//
// A .tar.gz is ONE gzip member: it goes through zippy::uncompress (GPU path; large members made
// of independent pieces are decoded in parallel, see DESIGN.md row f-1), then the 512-byte header walk
// runs on the host as in the reference: ustar prefix, GNU 'L' long names, files / directories /
// symlinks, pax and vendor records skipped, anything else is an error, unsafe paths rejected.
// writeTarball builds the reference's ustar layout on the host; a .tar.gz is that image compressed as
// ONE gzip member at DefaultCompression through zippy::compress (the GPU path).
// The Python form (with extraction to disk) is zippy_b200/tarballs.py.
#pragma once
#include <sys/stat.h>

#include <filesystem>
#include <fstream>
#include <iterator>
#include <string>
#include <utility>
#include <vector>

#include "zippy_b200.hpp"

namespace zippy {

struct TarEntry {
  enum Kind { File, Directory, Symlink } kind = File;
  std::string path;      // prefix/name, or the preceding 'L' record
  std::string contents;  // file bytes, or the link target
  uint32_t mode = 0;
  uint64_t mtime = 0;
};

namespace tardetail {
[[noreturn]] inline void fail(const std::string &msg) { throw ZippyError(ZB200_ERR_UNCOMPRESS, msg); }
// tarballs.nim:5-23: the first run of ASCII digits in the field, base 8 (0 if there is none)
inline uint64_t oct(const std::string &d, size_t pos, size_t n) {
  size_t i = pos, end = pos + n;
  while (i < end && !(d[i] >= '0' && d[i] <= '9')) i++;
  uint64_t v = 0;
  for (; i < end && d[i] >= '0' && d[i] <= '9'; i++) {
    if (d[i] > '7') fail("invalid octal digit");
    v = v * 8 + (uint64_t)(d[i] - '0');
  }
  return v;
}
inline std::string cstr(const std::string &d, size_t pos, size_t n) {
  size_t k = 0;
  while (k < n && d[pos + k] != '\0') k++;
  return d.substr(pos, k);
}
inline void check_safe(const std::string &path) {  // internal.nim verifyPathIsSafeToExtract
  if (!path.empty() && (path[0] == '/' || path[0] == '\\')) fail("Absolute path not allowed " + path);
  if (path.size() > 1 && path[1] == ':') fail("Absolute path not allowed " + path);
  size_t a = 0;
  while (a <= path.size()) {
    size_t b = path.find_first_of("/\\", a);
    if (b == std::string::npos) b = path.size();
    if (path.compare(a, b - a, "..") == 0) fail("Path ../ not allowed " + path);
    a = b + 1;
  }
}
// strutils.toOct(x, n): the low n octal digits of x, zero-padded
inline std::string toOct(uint64_t x, int n) {
  std::string s((size_t)n, '0');
  for (int j = n - 1; j >= 0; j--, x >>= 3) s[(size_t)j] = (char)('0' + (x & 7));
  return s;
}
// Nim's os.splitPath: (head, tail) around the last '/'
inline std::pair<std::string, std::string> splitPath(const std::string &p) {
  const size_t i = p.rfind('/');
  if (i == std::string::npos) return {std::string(), p};
  return {i ? p.substr(0, i) : std::string("/"), p.substr(i + 1)};
}
// Nim's os.splitFile(path).ext: the last '.' suffix of the last path component ("" for a dotfile)
inline std::string ext(const std::string &path) {
  const size_t s = path.rfind('/');
  const std::string name = s == std::string::npos ? path : path.substr(s + 1);
  for (size_t k = name.size(); k > 2; k--)
    if (name[k - 2] == '.' && name[k - 1] != '.') return name.substr(k - 2);
  return std::string();
}
inline bool supportedExt(const std::string &e) { return e == ".tar" || e == ".gz" || e == ".taz" || e == ".tgz"; }
// tarballs_v1.nim:210-261: per entry, one 512-byte ustar header and the contents zero-padded to 512 bytes;
// then two zero records
inline std::string image(const std::vector<TarEntry> &entries) {
  if (entries.empty()) fail("Tarball has no contents");
  std::string data;
  for (const TarEntry &e : entries) {
    const std::pair<std::string, std::string> ht = splitPath(e.path);
    if (ht.first.size() >= 155) fail("File path " + ht.first + " too long, must be < 155 characters");
    if (ht.second.size() >= 100) fail("File name " + ht.second + " too long, must be < 100 characters");
    if (e.kind == TarEntry::Symlink) fail("Unsupported tarball entry kind symlink");
    std::string h = ht.second;
    h.resize(100);
    h += std::string("000777 \0", 8);
    h += toOct(0, 6) + std::string(" \0", 2);
    h += toOct(0, 6) + std::string(" \0", 2);
    h += toOct(e.contents.size(), 11) + ' ';
    h += toOct(e.mtime, 11) + ' ';
    h += "        ";  // the checksum field counts as spaces
    h += e.kind == TarEntry::File ? '0' : '5';
    h.resize(257);
    h += std::string("ustar\0", 6) + toOct(0, 2);
    h.resize(329);
    h += toOct(0, 6) + std::string("\0 ", 2);
    h += toOct(0, 6) + std::string("\0 ", 2);
    h += ht.first;
    h.resize(512);
    uint64_t sum = 0;
    for (unsigned char c : h) sum += c;
    h.replace(148, 7, toOct(sum, 6) + '\0');  // byte 155 stays a space
    data += h;
    data += e.contents;
    data.resize((data.size() + 511) & ~(size_t)511);
  }
  data.resize(data.size() + 1024);
  return data;
}
// tarballs_v1.nim:21-43: relative itself, every directory and regular file under base/relative
inline void addDir(std::vector<TarEntry> &out, const std::string &base, const std::string &relative) {
  namespace fs = std::filesystem;
  const fs::path full = fs::path(base) / relative;
  std::error_code ec;
  if (!fs::exists(full, ec)) fail("Path " + full.string() + " does not exist");
  if (!relative.empty()) {
    TarEntry d;
    d.kind = TarEntry::Directory;
    d.path = relative;
    out.push_back(d);
  }
  if (!fs::is_directory(full, ec)) return;
  for (const fs::directory_entry &d : fs::directory_iterator(full)) {
    const std::string name = d.path().filename().string();
    const std::string rel = relative.empty() ? name : relative + "/" + name;
    const fs::file_status st = d.symlink_status();
    if (fs::is_regular_file(st)) {
      struct stat sb;
      if (::lstat(d.path().c_str(), &sb) != 0) fail("Unable to stat " + d.path().string());
      std::ifstream f(d.path(), std::ios::binary);
      TarEntry e;
      e.path = rel;
      e.contents.assign(std::istreambuf_iterator<char>(f), std::istreambuf_iterator<char>());
      e.mode = (uint32_t)(sb.st_mode & 0777);
      e.mtime = (uint64_t)(int64_t)sb.st_mtime;
      out.push_back(e);
    } else if (fs::is_directory(st)) {
      addDir(out, base, rel);
    }  // symlinks and other kinds are skipped
  }
}
}  // namespace tardetail

// tarballs_v1.nim:203-269: the tarball of `entries` (File and Directory only; a path's head must be < 155
// bytes and its tail < 100), gzip-compressed as one member at DefaultCompression when `gzip` is set.
inline std::string writeTarball(const std::vector<TarEntry> &entries, bool gzip) {
  std::string data = tardetail::image(entries);
  return gzip ? compress(data, DefaultCompression, dfGzip) : data;
}

// tarballs_v1.nim:333-342: every directory and regular file inside source (paths relative to source's
// parent) written to dest as .tar, or as .gz / .taz / .tgz through the GPU compressor.  Nothing is
// written to dest on error.
inline void createTarball(const std::string &source, const std::string &dest) {
  using namespace tardetail;
  if (!ext(source).empty()) fail("Error adding dir " + source + " to tarball, appears to be a file?");
  const std::pair<std::string, std::string> ht = splitPath(source);
  std::vector<TarEntry> entries;
  addDir(entries, ht.first, ht.second);
  std::string data = image(entries);
  const std::string e = ext(dest);
  if (!supportedExt(e)) fail("Unsupported tarball extension " + e);
  if (e != ".tar") data = compress(data, DefaultCompression, dfGzip);
  std::ofstream f(dest, std::ios::binary);
  f.write(data.data(), (std::streamsize)data.size());
  if (!f) throw std::runtime_error("Unable to write " + dest);
}

// The entries of a .tar or .tar.gz held in memory (tarballs.nim:40-123 without the file system part).
inline std::vector<TarEntry> readTarball(const std::string &file) {
  using namespace tardetail;
  if (file.size() < 2) fail("Invalid buffer, unable to uncompress");
  const bool gz = (unsigned char)file[0] == 31 && (unsigned char)file[1] == 139;
  const std::string data = gz ? uncompress(file, dfGzip) : file;
  std::vector<TarEntry> out;
  std::string longName;
  size_t pos = 0;
  while (pos < data.size()) {
    if (pos + 512 > data.size()) fail("Attempted to read past end of file, corrupted tarball?");
    const std::string name = cstr(data, pos, 100);
    const uint64_t mode = oct(data, pos + 100, 7), size = oct(data, pos + 124, 11), mtime = oct(data, pos + 136, 11);
    const char typeflag = data[pos + 156];
    const std::string linkname = cstr(data, pos + 157, 100);
    const std::string prefix = cstr(data, pos + 257, 6) == "ustar" ? cstr(data, pos + 345, 155) : std::string();
    pos += 512;
    if (pos + size > data.size()) fail("Attempted to read past end of file, corrupted tarball?");
    if (!name.empty() || !longName.empty()) {
      TarEntry e;
      if (!longName.empty()) {
        e.path = longName;
        longName.clear();
      } else {
        e.path = prefix.empty() ? name : prefix + "/" + name;
      }
      check_safe(e.path);
      e.mode = (uint32_t)mode;
      e.mtime = mtime;
      if (typeflag == '0' || typeflag == '\0') {
        e.kind = TarEntry::File;
        e.contents = data.substr(pos, (size_t)size);
        out.push_back(e);
      } else if (typeflag == '5') {
        e.kind = TarEntry::Directory;
        out.push_back(e);
      } else if (typeflag == '2') {
        e.kind = TarEntry::Symlink;
        e.contents = linkname;
        out.push_back(e);
      } else if (typeflag == 'L') {
        longName = cstr(data, pos, (size_t)size);
      } else if (typeflag == 'g' || typeflag == 'x' || (typeflag >= 'A' && typeflag <= 'Z')) {
        // pax and vendor records: skipped, as in the reference
      } else {
        fail(std::string("Unsupported header type ") + typeflag);
      }
    }
    pos += (size_t)((size + 511) & ~(uint64_t)511);
  }
  return out;
}

}  // namespace zippy
