// zippy_b200_zip.hpp -- header-only C++ form of the reference's ZIP layer (src/zippy/ziparchives.nim)
// over the batch entry points of include/zippy_b200.h (SURVEY.md 8(f-2)).
//
// The reference's createZipArchive (:458-634) is a loop of crc32 + compress(BestSpeed, dfDeflate)
// over the entries and extractFile (:37-93) a loop of uncompress(dfDeflate) + crc32; here each loop is
// ONE batched call (zb200_compress_batch / zb200_uncompress_batch / zb200_checksum_batch).  The
// container format -- local headers, central directory, ZIP64 records -- stays on the host as in the
// reference; same acceptance checks and error texts.  The Python form is zippy_b200/ziparchives.py.
//
// ZipArchive is the object API of ziparchives_v1.nim (addDir / addFile / open / writeZipArchive / extractAll,
// createZipArchive(source, dest)): its reader decodes every deflated entry in ONE zb200_inflate_batch_crc32 call,
// which also returns each output's CRC-32, and its writer compresses and checksums every entry in one batch each.
#pragma once
#include <fcntl.h>
#include <sys/stat.h>

#include <algorithm>
#include <cstring>
#include <ctime>
#include <filesystem>
#include <fstream>
#include <iterator>
#include <map>
#include <string>
#include <utility>
#include <vector>

#include "zippy_b200.hpp"

namespace zippy {

namespace zipdetail {
constexpr uint32_t kLocal = 0x04034b50u, kCentral = 0x02014b50u, kEocd = 0x06054b50u, kEocd64 = 0x06064b50u,
                   kLoc64 = 0x07064b50u;
constexpr uint64_t kMaxExtractBytes = 1ull << 40;  // one extract call never sizes a buffer beyond this
[[noreturn]] inline void fail(const std::string &msg) { throw ZippyError(ZB200_ERR_UNCOMPRESS, msg); }
[[noreturn]] inline void eof() { fail("Attempted to read past end of file, corrupted archive?"); }
inline uint16_t u16(const std::string &d, size_t p) {
  if (p + 2 > d.size()) eof();
  return (uint16_t)((uint8_t)d[p] | ((uint8_t)d[p + 1] << 8));
}
inline uint32_t u32(const std::string &d, size_t p) {
  if (p + 4 > d.size()) eof();
  return (uint32_t)(uint8_t)d[p] | ((uint32_t)(uint8_t)d[p + 1] << 8) | ((uint32_t)(uint8_t)d[p + 2] << 16) |
         ((uint32_t)(uint8_t)d[p + 3] << 24);
}
inline uint64_t u64(const std::string &d, size_t p) { return (uint64_t)u32(d, p) | ((uint64_t)u32(d, p + 4) << 32); }
inline void put16(std::string &o, uint32_t v) {
  o.push_back((char)(v & 255));
  o.push_back((char)((v >> 8) & 255));
}
inline void put32(std::string &o, uint32_t v) {
  put16(o, v & 0xffffu);
  put16(o, v >> 16);
}
inline void put64(std::string &o, uint64_t v) {
  put32(o, (uint32_t)v);
  put32(o, (uint32_t)(v >> 32));
}
inline bool valid_utf8(const std::string &s) {
  for (size_t i = 0; i < s.size();) {
    unsigned char c = (unsigned char)s[i];
    int n = c < 0x80 ? 0 : (c >> 5) == 6 ? 1 : (c >> 4) == 14 ? 2 : (c >> 3) == 30 ? 3 : -1;
    if (n < 0 || i + n >= s.size() + (n == 0 ? 1 : 0)) return false;
    for (int k = 1; k <= n; k++)
      if (((unsigned char)s[i + k] >> 6) != 2) return false;
    i += n + 1;
  }
  return true;
}
// names that are not UTF-8 are CP437 (ziparchives.nim:116-155): the upper half mapped to Unicode
inline std::string cp437_to_utf8(const std::string &s) {
  static const uint16_t hi[128] = {
      0x00c7, 0x00fc, 0x00e9, 0x00e2, 0x00e4, 0x00e0, 0x00e5, 0x00e7, 0x00ea, 0x00eb, 0x00e8, 0x00ef, 0x00ee, 0x00ec, 0x00c4, 0x00c5,
      0x00c9, 0x00e6, 0x00c6, 0x00f4, 0x00f6, 0x00f2, 0x00fb, 0x00f9, 0x00ff, 0x00d6, 0x00dc, 0x00a2, 0x00a3, 0x00a5, 0x20a7, 0x0192,
      0x00e1, 0x00ed, 0x00f3, 0x00fa, 0x00f1, 0x00d1, 0x00aa, 0x00ba, 0x00bf, 0x2310, 0x00ac, 0x00bd, 0x00bc, 0x00a1, 0x00ab, 0x00bb,
      0x2591, 0x2592, 0x2593, 0x2502, 0x2524, 0x2561, 0x2562, 0x2556, 0x2555, 0x2563, 0x2551, 0x2557, 0x255d, 0x255c, 0x255b, 0x2510,
      0x2514, 0x2534, 0x252c, 0x251c, 0x2500, 0x253c, 0x255e, 0x255f, 0x255a, 0x2554, 0x2569, 0x2566, 0x2560, 0x2550, 0x256c, 0x2567,
      0x2568, 0x2564, 0x2565, 0x2559, 0x2558, 0x2552, 0x2553, 0x256b, 0x256a, 0x2518, 0x250c, 0x2588, 0x2584, 0x258c, 0x2590, 0x2580,
      0x03b1, 0x00df, 0x0393, 0x03c0, 0x03a3, 0x03c3, 0x00b5, 0x03c4, 0x03a6, 0x0398, 0x03a9, 0x03b4, 0x221e, 0x03c6, 0x03b5, 0x2229,
      0x2261, 0x00b1, 0x2265, 0x2264, 0x2320, 0x2321, 0x00f7, 0x2248, 0x00b0, 0x2219, 0x00b7, 0x221a, 0x207f, 0x00b2, 0x25a0, 0x00a0};
  std::string o;
  for (unsigned char c : s) {
    uint32_t u = c < 0x80 ? c : hi[c - 0x80];
    if (u < 0x80) o.push_back((char)u);
    else if (u < 0x800) {
      o.push_back((char)(0xc0 | (u >> 6)));
      o.push_back((char)(0x80 | (u & 63)));
    } else {
      o.push_back((char)(0xe0 | (u >> 12)));
      o.push_back((char)(0x80 | ((u >> 6) & 63)));
      o.push_back((char)(0x80 | (u & 63)));
    }
  }
  return o;
}
}  // namespace zipdetail

// ziparchives.nim:16-29: the records keep the central directory's order
class ZipArchiveReader {
 public:
  struct Record {
    bool isDir = false;
    uint64_t headerOffset = 0, compressedSize = 0, uncompressedSize = 0;
    uint32_t crc = 0;
    std::string path;
  };

  explicit ZipArchiveReader(std::string data) : d_(std::move(data)) { parse(); }

  std::vector<std::string> walkFiles() const {  // ziparchives.nim:31-35
    std::vector<std::string> v;
    for (const Record &r : order_)
      if (!r.isDir) v.push_back(r.path);
    return v;
  }
  const std::vector<Record> &records() const { return order_; }

  // every requested file through ONE batched inflate and ONE batched crc32
  std::map<std::string, std::string> extractFiles(const std::vector<std::string> &names) const {
    using namespace zipdetail;
    std::vector<const Record *> recs;
    for (const std::string &nme : names) {
      auto it = index_.find(nme);
      if (it == index_.end() || order_[it->second].isDir) fail("No file record found for " + nme);
      recs.push_back(&order_[it->second]);
    }
    std::map<std::string, std::string> out;
    std::string packed;
    std::vector<uint64_t> so(1, 0), dofs(1, 0);
    std::vector<const Record *> deflated;
    for (const Record *r : recs) {
      size_t pos = (size_t)r->headerOffset;
      if (pos > d_.size() || d_.size() - pos < 30) eof();
      if (u32(d_, pos) != kLocal) fail("Invalid file header");
      const uint16_t method = u16(d_, pos + 8);
      pos += 30 + (size_t)u16(d_, pos + 26) + u16(d_, pos + 28);
      // sizes come from the archive: no unchecked arithmetic on them
      if (pos > d_.size() || r->compressedSize > d_.size() - pos) eof();
      if (method == 0) out[r->path] = d_.substr(pos, (size_t)r->compressedSize);
      else if (method == 8) {
        packed.append(d_, pos, (size_t)r->compressedSize);
        so.push_back(packed.size());
        // DEFLATE cannot expand more than 1032:1: a larger directory claim can only end in a
        // failed inflate, so never size a buffer by it (same clamp as the Python mirror)
        const uint64_t lim = r->compressedSize * 1032ull + 1024ull;
        const uint64_t want = r->uncompressedSize < lim ? r->uncompressedSize : lim;
        if (want > (uint64_t)kMaxExtractBytes - dofs.back()) fail("Archive too large to extract in one call");
        dofs.push_back(dofs.back() + want);
        deflated.push_back(r);
      } else fail("Unsupported archive, compression method");
    }
    if (!deflated.empty()) {
      const size_t n = deflated.size();
      std::string dst((size_t)dofs.back() + 64, '\0');
      std::vector<uint64_t> lens(n, 0);
      std::vector<int> st(n, 0);
      if (packed.empty()) packed.push_back('\0');
      detail::check(zb200_uncompress_batch(detail::ctx(), detail::u8(packed), so.data(), n, dfDeflate,
                                           reinterpret_cast<uint8_t *>(&dst[0]), dofs.data(), lens.data(), st.data()));
      for (size_t i = 0; i < n; i++) {
        if (st[i] != ZB200_OK) throw ZippyError(st[i], zb200_strerror(st[i]));
        out[deflated[i]->path] = dst.substr((size_t)dofs[i], (size_t)lens[i]);
      }
    }
    // crc32 of every extracted file against the directory (ziparchives.nim:92-93)
    std::string all;
    std::vector<uint64_t> co(1, 0);
    for (const Record *r : recs) {
      all += out[r->path];
      co.push_back(all.size());
    }
    if (!recs.empty()) {
      std::vector<uint32_t> crcs(recs.size(), 0);
      if (all.empty()) all.push_back('\0');
      detail::check(zb200_checksum_batch(detail::ctx(), detail::u8(all), co.data(), recs.size(), 0, crcs.data()));
      for (size_t i = 0; i < recs.size(); i++)
        if (crcs[i] != recs[i]->crc) fail("Verifying crc32 failed");
    }
    return out;
  }
  std::string extractFile(const std::string &path) const { return extractFiles({path})[path]; }  // :37-93

 private:
  void parse() {  // ziparchives.nim:183-395
    using namespace zipdetail;
    const size_t size = d_.size();
    if (size < 22) eof();
    size_t eocd = std::string::npos;
    for (size_t p = size - 22 + 1; p-- > 0;)
      if (u32(d_, p) == kEocd) {
        eocd = p;
        break;
      }
    if (eocd == std::string::npos) eof();
    uint64_t disk, startDisk, nDisk, nTotal, cdSize, cdStart;
    if (eocd >= 20 && u32(d_, eocd - 20) == kLoc64) {
      if (u32(d_, eocd - 16) != 0) fail("Unsupported archive, disk number");
      const uint64_t pos = u64(d_, eocd - 12);
      if (u32(d_, eocd - 4) != 1) fail("Unsupported archive, num disks");
      if (pos > size || size - pos < 64) eof();
      if (u32(d_, (size_t)pos) != kEocd64) fail("Invalid central directory file header");
      disk = u32(d_, (size_t)pos + 16);
      startDisk = u32(d_, (size_t)pos + 20);
      nDisk = u64(d_, (size_t)pos + 24);
      nTotal = u64(d_, (size_t)pos + 32);
      cdSize = u64(d_, (size_t)pos + 40);
      cdStart = u64(d_, (size_t)pos + 48);
    } else {
      disk = u16(d_, eocd + 4);
      startDisk = u16(d_, eocd + 6);
      nDisk = u16(d_, eocd + 8);
      nTotal = u16(d_, eocd + 10);
      cdSize = u32(d_, eocd + 12);
      cdStart = u32(d_, eocd + 16);
    }
    if (disk != 0) fail("Unsupported archive, disk number");
    if (startDisk != 0) fail("Unsupported archive, start disk");
    if (nDisk != nTotal) fail("Unsupported archive, record number");
    // an archive may be appended to another file: find the directory by counting its records
    // backwards from the end, fall back to the recorded offset
    uint64_t socd = cdStart;
    {
      uint64_t found = 0;
      for (size_t p = eocd; nTotal && p-- > 0;)
        if (u32(d_, p) == kCentral && ++found == nTotal) {
          socd = p;
          break;
        }
    }
    const int64_t shift = (int64_t)socd - (int64_t)cdStart;
    size_t pos = (size_t)socd;
    for (uint64_t k = 0; k < nTotal; k++) {
      if (pos + 46 > size) eof();
      if (u32(d_, pos) != kCentral) fail("Invalid central directory file header");
      const uint16_t flags = u16(d_, pos + 8), method = u16(d_, pos + 10);
      Record r;
      r.crc = u32(d_, pos + 16);
      uint64_t csize = u32(d_, pos + 20), usize = u32(d_, pos + 24), hoff = u32(d_, pos + 42);
      const size_t nlen = u16(d_, pos + 28), xlen = u16(d_, pos + 30), clen = u16(d_, pos + 32);
      const uint32_t xattr = u32(d_, pos + 38);
      if (method != 0 && method != 8) fail("Unsupported archive, compression method");
      if (u16(d_, pos + 34) != 0) fail("Invalid file disk number");
      pos += 46;
      if (pos + nlen > size) eof();
      std::string name = d_.substr(pos, nlen);
      pos += nlen;
      for (size_t q = pos; q + 4 <= pos + xlen;) {  // ZIP64 extended information: only the saturated fields
        const uint16_t id = u16(d_, q);
        const size_t flen = u16(d_, q + 2);
        q += 4;
        if (id == 1) {
          size_t z = q;
          for (uint64_t *field : {&usize, &csize, &hoff})
            if (*field == 0xffffffffull) {
              if (z + 8 > q + flen) eof();
              *field = u64(d_, z);
              z += 8;
            }
          break;
        }
        q += flen;
      }
      pos += xlen + clen;
      if (pos > socd + cdSize) fail("Invalid central directory size");
      if (!(flags & 0x800) && !valid_utf8(name)) name = cp437_to_utf8(name);
      if (index_.count(name)) fail("Unsupported archive, duplicate entry");
      r.path = name;
      r.isDir = (xattr & 0x10u) || ((xattr >> 16) & 0040000u) || (!name.empty() && name.back() == '/');
      r.headerOffset = (uint64_t)((int64_t)hoff + shift);
      r.compressedSize = csize;
      r.uncompressedSize = usize;
      index_[name] = order_.size();
      order_.push_back(r);
    }
  }

  std::string d_;
  std::vector<Record> order_;
  std::map<std::string, size_t> index_;
};

// ziparchives.nim:458-634: version 45, UTF-8 flag, ZIP64 extra fields on every entry, entries written
// from the LAST to the first (the reference pops keys off the end of its table), empty files stored,
// everything else deflated at BestSpeed -- in one batch.
inline std::string createZipArchive(const std::vector<std::pair<std::string, std::string>> &entries) {
  using namespace zipdetail;
  std::vector<const std::pair<std::string, std::string> *> order;
  for (auto it = entries.rbegin(); it != entries.rend(); ++it) {
    if (it->first.empty()) fail("Invalid empty file name");
    if (it->first[0] == '/') fail("File paths must be relative");
    if (it->first.size() > 0xffff) fail("File name len > uint16.high");
    order.push_back(&*it);
  }
  const size_t n = order.size();
  std::string base;
  std::vector<uint64_t> so(n + 1, 0), co(n + 1, 0);
  size_t bound = 64;
  for (size_t i = 0; i < n; i++) {
    base += order[i]->second;
    so[i + 1] = base.size();
    bound += zb200_compress_bound(order[i]->second.size(), dfDeflate) + 64;
  }
  std::vector<uint32_t> crcs(n, 0);
  std::string comp(bound, '\0');
  if (n) {
    if (base.empty()) base.push_back('\0');
    detail::check(zb200_checksum_batch(detail::ctx(), detail::u8(base), so.data(), n, 0, crcs.data()));
    detail::check(zb200_compress_batch(detail::ctx(), detail::u8(base), so.data(), n, BestSpeed, dfDeflate, nullptr,
                                       reinterpret_cast<uint8_t *>(&comp[0]), comp.size(), co.data(), nullptr));
  }
  std::time_t now = std::time(nullptr);
  std::tm lt = *std::localtime(&now);
  const uint32_t tm = (uint32_t)((lt.tm_hour << 11) | (lt.tm_min << 5) | (lt.tm_sec / 2));
  const uint32_t dt = (uint32_t)((std::max(0, lt.tm_year + 1900 - 1980) << 9) | ((lt.tm_mon + 1) << 5) | lt.tm_mday);
  struct Rec {
    uint64_t hoff, ulen, clen;
    uint32_t method, crc;
  };
  std::vector<Rec> recs;
  std::string out;
  for (size_t i = 0; i < n; i++) {
    const std::string &nme = order[i]->first;
    const uint64_t ulen = order[i]->second.size();
    const uint64_t clen = ulen ? co[i + 1] - co[i] : 0;
    const uint32_t method = ulen ? 8 : 0;
    recs.push_back({out.size(), ulen, clen, method, crcs[i]});
    put32(out, kLocal);
    put16(out, 45);
    put16(out, 1u << 11);
    put16(out, method);
    put16(out, tm);
    put16(out, dt);
    put32(out, crcs[i]);
    put32(out, 0xffffffffu);
    put32(out, 0xffffffffu);
    put16(out, (uint32_t)nme.size());
    put16(out, 20);
    out += nme;
    put16(out, 1);
    put16(out, 16);
    put64(out, ulen);
    put64(out, clen);
    if (clen) out.append(comp, (size_t)co[i], (size_t)clen);
  }
  const uint64_t cdStart = out.size();
  for (size_t i = 0; i < n; i++) {
    const std::string &nme = order[i]->first;
    put32(out, kCentral);
    put16(out, 45);
    put16(out, 45);
    put16(out, 1u << 11);
    put16(out, recs[i].method);
    put16(out, tm);
    put16(out, dt);
    put32(out, recs[i].crc);
    put32(out, 0xffffffffu);
    put32(out, 0xffffffffu);
    put16(out, (uint32_t)nme.size());
    put16(out, 28);
    put16(out, 0);
    put16(out, 0);
    put16(out, 0);
    put32(out, 0);
    put32(out, 0xffffffffu);
    out += nme;
    put16(out, 1);
    put16(out, 24);
    put64(out, recs[i].ulen);
    put64(out, recs[i].clen);
    put64(out, recs[i].hoff);
  }
  const uint64_t cdEnd = out.size();
  put32(out, kEocd64);
  put64(out, 44);
  put16(out, 45);
  put16(out, 45);
  put32(out, 0);
  put32(out, 0);
  put64(out, n);
  put64(out, n);
  put64(out, cdEnd - cdStart);
  put64(out, cdStart);
  put32(out, kLoc64);
  put32(out, 0);
  put64(out, cdEnd);
  put32(out, 1);
  put32(out, kEocd);
  put16(out, 0);
  put16(out, 0);
  put16(out, 0xffff);
  put16(out, 0xffff);
  put32(out, 0xffffffffu);
  put32(out, 0xffffffffu);
  put16(out, 0);
  return out;
}

// ---- the ZipArchive object (ziparchives_v1.nim) ----
struct ArchiveEntry {  // ziparchives_v1.nim:15-19
  enum Kind { File, Directory } kind = File;
  std::string contents;
  int64_t lastModified = 0;  // Unix seconds
  uint32_t permissions = 0;  // mode bits
};

namespace zipv1 {
[[noreturn]] inline void failEof() { zipdetail::fail("Attempted to read past end of file, corrupted zip archive?"); }
[[noreturn]] inline void failOpen() { zipdetail::fail("Unexpected error opening zip archive"); }
// Nim's os.splitPath: (head, tail) around the last '/'
inline std::pair<std::string, std::string> splitPath(const std::string &p) {
  const size_t i = p.rfind('/');
  if (i == std::string::npos) return {"", p};
  return {i ? p.substr(0, i) : "/", p.substr(i + 1)};
}
// Nim's os.splitFile(path).ext: the last '.' suffix of the last component ("" for a dotfile)
inline std::string ext(const std::string &p) {
  const std::string name = p.substr(p.rfind('/') == std::string::npos ? 0 : p.rfind('/') + 1);
  for (size_t j = name.size() >= 2 ? name.size() - 2 : 0; j > 0; j--)
    if (name[j] == '.' && name[j + 1] != '.') return name.substr(j);
  return "";
}
inline std::string join(const std::string &a, const std::string &b) {
  if (a.empty()) return b;
  if (b.empty()) return a;
  return a.back() == '/' ? a + b : a + "/" + b;
}
inline bool dirExists(const std::string &p) {
  struct stat sb;
  return !p.empty() && ::stat(p.c_str(), &sb) == 0 && S_ISDIR(sb.st_mode);
}
// toMsDos (ziparchives_v1.nim:351-369)
inline std::pair<uint32_t, uint32_t> toMsDos(int64_t t) {
  const std::time_t tt = (std::time_t)t;
  std::tm lt;
  localtime_r(&tt, &lt);
  return {(uint32_t)((lt.tm_hour << 11) | (lt.tm_min << 5) | (lt.tm_sec / 2)) & 0xffffu,
          (uint32_t)((std::max(0, lt.tm_year + 1900 - 1980) << 9) | ((lt.tm_mon + 1) << 5) | lt.tm_mday) & 0xffffu};
}
// ziparchives_v1.nim:161-179; 0 for out-of-range fields and for a date initDateTime rejects
inline int64_t fromMsDos(uint32_t tm, uint32_t dt) {
  const int sec = (tm & 31) * 2, mi = (tm >> 5) & 63, ho = (tm >> 11) & 31;
  const int day = dt & 31, mon = (dt >> 5) & 15, yr = ((dt >> 9) & 127) + 1980;
  static const int dim[12] = {31, 28, 31, 30, 31, 30, 31, 31, 30, 31, 30, 31};
  const bool leap = yr % 4 == 0 && (yr % 100 != 0 || yr % 400 == 0);
  if (sec > 59 || mi > 59 || ho > 23 || mon < 1 || mon > 12 || day < 1 || day > dim[mon - 1] + (mon == 2 && leap))
    return 0;
  std::tm lt{};
  lt.tm_year = yr - 1900;
  lt.tm_mon = mon - 1;
  lt.tm_mday = day;
  lt.tm_hour = ho;
  lt.tm_min = mi;
  lt.tm_sec = sec;
  lt.tm_isdst = -1;
  return (int64_t)std::mktime(&lt);
}
inline std::string readFile(const std::string &path) {
  std::ifstream f(path, std::ios::binary);
  if (!f) throw std::runtime_error("Unable to read " + path);
  return std::string(std::istreambuf_iterator<char>(f), std::istreambuf_iterator<char>());
}
inline void writeFile(const std::string &path, const std::string &data) {
  std::ofstream f(path, std::ios::binary);
  f.write(data.data(), (std::streamsize)data.size());
  if (!f) throw std::runtime_error("Unable to write " + path);
}
}  // namespace zipv1

// ziparchives_v1.nim:21-22: path -> entry in insertion order; directory keys end in '/'
class ZipArchive {
 public:
  const std::vector<std::pair<std::string, ArchiveEntry>> &entries() const { return order_; }
  ArchiveEntry *find(const std::string &path) {
    auto it = index_.find(path);
    return it == index_.end() ? nullptr : &order_[it->second].second;
  }
  // contents[path] = entry: a new path goes to the end, an existing one keeps its place
  void set(const std::string &path, ArchiveEntry e) {
    if (ArchiveEntry *old = find(path)) *old = std::move(e);
    else {
      index_[path] = order_.size();
      order_.emplace_back(path, std::move(e));
    }
  }
  void clear() {
    order_.clear();
    index_.clear();
  }

  // ziparchives_v1.nim:24-54
  void addDir(const std::string &dir) {
    if (!zipv1::ext(dir).empty()) zipdetail::fail("Error adding dir " + dir + " to archive, appears to be a file?");
    const auto ht = zipv1::splitPath(dir);
    addDir(ht.first, ht.second);
  }
  // ziparchives_v1.nim:56-74 (a symlink is followed)
  void addFile(const std::string &path) {
    struct stat sb;
    if (::stat(path.c_str(), &sb) != 0) throw std::runtime_error("Unable to stat " + path);
    if (!S_ISREG(sb.st_mode)) zipdetail::fail("Error adding file " + path + " to archive, appears to be a directory?");
    ArchiveEntry e;
    e.contents = zipv1::readFile(path);
    e.lastModified = (int64_t)sb.st_mtime;
    e.permissions = (uint32_t)(sb.st_mode & 0777);
    set(zipv1::splitPath(path).second, std::move(e));
  }

  // ziparchives_v1.nim:371-481: the archive bytes (see zippy_b200/ziparchives.py ZipArchive.zip_image)
  std::string zipImage() const {
    using namespace zipdetail;
    if (order_.empty()) fail("Zip archive has no contents");
    const size_t n = order_.size();
    std::string base, fullBase;
    std::vector<uint64_t> so(n + 1, 0), fo(1, 0), co;
    std::vector<size_t> full;
    size_t bound = 64;
    for (size_t i = 0; i < n; i++) {
      const std::string &c = order_[i].second.contents;
      base += c;
      so[i + 1] = base.size();
      if (!c.empty()) {
        full.push_back(i);
        fullBase += c;
        fo.push_back(fullBase.size());
        bound += zb200_compress_bound(c.size(), dfDeflate) + 64;
      }
    }
    std::vector<uint32_t> crcs(n, 0);
    if (base.empty()) base.push_back('\0');
    detail::check(zb200_checksum_batch(detail::ctx(), detail::u8(base), so.data(), n, 0, crcs.data()));
    std::string comp(bound, '\0');
    co.assign(full.size() + 1, 0);
    if (!full.empty())
      detail::check(zb200_compress_batch(detail::ctx(), detail::u8(fullBase), fo.data(), full.size(), DefaultCompression,
                                         dfDeflate, nullptr, reinterpret_cast<uint8_t *>(&comp[0]), comp.size(),
                                         co.data(), nullptr));
    std::vector<std::string> data(n);
    for (size_t k = 0; k < full.size(); k++) data[full[k]] = comp.substr((size_t)co[k], (size_t)(co[k + 1] - co[k]));
    std::string out, cd;
    for (size_t i = 0; i < n; i++) {
      const std::string &path = order_[i].first;
      const ArchiveEntry &e = order_[i].second;
      // the method is 0 when splitFile(path).name is empty (a "dir/" key) or there are no contents; the data is
      // the deflate stream whenever there are contents, as the reference writes it
      const uint32_t method = (path.empty() || path.back() == '/' || e.contents.empty()) ? 0 : 8;
      const auto td = zipv1::toMsDos(e.lastModified);
      std::string fixed;
      put16(fixed, 0x800);
      put16(fixed, method);
      put16(fixed, td.first);
      put16(fixed, td.second);
      put32(fixed, crcs[i]);
      put32(fixed, (uint32_t)data[i].size());
      put32(fixed, (uint32_t)e.contents.size());
      put16(fixed, (uint32_t)path.size() & 0xffffu);
      put16(fixed, 0);
      put32(cd, kCentral);
      put16(cd, 63);
      put16(cd, 20);
      cd += fixed;
      put16(cd, 0);
      put16(cd, 0);
      put16(cd, 0);
      put32(cd, e.kind == ArchiveEntry::Directory ? 0x10 : 0x20);
      put32(cd, (uint32_t)out.size());
      cd += path;
      put32(out, kLocal);
      put16(out, 20);
      out += fixed;
      out += path;
      out += data[i];
    }
    const uint64_t cdStart = out.size(), cdSize = cd.size();
    out += cd;
    put32(out, kEocd);
    put16(out, 0);
    put16(out, 0);
    put16(out, (uint32_t)n & 0xffffu);
    put16(out, (uint32_t)n & 0xffffu);
    put32(out, (uint32_t)cdSize);
    put32(out, (uint32_t)cdStart);
    put16(out, 0);
    return out;
  }
  // ziparchives_v1.nim:371-486: nothing is written on error
  void writeZipArchive(const std::string &path) const { zipv1::writeFile(path, zipImage()); }

  // ziparchives_v1.nim:105-349 (see zippy_b200/ziparchives.py ZipArchive.open): walk the headers, decode every
  // entry before the first header error, then raise in archive order
  void openData(const std::string &d) {
    using namespace zipdetail;
    clear();
    struct Local {
      std::string name;
      uint32_t method, crc, usize;
      int64_t mtime;
      size_t pos, csize;
    };
    struct Step {
      bool local;
      size_t idx;
      std::string name;
      uint32_t xattr;
    };
    std::vector<Local> locals;
    std::vector<Step> steps;
    std::string headerError;
    const size_t size = d.size();
    try {
      for (size_t pos = 0;;) {
        if (pos + 4 > size) zipv1::failEof();
        const uint32_t sig = u32(d, pos);
        if (sig == kLocal) {
          if (pos + 30 > size) zipv1::failEof();
          const uint32_t flag = u16(d, pos + 6), method = u16(d, pos + 8);
          Local l;
          l.mtime = zipv1::fromMsDos(u16(d, pos + 10), u16(d, pos + 12));
          l.method = method;
          l.crc = u32(d, pos + 14);
          l.csize = u32(d, pos + 18);
          l.usize = u32(d, pos + 22);
          const size_t nlen = u16(d, pos + 26), xlen = u16(d, pos + 28);
          pos += 30;
          if (flag & 4) fail("Unsupported zip archive, data descriptor bit set");
          if (flag & 8) fail("Unsupported zip archive, uses deflate64");
          if (method != 0 && method != 8) fail("Unsupported zip archive compression method " + std::to_string(method));
          if (pos + nlen + xlen > size) zipv1::failEof();
          l.name = d.substr(pos, nlen);
          pos += nlen + xlen;
          if (pos + l.csize > size) zipv1::failEof();
          l.pos = pos;
          steps.push_back({true, locals.size(), "", 0});
          locals.push_back(l);
          pos += l.csize;
        } else if (sig == kCentral) {
          if (pos + 46 > size) zipv1::failEof();
          const size_t nlen = u16(d, pos + 28), xlen = u16(d, pos + 30), clen = u16(d, pos + 32);
          const uint32_t xattr = u32(d, pos + 38);
          pos += 46;
          if (pos + nlen + xlen + clen > size) zipv1::failEof();
          steps.push_back({false, 0, d.substr(pos, nlen), xattr});
          pos += nlen + xlen + clen;
        } else if (sig == kEocd) {
          if (pos + 22 > size) zipv1::failEof();
          if (pos + 22 + u16(d, pos + 20) > size) zipv1::failEof();
          break;
        } else {
          zipv1::failOpen();
        }
      }
    } catch (const ZippyError &e) {
      headerError = e.what();
    }
    // decode: deflated entries in one inflate_batch_crc32, stored ones in one checksum_batch
    const size_t n = locals.size();
    std::vector<std::string> outs(n);
    std::vector<uint32_t> crcs(n, 0);
    std::vector<int> status(n, 0);
    for (int method : {8, 0}) {
      std::vector<size_t> idx;
      std::string packed;
      std::vector<uint64_t> so(1, 0), dofs(1, 0);
      for (size_t i = 0; i < n; i++)
        if ((int)locals[i].method == method) {
          idx.push_back(i);
          packed.append(d, locals[i].pos, locals[i].csize);
          so.push_back(packed.size());
          const uint64_t lim = (uint64_t)locals[i].csize * 1032ull + 1024ull;
          dofs.push_back(dofs.back() + std::min<uint64_t>(locals[i].usize, lim));
        }
      if (idx.empty()) continue;
      const size_t m = idx.size();
      if (packed.empty()) packed.push_back('\0');
      std::vector<uint32_t> c(m, 0);
      if (method == 0) {
        detail::check(zb200_checksum_batch(detail::ctx(), detail::u8(packed), so.data(), m, 0, c.data()));
        for (size_t k = 0; k < m; k++) {
          outs[idx[k]] = d.substr(locals[idx[k]].pos, locals[idx[k]].csize);
          crcs[idx[k]] = c[k];
        }
        continue;
      }
      std::string dst((size_t)dofs.back() + 64, '\0');
      std::vector<uint64_t> lens(m, 0);
      std::vector<int> st(m, 0);
      detail::check(zb200_inflate_batch_crc32(detail::ctx(), detail::u8(packed), so.data(), m,
                                              reinterpret_cast<uint8_t *>(&dst[0]), dofs.data(), lens.data(), c.data(),
                                              st.data()));
      for (size_t k = 0; k < m; k++) {
        const size_t i = idx[k];
        if (st[k] == ZB200_ERR_DST_TOO_SMALL) {  // the header's size understated the content: decode it alone
          try {
            outs[i] = uncompress(d.data() + locals[i].pos, locals[i].csize, dfDeflate);
            crcs[i] = crc32(outs[i]);
          } catch (const ZippyError &e) {
            status[i] = e.code;
          }
        } else if (st[k] != ZB200_OK) {
          status[i] = st[k];
        } else {
          outs[i] = dst.substr((size_t)dofs[k], (size_t)lens[k]);
          crcs[i] = c[k];
        }
      }
    }
    for (const Step &s : steps) {
      if (s.local) {
        const Local &l = locals[s.idx];
        if (status[s.idx]) throw ZippyError(status[s.idx], zb200_strerror(status[s.idx]));
        if (crcs[s.idx] != l.crc) fail("Verifying archive entry " + l.name + " CRC-32 failed");
        if (outs[s.idx].size() != l.usize) fail("Unexpected error verifying " + l.name + " uncompressed size");
        ArchiveEntry e;
        e.contents = std::move(outs[s.idx]);
        e.lastModified = l.mtime;
        std::string key = l.name;
        std::replace(key.begin(), key.end(), '\\', '/');
        set(key, std::move(e));
      } else {
        ArchiveEntry *e = find(s.name);  // looked up as written, not unix-pathed
        if (!e) zipv1::failOpen();
        if (s.xattr & 0x10) e->kind = ArchiveEntry::Directory;
        const uint32_t perms = s.xattr >> 16;
        e->permissions = perms == 0 ? 0664 : perms & 0777;  // extractPermissions, ziparchives_v1.nim:84-103
      }
    }
    if (!headerError.empty()) fail(headerError);
  }
  void open(const std::string &path) { openData(zipv1::readFile(path)); }

  // ziparchives_v1.nim:488-546
  void extractAll(const std::string &dest) const {
    namespace fs = std::filesystem;
    if (zipv1::dirExists(dest)) zipdetail::fail("Destination " + dest + " already exists");
    const auto ht = zipv1::splitPath(dest);
    if (!ht.second.empty() && !zipv1::dirExists(ht.first))
      zipdetail::fail("Path to destination " + dest + " does not exist");
    try {
      for (const auto &pe : order_) {
        const std::string &path = pe.first;
        const ArchiveEntry &e = pe.second;
        if (!path.empty() && path[0] == '/')
          zipdetail::fail("Extracting absolute paths is not supported (" + path + ")");
        if (path.rfind("../", 0) == 0 || path.rfind("..\\", 0) == 0)
          zipdetail::fail("Extracting paths starting with `..` is not supported (" + path + ")");
        if (path.find("/../") != std::string::npos || path.find("\\..\\") != std::string::npos)
          zipdetail::fail("Extracting paths containing `/../` is not supported (" + path + ")");
        const std::string target = zipv1::join(dest, path);
        if (e.kind == ArchiveEntry::Directory) {
          fs::create_directories(target);
        } else {
          fs::create_directories(zipv1::join(dest, zipv1::splitPath(path).first));
          zipv1::writeFile(target, e.contents);
          if (e.lastModified > 0) {
            struct timespec ts[2];
            ts[0].tv_sec = ts[1].tv_sec = (time_t)e.lastModified;
            ts[0].tv_nsec = ts[1].tv_nsec = 0;
            if (::utimensat(AT_FDCWD, target.c_str(), ts, 0) != 0) throw std::runtime_error("Unable to set the time of " + target);
          }
          fs::permissions(target, (fs::perms)e.permissions, fs::perm_options::replace);
        }
      }
    } catch (...) {
      std::error_code ec;
      fs::remove_all(dest, ec);
      throw;
    }
  }

 private:
  void addDir(const std::string &base, const std::string &relative) {
    namespace fs = std::filesystem;
    if (!relative.empty() && !index_.count(relative)) {
      ArchiveEntry d;
      d.kind = ArchiveEntry::Directory;
      set(relative + "/", d);
    }
    std::error_code ec;
    fs::directory_iterator it(zipv1::join(base, relative), ec);
    if (ec) return;  // walkDir yields nothing for a path it cannot open
    for (const fs::directory_entry &de : it) {
      const std::string rel = zipv1::join(relative, de.path().filename().string());
      const fs::file_status st = de.symlink_status();
      if (fs::is_regular_file(st)) {
        struct stat sb;
        if (::lstat(de.path().c_str(), &sb) != 0) throw std::runtime_error("Unable to stat " + de.path().string());
        ArchiveEntry e;
        e.contents = zipv1::readFile(de.path().string());
        e.lastModified = (int64_t)sb.st_mtime;
        e.permissions = (uint32_t)(sb.st_mode & 0777);
        set(rel, std::move(e));
      } else if (fs::is_directory(st)) {
        addDir(base, rel);
      }  // symlinks and other kinds are skipped
    }
  }

  std::vector<std::pair<std::string, ArchiveEntry>> order_;
  std::map<std::string, size_t> index_;
};

// ziparchives_v1.nim:548-555: every directory and file inside source, written to the file dest
inline void createZipArchive(const std::string &source, const std::string &dest) {
  ZipArchive a;
  a.addDir(source);
  a.writeZipArchive(dest);
}

}  // namespace zippy
