// Per-member preset dictionaries through include/zippy_b200.hpp: compressBatch with a window, a dictionary table and
// dictOf, written to OUT (to be compared with Python's bytes); uncompressBatch of Python's members PY must give back
// the items.  ITEMS, DICTS, PY and OUT hold (u64 little-endian length, bytes) records; OF holds int32 dictOf.
// Usage: cpp_dicts_test ITEMS DICTS OF LEVEL FORMAT WINDOW_BITS PY OUT
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iterator>

#include "../../include/zippy_b200.hpp"

static std::string slurp(const char *path) {
  std::ifstream in(path, std::ios::binary);
  return std::string((std::istreambuf_iterator<char>(in)), std::istreambuf_iterator<char>());
}

static std::vector<std::string> records(const std::string &s) {
  std::vector<std::string> r;
  for (size_t p = 0; p + 8 <= s.size();) {
    uint64_t n = 0;
    memcpy(&n, s.data() + p, 8);
    r.push_back(s.substr(p + 8, n));
    p += 8 + n;
  }
  return r;
}

int main(int argc, char **argv) {
  if (argc != 9) {
    fprintf(stderr, "usage: %s ITEMS DICTS OF LEVEL FORMAT WINDOW_BITS PY OUT\n", argv[0]);
    return 2;
  }
  const std::vector<std::string> items = records(slurp(argv[1])), dicts = records(slurp(argv[2])),
                                  py = records(slurp(argv[7]));
  const std::string ofs = slurp(argv[3]);
  std::vector<int32_t> of(ofs.size() / 4);
  memcpy(of.data(), ofs.data(), of.size() * 4);
  const int level = atoi(argv[4]), windowBits = atoi(argv[6]);
  const auto fmt = (zippy::CompressedDataFormat)atoi(argv[5]);
  try {
    const std::vector<std::string> c = zippy::compressBatch(items, level, fmt, windowBits, dicts, of);
    if (zippy::uncompressBatch(py, fmt, dicts, of) != items || zippy::uncompressBatch(c, fmt, dicts, of) != items) {
      fprintf(stderr, "uncompressBatch differs from the items\n");
      return 1;
    }
    std::ofstream out(argv[8], std::ios::binary);
    for (const std::string &m : c) {
      const uint64_t n = m.size();
      out.write(reinterpret_cast<const char *>(&n), 8);
      out << m;
    }
  } catch (const zippy::ZippyError &e) {
    fprintf(stderr, "ZippyError %d: %s\n", e.code, e.what());
    return 1;
  }
  return 0;
}
