// zippy::Index (include/zippy_b200.hpp) from C++: build the index of a member, write its exported bytes, read it
// back with fromBytes and check that both give the same points and the same range.  Writes the range to OUT_RANGE.
// Usage: cpp_index_test MEMBER FORMAT SPAN OUT_INDEX OFFSET LENGTH OUT_RANGE
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <iterator>

#include "../../include/zippy_b200.hpp"

int main(int argc, char **argv) {
  if (argc != 8) {
    fprintf(stderr, "usage: %s MEMBER FORMAT SPAN OUT_INDEX OFFSET LENGTH OUT_RANGE\n", argv[0]);
    return 2;
  }
  std::ifstream in(argv[1], std::ios::binary);
  const std::string member((std::istreambuf_iterator<char>(in)), std::istreambuf_iterator<char>());
  try {
    zippy::Index idx = zippy::Index::build(member, (zippy::CompressedDataFormat)atoi(argv[2]), strtoull(argv[3], 0, 10));
    const std::string bytes = idx.toBytes();
    std::ofstream(argv[4], std::ios::binary) << bytes;
    zippy::Index back = zippy::Index::fromBytes(bytes);
    const auto a = idx.points(), b = back.points();
    if (a.size() != b.size() || back.size() != idx.size() || back.toBytes() != bytes) {
      fprintf(stderr, "the imported index differs\n");
      return 1;
    }
    for (size_t i = 0; i < a.size(); i++)
      if (a[i].bit != b[i].bit || a[i].out != b[i].out || a[i].crc != b[i].crc || a[i].window != b[i].window) {
        fprintf(stderr, "point %zu differs\n", i);
        return 1;
      }
    const uint64_t off = strtoull(argv[5], 0, 10), len = strtoull(argv[6], 0, 10);
    const std::string r = idx.extract(member, off, len);
    if (back.extract(member, off, len) != r) {
      fprintf(stderr, "the imported index reads other bytes\n");
      return 1;
    }
    std::ofstream(argv[7], std::ios::binary) << r;
  } catch (const zippy::ZippyError &e) {
    fprintf(stderr, "ZippyError %d: %s\n", e.code, e.what());
    return 1;
  }
  return 0;
}
