// zippy::compressWithIndex and an indexing zippy::CompressStream (include/zippy_b200.hpp) from C++: compress INPUT
// as one gzip / zlib / raw member with its index, and as a stream written in WRITE-byte pieces with a sync flush
// after the first piece.  Writes both members and both exported indexes; the caller compares them with Python's.
// Usage: cpp_compress_index_test INPUT LEVEL FORMAT SPAN FNAME_LEN WRITE OUT_MEMBER OUT_INDEX OUT_SMEMBER OUT_SINDEX
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <iterator>

#include "../../include/zippy_b200.hpp"

int main(int argc, char **argv) {
  if (argc != 11) {
    fprintf(stderr, "usage: %s INPUT LEVEL FORMAT SPAN FNAME_LEN WRITE OUT_MEMBER OUT_INDEX OUT_SMEMBER OUT_SINDEX\n",
            argv[0]);
    return 2;
  }
  std::ifstream in(argv[1], std::ios::binary);
  const std::string input((std::istreambuf_iterator<char>(in)), std::istreambuf_iterator<char>());
  const int level = atoi(argv[2]), fl = atoi(argv[5]);
  const auto fmt = (zippy::CompressedDataFormat)atoi(argv[3]);
  const uint64_t span = strtoull(argv[4], 0, 10), piece = strtoull(argv[6], 0, 10);
  try {
    auto r = zippy::compressWithIndex(input, level, fmt, span, fl);
    std::ofstream(argv[7], std::ios::binary) << r.first;
    std::ofstream(argv[8], std::ios::binary) << r.second.toBytes();
    zippy::CompressStream s(level, fmt, fl, span);
    std::string m;
    for (size_t off = 0; off < input.size(); off += piece) {
      m += s.write(input.substr(off, piece));
      if (off == 0) m += s.flush();
    }
    m += s.finish();
    std::ofstream(argv[9], std::ios::binary) << m;
    std::ofstream(argv[10], std::ios::binary) << s.index().toBytes();
  } catch (const zippy::ZippyError &e) {
    fprintf(stderr, "ZippyError %d: %s\n", e.code, e.what());
    return 1;
  }
  return 0;
}
