// zippy::compressOptimal and zippy::CompressStream(CompressStream::Optimal{}, ...) (include/zippy_b200.hpp) from C++:
// compress INPUT as one member, and as a stream written in WRITE-byte pieces with a sync flush after the first piece.
// Writes both members; the caller compares them with Python's.
// Usage: cpp_optimal_test INPUT WINDOW_BITS FORMAT FNAME_LEN WRITE OUT_MEMBER OUT_SMEMBER
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <iterator>

#include "../../include/zippy_b200.hpp"

int main(int argc, char **argv) {
  if (argc != 8) {
    fprintf(stderr, "usage: %s INPUT WINDOW_BITS FORMAT FNAME_LEN WRITE OUT_MEMBER OUT_SMEMBER\n", argv[0]);
    return 2;
  }
  std::ifstream in(argv[1], std::ios::binary);
  const std::string input((std::istreambuf_iterator<char>(in)), std::istreambuf_iterator<char>());
  const int window_bits = atoi(argv[2]), fl = atoi(argv[4]);
  const auto fmt = (zippy::CompressedDataFormat)atoi(argv[3]);
  const size_t piece = strtoull(argv[5], 0, 10);
  try {
    // the one-shot form draws a gzip FNAME length at random: raw and zlib members only
    if (fmt != zippy::dfGzip) std::ofstream(argv[6], std::ios::binary) << zippy::compressOptimal(input, fmt, window_bits);
    zippy::CompressStream s(zippy::CompressStream::Optimal{}, fmt, window_bits, fl);
    std::string m;
    for (size_t off = 0; off < input.size(); off += piece) {
      m += s.write(input.substr(off, piece));
      if (off == 0) m += s.flush();
    }
    m += s.finish();
    std::ofstream(argv[7], std::ios::binary) << m;
  } catch (const zippy::ZippyError &e) {
    fprintf(stderr, "ZippyError %d: %s\n", e.code, e.what());
    return 1;
  }
  return 0;
}
