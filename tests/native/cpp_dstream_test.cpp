// zippy::DecompressStream (include/zippy_b200.hpp) from C++: decode a compressed file in pieces of a given size and
// write the concatenated output.  Usage: cpp_dstream_test IN OUT FORMAT PIECE
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <iterator>

#include "../../include/zippy_b200.hpp"

int main(int argc, char **argv) {
  if (argc != 5) {
    fprintf(stderr, "usage: %s IN OUT FORMAT PIECE\n", argv[0]);
    return 2;
  }
  std::ifstream in(argv[1], std::ios::binary);
  const std::string src((std::istreambuf_iterator<char>(in)), std::istreambuf_iterator<char>());
  const size_t piece = (size_t)atol(argv[4]);
  std::string out;
  try {
    zippy::DecompressStream s((zippy::CompressedDataFormat)atoi(argv[3]));
    for (size_t off = 0; off < src.size(); off += piece) out += s.write(src.substr(off, piece));
    out += s.finish();
  } catch (const zippy::ZippyError &e) {
    fprintf(stderr, "ZippyError %d: %s\n", e.code, e.what());
    return 1;
  }
  std::ofstream(argv[2], std::ios::binary).write(out.data(), (std::streamsize)out.size());
  return 0;
}
