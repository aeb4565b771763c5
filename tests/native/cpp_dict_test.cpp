// Preset dictionaries through include/zippy_b200.hpp: compress INPUT against DICT (zippy::compress with a dictionary,
// and a CompressStream with it), decode MEMBER (bytes Python wrote) against DICT (zippy::uncompress and a
// DecompressStream fed one byte at a time).  Writes the C++ member to OUT_MEMBER and the decoded MEMBER to OUT_DATA.
// Usage: cpp_dict_test INPUT DICT LEVEL FORMAT MEMBER OUT_MEMBER OUT_DATA
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <iterator>

#include "../../include/zippy_b200.hpp"

static std::string slurp(const char *path) {
  std::ifstream in(path, std::ios::binary);
  return std::string((std::istreambuf_iterator<char>(in)), std::istreambuf_iterator<char>());
}

int main(int argc, char **argv) {
  if (argc != 8) {
    fprintf(stderr, "usage: %s INPUT DICT LEVEL FORMAT MEMBER OUT_MEMBER OUT_DATA\n", argv[0]);
    return 2;
  }
  const std::string input = slurp(argv[1]), dict = slurp(argv[2]), member = slurp(argv[5]);
  const int level = atoi(argv[3]);
  const auto fmt = (zippy::CompressedDataFormat)atoi(argv[4]);
  try {
    const std::string c = zippy::compress(input, level, fmt, dict);
    zippy::CompressStream cs(level, fmt, dict);
    std::string s;
    for (size_t i = 0; i < input.size(); i += 100000) s += cs.write(input.substr(i, 100000));
    s += cs.finish();
    if (s != c) {
      fprintf(stderr, "the compress stream differs from compress\n");
      return 1;
    }
    if (zippy::uncompress(c, fmt, dict) != input) {
      fprintf(stderr, "uncompress of the C++ member differs from the input\n");
      return 1;
    }
    std::ofstream(argv[6], std::ios::binary) << c;
    const std::string d = zippy::uncompress(member, fmt, dict);
    zippy::DecompressStream ds(fmt, dict);
    std::string r;
    for (char ch : member) r += ds.write(&ch, 1);
    r += ds.finish();
    if (r != d) {
      fprintf(stderr, "the decompress stream differs from uncompress\n");
      return 1;
    }
    std::ofstream(argv[7], std::ios::binary) << d;
  } catch (const zippy::ZippyError &e) {
    fprintf(stderr, "ZippyError %d: %s\n", e.code, e.what());
    return 1;
  }
  return 0;
}
