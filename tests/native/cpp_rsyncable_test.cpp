// zippy::compressRsyncable and zippy::compressRsyncableBatch (include/zippy_b200.hpp) from C++: compress INPUT as one
// member, and INPUT and its first half as a batch.  Writes the three members; the caller compares them with Python's.
// Usage: cpp_rsyncable_test INPUT LEVEL FORMAT FNAME_LEN OUT_MEMBER OUT_BATCH0 OUT_BATCH1
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <iterator>

#include "../../include/zippy_b200.hpp"

int main(int argc, char **argv) {
  if (argc != 8) {
    fprintf(stderr, "usage: %s INPUT LEVEL FORMAT FNAME_LEN OUT_MEMBER OUT_BATCH0 OUT_BATCH1\n", argv[0]);
    return 2;
  }
  std::ifstream in(argv[1], std::ios::binary);
  const std::string input((std::istreambuf_iterator<char>(in)), std::istreambuf_iterator<char>());
  const int level = atoi(argv[2]), fl = atoi(argv[4]);
  const auto fmt = (zippy::CompressedDataFormat)atoi(argv[3]);
  try {
    std::ofstream(argv[5], std::ios::binary) << zippy::compressRsyncable(input, level, fmt, fl);
    const auto b = zippy::compressRsyncableBatch({input, input.substr(0, input.size() / 2)}, level, fmt,
                                                 {(uint8_t)fl, (uint8_t)fl});
    std::ofstream(argv[6], std::ios::binary) << b[0];
    std::ofstream(argv[7], std::ios::binary) << b[1];
  } catch (const zippy::ZippyError &e) {
    fprintf(stderr, "ZippyError %d: %s\n", e.code, e.what());
    return 1;
  }
  return 0;
}
