// zippy::CompressStream::flush and zippy::DecompressStream::drain (include/zippy_b200.hpp) from C++: compress a
// file as messages of a given size, each followed by a sync flush; a receiver writes what each flush emitted and
// drains.  Fails unless it has then read exactly the messages so far.  Writes the compressed member to OUT.
// Usage: cpp_flush_test IN OUT LEVEL FORMAT MSG
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <iterator>

#include "../../include/zippy_b200.hpp"

int main(int argc, char **argv) {
  if (argc != 6) {
    fprintf(stderr, "usage: %s IN OUT LEVEL FORMAT MSG\n", argv[0]);
    return 2;
  }
  std::ifstream in(argv[1], std::ios::binary);
  const std::string src((std::istreambuf_iterator<char>(in)), std::istreambuf_iterator<char>());
  const auto fmt = (zippy::CompressedDataFormat)atoi(argv[4]);
  const size_t msg = (size_t)atol(argv[5]);
  // member bytes from which the receiver's header is decided: 19, and for gzip (FNAME of length 0 here: 11 bytes of
  // header) the header and 9 bytes more; raw streams at once
  const size_t decided = fmt == zippy::dfDeflate ? 0 : fmt == zippy::dfGzip ? 20 : 19;
  std::string member, got;
  try {
    zippy::CompressStream tx(atoi(argv[3]), fmt, 0);
    zippy::DecompressStream rx(fmt);
    for (size_t off = 0; off < src.size(); off += msg) {
      std::string piece = tx.write(src.substr(off, msg));
      piece += tx.flush();
      member += piece;
      got += rx.write(piece);
      got += rx.drain();
      const size_t upto = std::min(src.size(), off + msg);
      if (member.size() >= decided && got != src.substr(0, upto)) {
        fprintf(stderr, "after %zu bytes: read %zu bytes\n", upto, got.size());
        return 1;
      }
    }
    const std::string tail = tx.finish();
    member += tail;
    got += rx.write(tail);
    got += rx.finish();
    if (got != src) {
      fprintf(stderr, "finish: read %zu bytes of %zu\n", got.size(), src.size());
      return 1;
    }
  } catch (const zippy::ZippyError &e) {
    fprintf(stderr, "ZippyError %d: %s\n", e.code, e.what());
    return 1;
  }
  std::ofstream(argv[2], std::ios::binary).write(member.data(), (std::streamsize)member.size());
  return 0;
}
