// Exercises the ZipArchive of include/zippy_b200_zip.hpp.  argv[1] = a manifest (one entry per line:
// kind<TAB>mtime<TAB>octal permissions<TAB>path<TAB>file holding the contents), argv[2] = an output directory,
// argv[3] = a source tree.  Writes the manifest's archive (cpp.zip) and createZipArchive's archive of the tree
// (create.zip) for the Python test to compare with zippy_b200/ziparchives.py, opens both again, extracts the tree
// (extracted/), checks the error contract, and prints OK.  Linked against libzippy_b200.so on a GPU box, or
// against mock_abi_zlib.cpp + mock_abi_deflate.cpp + mock_abi_inflate_crc32.cpp on a CPU-only machine.
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <sstream>

#include "../../include/zippy_b200_zip.hpp"

static std::string slurp(const std::string &path) {
  std::ifstream f(path, std::ios::binary);
  std::stringstream ss;
  ss << f.rdbuf();
  return ss.str();
}

static int expect_error(const char *what, const std::string &msg, void (*fn)(const std::string &), const std::string &arg) {
  try {
    fn(arg);
  } catch (const zippy::ZippyError &e) {
    if (msg == e.what()) return 0;
    std::printf("FAILED %s: got \"%s\"\n", what, e.what());
    return 1;
  }
  std::printf("FAILED %s: no error\n", what);
  return 1;
}

static std::string g_out;
static void write_empty(const std::string &path) { zippy::ZipArchive().writeZipArchive(path); }
static void open_data(const std::string &data) { zippy::ZipArchive().openData(data); }
static void add_dir(const std::string &dir) { zippy::ZipArchive().addDir(dir); }
static void add_file(const std::string &path) { zippy::ZipArchive().addFile(path); }
static void extract_into(const std::string &dest) {
  zippy::ZipArchive a;
  zippy::ArchiveEntry e;
  a.set("ok.txt", e);
  a.set("../up", e);
  a.extractAll(dest);
}

int main(int argc, char **argv) {
  if (argc < 4) return 2;
  zippy::ZipArchive archive;
  std::istringstream manifest(slurp(argv[1]));
  for (std::string line; std::getline(manifest, line);) {
    std::istringstream f(line);
    std::string kind, mtime, perms, path, data;
    std::getline(f, kind, '\t');
    std::getline(f, mtime, '\t');
    std::getline(f, perms, '\t');
    std::getline(f, path, '\t');
    std::getline(f, data, '\t');
    zippy::ArchiveEntry e;
    e.kind = kind == "dir" ? zippy::ArchiveEntry::Directory : zippy::ArchiveEntry::File;
    e.lastModified = std::strtoll(mtime.c_str(), nullptr, 10);
    e.permissions = (uint32_t)std::strtoul(perms.c_str(), nullptr, 8);
    e.contents = slurp(data);
    archive.set(path, e);
  }
  const std::string out = argv[2], source = argv[3];
  g_out = out;
  archive.writeZipArchive(out + "/cpp.zip");
  zippy::createZipArchive(source, out + "/create.zip");
  int bad = 0;
  zippy::ZipArchive back;
  back.open(out + "/cpp.zip");
  if (back.entries().size() != archive.entries().size()) {
    std::printf("FAILED read back: %zu entries\n", back.entries().size());
    bad++;
  }
  for (size_t i = 0; i < back.entries().size() && i < archive.entries().size(); i++) {
    const auto &a = archive.entries()[i], &b = back.entries()[i];
    if (a.first != b.first || a.second.contents != b.second.contents || a.second.kind != b.second.kind ||
        b.second.permissions != 0664) {
      std::printf("FAILED read back: entry %s\n", a.first.c_str());
      bad++;
    }
  }
  zippy::ZipArchive tree;
  tree.addDir(source);
  tree.extractAll(out + "/extracted");

  const std::string data = slurp(out + "/cpp.zip");
  std::string crcBad = data;
  crcBad[14] ^= 1;   // the first entry's CRC-32
  bad += expect_error("empty", "Zip archive has no contents", write_empty, out + "/empty.zip");
  bad += expect_error("eof", "Attempted to read past end of file, corrupted zip archive?", open_data, data.substr(0, 40));
  bad += expect_error("crc", "Verifying archive entry a.txt CRC-32 failed", open_data, crcBad);
  bad += expect_error("signature", "Unexpected error opening zip archive", open_data, "PK\x05\x05 and more");
  std::string flag = data;
  flag[6] |= 8;
  bad += expect_error("deflate64", "Unsupported zip archive, uses deflate64", open_data, flag);
  bad += expect_error("dir", "Error adding dir " + out + "/x.d to archive, appears to be a file?", add_dir, out + "/x.d");
  bad += expect_error("file", "Error adding file " + out + " to archive, appears to be a directory?", add_file, out);
  bad += expect_error("exists", "Destination " + out + " already exists", extract_into, out);
  bad += expect_error("relative", "Path to destination rel_out does not exist", extract_into, "rel_out");
  bad += expect_error("dotdot", "Extracting paths starting with `..` is not supported (../up)", extract_into,
                      out + "/bad");
  if (std::ifstream(out + "/empty.zip") || std::ifstream(out + "/bad/ok.txt")) {
    std::printf("FAILED a failed call left its destination\n");
    bad++;
  }
  if (bad) return 1;
  std::printf("OK\n");
  return 0;
}
