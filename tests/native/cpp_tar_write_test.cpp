// Exercises the writer of include/zippy_b200_tar.hpp.  argv[1] = a manifest (one entry per line:
// kind<TAB>mtime<TAB>path<TAB>file holding the contents, "-" for none), argv[2] = an output directory,
// argv[3] = a source tree.  Writes writeTarball's .tar and .tar.gz of the manifest and createTarball's
// .tar and .tgz of the tree for the Python test to compare with zippy_b200/tarballs.py, checks the
// error contract, and prints OK.  Linked against libzippy_b200.so on a GPU box, or against
// mock_abi_zlib.cpp + mock_abi_deflate.cpp on a CPU-only machine.
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <sstream>

#include "../../include/zippy_b200_tar.hpp"

static std::string slurp(const std::string &path) {
  std::ifstream f(path, std::ios::binary);
  std::stringstream ss;
  ss << f.rdbuf();
  return ss.str();
}

static void put(const std::string &path, const std::string &data) {
  std::ofstream f(path, std::ios::binary);
  f.write(data.data(), (std::streamsize)data.size());
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

static void write_one(const std::string &path) {
  zippy::TarEntry e;
  e.path = path;
  zippy::writeTarball(std::vector<zippy::TarEntry>(path.empty() ? 0 : 1, e), false);
}

static std::string g_out;
static void create_into(const std::string &name) { zippy::createTarball(g_out, g_out + "/" + name); }
static void create_from(const std::string &source) { zippy::createTarball(source, g_out + "/from.tar"); }

int main(int argc, char **argv) {
  if (argc < 4) return 2;
  std::vector<zippy::TarEntry> entries;
  std::istringstream manifest(slurp(argv[1]));
  for (std::string line; std::getline(manifest, line);) {
    std::istringstream f(line);
    std::string kind, mtime, path, data;
    std::getline(f, kind, '\t');
    std::getline(f, mtime, '\t');
    std::getline(f, path, '\t');
    std::getline(f, data, '\t');
    zippy::TarEntry e;
    e.kind = kind == "dir" ? zippy::TarEntry::Directory : zippy::TarEntry::File;
    e.mtime = std::strtoull(mtime.c_str(), nullptr, 10);
    e.path = path;
    if (data != "-") e.contents = slurp(data);
    entries.push_back(e);
  }
  const std::string out = argv[2], source = argv[3];
  put(out + "/cpp.tar", zippy::writeTarball(entries, false));
  put(out + "/cpp.tar.gz", zippy::writeTarball(entries, true));
  zippy::createTarball(source, out + "/create.tar");
  zippy::createTarball(source, out + "/create.tgz");

  g_out = out;
  const std::string tail99(99, 't'), head154(154, 'h');
  int bad = 0;
  bad += expect_error("empty", "Tarball has no contents", write_one, "");
  bad += expect_error("tail", "File name " + tail99 + "t too long, must be < 100 characters", write_one, tail99 + "t");
  bad += expect_error("head", "File path " + head154 + "h too long, must be < 155 characters", write_one,
                      head154 + "h/x");
  bad += expect_error("extension", "Unsupported tarball extension .zip", create_into, "bad.zip");
  bad += expect_error("missing", "Path " + out + "/missing does not exist", create_from, out + "/missing");
  bad += expect_error("file", "Error adding dir " + out + "/x.d to tarball, appears to be a file?", create_from,
                      out + "/x.d");
  write_one(tail99);                // the longest name and path the reference accepts
  write_one(head154 + "/" + tail99);
  if (std::ifstream(out + "/bad.zip") || std::ifstream(out + "/from.tar")) {
    std::printf("FAILED a failed call wrote its destination\n");
    bad++;
  }
  if (bad) return 1;
  std::printf("OK\n");
  return 0;
}
