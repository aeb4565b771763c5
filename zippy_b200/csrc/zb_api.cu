// zb_api.cu -- the C ABI (include/zippy_b200.h): context, device scratch, host<->device
// staging and the launch sequences.  No codec logic lives here and nothing here falls
// back to the CPU: every data byte is produced by the kernels in zb_deflate.cu /
// zb_inflate.cu.
#include <cuda.h>
#include <cuda_runtime.h>
#include <execinfo.h>
#include <signal.h>
#include <stdio.h>
#include <unistd.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <condition_variable>
#include <deque>
#include <functional>
#include <memory>
#include <mutex>
#include <thread>
#include <unordered_map>
#include <string>
#include <vector>

#include "../../include/zippy_b200.h"
#include "zb_kernels.h"
#include "zb_wrapper.h"

namespace {

struct DevBuf {
  void *p = nullptr;
  size_t cap = 0;
};

// Stream memory operations (driver API, fetched at run time: the library links the runtime only).  A wait on a
// device word lets the D2H stream follow the progress of ONE persistent inflate launch, group by group.
struct StreamMemOps {
  CUresult (*wait32)(CUstream, CUdeviceptr, cuuint32_t, unsigned int) = nullptr;
  CUresult (*write32)(CUstream, CUdeviceptr, cuuint32_t, unsigned int) = nullptr;
  bool ok = false;
};
StreamMemOps load_stream_memops() {
  StreamMemOps m;
  void *f1 = nullptr, *f2 = nullptr;
  cudaDriverEntryPointQueryResult q1, q2;
  if (cudaGetDriverEntryPoint("cuStreamWaitValue32", &f1, cudaEnableDefault, &q1) == cudaSuccess && q1 == cudaDriverEntryPointSuccess &&
      cudaGetDriverEntryPoint("cuStreamWriteValue32", &f2, cudaEnableDefault, &q2) == cudaSuccess && q2 == cudaDriverEntryPointSuccess &&
      f1 && f2) {
    m.wait32 = reinterpret_cast<decltype(m.wait32)>(f1);
    m.write32 = reinterpret_cast<decltype(m.write32)>(f2);
    m.ok = true;
  } else {
    (void)cudaGetLastError();
  }
  return m;
}

constexpr size_t kMaxChunksPerGroup = 32768;  // device-resident batches: 2 GiB of input per launch group
constexpr size_t kHostGroupChunks = 4096;     // host batches: 256 MiB groups so transfers overlap the kernels
// A compress stream launches once this much input is pending: smaller writes are gathered, as every launch costs
// five kernels and a sync.  Of 16 / 64 / 256 MiB, 64 was the fastest at levels 1 and Default on one H100 80GB HBM3
// at 700 W (tools/bench_compress_stream.py, DESIGN.md section 8 "Compress streams").
constexpr size_t ZB_STREAM_BATCH_BYTES = 64u << 20;
// A decompress stream launches once this much compressed payload is pending (tools/bench_decompress_stream.py,
// DESIGN.md section 8 "Decompress streams"), and one launch produces at most about kDstreamMaxOut bytes.
constexpr size_t ZB_DSTREAM_BATCH_BYTES = 64u << 20;
constexpr uint64_t kDstreamMaxOut = 1ull << 30;

}  // namespace

// ---- pageable host memory ----
// cudaMemcpyAsync only overlaps with kernels for page-locked memory; a caller's ordinary buffer (a Nim
// string, malloc, numpy) would make every copy block.  Such buffers are staged through a ring of pinned
// slots: a few host threads memcpy a slice into a slot while the DMA engine drains the previous one.
class CopyPool {
 public:
  ~CopyPool() { stop(); }
  void start(int n) {
    if (!th_.empty()) return;
    for (int i = 0; i < n; i++) th_.emplace_back([this] { work(); });
  }
  void stop() {
    {
      std::lock_guard<std::mutex> lk(m_);
      quit_ = true;
    }
    cv_.notify_all();
    for (std::thread &t : th_) t.join();
    th_.clear();
  }
  // copy n bytes with all workers (plus the caller); returns when done
  void copy(uint8_t *dst, const uint8_t *src, size_t n) {
    const size_t piece = 1 << 20;
    if (th_.empty() || n < 2 * piece) {
      memcpy(dst, src, n);
      return;
    }
    {
      std::lock_guard<std::mutex> lk(m_);
      dst_ = dst;
      src_ = src;
      n_ = n;
      next_ = 0;
      left_ = (n + piece - 1) / piece;
    }
    cv_.notify_all();
    help(piece);
    std::unique_lock<std::mutex> lk(m_);
    done_.wait(lk, [this] { return left_ == 0; });
  }

 private:
  bool take(size_t piece, size_t &off, size_t &len) {
    std::lock_guard<std::mutex> lk(m_);
    if (next_ >= n_) return false;
    off = next_;
    len = std::min(piece, n_ - next_);
    next_ += len;
    return true;
  }
  void finish_one() {
    std::lock_guard<std::mutex> lk(m_);
    if (--left_ == 0) done_.notify_all();
  }
  void help(size_t piece) {
    size_t off, len;
    while (take(piece, off, len)) {
      memcpy(dst_ + off, src_ + off, len);
      finish_one();
    }
  }
  void work() {
    for (;;) {
      {
        std::unique_lock<std::mutex> lk(m_);
        cv_.wait(lk, [this] { return quit_ || next_ < n_; });
        if (quit_) return;
      }
      help(1 << 20);
    }
  }
  std::vector<std::thread> th_;
  std::mutex m_;
  std::condition_variable cv_, done_;
  uint8_t *dst_ = nullptr;
  const uint8_t *src_ = nullptr;
  size_t n_ = 0, next_ = 0, left_ = 0;
  bool quit_ = false;
};

constexpr size_t kStageSlotBytes = 32u << 20;
constexpr int kStageSlots = 4;
struct StageRing {
  uint8_t *slot[kStageSlots] = {nullptr, nullptr, nullptr, nullptr};
  cudaEvent_t ev[kStageSlots] = {nullptr, nullptr, nullptr, nullptr};
  bool busy[kStageSlots] = {false, false, false, false};
  uint8_t *out_dst[kStageSlots] = {nullptr, nullptr, nullptr, nullptr};  // D2H ring: where the slot's bytes go
  size_t out_n[kStageSlots] = {0, 0, 0, 0};
  size_t next = 0;
};

// The small device words of the decode paths (zb200_ctx::counter).  Whoever uses a word sets it before a kernel reads
// it; the launch wrappers zero the work-queue counters and candidate counts themselves.
struct ZbCounters {
  uint32_t member;      // work-queue counter of a whole-member inflate launch
  uint32_t segment;     // work-queue counter of a segment launch (seg_pass)
  uint32_t cand;        // candidates found by k_find_sync / k_find_blocks (find_candidates)
  int bad;              // the marker resolve: a marker points before the start of the stream
  uint64_t resume[2];   // ZbInflateWork::resume of a decompress stream's counting pass
};

struct zb200_ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  cudaStream_t own_stream = nullptr;
  ZbCrcTables *d_tabs = nullptr;
  DevBuf desc, member_first, fname, masks, recs, hist, chk, cb, chunk_off, member_off, member_check, member_isize;
  DevBuf src_off, dst_off, out_len, status, expect, kind, ck_out, ck_pieces, ck_first, ck_piece_out, ck_partials;
  DevBuf counter;           // ZbCounters (allocated with the ctx), then uncompress_host_pipelined's per-group counters
  DevBuf in_stage, out_stage, lz2_tables;
  DevBuf opt_scratch;       // k_opt's per-CTA scratch (the _optimal calls)
  DevBuf rs_meta, rs_tiles, rs_counts, rs_starts;  // the rsyncable chunk map (rsync_chunks_locked)
  DevBuf carry;             // a compress stream's member carry: [0] in, [1] out
  size_t stream_batch_bytes = ZB_STREAM_BATCH_BYTES;  // pending input at which a stream write launches
  size_t dstream_batch_bytes = ZB_DSTREAM_BATCH_BYTES;  // pending compressed input at which a decompress stream launches
  bool dstream_log = false;
  DevBuf seg_src, seg_dst, seg_len, seg_status, seg_kind, seg_expect, seg_cand, skip_mask;  // large-member segments
  DevBuf mark_scratch, mark_segs, seg_bits;  // speculative segments of a large member (uint16 symbols, descriptors)
  DevBuf mark_win;          // window resolve scratch of the joint segments: group window maps (uint16) + incoming windows
  DevBuf order;             // work-queue order of an inflate launch (longest members first)
  DevBuf gate;              // gated inflate launch: [0] groups copied in, [1 .. ng] members done per group, then the group starts
  StreamMemOps memops;      // stream wait / write on device words (null: group-by-group launches instead)
  bool gated_unc = true;    // env ZB200_UNC_GATED=0 forces the group-by-group launches
  StageRing ring_in, ring_out;   // pinned slots for pageable callers (allocated on first use)
  CopyPool pool;
  uint64_t pending_len = 0;     // zb200_decode_begin's result, waiting in out_stage for zb200_decode_finish
  bool pending = false;
  uint64_t big_member_bytes = 512ull << 10;  // members at least this long are tried as parallel segments
  uint64_t single_member_bytes = 512ull << 10; // threshold when the call holds ONE input.  (24 KiB was tried: alice29.txt.gz has three blocks,
                                               // two decode passes over three segments cost what one serial pass costs, so no gain)
  bool big_env = false;
  bool joint_markers = true;       // env ZB200_JOINT_MARKERS=0 turns the marker segments at sync joints off (A/B timing)
  uint32_t mark_window_segs = 8192;  // segments per window of the joint marker decode (env ZB200_MARK_WINDOW_SEGS)
  DevBuf idx_desc, idx_out;          // index build / extraction: gather descriptors, gathered bytes
  DevBuf cix_rec, cix_crc, cix_first, cix_out;  // a compress-time index: ZbIndexWork's arrays
  uint64_t index_group_bytes = kDstreamMaxOut;  // output budget of one extraction launch group (env ZB200_INDEX_GROUP_BYTES)
  bool index_log = false;            // env ZB200_INDEX_LOG: one stderr line per extraction launch group
  // the dictionary table of the *_dict / *_dicts call in progress (DictScope, the caller's dict_base / dict_offsets):
  // dict_win holds the windows of the launch groups in flight (DictWindows), dict_md the ZbMemberDict per member.
  // dict_member / dict_entry: per member of the call, its ZbMemberDict (wend set by DictWindows::plan) and its table
  // entry (-1: none, or an empty one).  dict_on is false outside such a call, and in a call where no member names a
  // non-empty dictionary: every such call runs exactly as without them
  DevBuf dict_win, dict_md;
  std::vector<ZbMemberDict> dict_member;
  std::vector<int32_t> dict_entry;
  const uint8_t *dict_base = nullptr;
  const uint64_t *dict_offs = nullptr;
  size_t dict_k = 0;
  bool dict_on = false;
  uint64_t pending_skip = 0;         // zb200_decode_begin_dict: output bytes in front of the result (the window)
  cudaEvent_t ev[10] = {};
  cudaStream_t h2d_stream = nullptr, d2h_stream = nullptr;
  std::vector<cudaEvent_t> gev;   // per-group events (H2D done, compute done, offsets ready)
  void *pin = nullptr;            // pinned host scratch for descriptors / offsets
  size_t pin_cap = 0;
  DevBuf group_end;               // device u64 per group: end offset of the group's output
  size_t dev_group_chunks = kMaxChunksPerGroup, host_group_chunks = kHostGroupChunks;
  uint64_t unc_group_out_bytes = 0;  // host uncompress: output bytes per pipelined member group (0: a quarter of the batch)
  zb200_timing timing;
  std::string last_err;
  std::mutex mu;
};

// Segment points: for k = 0, 1, ..., the first block start whose output offset is >= k * 32768 (duplicates removed).
// Window points: for j = 0, 1, ..., the first segment point whose output offset is >= j * span; each keeps the 32 KiB
// of output in front of it.  Every segment point keeps the CRC-32 of its interval (up to the next point, the last one
// to the end of the member).  All of it is host memory, tied to no ctx.
struct zb200_index {
  int fmt = 0;
  uint64_t payload = 0, len = 0, size = 0, span = 0;
  uint8_t head[32] = {}, tail[32] = {};
  std::vector<uint64_t> bit, out;   // per point: absolute bit position in the member, output offset
  std::vector<uint32_t> crc;        // per point: CRC-32 of its interval
  std::vector<uint8_t> win;         // per point: 1 = window point
  std::vector<uint64_t> win_at;     // per point: offset of its window in `windows` (window points with out > 0)
  std::vector<uint8_t> windows;
};

// One member compressed from input that arrives piece by piece.  All of its state is on the host; the
// kernels run on its ctx's scratch, so any number of streams and other calls can share a ctx.
struct zb200_compress_stream {
  zb200_ctx *ctx = nullptr;
  int level = 0, data_format = 0;
  int strategy = ZB_STRATEGY_DEFAULT;  // folded with the level by zb_strategy_level
  bool optimal = false;        // begun by zb200_compress_stream_begin_optimal (level 9's history rules, k_opt's parse)
  int window_bits = 15;        // after zb_window_bits: every launch, flush and carried history keeps to it
  uint8_t fname_len = 0;
  size_t batch_bytes = 0;      // launch once this much input is pending
  std::vector<uint8_t> buf;    // [history | pending input]: pending starts at a chunk boundary of its flush segment
  size_t hist = 0;             // bytes of history (the LZ levels: the last <= 32 KiB compressed since the member
                               // start or the last full flush)
  ZbMemberCarry carry{0u, 1u, 0ull};  // the input compressed so far: raw CRC-32, Adler-32, bytes
  bool has_dict = false;       // zlib: the header carries FDICT and dict_id
  uint32_t dict_id = 0;
  bool head_done = false, finished = false;
  int err = ZB200_OK;          // a CUDA failure: the stream is unusable
  // begun with an index (zb200_compress_stream_begin_index): the points so far, written launch by launch
  std::unique_ptr<zb200_index> ix;
  uint64_t ix_next = 0;        // the next window point is the first point at or past this output offset
  uint64_t ix_lo = 0;          // the first output offset the next launch's first block start may own
  uint32_t ix_raw = 0;         // ix_open: the raw CRC-32 of the last point's interval so far
  bool ix_open = false;
  std::vector<uint8_t> ix_in;  // the last <= 32 KiB of input compressed (windows need input, not history)
  std::vector<uint8_t> ix_tail;  // the last <= 32 bytes of the member written
};

// One member decoded from compressed input that arrives piece by piece.  All of its state is on the host; the
// kernels run on its ctx's scratch, so any number of streams and other calls can share a ctx.
struct zb200_decompress_stream {
  zb200_ctx *ctx = nullptr;
  int data_format = 0;         // as requested (DETECT too)
  int fmt = -1;                // the resolved format once the header is decided, -1 before
  size_t batch_bytes = 0;      // a write launches once this much compressed payload is pending
  std::vector<uint8_t> in;     // held input: in[in_head ..) are member bytes from in_off on, from a block boundary on
  size_t in_head = 0;          // in[0 .. in_head) is decoded already (dropped once it is half of the vector)
  uint64_t in_off = 0;
  uint32_t bit0 = 0;           // the decode resumes at bit bit0 of in[in_head]
  uint64_t total_in = 0;       // member bytes written
  uint8_t tail[8] = {};        // the last 8 member bytes written (the trailer once the input has ended)
  std::vector<uint8_t> win;    // the last 32 KiB of output in front of the resume point (when base_out > 0)
  uint64_t base_out = 0;       // output position of the resume point: 0, or >= 32768 (see dstream_run)
  uint64_t out_total = 0;      // output produced so far (64-bit; gzip ISIZE is compared mod 2^32)
  uint32_t check = 0;          // CRC-32 (gzip) or Adler-32 (zlib) of that output
  std::vector<uint8_t> q;      // decoded bytes not read yet: q[q_head ..)
  size_t q_head = 0;
  bool done = false;           // the final block is decoded: the rest of the payload is ignored
  bool finished = false;
  bool log = false;            // env ZB200_DSTREAM_LOG: one line per launch on stderr (which decode path ran)
  int err = ZB200_OK;          // once a write or finish failed, every later call reports it
  // a preset dictionary (zb200_decompress_stream_begin_dict): its window W and DICTID; once the header is decided a raw
  // stream, or a zlib member whose FDICT carries dict_id, holds stored(W) in front of its payload (dstream_header)
  std::vector<uint8_t> dict_win;
  uint32_t dict_id = 0;
  bool has_dict = false;
};

namespace {

bool cuda_ok(zb200_ctx *c, cudaError_t e, const char *what) {
  if (e == cudaSuccess) return true;
  c->last_err = std::string(what) + ": " + cudaGetErrorString(e);
  return false;
}
#define CK(call)                                      \
  do {                                                \
    if (!cuda_ok(ctx, (call), #call)) return ZB200_ERR_CUDA; \
  } while (0)

int ensure(zb200_ctx *ctx, DevBuf &b, size_t bytes) {
  if (bytes <= b.cap) return ZB200_OK;
  if (b.p) cudaFree(b.p);
  b.p = nullptr;
  b.cap = 0;
  size_t want = bytes + bytes / 8 + 256;
  cudaError_t e = cudaMalloc(&b.p, want);
  if (e != cudaSuccess) {
    cudaGetLastError();
    e = cudaMalloc(&b.p, bytes);
    want = bytes;
  }
  if (e != cudaSuccess) {
    ctx->last_err = std::string("cudaMalloc: ") + cudaGetErrorString(e);
    cudaGetLastError();
    return ZB200_ERR_NOMEM;
  }
  b.cap = want;
  return ZB200_OK;
}
#define ENSURE(buf, bytes)                         \
  do {                                             \
    int _rc = ensure(ctx, (buf), (bytes));         \
    if (_rc != ZB200_OK) return _rc;               \
  } while (0)

ZbCounters *counters(zb200_ctx *ctx) { return (ZbCounters *)ctx->counter.p; }

struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev) {
    cudaGetDevice(&prev);
    if (prev != dev) cudaSetDevice(dev);
    else prev = -1;
  }
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};


float ev_ms(cudaEvent_t a, cudaEvent_t b) {
  float ms = 0.f;
  if (cudaEventElapsedTime(&ms, a, b) != cudaSuccess) {
    cudaGetLastError();
    return 0.f;
  }
  return ms;
}

int ensure_pinned(zb200_ctx *ctx, size_t bytes) {
  if (bytes <= ctx->pin_cap) return ZB200_OK;
  if (ctx->pin) cudaFreeHost(ctx->pin);
  ctx->pin = nullptr;
  ctx->pin_cap = 0;
  size_t want = bytes + bytes / 4 + 4096;
  if (cudaMallocHost(&ctx->pin, want) != cudaSuccess) {
    cudaGetLastError();
    ctx->last_err = "cudaMallocHost failed";
    return ZB200_ERR_NOMEM;
  }
  ctx->pin_cap = want;
  return ZB200_OK;
}

int ensure_group_events(zb200_ctx *ctx, size_t n) {
  while (ctx->gev.size() < n) {
    cudaEvent_t e;
    if (cudaEventCreateWithFlags(&e, cudaEventDisableTiming) != cudaSuccess) return ZB200_ERR_CUDA;
    ctx->gev.push_back(e);
  }
  return ZB200_OK;
}

bool is_pageable(const void *p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return true;
  }
  return a.type == cudaMemoryTypeUnregistered;
}

int ring_ready(zb200_ctx *ctx, StageRing &r) {
  if (r.slot[0]) return ZB200_OK;
  for (int i = 0; i < kStageSlots; i++) {
    if (cudaMallocHost((void **)&r.slot[i], kStageSlotBytes) != cudaSuccess ||
        cudaEventCreateWithFlags(&r.ev[i], cudaEventDisableTiming) != cudaSuccess) {
      cudaGetLastError();
      ctx->last_err = "pinned staging ring: allocation failed";
      return ZB200_ERR_NOMEM;
    }
  }
  unsigned hc = std::thread::hardware_concurrency();
  ctx->pool.start((int)std::min<unsigned>(7, hc > 2 ? hc / 2 : 1));
  return ZB200_OK;
}

// host -> device on `st`: asynchronous for page-locked memory, staged through the pinned ring otherwise
int h2d_copy(zb200_ctx *ctx, uint8_t *d_dst, const uint8_t *h_src, size_t n, cudaStream_t st, bool pageable) {
  if (!n) return ZB200_OK;
  if (!pageable) {
    CK(cudaMemcpyAsync(d_dst, h_src, n, cudaMemcpyHostToDevice, st));
    return ZB200_OK;
  }
  StageRing &r = ctx->ring_in;
  int rc = ring_ready(ctx, r);
  if (rc) return rc;
  for (size_t off = 0; off < n; off += kStageSlotBytes) {
    const size_t len = std::min(kStageSlotBytes, n - off);
    const size_t k = r.next++ % kStageSlots;
    if (r.busy[k]) CK(cudaEventSynchronize(r.ev[k]));   // the DMA that last read this slot is done
    ctx->pool.copy(r.slot[k], h_src + off, len);
    CK(cudaMemcpyAsync(d_dst + off, r.slot[k], len, cudaMemcpyHostToDevice, st));
    CK(cudaEventRecord(r.ev[k], st));
    r.busy[k] = true;
  }
  return ZB200_OK;
}

// finish the oldest / all pending device -> pageable copies (the slot's bytes go to their place)
int d2h_complete(zb200_ctx *ctx, size_t k) {
  StageRing &r = ctx->ring_out;
  if (!r.busy[k]) return ZB200_OK;
  CK(cudaEventSynchronize(r.ev[k]));
  ctx->pool.copy(r.out_dst[k], r.slot[k], r.out_n[k]);
  r.busy[k] = false;
  return ZB200_OK;
}
int d2h_flush(zb200_ctx *ctx) {
  if (!ctx->ring_out.slot[0]) return ZB200_OK;
  for (size_t i = 0; i < (size_t)kStageSlots; i++) {
    int rc = d2h_complete(ctx, (ctx->ring_out.next + i) % kStageSlots);   // oldest first
    if (rc) return rc;
  }
  return ZB200_OK;
}
// device -> host on `st`; for pageable memory the bytes land when d2h_flush (or a later d2h_copy) says so
int d2h_copy(zb200_ctx *ctx, uint8_t *h_dst, const uint8_t *d_src, size_t n, cudaStream_t st, bool pageable) {
  if (!n) return ZB200_OK;
  if (!pageable) {
    CK(cudaMemcpyAsync(h_dst, d_src, n, cudaMemcpyDeviceToHost, st));
    return ZB200_OK;
  }
  StageRing &r = ctx->ring_out;
  int rc = ring_ready(ctx, r);
  if (rc) return rc;
  for (size_t off = 0; off < n; off += kStageSlotBytes) {
    const size_t len = std::min(kStageSlotBytes, n - off);
    const size_t k = r.next++ % kStageSlots;
    rc = d2h_complete(ctx, k);
    if (rc) return rc;
    CK(cudaMemcpyAsync(r.slot[k], d_src + off, len, cudaMemcpyDeviceToHost, st));
    CK(cudaEventRecord(r.ev[k], st));
    r.busy[k] = true;
    r.out_dst[k] = h_dst + off;
    r.out_n[k] = len;
  }
  return ZB200_OK;
}

struct Group {
  size_t m0, m1;        // members [m0, m1)
  size_t c0, nc;        // chunks [c0, c0 + nc) in the batch-wide descriptor array
  size_t first0;        // start of this group's (nm + 1) entries in the member_first / member_off arrays
  uint64_t in_lo, in_hi;  // source byte range
};

// The chunk starts of an rsyncable batch (rsync_chunks_locked): member i's count[i] starts, member positions in
// ascending order from 0, are starts[off[i]] .. starts[off[i] + count[i] - 1]; off[i + 1] - off[i] = zb_rsync_cap.
struct RsyncMap {
  std::vector<uint64_t> count, off, starts;
};

// One launch of a compress stream (zb200_compress_stream_*): a run of chunks of ONE member that continues
// what earlier launches compressed; only the run's last chunk may be short (the end of a flush segment, or of
// the member).  The source holds `hist` bytes (0..32768) of the member's preceding input in front of the run
// (k_lz2's history for the first chunk); `head`: the run starts the member (header);
// `last`: the run ends it (BFINAL, trailer).  carry_in is the member's bytes before the run, carry_out
// receives the bytes through its end.
struct StreamPart {
  uint32_t hist;
  bool head, last;
  ZbMemberCarry carry_in, carry_out;
  bool has_dict;       // a zlib header with FDICT and dict_id
  uint32_t dict_id;
};

// Adler-32 on the host: the DICTID of a dictionary (zlib: the Adler-32 of all of it)
uint32_t host_adler32(const uint8_t *p, size_t n) {
  uint64_t a = 1, b = 0;
  while (n) {
    const size_t k = std::min<size_t>(n, 5552);
    for (size_t i = 0; i < k; i++) {
      a += p[i];
      b += a;
    }
    a %= 65521;
    b %= 65521;
    p += k;
    n -= k;
  }
  return (uint32_t)(b << 16 | a);
}

int checksum_device_locked(zb200_ctx *ctx, const uint8_t *d_src, const uint64_t *src_offsets, size_t n, int kind,
                           uint32_t *out);

// A call's dictionary table (zb200_*_dicts; the *_dict calls are its k = 1 case with every member naming entry 0, of
// == null): entry j is base[offs[j] .. offs[j + 1]), member i names of[i] in -1 .. k - 1.  ZB200_ERR_ARG for a name
// out of range, offsets that decrease, or bytes without a base; *any: some member names a non-empty entry.
static int check_dicts(const uint8_t *base, const uint64_t *offs, size_t k, const int32_t *of, size_t n, bool &any) {
  any = false;
  if (k && !offs) return ZB200_ERR_ARG;
  for (size_t j = 0; j < k; j++)
    if (offs[j + 1] < offs[j]) return ZB200_ERR_ARG;
  if (!of) return n && k ? ZB200_ERR_ARG : ZB200_OK;   // (no table: the calls without dictionaries)
  for (size_t i = 0; i < n; i++) {
    if (of[i] < -1 || of[i] >= (int64_t)k) return ZB200_ERR_ARG;
    any = any || (of[i] >= 0 && offs[of[i] + 1] > offs[of[i]]);
  }
  if (any && !base) return ZB200_ERR_ARG;
  return ZB200_OK;
}

// Above this many bytes of named dictionaries the DICTIDs come from the batched Adler-32 on the device, below it from
// a host loop.  The device pass uploads runs of consecutive named entries, at most kDictSlabBytes at a time (an entry
// larger than that alone), into dict_win before any window needs it.
constexpr uint64_t kDictHostAdlerBytes = 256u << 10;
constexpr uint64_t kDictSlabBytes = 256ull << 20;

// A call's dictionary table (check_dicts has passed).  Every entry that a member names and that is not empty gets its
// DICTID (the Adler-32 of all of it) once; each member gets its ZbMemberDict in ctx->dict_member without a window
// (DictWindows places the windows launch group by launch group).  A table no member names non-empty leaves the ctx
// as it is (the call is the one without dictionaries).  The destructor turns the table off again.
struct DictScope {
  zb200_ctx *ctx;
  explicit DictScope(zb200_ctx *c) : ctx(c) {}
  int set(const uint8_t *base, const uint64_t *offs, size_t k, const int32_t *of, size_t n) {
    zb200_ctx *ctx = this->ctx;   // (CK / ENSURE)
    ctx->dict_entry.assign(n, -1);
    uint64_t named = 0;
    std::vector<uint8_t> is_named(k, 0);
    bool any = false;
    for (size_t i = 0; i < n; i++) {
      const int32_t j = of ? of[i] : 0;
      if (j < 0 || offs[j + 1] == offs[j]) continue;
      ctx->dict_entry[i] = j;
      if (!is_named[j]) named += offs[j + 1] - offs[j];
      is_named[j] = 1;
      any = true;
    }
    if (!any) return ZB200_OK;
    auto len = [&](size_t j) { return offs[j + 1] - offs[j]; };
    std::vector<uint32_t> ids(k, 0);
    if (named > kDictHostAdlerBytes) {
      for (size_t ja = 0; ja < k;) {
        if (!is_named[ja]) {
          ja++;
          continue;
        }
        size_t jb = ja + 1;
        uint64_t bytes = len(ja);
        while (jb < k && is_named[jb] && bytes + len(jb) <= kDictSlabBytes) bytes += len(jb++);
        std::vector<uint64_t> rel(jb - ja + 1);
        for (size_t j = ja; j <= jb; j++) rel[j - ja] = offs[j] - offs[ja];
        ENSURE(ctx->dict_win, (size_t)bytes + 64);
        CK(cudaMemcpyAsync(ctx->dict_win.p, base + offs[ja], (size_t)bytes, cudaMemcpyHostToDevice, ctx->stream));
        if (int rc = checksum_device_locked(ctx, (const uint8_t *)ctx->dict_win.p, rel.data(), jb - ja, 1, ids.data() + ja))
          return rc;
        ja = jb;
      }
    } else {
      for (size_t j = 0; j < k; j++)
        if (is_named[j]) ids[j] = host_adler32(base + offs[j], (size_t)len(j));
    }
    ctx->dict_member.assign(n, ZbMemberDict{nullptr, 0u, 0u});
    for (size_t i = 0; i < n; i++) {
      const int32_t j = ctx->dict_entry[i];
      if (j < 0) continue;
      ctx->dict_member[i].win_len = (uint32_t)std::min<uint64_t>(len((size_t)j), 32768);
      ctx->dict_member[i].dict_id = ids[(size_t)j];
    }
    ctx->dict_base = base;
    ctx->dict_offs = offs;
    ctx->dict_k = k;
    ctx->dict_on = true;
    return ZB200_OK;
  }
  ~DictScope() { ctx->dict_on = false; }
};

// The windows of the call's members, launch group by launch group, so that device memory for windows is bounded by
// the groups in flight and not by the batch.  Group g (members [gb[g], gb[g + 1])) gets slot g % slots of
// ctx->dict_win: one copy of W per (entry, class) its members use, class being the member's first-chunk address
// modulo 16 for k_lz2 (stage_dict_chunk needs W to end at an address congruent to it) and 0 for k_inflate, each copy
// zb_win_stride(|W|) bytes with W ending at an address congruent to its class.  plan() sizes the slots and sets every
// member's ZbMemberDict::wend in ctx->dict_member; upload(g) packs the group's windows on the host and copies them into
// its slot on a stream, which the caller orders after the last reader of the slot's previous group.
constexpr uint64_t kDictGroupWindowBytes = 256ull << 20;   // a decode group's windows (uncompress_batch_host)
constexpr size_t kDictSlots = 3;
struct DictWindows {
  struct Copy {
    int32_t entry;
    uint64_t end;   // of W in the slot
  };
  std::vector<size_t> gb, c0;   // per group: members, first copy
  std::vector<Copy> copies;
  std::vector<uint64_t> bytes;  // per group
  std::vector<uint8_t> host;
  uint64_t slot_cap = 0;
  size_t slots = 1;

  std::vector<uint64_t> end_of;   // per member: W's end in its group's slot

  // cls: per member (null: 0).  nslots: slots in ctx->dict_win (place(), at most one per group)
  int plan(zb200_ctx *ctx, const std::vector<size_t> &groups, const uint8_t *cls, size_t nslots) {
    layout(ctx, groups, cls);
    return place(ctx, nslots);
  }
  void layout(zb200_ctx *ctx, const std::vector<size_t> &groups, const uint8_t *cls) {
    gb = groups;
    const size_t ng = gb.size() - 1;
    c0.assign(1, 0);
    bytes.clear();
    copies.clear();
    end_of.assign(ctx->dict_member.size(), 0);
    std::unordered_map<uint64_t, uint64_t> seen;
    for (size_t g = 0; g < ng; g++) {
      seen.clear();
      uint64_t b = 0;
      for (size_t i = gb[g]; i < gb[g + 1]; i++) {
        const int32_t j = ctx->dict_entry[i];
        if (j < 0) continue;
        const uint32_t c = cls ? cls[i] : 0u, wl = ctx->dict_member[i].win_len;
        auto it = seen.find((uint64_t)j * 16u + c);
        if (it == seen.end()) {
          const uint64_t end = b + ZB_WIN_SLACK + ((c - wl) & 15u) + wl;
          copies.push_back(Copy{j, end});
          b += zb_win_stride(wl);
          it = seen.emplace((uint64_t)j * 16u + c, end).first;
        }
        end_of[i] = it->second;
      }
      bytes.push_back(b);
      c0.push_back(copies.size());
      slot_cap = std::max(slot_cap, b);
    }
  }
  int place(zb200_ctx *ctx, size_t nslots) {
    const size_t ng = gb.size() - 1;
    slots = std::max<size_t>(1, std::min(nslots, ng));
    ENSURE(ctx->dict_win, (size_t)(slots * slot_cap) + 64);
    for (size_t g = 0; g < ng; g++)
      for (size_t i = gb[g]; i < gb[g + 1]; i++)
        if (ctx->dict_entry[i] >= 0)
          ctx->dict_member[i].wend = (const uint8_t *)ctx->dict_win.p + (g % slots) * slot_cap + end_of[i];
    return ZB200_OK;
  }

  int upload(zb200_ctx *ctx, size_t g, cudaStream_t st) {
    if (!bytes[g]) return ZB200_OK;
    host.resize(bytes[g]);
    for (size_t t = c0[g]; t < c0[g + 1]; t++) {
      const size_t j = (size_t)copies[t].entry;
      const uint64_t wl = std::min<uint64_t>(ctx->dict_offs[j + 1] - ctx->dict_offs[j], 32768);
      memcpy(host.data() + copies[t].end - wl, ctx->dict_base + ctx->dict_offs[j + 1] - wl, (size_t)wl);
    }
    // through the pinned staging ring: `host` may be refilled as soon as this returns
    return h2d_copy(ctx, (uint8_t *)ctx->dict_win.p + (g % slots) * slot_cap, host.data(), (size_t)bytes[g], st, true);
  }
};

// A compression strategy (ZB_STRATEGY_*) folded into the level, in zlib's order: stored at level 0 whatever the
// strategy, then Huffman-only (= level -2), then the run-length parse, then the level's own parse.  Afterwards the
// work's strategy is RLE only at level 1 (RLE's bytes do not depend on the level), FILTERED only at the LZ levels
// (level 1 ignores it, as zlib's fast levels do), FIXED at any level but 0, and nothing else changes the parse.
// ZB200_ERR_ARG: not a strategy.
static int zb_strategy_level(int &level, int &strategy) {
  if (strategy < ZB_STRATEGY_DEFAULT || strategy > ZB_STRATEGY_FIXED) return ZB200_ERR_ARG;
  if (level < -2 || level > 9) return ZB200_ERR_INVALID_LEVEL;
  if (level == 0 || level == -2) {
    if (strategy != ZB_STRATEGY_FIXED || level == 0) strategy = ZB_STRATEGY_DEFAULT;
  } else if (strategy == ZB_STRATEGY_HUFFMAN_ONLY) {
    level = -2;
    strategy = ZB_STRATEGY_DEFAULT;
  } else if (strategy == ZB_STRATEGY_RLE) {
    level = 1;
  } else if (strategy == ZB_STRATEGY_FILTERED && level == 1) {
    strategy = ZB_STRATEGY_DEFAULT;
  }
  return ZB200_OK;
}

// zlib's window size (deflateInit2's windowBits, zlib.compressobj's wbits): 9..15, and 8 for the zlib format, where it
// means 9 as in zlib.  ZB200_ERR_ARG for anything else.
static int zb_window_bits(int &window_bits, int data_format) {
  if (window_bits == 8 && data_format == ZB200_DF_ZLIB) window_bits = 9;
  return window_bits < 9 || window_bits > 15 ? ZB200_ERR_ARG : ZB200_OK;
}

// ---- compress: device-resident (h_src == h_dst == nullptr) or pipelined host buffers ----
// With host buffers the batch is cut into groups and H2D(g+1) || kernels(g) || D2H(g-1) run
// on three streams; each group's output offset is chained on the device (out_base_ptr), so
// the only host waits are for the small per-group offset arrays that size the D2H copies.
// sp (host buffers, n == 1 only): the member is one part of a stream; null for every batch call.
// ix: null, or the records of a compress-time index (k_index_rec after k_scan; ix->rec_first counts the batch's members).
// optimal: the optimal parse (k_opt); the caller passes level 9, whose history rules it keeps.
// rs (batch calls only): the members' chunk starts (an rsyncable batch) instead of the 64 KiB grid; at the LZ levels a
// chunk sees up to 32 KiB of the member in front of its start as history.
int compress_locked(zb200_ctx *ctx, const uint8_t *d_src, const uint8_t *h_src, const uint64_t *src_offsets,
                    size_t n, int level, int data_format, const uint8_t *fname_lens, uint8_t *d_dst,
                    size_t dst_cap, uint8_t *h_dst, size_t h_dst_cap, uint64_t *dst_offsets, int *statuses,
                    size_t max_group_chunks, StreamPart *sp = nullptr, const ZbIndexWork *ix = nullptr,
                    int strategy = ZB_STRATEGY_DEFAULT, int window_bits = 15, bool optimal = false,
                    const RsyncMap *rs = nullptr) {
  const auto t_entry = std::chrono::steady_clock::now();
  if (int rc = zb_strategy_level(level, strategy)) return rc;
  if (optimal) strategy = ZB_STRATEGY_OPTIMAL;
  if (int rc = zb_window_bits(window_bits, data_format)) return rc;
  if (data_format != ZB200_DF_GZIP && data_format != ZB200_DF_ZLIB && data_format != ZB200_DF_DEFLATE)
    return ZB200_ERR_INVALID_FORMAT;
  if (fname_lens)
    for (size_t i = 0; i < n; i++)
      if (fname_lens[i] > 25) return ZB200_ERR_ARG;
  if (((uintptr_t)d_dst & 3u) != 0) return ZB200_ERR_ARG;
  dst_cap &= ~(size_t)3;  // the packer writes whole 32-bit words: never touch a word that straddles the end
  if (src_offsets[n] < src_offsets[0]) return ZB200_ERR_ARG;  // each member's offsets are checked by the plan
  ctx->timing.lz_ms = ctx->timing.huff_ms = ctx->timing.scan_ms = ctx->timing.pack_ms = ctx->timing.plan_ms = 0.f;
  ctx->timing.n_chunks = 0;
  dst_offsets[0] = 0;
  if (n == 0) return ZB200_OK;
  const uint64_t hist = sp ? sp->hist : 0;
  const bool head = !sp || sp->head, last = !sp || sp->last;
  const bool lz = level == -1 || level >= 2;
  // a batch's dictionaries: a member's first chunk sees its window as its history (LZ levels), and zlib headers
  // carry FDICT; a stream's dictionary is history in its own buffer, so only its header is the stream's business
  // (any non-zero win_len marks FDICT)
  const bool dict_hist = !sp && ctx->dict_on && lz && h_src;
  std::vector<ZbMemberDict> mdict;   // set once the windows are placed (dict_hist) or now
  if (sp && sp->has_dict && data_format == ZB200_DF_ZLIB) mdict.assign(1, ZbMemberDict{nullptr, 1u, sp->dict_id});
  else if (!sp && ctx->dict_on && !dict_hist) mdict = ctx->dict_member;
  DictWindows dw;
  const uint64_t src_lo = src_offsets[0] - hist;  // d_src holds [src_lo, src_hi) rebased to 0 when staging from the host
  const bool src_pageable = h_src && is_pageable(h_src + src_lo), dst_pageable = h_dst && is_pageable(h_dst);

  // ---- plan: groups, descriptors ----
  // One pass over the members validates their offsets and writes the descriptors and member_first entries straight
  // into pinned memory, so that their upload is a true asynchronous copy; the member offsets come back at its
  // start.  With offsets that do not decrease a member of len bytes has at most len / 64 KiB + 1 chunks, so the
  // batch at most nc_cap (rsyncable: len / MIN more, zb_rsync_cap); member_first holds n entries plus one per group,
  // and a group holds at least one member.
  auto chunks_of = [](uint64_t len) { return len == 0 ? (size_t)1 : (size_t)((len + ZB_CHUNK_BYTES - 1) / ZB_CHUNK_BYTES); };
  const uint64_t total_in = src_offsets[n] - src_offsets[0];
  const size_t nc_cap = n + (size_t)(total_in / ZB_CHUNK_BYTES) + (rs ? (size_t)(total_in / ZB_RSYNC_MIN) : 0),
               nfirst_cap = 2 * n;
  {
    int rc = ensure_pinned(ctx, nfirst_cap * (sizeof(uint64_t) + sizeof(uint32_t)) + sizeof(ZbMemberCarry) +
                                    nc_cap * sizeof(ZbChunkDesc) + 64);
    if (rc) return rc;
  }
  uint64_t *pin_off = (uint64_t *)ctx->pin;
  ZbMemberCarry *pin_carry = (ZbMemberCarry *)(pin_off + nfirst_cap);  // a stream's carry-out comes back behind the offsets
  ZbChunkDesc *desc = (ZbChunkDesc *)(pin_carry + 1);
  uint32_t *first = (uint32_t *)(desc + nc_cap);
  std::vector<Group> groups;
  size_t max_nc = 0, max_nm = 0;
  size_t nd = 0, nfirst = 0;  // entries of desc / first written so far
  // the host pipeline sizes its groups by the chunks still to come (a wrong count from decreasing offsets is never
  // used: the plan stops at the first such member)
  size_t chunks_left = 0;
  if (h_src)
    for (size_t i = 0; i < n; i++) chunks_left += rs ? (size_t)rs->count[i] : chunks_of(src_offsets[i + 1] - src_offsets[i]);
  const size_t group_cap = max_group_chunks;
  for (size_t m0 = 0; m0 < n;) {
    // host pipeline: the work after the last H2D (kernels + D2H of the last group) is not overlapped
    // with anything, so the groups shrink geometrically towards the end of the batch
    if (h_src) max_group_chunks = std::min(group_cap, std::max<size_t>(512, chunks_left / 2));
    Group g;
    g.m0 = m0;
    g.c0 = nd;
    g.first0 = nfirst;
    size_t m1 = m0;
    while (m1 < n) {
      if (src_offsets[m1 + 1] < src_offsets[m1]) return ZB200_ERR_ARG;
      uint64_t len = src_offsets[m1 + 1] - src_offsets[m1];
      size_t nc = rs ? (size_t)rs->count[m1] : chunks_of(len);
      if (nd + nc > nc_cap) return ZB200_ERR_ARG;  // only offsets that decrease further on get here
      if (nd > g.c0 && nd - g.c0 + nc > max_group_chunks) break;
      if (statuses) statuses[m1] = ZB200_OK;
      first[nfirst++] = (uint32_t)(nd - g.c0);
      const uint64_t *rs_starts = rs ? rs->starts.data() + rs->off[m1] : nullptr;
      for (size_t k = 0; k < nc; k++) {
        ZbChunkDesc &d = desc[nd++];
        const uint64_t at = rs ? rs_starts[k] : (uint64_t)k * ZB_CHUNK_BYTES;
        d.src_off = src_offsets[m1] - (h_src ? src_lo : 0) + at;
        d.len = (uint32_t)(rs ? (k + 1 < nc ? rs_starts[k + 1] : len) - at
                              : std::min<uint64_t>(ZB_CHUNK_BYTES, len - at));
        d.member = (uint32_t)(m1 - m0);
        d.flags = (k == 0 ? ZB_CHUNK_FIRST | (head ? ZB_CHUNK_HEAD : 0u) : 0u) | (k == nc - 1 && last ? ZB_CHUNK_LAST : 0u);
        d.pad = lz ? (uint32_t)std::min<uint64_t>(32768, hist + at) : 0u;
        if (dict_hist && k == 0 && ctx->dict_member[m1].win_len) {
          d.pad = ctx->dict_member[m1].win_len;
          d.flags |= ZB_CHUNK_DICT;
        }
      }
      m1++;
    }
    g.m1 = m1;
    g.nc = nd - g.c0;
    chunks_left -= std::min(chunks_left, g.nc);
    first[nfirst++] = (uint32_t)g.nc;
    g.in_lo = m0 == 0 ? 0 : src_offsets[m0] - src_lo;  // the first group also copies a stream's history
    g.in_hi = src_offsets[m1] - src_lo;
    max_nc = std::max(max_nc, g.nc);
    max_nm = std::max(max_nm, g.m1 - g.m0);
    groups.push_back(g);
    m0 = m1;
  }
  const size_t ng = groups.size(), nc_all = nd;
  if (dict_hist) {
    // each launch group's windows go up with its input (DictWindows), in slots reused kDictSlots groups later
    std::vector<size_t> gbounds(1, 0);
    std::vector<uint8_t> cls(n);
    for (const Group &g : groups) gbounds.push_back(g.m1);
    for (size_t i = 0; i < n; i++) cls[i] = (uint8_t)((uintptr_t)(d_src + src_offsets[i] - src_lo) & 15u);
    if (int rc = dw.plan(ctx, gbounds, cls.data(), kDictSlots)) return rc;
    mdict = ctx->dict_member;
  }
  if (!mdict.empty()) ENSURE(ctx->dict_md, mdict.size() * sizeof(ZbMemberDict));

  ENSURE(ctx->desc, nc_all * sizeof(ZbChunkDesc));
  ENSURE(ctx->member_first, nfirst * sizeof(uint32_t));
  ENSURE(ctx->member_off, nfirst * sizeof(uint64_t));
  ENSURE(ctx->fname, n + 16);
  ENSURE(ctx->group_end, (ng + 1) * sizeof(uint64_t));
  ENSURE(ctx->masks, max_nc * ZB_WINDOWS_PER_CHUNK * sizeof(uint2));
  ENSURE(ctx->recs, max_nc * (size_t)ZB_RECS_PER_CHUNK * sizeof(uint32_t));
  ENSURE(ctx->hist, max_nc * (size_t)ZB_WARPS_PER_CHUNK * ZB_HIST_SYMS * sizeof(uint16_t));
  ENSURE(ctx->chk, max_nc * sizeof(ZbChunkCheck));
  ENSURE(ctx->cb, max_nc * sizeof(ZbCodebook));
  ENSURE(ctx->chunk_off, max_nc * sizeof(uint64_t));
  ENSURE(ctx->member_check, max_nm * sizeof(uint32_t));
  ENSURE(ctx->member_isize, max_nm * sizeof(uint32_t));
  if (optimal) ENSURE(ctx->opt_scratch, zb_opt_scratch_bytes(nullptr));
  else if (lz) ENSURE(ctx->lz2_tables, zb_lz2_table_bytes(nullptr));
  if (sp) ENSURE(ctx->carry, 2 * sizeof(ZbMemberCarry));
  {
    int rc = ensure_group_events(ctx, 3 * ng + 1);
    if (rc) return rc;
  }
  ZbMemberCarry *d_carry = (ZbMemberCarry *)ctx->carry.p;          // [0] in, [1] out

  cudaStream_t s = ctx->stream;
  cudaStream_t sh = h_src ? ctx->h2d_stream : s, sd = h_dst ? ctx->d2h_stream : s;
  // the next call writes its plan into the same pinned memory: no return, an early one included, leaves a copy
  // from or to it running on s
  struct SyncOnReturn {
    cudaStream_t s;
    ~SyncOnReturn() { cudaStreamSynchronize(s); }
  } sync_on_return{s};
  CK(cudaMemcpyAsync(ctx->desc.p, desc, nc_all * sizeof(ZbChunkDesc), cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(ctx->member_first.p, first, nfirst * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
  if (!mdict.empty())
    CK(cudaMemcpyAsync(ctx->dict_md.p, mdict.data(), mdict.size() * sizeof(ZbMemberDict), cudaMemcpyHostToDevice, s));
  if (fname_lens && data_format == ZB200_DF_GZIP)
    CK(cudaMemcpyAsync(ctx->fname.p, fname_lens, n, cudaMemcpyHostToDevice, s));
  if (sp) CK(cudaMemcpyAsync(d_carry, &sp->carry_in, sizeof(ZbMemberCarry), cudaMemcpyHostToDevice, s));
  CK(cudaMemsetAsync(ctx->group_end.p, 0, sizeof(uint64_t), s));
  if (h_src || h_dst) {
    // the transfer streams must not run ahead of the setup above
    CK(cudaEventRecord(ctx->gev[3 * ng], s));
    if (h_src) CK(cudaStreamWaitEvent(sh, ctx->gev[3 * ng], 0));
    if (h_dst) CK(cudaStreamWaitEvent(sd, ctx->gev[3 * ng], 0));
  }
  CK(cudaEventRecord(ctx->ev[6], sh));

  auto make_work = [&](const Group &g, size_t gi) {
    ZbCompressWork w;
    w.src = d_src;
    w.dst = d_dst;
    w.dst_cap = dst_cap;
    w.desc = (const ZbChunkDesc *)ctx->desc.p + g.c0;
    w.member_first = (const uint32_t *)ctx->member_first.p + g.first0;
    w.fname_len = (fname_lens && data_format == ZB200_DF_GZIP) ? (const uint8_t *)ctx->fname.p + g.m0 : nullptr;
    w.masks = (uint2 *)ctx->masks.p;
    w.recs = (uint32_t *)ctx->recs.p;
    w.hist = (uint16_t *)ctx->hist.p;
    w.chk = (ZbChunkCheck *)ctx->chk.p;
    w.cb = (ZbCodebook *)ctx->cb.p;
    w.chunk_off = (uint64_t *)ctx->chunk_off.p;
    w.member_off = (uint64_t *)ctx->member_off.p + g.first0;
    w.member_check = (uint32_t *)ctx->member_check.p;
    w.member_isize = (uint32_t *)ctx->member_isize.p;
    w.carry_in = sp ? d_carry : nullptr;
    w.carry_out = sp ? d_carry + 1 : nullptr;
    w.tabs = ctx->d_tabs;
    w.lz2_tables = (uint2 *)ctx->lz2_tables.p;
    w.n_chunks = (uint32_t)g.nc;
    w.n_members = (uint32_t)(g.m1 - g.m0);
    w.level = level;
    w.strategy = strategy;
    w.max_dist = 1u << window_bits;
    w.data_format = data_format;
    w.out_base = 0;
    w.out_base_ptr = (const uint64_t *)ctx->group_end.p + gi;
    w.mdict = mdict.empty() ? nullptr : (const ZbMemberDict *)ctx->dict_md.p + g.m0;
    w.dict_hist = dict_hist ? 1 : 0;
    w.opt_scratch = (uint8_t *)ctx->opt_scratch.p;
    return w;
  };

  // ---- enqueue every group ----
  size_t d2h_done = 0;  // groups whose output has been handed to the D2H stream
  uint64_t total_out = 0;
  auto drain_d2h = [&](size_t upto) -> int {  // enqueue D2H for groups [d2h_done, upto)
    for (; d2h_done < upto; d2h_done++) {
      const Group &g = groups[d2h_done];
      CK(cudaEventSynchronize(ctx->gev[3 * d2h_done + 2]));  // offsets of this group are in pin_off
      const size_t nm = g.m1 - g.m0;
      const uint64_t lo = pin_off[g.first0], hi = pin_off[g.first0 + nm];
      for (size_t j = 0; j <= nm; j++) dst_offsets[g.m0 + j] = pin_off[g.first0 + j];
      total_out = hi;
      if (h_dst) {
        if (hi > h_dst_cap) return ZB200_ERR_DST_TOO_SMALL;
        CK(cudaStreamWaitEvent(sd, ctx->gev[3 * d2h_done + 1], 0));
        if (d2h_done == 0) CK(cudaEventRecord(ctx->ev[8], sd));
        if (hi > lo) {
          int rc2 = d2h_copy(ctx, h_dst + lo, d_dst + lo, (size_t)(hi - lo), sd, dst_pageable);
          if (rc2) return rc2;
        }
      }
    }
    return ZB200_OK;
  };

  for (size_t gi = 0; gi < ng; gi++) {
    const Group &g = groups[gi];
    if (h_src) {
      if (dict_hist) {   // the slot's previous group has been packed (its k_lz2 is done)
        if (gi >= dw.slots) CK(cudaStreamWaitEvent(sh, ctx->gev[3 * (gi - dw.slots) + 1], 0));
        if (int rc2 = dw.upload(ctx, gi, sh)) return rc2;
      }
      if (g.in_hi > g.in_lo) {
        int rc2 = h2d_copy(ctx, (uint8_t *)d_src + g.in_lo, h_src + src_lo + g.in_lo, (size_t)(g.in_hi - g.in_lo), sh, src_pageable);
        if (rc2) return rc2;
      }
      CK(cudaEventRecord(ctx->gev[3 * gi + 0], sh));
      CK(cudaStreamWaitEvent(s, ctx->gev[3 * gi + 0], 0));
    }
    ZbCompressWork w = make_work(g, gi);
    const bool timed = (gi == 0);  // per-kernel events on the first group; totals are scaled by chunk count
    if (timed) {
      ctx->timing.plan_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t_entry).count();
      CK(cudaEventRecord(ctx->ev[0], s));
    }
    CK(zb_launch_lz(w, s, ix != nullptr));
    if (timed) CK(cudaEventRecord(ctx->ev[1], s));
    CK(zb_launch_huff(w, s));
    if (timed) CK(cudaEventRecord(ctx->ev[2], s));
    CK(zb_launch_scan(w, s));
    if (timed) CK(cudaEventRecord(ctx->ev[3], s));
    // chain: the next group starts where this one ended
    CK(cudaMemcpyAsync((uint64_t *)ctx->group_end.p + gi + 1, w.member_off + w.n_members, sizeof(uint64_t),
                       cudaMemcpyDeviceToDevice, s));
    CK(cudaMemcpyAsync(pin_off + g.first0, w.member_off, (w.n_members + 1) * sizeof(uint64_t),
                       cudaMemcpyDeviceToHost, s));
    if (sp) CK(cudaMemcpyAsync(pin_carry, w.carry_out, sizeof(ZbMemberCarry), cudaMemcpyDeviceToHost, s));
    CK(cudaEventRecord(ctx->gev[3 * gi + 2], s));
    if (ix) {
      ZbIndexWork x = *ix;
      x.rec_first += g.m0;
      CK(zb_launch_index_rec(w, x, s));
      ctx->timing.kernel_launches += 1;
    }
    if (timed) CK(cudaEventRecord(ctx->ev[4], s));
    CK(zb_launch_pack(w, s));
    if (timed) CK(cudaEventRecord(ctx->ev[5], s));
    CK(cudaEventRecord(ctx->gev[3 * gi + 1], s));
    ctx->timing.kernel_launches += 5;
    ctx->timing.n_chunks += (uint32_t)g.nc;
    // keep at most two groups of output waiting on the device before draining to the host
    if (h_dst && gi >= 2) {
      int rc = drain_d2h(gi - 1);
      if (rc) return rc;
    }
  }
  if (h_src) CK(cudaEventRecord(ctx->ev[7], sh));
  {
    int rc = drain_d2h(ng);
    if (rc) return rc;
  }
  if (h_dst) CK(cudaEventRecord(ctx->ev[9], sd));
  if (dst_pageable) {
    int rc = d2h_flush(ctx);
    if (rc) return rc;
  }
  CK(cudaStreamSynchronize(s));
  if (h_src) CK(cudaStreamSynchronize(sh));
  if (h_dst) CK(cudaStreamSynchronize(sd));
  if (total_out > dst_cap) return ZB200_ERR_DST_TOO_SMALL;
  if (sp) sp->carry_out = *pin_carry;
  // per-kernel times: measured on the first group, scaled to the batch by chunk count
  const float scale = groups[0].nc ? (float)nc_all / (float)groups[0].nc : 1.f;
  ctx->timing.lz_ms = ev_ms(ctx->ev[0], ctx->ev[1]) * scale;
  ctx->timing.huff_ms = ev_ms(ctx->ev[1], ctx->ev[2]) * scale;
  ctx->timing.scan_ms = ev_ms(ctx->ev[2], ctx->ev[3]) * scale;
  ctx->timing.pack_ms = ev_ms(ctx->ev[4], ctx->ev[5]) * scale;
  return ZB200_OK;
}

// ---- compress-time index ----
// The rule that turns access-point records into an index's points, shared by zb200_index_build and the compress
// calls that write an index: (b, o) is the point recorded for the next multiple k * 32768, k increasing.  A record
// that repeats the last point adds nothing.  A new point is a window point when it is the first at or past
// next_win (the next multiple of the span); one with o > 0 gets 32 KiB of idx->windows (win_at) that the caller
// fills with the output in front of it.  Returns 1 for a new point, 0 for a repeat, -1 for records out of order.
int index_add_point(zb200_index *idx, uint64_t b, uint64_t o, uint64_t &next_win) {
  if (!idx->bit.empty() && idx->bit.back() == b) return 0;
  if (!idx->bit.empty() && (b < idx->bit.back() || o <= idx->out.back())) return -1;
  idx->bit.push_back(b);
  idx->out.push_back(o);
  const bool win = o >= next_win;
  idx->win.push_back(win ? 1 : 0);
  idx->win_at.push_back(~0ull);
  if (win) {
    next_win = (o / idx->span + 1) * idx->span;
    if (o > 0) {
      idx->win_at.back() = idx->windows.size();
      idx->windows.resize(idx->windows.size() + 32768);
    }
  }
  return 1;
}

// the header bytes in front of a member's first block
uint64_t frame_head(int data_format, uint8_t fname_len) {
  return data_format == ZB200_DF_GZIP ? 11u + fname_len : data_format == ZB200_DF_ZLIB ? 2u : 0u;
}

// ZbIndexWork's device arrays for nrec records of the members whose first records are rec_first: the records
// prefilled with ~0, the launch words zeroed (k0, lo0 and byte_base are the caller's)
int index_rec_prepare(zb200_ctx *ctx, const std::vector<uint64_t> &rec_first, size_t nrec, ZbIndexWork &x) {
  ENSURE(ctx->cix_rec, nrec * 16 + 16);
  ENSURE(ctx->cix_crc, nrec * 4 + 4);
  ENSURE(ctx->cix_first, rec_first.size() * 8 + 8);
  ENSURE(ctx->cix_out, 16);
  CK(cudaMemcpyAsync(ctx->cix_first.p, rec_first.data(), rec_first.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemsetAsync(ctx->cix_rec.p, 0xff, nrec * 16, ctx->stream));
  CK(cudaMemsetAsync(ctx->cix_out.p, 0, 16, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));   // rec_first is pageable host memory
  memset(&x, 0, sizeof(x));
  x.rec = (uint64_t *)ctx->cix_rec.p;
  x.crc = (uint32_t *)ctx->cix_crc.p;
  x.rec_first = (const uint64_t *)ctx->cix_first.p;
  x.launch_out = (uint64_t *)ctx->cix_out.p;
  return ZB200_OK;
}

int index_rec_fetch(zb200_ctx *ctx, size_t nrec, std::vector<uint64_t> &rec, std::vector<uint32_t> &crc, uint64_t *launch_out) {
  rec.resize(nrec * 2);
  crc.resize(nrec);
  CK(cudaMemcpyAsync(rec.data(), ctx->cix_rec.p, nrec * 16, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(crc.data(), ctx->cix_crc.p, nrec * 4, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(launch_out, ctx->cix_out.p, 16, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return ZB200_OK;
}

// A stream launch that wrote the member's input [start, start + nbytes) (`in`) and dst_len bytes at dst, with
// nrec records from multiple k0 on: its points join the stream's index.  The interval of the last point stays open
// (a raw CRC) until a later launch records the next point or ends the member.
int stream_index_launch(zb200_compress_stream *st, const uint8_t *in, size_t nbytes, bool last, const uint8_t *dst,
                        size_t dst_len, size_t nrec) {
  zb200_ctx *ctx = st->ctx;
  std::vector<uint64_t> rec;
  std::vector<uint32_t> crc;
  uint64_t lout[2];
  int rc = index_rec_fetch(ctx, nrec, rec, crc, lout);
  if (rc) return rc;
  zb200_index *idx = st->ix.get();
  const uint64_t start = st->carry.bytes, end = start + nbytes;
  bool none = true;
  for (size_t r = 0; r < nrec; r++) {
    const uint64_t b = rec[2 * r], o = rec[2 * r + 1];
    if (b == ~0ull) continue;
    const size_t before = idx->bit.size();
    const int a = index_add_point(idx, b, o, st->ix_next);
    if (a < 0) {
      ctx->last_err = "compress-time index: records out of order";
      return ZB200_ERR_CUDA;
    }
    if (!a) continue;
    if (none) {  // the open interval ends here
      none = false;
      st->ix_raw = zb_gf2_mul(st->ix_raw, zb_xpow8(o - start)) ^ (uint32_t)lout[1];
      if (st->ix_open) idx->crc.back() = zb_crc32_finalize(st->ix_raw, o - idx->out[before - 1]);
    }
    idx->crc.push_back(crc[r]);
    if (idx->win_at.back() != ~0ull) {   // the 32 KiB of input in front of the point: held input, then this launch's
      uint8_t *w = idx->windows.data() + idx->win_at.back();
      const uint64_t lo = o - 32768ull;
      const size_t held = lo < start ? (size_t)(start - lo) : 0;
      if (held) memcpy(w, st->ix_in.data() + st->ix_in.size() - held, held);
      memcpy(w + held, in + (lo + held - start), 32768 - held);
    }
  }
  if (none) {
    st->ix_raw = zb_gf2_mul(st->ix_raw, zb_xpow8(nbytes)) ^ (uint32_t)lout[1];
  } else {
    st->ix_open = !last;
    if (!last) st->ix_raw = idx->crc.back();
  }
  if (last && st->ix_open) {
    idx->crc.back() = zb_crc32_finalize(st->ix_raw, end - idx->out.back());
    st->ix_open = false;
  }
  st->ix_lo = lout[0] + 1;
  if (nbytes >= 32768) {
    st->ix_in.assign(in + nbytes - 32768, in + nbytes);
  } else {
    st->ix_in.insert(st->ix_in.end(), in, in + nbytes);
    if (st->ix_in.size() > 32768) st->ix_in.erase(st->ix_in.begin(), st->ix_in.end() - 32768);
  }
  for (size_t i = 0; i < dst_len && idx->len + i < 32; i++) idx->head[idx->len + i] = dst[i];
  st->ix_tail.insert(st->ix_tail.end(), dst + (dst_len > 32 ? dst_len - 32 : 0), dst + dst_len);
  if (st->ix_tail.size() > 32) st->ix_tail.erase(st->ix_tail.begin(), st->ix_tail.end() - 32);
  idx->len += dst_len;
  if (last) {
    idx->size = end;
    memset(idx->tail, 0, 32);
    memcpy(idx->tail, st->ix_tail.data(), st->ix_tail.size());
  }
  return ZB200_OK;
}

// Compress the stream's next `nbytes` pending bytes into dst; ctx locked.  They are whole chunks, unless the run
// ends the member (`last`) or a flush segment (a flush: every pending byte, last = false).  On success the carry
// advances and the compressed input leaves the buffer: its last 32 KiB stay as history, none after a full flush
// (`reset`).  On failure nothing changes.
int stream_run(zb200_compress_stream *st, size_t nbytes, bool last, uint8_t *dst, size_t dst_cap, size_t *dst_len,
               bool reset = false) {
  zb200_ctx *ctx = st->ctx;
  if (!dst) return ZB200_ERR_DST_TOO_SMALL;  // every run emits at least one byte
  const size_t in_end = st->hist + nbytes;
  ENSURE(ctx->in_stage, in_end + 64);
  ENSURE(ctx->out_stage, zb200_compress_bound(nbytes, st->data_format) + 128);
  const uint64_t offs[2] = {st->hist, in_end};
  uint64_t dst_offs[2] = {0, 0};
  StreamPart sp;
  sp.hist = (uint32_t)st->hist;
  sp.head = !st->head_done;
  sp.last = last;
  sp.carry_in = st->carry;
  sp.has_dict = st->has_dict;
  sp.dict_id = st->dict_id;
  ZbIndexWork x;
  size_t nrec = 0;
  if (st->ix) {   // the multiples this launch's block starts can own: from the first one past the last block start on
    const uint64_t k0 = (st->ix_lo + 32767ull) >> 15, kend = (st->carry.bytes + nbytes) >> 15;
    nrec = kend >= k0 ? (size_t)(kend - k0 + 1) : 0;
    int rc = index_rec_prepare(ctx, std::vector<uint64_t>(1, 0), nrec, x);
    if (rc) return rc;
    x.k0 = k0;
    x.lo0 = st->ix_lo;
    x.byte_base = st->ix->len;
  }
  int rc = compress_locked(ctx, (const uint8_t *)ctx->in_stage.p, st->buf.data(), offs, 1, st->level, st->data_format,
                           &st->fname_len, (uint8_t *)ctx->out_stage.p, ctx->out_stage.cap & ~(size_t)3, dst, dst_cap,
                           dst_offs, nullptr, ctx->host_group_chunks, &sp, st->ix ? &x : nullptr, st->strategy,
                           st->window_bits, st->optimal);
  if (rc) return rc;
  *dst_len = (size_t)dst_offs[1];
  if (st->ix) {
    rc = stream_index_launch(st, st->buf.data() + st->hist, nbytes, last, dst, *dst_len, nrec);
    if (rc) return rc;
  }
  st->carry = sp.carry_out;
  st->head_done = true;
  const bool lz = st->level == -1 || st->level >= 2;
  const size_t keep = lz && !reset ? std::min<size_t>(32768, in_end) : 0;
  st->buf.erase(st->buf.begin(), st->buf.begin() + (in_end - keep));
  st->hist = keep;
  return ZB200_OK;
}

// ZB_CK_PIECE_BYTES pieces covering the capacity [offs[i], offs[i+1]) of every buffer (at least one per buffer)
int upload_pieces(zb200_ctx *ctx, const uint64_t *offs, size_t n, ZbChecksumWork &w) {
  std::vector<ZbPiece> pieces;
  std::vector<uint32_t> first(n + 1);
  for (size_t i = 0; i < n; i++) {
    first[i] = (uint32_t)pieces.size();
    uint64_t cap = offs[i + 1] - offs[i];
    uint64_t rel = 0;
    do {
      ZbPiece p;
      p.rel = rel;
      p.buf = (uint32_t)i;
      p.pad = 0;
      pieces.push_back(p);
      rel += ZB_CK_PIECE_BYTES;
    } while (rel < cap);
  }
  first[n] = (uint32_t)pieces.size();
  w.big_pieces = 0;
  for (size_t i = 0; i < n; i++)
    if (first[i + 1] - first[i] > ZB_CK_BIG_PIECES) w.big_pieces = ZB_CK_BIG_PIECES;
  ENSURE(ctx->ck_pieces, pieces.size() * sizeof(ZbPiece));
  ENSURE(ctx->ck_first, (n + 1) * sizeof(uint32_t));
  ENSURE(ctx->ck_piece_out, pieces.size() * sizeof(ZbChunkCheck));
  ENSURE(ctx->ck_partials, pieces.size() * (size_t)ZB_CK_PARTIAL_BYTES);
  w.partials = (uint32_t *)ctx->ck_partials.p;
  CK(cudaMemcpyAsync(ctx->ck_pieces.p, pieces.data(), pieces.size() * sizeof(ZbPiece), cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(ctx->ck_first.p, first.data(), (n + 1) * sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));  // the host vectors go out of scope
  w.pieces = (const ZbPiece *)ctx->ck_pieces.p;
  w.first = (const uint32_t *)ctx->ck_first.p;
  w.piece_out = (ZbChunkCheck *)ctx->ck_piece_out.p;
  w.n_pieces = (uint32_t)pieces.size();
  w.tabs = ctx->d_tabs;
  w.n = (uint32_t)n;
  return ZB200_OK;
}


// ---- large members as parallel segments (SURVEY 8f-1) ----
// A DEFLATE stream is serial, and one member is decoded by one 8-lane group: a single multi-MiB
// member would crawl.  But this library's own multi-chunk members (and zlib's Z_FULL_FLUSH /
// pigz -i streams) are chains of INDEPENDENT, byte-aligned pieces, each ending with the empty
// stored block 00 00 ff ff.  So a large member is handled speculatively: find every 00 00 ff ff
// in its payload, decode the pieces between them as separate raw-deflate segments (a count pass
// for the sizes, then the real pass at the prefix-summed positions), and accept the result only
// if every segment decodes cleanly, only the last one holds the final block, and the sizes add up
// inside the member's capacity.  Anything else (a false 00 00 ff ff inside data, a back-reference
// across a boundary, a corrupt stream) leaves the member to the ordinary serial decode, which
// also produces the reference's error for it.  The trailer check runs on the output either way.
struct HostWrapper {
  int fmt;
  uint64_t pos, end;  // payload [pos, end) inside the member
  uint32_t expect, isize;
};

// zippy.nim:100-165 + gzip.nim:3-66 on the first hn bytes / last 8 bytes of a member; false when
// the member is not acceptable or the header does not fit in hn (then the serial path decides).
bool host_parse_wrapper(const uint8_t *h, size_t hn, const uint8_t *t8, uint64_t len, int fmt, uint64_t raw_pos,
                        HostWrapper &w) {
  auto le32 = [](const uint8_t *p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); };
  if (fmt == ZB200_DF_DETECT) {
    if (len > 18 && hn >= 4 && h[0] == 31 && h[1] == 139 && h[2] == 8 && (h[3] & 0xe0) == 0) fmt = ZB200_DF_GZIP;
    else if (len > 6 && hn >= 2 && (h[0] & 0x0f) == 8 && (h[0] >> 4) <= 7 && (((uint32_t)h[0] * 256u) + h[1]) % 31u == 0)
      fmt = ZB200_DF_ZLIB;
    else return false;
  }
  w.fmt = fmt;
  w.expect = w.isize = 0;
  if (fmt == ZB200_DF_GZIP) {
    if (len < 18 || hn < 10) return false;
    uint32_t flg = h[3];
    if (h[0] != 31 || h[1] != 139 || h[2] != 8 || (flg & 0xe0) || (flg & 4)) return false;
    uint64_t p = 10;
    for (int pass = 0; pass < 2; pass++)
      if ((pass == 0 && (flg & 8)) || (pass == 1 && (flg & 16))) {
        while (p < hn && h[p] != 0) p++;
        if (p >= hn) return false;
        p++;
      }
    if (flg & 2) p += 2;
    if (p + 8 >= len) return false;
    w.pos = p;
    w.end = len - 8;
    w.expect = le32(t8);
    w.isize = le32(t8 + 4);
    return true;
  }
  if (fmt == ZB200_DF_ZLIB) {
    if (len < 6 || hn < 2) return false;
    uint32_t cmf = h[0], flg = h[1];
    if ((cmf & 0x0f) != 8 || (cmf >> 4) > 7 || (cmf * 256u + flg) % 31u != 0 || (flg & 0x20)) return false;
    w.pos = 2;
    w.end = len - 4;
    w.expect = ((uint32_t)t8[4] << 24) | ((uint32_t)t8[5] << 16) | ((uint32_t)t8[6] << 8) | t8[7];
    return true;
  }
  if (fmt == ZB200_DF_DEFLATE) {
    if (raw_pos > len) return false;
    w.pos = raw_pos;
    w.end = len;
    return true;
  }
  return false;
}

struct BigResult {
  size_t member;
  uint64_t out_len;
  uint32_t kind, expect;
  int status = ZB200_OK;
};

// ---- the mechanics every parallel segment decode shares ----
// (The large-member, decompress stream and index paths decide what to launch; the helpers launch it.  Launch counts
// stay with the callers, in timing.kernel_launches, where each path keeps its own convention.)

// Segment start candidates in src, sorted: with `blocks`, the bit positions in [lo, hi) where a dynamic block could
// start (k_find_blocks; bytes from limit_byte on read as zero), else the byte positions in [lo, hi) just past a
// 00 00 ff ff (k_find_sync).  Empty when there are none, or more than cap (then the list is incomplete).
int find_candidates(zb200_ctx *ctx, bool blocks, const uint8_t *src, uint64_t lo, uint64_t hi, uint64_t limit_byte,
                    uint32_t cap, std::vector<uint64_t> &cand) {
  cudaStream_t s = ctx->stream;
  cand.clear();
  ENSURE(ctx->seg_cand, (size_t)cap * 8 + 16);
  uint32_t *d_cnt = &counters(ctx)->cand;
  if (blocks) CK(zb_launch_find_blocks(src, lo, hi, limit_byte, (uint64_t *)ctx->seg_cand.p, cap, d_cnt, s));
  else CK(zb_launch_find_sync(src, lo, hi, (uint64_t *)ctx->seg_cand.p, cap, d_cnt, s));
  uint32_t cnt = 0;
  CK(cudaMemcpyAsync(&cnt, d_cnt, 4, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  if (cnt == 0 || cnt > cap) return ZB200_OK;
  cand.resize(cnt);
  CK(cudaMemcpyAsync(cand.data(), ctx->seg_cand.p, (size_t)cnt * 8, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  std::sort(cand.begin(), cand.end());
  return ZB200_OK;
}

// Uploads segment (start, end) bit pairs to seg_bits, for w.seg_bits.
int seg_bits_upload(zb200_ctx *ctx, const std::vector<uint64_t> &pairs, ZbInflateWork &w) {
  ENSURE(ctx->seg_bits, pairs.size() * 8);
  CK(cudaMemcpyAsync(ctx->seg_bits.p, pairs.data(), pairs.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
  w.seg_bits = (const uint64_t *)ctx->seg_bits.p;
  return ZB200_OK;
}

// The n segments [b[0], b[1]), ..., [b[n - 1], end) of n consecutive boundaries and an end (bit positions), uploaded.
int seg_bounds_upload(zb200_ctx *ctx, const uint64_t *b, size_t n, uint64_t end, ZbInflateWork &w) {
  std::vector<uint64_t> pairs(2 * n);
  for (size_t i = 0; i < n; i++) {
    pairs[2 * i] = b[i];
    pairs[2 * i + 1] = i + 1 < n ? b[i + 1] : end;
  }
  return seg_bits_upload(ctx, pairs, w);
}

// One segment-mode k_inflate launch over n segments of the raw DEFLATE stream at w.src.  w holds only what the caller
// decides: src, seg_bits (uploaded) or src_off, seg_limit, seg_win0, dst (its offsets are seg_dst), count_only / mark,
// rec*.  Returns every segment's output length, status and kind after one synchronise.  resume: null, or host [2]
// uploaded as ZbInflateWork::resume before the launch and read back with the rest.
int seg_pass(zb200_ctx *ctx, ZbInflateWork w, size_t n, std::vector<uint64_t> &sl, std::vector<int> &sst,
             std::vector<uint32_t> &sk, uint64_t *resume = nullptr) {
  cudaStream_t s = ctx->stream;
  ENSURE(ctx->seg_len, n * 8);
  ENSURE(ctx->seg_status, n * 4);
  ENSURE(ctx->seg_kind, n * 4);
  ENSURE(ctx->seg_expect, n * 4);
  if (resume) {
    w.resume = counters(ctx)->resume;
    CK(cudaMemcpyAsync(w.resume, resume, 16, cudaMemcpyHostToDevice, s));
  }
  w.dst_off = (const uint64_t *)ctx->seg_dst.p;
  w.out_len = (uint64_t *)ctx->seg_len.p;
  w.status = (int *)ctx->seg_status.p;
  w.expect = (uint32_t *)ctx->seg_expect.p;
  w.kind = (uint32_t *)ctx->seg_kind.p;
  w.counter = &counters(ctx)->segment;
  w.tabs = ctx->d_tabs;
  w.n = (uint32_t)n;
  w.data_format = ZB200_DF_DEFLATE;
  w.seg_mode = 1;
  CK(zb_launch_inflate(w, s));
  sl.resize(n);
  sst.resize(n);
  sk.resize(n);
  CK(cudaMemcpyAsync(sl.data(), ctx->seg_len.p, n * 8, cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(sst.data(), ctx->seg_status.p, n * 4, cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(sk.data(), ctx->seg_kind.p, n * 4, cudaMemcpyDeviceToHost, s));
  if (resume) CK(cudaMemcpyAsync(resume, w.resume, 16, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  return ZB200_OK;
}

// Uploads a marker layout for a marker pass and the resolve -- segs to mark_segs, every segment's first element
// offset in the scratch to seg_dst (dof.back(): the scratch's size in elements) -- and fills the marker symbols in
// front of every segment (k_mark_prefill).
int mark_upload(zb200_ctx *ctx, const std::vector<ZbMarkSegHost> &segs, const std::vector<uint64_t> &dof) {
  cudaStream_t s = ctx->stream;
  ENSURE(ctx->mark_scratch, (size_t)dof.back() * 2 + 64);
  ENSURE(ctx->mark_segs, segs.size() * sizeof(ZbMarkSegHost) + 16);
  ENSURE(ctx->seg_dst, dof.size() * 8);
  CK(cudaMemcpyAsync(ctx->seg_dst.p, dof.data(), dof.size() * 8, cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(ctx->mark_segs.p, segs.data(), segs.size() * sizeof(ZbMarkSegHost), cudaMemcpyHostToDevice, s));
  CK(zb_launch_mark_prefill((uint16_t *)ctx->mark_scratch.p, ctx->mark_segs.p, (uint32_t)segs.size(), s));
  return ZB200_OK;
}

// The marker layout of n consecutive segments of sizes[i] output bytes, [32768 markers | sizes[i] symbols] each, whose
// bytes go to dst0 on in order; uploaded and prefilled (mark_upload).  max_n: the largest size.
int mark_segments(zb200_ctx *ctx, const uint64_t *sizes, size_t n, uint64_t dst0, std::vector<ZbMarkSegHost> &segs,
                  uint32_t &max_n) {
  segs.resize(n);
  std::vector<uint64_t> dof(n + 1);
  uint64_t se = 0, de = dst0;
  max_n = 0;
  for (size_t i = 0; i < n; i++) {
    se += 32768ull;
    segs[i].scr = se;
    segs[i].dst = de;
    segs[i].n = (uint32_t)sizes[i];
    segs[i].pad = 0;
    dof[i] = se;
    se += sizes[i];
    de += sizes[i];
    max_n = std::max<uint32_t>(max_n, (uint32_t)sizes[i]);
  }
  dof[n] = se;
  return mark_upload(ctx, segs, dof);
}

// The parallel window resolve (zb_resolve.h) of the n segments in mark_segs into dst, in groups of ceil(sqrt(n))
// segments; base / w0 as in zb_kernels.h.  bad: null, or where to read the `bad` flag after the resolve (one
// synchronise); the flag is cleared by the caller, once for all the windows it gathers.
int resolve_window(zb200_ctx *ctx, size_t n, uint32_t max_n, uint64_t base, uint64_t w0, uint8_t *dst, int *bad) {
  cudaStream_t s = ctx->stream;
  const uint32_t gsz = std::max<uint32_t>(1u, (uint32_t)std::ceil(std::sqrt((double)n)));
  const size_t ngroups = (n + gsz - 1) / gsz;
  ENSURE(ctx->mark_win, ngroups * 32768ull * 3);
  int *d_bad = &counters(ctx)->bad;
  CK(zb_launch_resolve_groups((uint16_t *)ctx->mark_scratch.p, ctx->mark_segs.p, (uint32_t)n, max_n, gsz, base, w0,
                              (uint16_t *)ctx->mark_win.p, (uint8_t *)ctx->mark_win.p + ngroups * 65536ull, dst, d_bad, s));
  if (bad) {
    CK(cudaMemcpyAsync(bad, d_bad, 4, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
  }
  return ZB200_OK;
}

// ---- a large member WITHOUT sync markers (any foreign gzip / zlib / raw stream) ----
// 1. k_find_blocks lists every plausible dynamic-block start in the payload; the list is thinned to one
//    boundary per >= 16 KiB of input.  2. A counting pass decodes every segment [boundary i, boundary i+1)
//    in parallel, each from its own block start with an UNKNOWN 32 KiB window (back-references before the
//    segment's start are allowed, nothing is written): it must end exactly on the next boundary, and only the
//    last segment may hold the final block -- this is what exposes a false boundary.  3. The sizes give every
//    segment its place; the segments are decoded again into uint16 symbols, with marker symbols standing in
//    for the bytes of the unknown window.  4. The markers are resolved: the last 32 KiB of every segment in
//    order (one CTA), then everything else in parallel.  Anything irregular -- a decode error, a boundary
//    that is not hit, a marker that points before the start of the stream -- leaves the member to the serial
//    decode, which also produces the reference's verdict for it.  The trailer check runs on the output
//    either way.
int inflate_member_speculative(zb200_ctx *ctx, const uint8_t *d_src, uint64_t m0, const HostWrapper &hw, uint8_t *d_dst,
                               uint64_t dst0, uint64_t mcap, bool count_only, bool latency, bool &ok, uint64_t &out_len,
                               bool &too_small) {
  ok = false;
  too_small = false;
  cudaStream_t s = ctx->stream;
  const uint64_t lo_bit = (m0 + hw.pos) * 8ull, hi_bit = (m0 + hw.end) * 8ull, limit_byte = m0 + hw.end;
  const uint32_t cap = (uint32_t)std::min<uint64_t>((hw.end - hw.pos) / 64 + 1024, 1u << 24);
  std::vector<uint64_t> cand;
  int rc = find_candidates(ctx, true, d_src, lo_bit, hi_bit, limit_byte, cap, cand);
  if (rc) return rc;
  ctx->timing.kernel_launches += 1;
  if (cand.empty()) return ZB200_OK;
  // boundaries: the payload start, then candidates at least min_gap apart (a segment costs a 64 KiB marker prefill)
  // (at most 60000 segments: the resolve kernels index them with a grid dimension)
  // a single input is all the GPU has: cut it as finely as its blocks allow
  const uint64_t min_gap = std::max<uint64_t>((latency ? 2048ull : 16384ull) * 8ull, (hi_bit - lo_bit) / 60000ull);
  std::vector<uint64_t> bits(1, lo_bit);
  for (uint64_t c : cand)
    if (c >= bits.back() + min_gap && c + min_gap / 4 < hi_bit) bits.push_back(c);
  const size_t S = bits.size();
  if (S < 2) return ZB200_OK;
  ZbInflateWork w;
  memset(&w, 0, sizeof(w));
  w.src = d_src;
  w.seg_limit = limit_byte;
  rc = seg_bounds_upload(ctx, bits.data(), S, hi_bit, w);
  if (rc) return rc;
  std::vector<uint64_t> sl;
  std::vector<int> sst;
  std::vector<uint32_t> sk;
  // 2. the counting pass
  w.count_only = 1;
  rc = seg_pass(ctx, w, S, sl, sst, sk);
  if (rc) return rc;
  ctx->timing.kernel_launches += 1;
  uint64_t total = 0;
  for (size_t i = 0; i < S; i++) {
    if (sst[i] != ZB200_OK || (sk[i] != 0) != (i + 1 == S) || sl[i] > 0xf0000000ull) return ZB200_OK;
    total += sl[i];
  }
  if (count_only) {
    ok = true;
    out_len = total;
    return ZB200_OK;
  }
  if (total > mcap) {   // the whole stream decodes, so the serial decode could only run out of room: say so now
    too_small = true;
    return ZB200_OK;
  }
  // 3. uint16 symbols, markers in front of every segment
  const std::vector<uint64_t> want = sl;
  int *d_bad = &counters(ctx)->bad;
  CK(cudaMemsetAsync(d_bad, 0, 4, s));
  std::vector<ZbMarkSegHost> segs;
  uint32_t max_n = 0;
  rc = mark_segments(ctx, want.data(), S, dst0, segs, max_n);
  if (rc) return rc;
  w.count_only = 0;
  w.mark = 1;
  w.dst = (uint8_t *)ctx->mark_scratch.p;
  rc = seg_pass(ctx, w, S, sl, sst, sk);
  if (rc) return rc;
  ctx->timing.kernel_launches += 2;
  for (size_t i = 0; i < S; i++)
    if (sst[i] != ZB200_OK || sl[i] != want[i]) return ZB200_OK;
  // 4. markers -> bytes
  CK(zb_launch_resolve((const uint16_t *)ctx->mark_scratch.p, ctx->mark_segs.p, (uint32_t)S, max_n, dst0, d_dst, d_bad, s));
  int bad = 0;
  CK(cudaMemcpyAsync(&bad, d_bad, 4, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  ctx->timing.kernel_launches += 2;
  if (bad) return ZB200_OK;
  ok = true;
  out_len = total;
  return ZB200_OK;
}

// ---- a large member cut at its sync joints, whose pieces refer back across them ----
// This library's levels -1 and 2..9 stage every 64 KiB chunk with the member's previous 32 KiB, so its matches
// reach back across the 00 00 ff ff joints and the pieces between them are not independent.  The joints are
// still exact block boundaries: every segment is decoded from its joint (bit-exact seg_bits) straight into
// uint16 symbols, with marker symbols for the unknown 32 KiB in front of it, and the markers are resolved.
// Sizes: first the 64 KiB-per-segment guess (what this library's chunks produce) with no count pass; if a
// segment disagrees, a count pass in marker mode.  A count pass whose segments on both sides of a joint fail
// drops that joint (a 00 00 ff ff inside stored data or inside Huffman bits) and counts again, at most twice.
// The member is processed in windows of segments (ctx->mark_window_segs, and about as much output as that many
// full chunks): every window starts from the resolved output in front of it, so the scratch depends on the
// window, not on the member.  Anything irregular leaves the member to the speculative and serial paths.
// bounds: absolute bit offsets of the S + 1 (byte-aligned) segment boundaries in d_src.
int inflate_member_joints(zb200_ctx *ctx, const uint8_t *d_src, uint64_t limit_byte, std::vector<uint64_t> bounds,
                          uint8_t *d_dst, uint64_t dst0, uint64_t mcap, bool count_only, bool guess, bool &ok,
                          uint64_t &out_len, bool &too_small) {
  ok = false;
  too_small = false;
  cudaStream_t s = ctx->stream;
  ZbInflateWork w;
  memset(&w, 0, sizeof(w));
  w.src = d_src;
  w.seg_limit = limit_byte;
  std::vector<uint64_t> sl;
  std::vector<int> sst;
  std::vector<uint32_t> sk;
  // one decode launch over segments [a, b): counting, or marker symbols into mark_scratch at seg_dst
  auto run = [&](size_t a, size_t b, bool count) -> int {
    int rc = seg_bounds_upload(ctx, bounds.data() + a, b - a, bounds[b], w);
    if (rc) return rc;
    w.dst = count ? nullptr : (uint8_t *)ctx->mark_scratch.p;
    w.seg_win0 = a > 0;
    w.count_only = count ? 1 : 0;
    w.mark = count ? 0 : 1;
    return seg_pass(ctx, w, b - a, sl, sst, sk);
  };
  // exact sizes of every segment, with the repair rounds; counted = false: give up on this path
  std::vector<uint64_t> size;
  bool counted = false;
  auto count_all = [&]() -> int {
    for (int round = 0;; round++) {
      const size_t S = bounds.size() - 1;
      int rc = run(0, S, true);
      if (rc) return rc;
      ctx->timing.kernel_launches += 1;
      std::vector<char> fail(S);
      bool any = false;
      for (size_t i = 0; i < S; i++) {
        fail[i] = sst[i] != ZB200_OK || (sk[i] != 0) != (i + 1 == S) || sl[i] > 0xf0000000ull;
        any = any || fail[i];
      }
      std::vector<uint64_t> nb(1, bounds[0]);
      if (any) {   // a false joint: both segments around it fail
        for (size_t k = 1; k < S; k++)
          if (!(fail[k - 1] && fail[k])) nb.push_back(bounds[k]);
      } else {     // a segment that starts before output byte 32768 could reach before the stream: join it to segment 0
        uint64_t p = sl[0];
        for (size_t k = 1; k < S; k++) {
          if (p >= 32768ull) nb.push_back(bounds[k]);
          p += sl[k];
        }
      }
      nb.push_back(bounds[S]);
      if (nb.size() == bounds.size()) {
        counted = !any;
        size = sl;
        return ZB200_OK;
      }
      if (round == 2) return ZB200_OK;
      bounds.swap(nb);
    }
  };
  if (count_only || !guess) {
    int rc = count_all();
    if (rc || !counted) return rc;
    uint64_t total = 0;
    for (uint64_t v : size) total += v;
    if (count_only) {
      ok = true;
      out_len = total;
      return ZB200_OK;
    }
    if (total > mcap) {   // the whole stream decodes, so the serial decode could only run out of room: say so now
      too_small = true;
      return ZB200_OK;
    }
  } else if ((uint64_t)(bounds.size() - 2) * ZB_CHUNK_BYTES >= mcap) {
    return ZB200_OK;
  }
  const uint64_t W = ctx->mark_window_segs, win_elems = W * (32768ull + ZB_CHUNK_BYTES);
  CK(cudaMemsetAsync(&counters(ctx)->bad, 0, 4, s));
  int bad = 0;   // every window's resolve sets the flag; it is read after the last one
  std::vector<ZbMarkSegHost> segs;
  uint64_t dpos = dst0;
  for (size_t a = 0; a < bounds.size() - 1;) {
    const size_t S = bounds.size() - 1;
    size_t b = a;
    uint64_t el = 0;
    while (b < S && b - a < W) {
      const uint64_t e = 32768ull + (counted ? size[b] : ZB_CHUNK_BYTES);
      if (b > a && el + e > win_elems) break;
      el += e;
      b++;
    }
    const size_t nw = b - a;
    std::vector<uint64_t> guessed;
    if (!counted) guessed.assign(nw, ZB_CHUNK_BYTES);
    uint32_t max_n = 0;
    int rc = mark_segments(ctx, counted ? size.data() + a : guessed.data(), nw, dpos, segs, max_n);
    if (rc) return rc;
    uint64_t dp = segs[nw - 1].dst + segs[nw - 1].n;
    rc = run(a, b, false);
    if (rc) return rc;
    ctx->timing.kernel_launches += 2;
    bool wok = true;
    for (size_t i = 0; i < nw && wok; i++) {
      const bool last = a + i + 1 == S;
      wok = sst[i] == ZB200_OK && (sk[i] != 0) == last &&
            (counted ? sl[i] == size[a + i] : (last ? sl[i] <= (uint64_t)ZB_CHUNK_BYTES : sl[i] == (uint64_t)ZB_CHUNK_BYTES));
    }
    if (!wok) {
      if (counted) return ZB200_OK;
      // the 64 KiB guess does not hold: exact sizes, then this window again.  (The windows before decoded as
      // guessed, so their segments pass the count too and no joint before `a` is dropped.)
      rc = count_all();
      if (rc || !counted) return rc;
      uint64_t total = 0;
      for (uint64_t v : size) total += v;
      if (total > mcap) {
        too_small = true;
        return ZB200_OK;
      }
      continue;
    }
    if (!counted && b == S) {   // the member's last segment: its size is known now
      dp = segs[nw - 1].dst + sl[nw - 1];
      if (dp - dst0 > mcap) {
        too_small = true;
        return ZB200_OK;
      }
      segs[nw - 1].n = (uint32_t)sl[nw - 1];
      CK(cudaMemcpyAsync((ZbMarkSegHost *)ctx->mark_segs.p + (nw - 1), &segs[nw - 1], sizeof(ZbMarkSegHost),
                         cudaMemcpyHostToDevice, s));
    }
    rc = resolve_window(ctx, nw, max_n, dst0, dpos - dst0, d_dst, b == S ? &bad : nullptr);
    if (rc) return rc;
    ctx->timing.kernel_launches += 4;
    dpos = dp;
    a = b;
  }
  if (bad) return ZB200_OK;
  ok = true;
  out_len = dpos - dst0;
  return ZB200_OK;
}

// Tries every large member; `done` gets the members that were fully decoded here (their output
// is in place; status / length / kind / expect still have to be written to the device arrays).
int inflate_big_members(zb200_ctx *ctx, const uint8_t *d_src, const uint64_t *src_offsets, size_t n, int data_format,
                        uint64_t raw_pos, uint8_t *d_dst, const uint64_t *dst_offsets, bool count_only,
                        std::vector<BigResult> &done) {
  cudaStream_t s = ctx->stream;
  // Every large member costs a few host round trips here, while a batch of thousands of members
  // already fills the GPU with one group per member: with many large members only the huge ones
  // (minutes of serial decode) take this path.
  uint64_t min_len = (n == 1 && !ctx->big_env) ? ctx->single_member_bytes : ctx->big_member_bytes;
  {
    size_t count = 0;
    for (size_t m = 0; m < n; m++) count += (src_offsets[m + 1] - src_offsets[m]) >= min_len;
    if (count == 0) return ZB200_OK;
    if (count > 256) min_len = std::max<uint64_t>(min_len, 64ull << 20);
  }
  for (size_t m = 0; m < n; m++) {
    const uint64_t m0 = src_offsets[m], len = src_offsets[m + 1] - m0;
    if (len < min_len) continue;
    uint8_t head[1024], tail[8];
    const size_t hn = (size_t)std::min<uint64_t>(len, sizeof(head));
    CK(cudaMemcpyAsync(head, d_src + m0, hn, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(tail, d_src + m0 + len - 8, 8, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    HostWrapper hw;
    if (!host_parse_wrapper(head, hn, tail, len, data_format, raw_pos, hw)) continue;
    if (count_only && hw.fmt == ZB200_DF_GZIP) continue;  // ISIZE answers that (gzip.nim:66)
    if (hw.end <= hw.pos + 4) continue;
    const uint64_t dst0_m = count_only ? 0 : dst_offsets[m], mcap_m = count_only ? ~0ull : dst_offsets[m + 1] - dst_offsets[m];
    // streams without sync markers (or whose pieces are not independent): speculative segments
    auto speculative = [&]() -> int {
      bool sok = false, small = false;
      uint64_t slen = 0;
      int src_ = inflate_member_speculative(ctx, d_src, m0, hw, d_dst, dst0_m, mcap_m, count_only, n == 1, sok, slen, small);
      if (src_) return src_;
      if (sok || small) {
        BigResult r;
        r.member = m;
        r.out_len = sok ? slen : 0;
        r.kind = (uint32_t)hw.fmt;
        r.expect = hw.expect;
        r.status = small ? ZB200_ERR_DST_TOO_SMALL : ZB200_OK;
        done.push_back(r);
      }
      return ZB200_OK;
    };
#define ZB_TRY_SPECULATIVE()      \
  {                               \
    int _rc = speculative();      \
    if (_rc) return _rc;          \
    continue;                     \
  }
    // 1. candidate boundaries
    const uint32_t cap = (uint32_t)std::min<uint64_t>((hw.end - hw.pos) / 32 + 64, 1u << 24);
    std::vector<uint64_t> bounds;
    int rc = find_candidates(ctx, false, d_src + m0, hw.pos, hw.end, 0, cap, bounds);
    if (rc) return rc;
    if (bounds.empty()) ZB_TRY_SPECULATIVE();
    bounds.insert(bounds.begin(), hw.pos);
    if (bounds.back() < hw.end) bounds.push_back(hw.end);   // (a payload that ends with a marker: no trailing segment)
    const size_t S = bounds.size() - 1;
    if (S < 2) ZB_TRY_SPECULATIVE();
    for (size_t j = 0; j <= S; j++) bounds[j] += m0;  // absolute in d_src
    ENSURE(ctx->seg_src, (S + 1) * 8);
    ENSURE(ctx->seg_dst, (S + 1) * 8);
    CK(cudaMemcpyAsync(ctx->seg_src.p, bounds.data(), (S + 1) * 8, cudaMemcpyHostToDevice, s));
    ZbInflateWork w;
    memset(&w, 0, sizeof(w));
    w.src = d_src;
    w.src_off = (const uint64_t *)ctx->seg_src.p;
    w.dst = d_dst;
    std::vector<uint64_t> sl, dof(S + 1);
    std::vector<int> sst;
    std::vector<uint32_t> sk;
    const uint64_t dst0 = count_only ? 0 : dst_offsets[m], mcap = count_only ? ~0ull : dst_offsets[m + 1] - dst_offsets[m];
    bool ok = false;
    // segments that refer back across their joints: marker segments (inflate_member_joints); 1 = not handled there
    auto joints = [&](bool guess) -> int {
      if (!ctx->joint_markers) return 1;
      bool jok = false, small = false;
      uint64_t jlen = 0;
      std::vector<uint64_t> jb(S + 1);
      for (size_t j = 0; j <= S; j++) jb[j] = bounds[j] * 8ull;
      int rc_ = inflate_member_joints(ctx, d_src, m0 + hw.end, jb, d_dst, dst0, mcap, count_only, guess, jok, jlen, small);
      if (rc_) return -rc_;
      if (!jok && !small) return 1;
      BigResult r;
      r.member = m;
      r.out_len = jok ? jlen : 0;
      r.kind = (uint32_t)hw.fmt;
      r.expect = hw.expect;
      r.status = small ? ZB200_ERR_DST_TOO_SMALL : ZB200_OK;
      done.push_back(r);
      return 0;
    };
#define ZB_TRY_JOINTS(guess)         \
  {                                  \
    int _jr = joints(guess);         \
    if (_jr < 0) return -_jr;        \
    if (_jr == 0) continue;          \
    ZB_TRY_SPECULATIVE();            \
  }
    // a segment after the first that refers back across its joint fails on its own: no count pass can help
    bool back_refs = false, guess = false;
    // 2. the optimistic pass: this library's own members have 64 KiB of output per segment (the
    // last one takes what is left); if every segment agrees, one pass was enough
    if (!count_only && (S - 1) * (uint64_t)ZB_CHUNK_BYTES < mcap) {
      for (size_t j = 0; j < S; j++) dof[j] = dst0 + j * (uint64_t)ZB_CHUNK_BYTES;
      dof[S] = dst0 + mcap;
      CK(cudaMemcpyAsync(ctx->seg_dst.p, dof.data(), (S + 1) * 8, cudaMemcpyHostToDevice, s));
      w.count_only = 0;
      rc = seg_pass(ctx, w, S, sl, sst, sk);
      if (rc) return rc;
      ctx->timing.kernel_launches += 2;
      ok = true;
      for (size_t j = 0; j < S && ok; j++)
        ok = sst[j] == ZB200_OK && (sk[j] != 0) == (j + 1 == S) && (j + 1 == S || sl[j] == (uint64_t)ZB_CHUNK_BYTES);
      if (ok) dof[S] = dof[S - 1] + sl[S - 1];
      // the 64 KiB guess stays plausible for the marker segments while no segment is known to be larger or smaller
      guess = true;
      for (size_t j = 0; j < S; j++) {
        back_refs = back_refs || (j > 0 && sst[j] == ZB200_ERR_UNCOMPRESS);   // (distance beyond the segment start)
        if (j + 1 < S && ((sst[j] == ZB200_OK && sl[j] != (uint64_t)ZB_CHUNK_BYTES) || sst[j] == ZB200_ERR_DST_TOO_SMALL))
          guess = false;
      }
    }
    if (!ok && back_refs && ctx->joint_markers) ZB_TRY_JOINTS(guess);
    if (!ok) {
      // 3. sizes from a count pass, then the real pass with every segment at its place
      w.count_only = 1;
      rc = seg_pass(ctx, w, S, sl, sst, sk);
      if (rc) return rc;
      ctx->timing.kernel_launches += 2;
      ok = true;
      dof[0] = dst0;
      for (size_t j = 0; j < S && ok; j++) {
        ok = sst[j] == ZB200_OK && (sk[j] != 0) == (j + 1 == S);
        dof[j + 1] = dof[j] + sl[j];
      }
      if (!ok) ZB_TRY_JOINTS(false);
      if (dof[S] - dst0 > mcap) ZB_TRY_SPECULATIVE();
      if (!count_only) {
        std::vector<uint64_t> want = sl;
        CK(cudaMemcpyAsync(ctx->seg_dst.p, dof.data(), (S + 1) * 8, cudaMemcpyHostToDevice, s));
        w.count_only = 0;
        rc = seg_pass(ctx, w, S, sl, sst, sk);
        if (rc) return rc;
        ctx->timing.kernel_launches += 1;
        for (size_t j = 0; j < S && ok; j++) ok = sst[j] == ZB200_OK && sl[j] == want[j];
        if (!ok) ZB_TRY_SPECULATIVE();
      }
    }
    BigResult r;
    r.member = m;
    r.out_len = dof[S] - dst0;
    r.kind = (uint32_t)hw.fmt;
    r.expect = hw.expect;
    done.push_back(r);
  }
  return ZB200_OK;
}

// ---- decompress streams (zb200_decompress_stream_*) ----
// The wrapper waits until the input's length can no longer change its verdict: zb_parse_wrapper decides DETECT
// with len > 18 / len > 6 and checks the gzip header's length against len, so a header is decided once 19 bytes
// are held and zb_parse_wrapper accepts them, or when it rejects them for anything but their length, or at
// finish (`final`).  Raw streams start at byte 0 at once.
int dstream_header(zb200_decompress_stream *st, bool final) {
  if (st->data_format != ZB200_DF_DEFLATE && !final && st->total_in < 19) return ZB200_OK;
  uint64_t pos = 0;
  uint32_t kind = 0, expect = 0, isize = 0;
  uint8_t dummy = 0;
  const int r = zb_parse_wrapper(st->in.empty() ? &dummy : st->in.data(), st->in.size(), st->data_format, 0, pos, kind,
                                 expect, isize, st->has_dict ? &st->dict_id : nullptr);
  if (r == ZB200_ERR_UNCOMPRESS && !final) return ZB200_OK;   // a gzip header longer than what is held so far
  if (r) return r;
  st->fmt = (int)kind;
  st->check = kind == ZB200_DF_ZLIB ? 1u : 0u;   // Adler-32 / CRC-32 of no bytes
  st->in.erase(st->in.begin(), st->in.begin() + (ptrdiff_t)pos);
  st->in_off = pos;
  st->bit0 = 0;
  if (st->has_dict && (kind == ZB200_DF_DEFLATE || (kind == ZB200_DF_ZLIB && pos == 6))) {
    // the payload decodes as stored(W) || payload (zb200_decode_begin_dict's definition): the stored block counts
    // as held member bytes, and its |W| output bytes count as output already emitted, so dstream_run never emits
    // them or folds them into the checksum -- yet they are the window the first blocks may reach into
    const size_t wl = st->dict_win.size();
    const uint8_t head[5] = {0, (uint8_t)wl, (uint8_t)(wl >> 8), (uint8_t)~wl, (uint8_t)(~wl >> 8)};
    st->in.insert(st->in.begin(), st->dict_win.begin(), st->dict_win.end());
    st->in.insert(st->in.begin(), head, head + 5);
    st->total_in += 5 + wl;
    st->out_total = wl;
  }
  return ZB200_OK;
}

uint64_t dstream_reserve(const zb200_decompress_stream *st) {
  return st->fmt == ZB200_DF_GZIP ? 8 : st->fmt == ZB200_DF_ZLIB ? 4 : 0;
}

// A dynamic block header is at most 14 + 19 * 3 + 320 * 14 bits.  Its decode reads bits past the input as zeros and
// rejects some headers before it asks whether it ran past the end, so an error in a block that starts less than this
// before the end of the input received so far is only believed at finish.
constexpr uint64_t kDstreamHeaderBits = 1024 * 8;

// Segment boundaries of a raw stream in d_src that starts at bit lo_bit and whose payload ends at byte pay_end:
// bits[0] = lo_bit, then this library's joints / zlib flushes (k_find_sync), else dynamic-block starts
// (k_find_blocks), at least 16 KiB apart.  They are candidates: every segment [bits[i], bits[i + 1]) still has to
// decode as a closed segment.  `path` names what was found ("joints", "blocks", or "serial": bits = {lo_bit}).
int find_segment_bits(zb200_ctx *ctx, const uint8_t *d_src, uint64_t lo_bit, uint64_t pay_end, std::vector<uint64_t> &bits,
                      const char *&path) {
  const uint64_t pay_bit = pay_end * 8ull;
  const uint64_t min_gap = std::max<uint64_t>(16384ull * 8ull, (pay_bit - std::min(pay_bit, lo_bit)) / 60000ull);
  bits.assign(1, lo_bit);
  path = "serial";
  if (pay_bit <= lo_bit + 2 * min_gap) return ZB200_OK;
  const uint64_t lo = (lo_bit + 7) / 8;
  std::vector<uint64_t> cand;
  int rc = find_candidates(ctx, false, d_src, lo, pay_end, 0,
                           (uint32_t)std::min<uint64_t>((pay_end - lo) / 32 + 64, 1u << 24), cand);
  if (rc) return rc;
  ctx->timing.kernel_launches += 1;
  if (!cand.empty()) {
    for (uint64_t c : cand)
      if (c * 8 >= bits.back() + min_gap && c * 8 < pay_bit) bits.push_back(c * 8);
    path = "joints";
  }
  if (bits.size() < 2) {
    rc = find_candidates(ctx, true, d_src, lo_bit, pay_bit, pay_end,
                         (uint32_t)std::min<uint64_t>((pay_end - lo) / 64 + 1024, 1u << 24), cand);
    if (rc) return rc;
    ctx->timing.kernel_launches += 1;
    if (!cand.empty()) {
      for (uint64_t c : cand)
        if (c >= bits.back() + min_gap && c + min_gap / 4 < pay_bit) bits.push_back(c);
      path = "blocks";
    }
  }
  if (bits.size() < 2) path = "serial";
  return ZB200_OK;
}

// One launch of a decompress stream (ctx locked): decode the held input from the resume point, bits [bit0, end),
// where end is the payload received so far (`last`: everything, the trailer included, as uncompress reads it).
//  1. Boundaries: this library's joints / zlib flushes (k_find_sync), else dynamic-block starts (k_find_blocks),
//     at least 16 KiB apart.  Segments [b_i, b_i+1) are CLOSED (they must end on the next boundary without a
//     final block); the last one is OPEN: it stops where the input runs out and says where to resume.
//  2. A counting pass, then the uint16 marker decode of the segments that fit in kDstreamMaxOut, then the window
//     resolve with the carried 32 KiB in front of the launch's output (dst = [window | output]).
//  3. The bytes go to the stream's queue; their checksum is folded into the running one, and the last 32 KiB, the
//     resume point and the output count are carried, all together once nothing can fail any more.
// One launch stages at most max(2 x the batching threshold, 64 KiB) of held input (one large write is decoded in
// several launches, each copying only its own slice); it takes the whole rest only if that slice holds no complete
// block (`uncapped`).
// Anything irregular (a closed segment that fails or misses its boundary, a bad marker, a marker before the start of
// the stream, an error in the open segment of several) redoes the launch as ONE open segment from bit0: the serial
// decode with the carried window, whose verdict is the reference's.  Until 32 KiB of output exist the resume point
// stays at the payload start (base_out = 0): a window shorter than 32 KiB would let a distance reach before the
// stream's start, which only a decode from the start rejects; the bytes already produced are not emitted twice.
// `progress`: the output or the resume point moved.  Returns a decode status (the stream's verdict) or a CUDA one.
// `drain` (zb200_decompress_stream_drain, not `last_in`): the bytes held back as the possible trailer are decoded
// too, as payload that may go on: a block that ends inside them counts, and only finish decides where the input
// ends.  If it does end there, the member has no final block before its trailer, and finish reports the error
// that uncompress (which reads the trailer as payload as well) reports.
int dstream_run(zb200_decompress_stream *st, bool last_in, bool &progress, bool drain = false, bool uncapped = false) {
  progress = false;
  zb200_ctx *ctx = st->ctx;
  cudaStream_t s = ctx->stream;
  const uint8_t *held = st->in.data() + st->in_head;
  const uint64_t held_n = st->in.size() - st->in_head;
  const uint64_t resv = drain ? 0 : dstream_reserve(st);
  uint64_t pay_end = st->total_in - resv > st->in_off ? st->total_in - resv - st->in_off : 0;  // local bytes
  const uint64_t max_in = std::max<uint64_t>(2 * (uint64_t)st->batch_bytes, 65536);
  const bool capped = !uncapped && (last_in ? held_n : pay_end) > max_in;
  bool last = last_in;
  if (capped) {   // a slice of the input: where it ends is not the end of the input
    pay_end = max_in;
    last = false;
  }
  const uint64_t dec_end = last ? held_n : pay_end;
  const uint64_t lo_bit = st->bit0, end_bit = dec_end * 8ull, pay_bit = pay_end * 8ull;
  if (!last && pay_bit <= lo_bit) return ZB200_OK;
  ENSURE(ctx->in_stage, dec_end + 64);
  const uint8_t *d_src = (const uint8_t *)ctx->in_stage.p;
  int rc = h2d_copy(ctx, (uint8_t *)ctx->in_stage.p, held, dec_end, s, true);
  if (rc) return rc;
  // 1. boundaries
  std::vector<uint64_t> bits;
  const char *path = "serial";
  rc = find_segment_bits(ctx, d_src, lo_bit, pay_end, bits, path);
  if (rc) return rc;
  ZbInflateWork w;
  memset(&w, 0, sizeof(w));
  w.src = d_src;
  w.seg_limit = dec_end;
  w.seg_win0 = st->base_out > 0;
  std::vector<uint64_t> sl;
  std::vector<int> sst;
  std::vector<uint32_t> sk;
  uint64_t res[2] = {0, 0};
  // one decode launch over the first n segments, the last of them ending at bit `last_end`: counting with the last
  // one open, or marker symbols (every segment closed)
  auto pass = [&](size_t n, bool count, uint64_t last_end) -> int {
    int rc_ = seg_bounds_upload(ctx, bits.data(), n, last_end, w);
    if (rc_) return rc_;
    w.dst = count ? nullptr : (uint8_t *)ctx->mark_scratch.p;
    w.count_only = count ? 1 : 0;
    w.mark = count ? 0 : 1;
    if (count) {
      res[0] = bits[n - 1];
      res[1] = 0;
    }
    rc_ = seg_pass(ctx, w, n, sl, sst, sk, count ? res : nullptr);
    if (rc_) return rc_;
    ctx->timing.kernel_launches += 1;
    return ZB200_OK;
  };
  // The open segment decodes up to lim_bit: the input's end, or (once) less of it when one serial segment would
  // produce more than kDstreamMaxOut (DEFLATE expands at most 1032:1, so 1 MiB of input stays near the bound).
  uint64_t lim_bit = end_bit;
  bool lim_last = last, cut = false;
  const uint64_t cut_bits = 8ull * (kDstreamMaxOut / 1032);
  for (;;) {
    const size_t S = bits.size();
    // 2. the counting pass
    rc = pass(S, true, lim_bit);
    if (rc) return rc;
    bool irregular = false;
    for (size_t i = 0; i + 1 < S; i++)
      irregular = irregular || sst[i] != ZB200_OK || sk[i] != 0 || sl[i] > 0xf0000000ull;
    // the open segment: its complete output, where it stopped, whether that was the final block
    uint64_t open_n = 0, open_stop = 0;
    bool open_fin = false;
    if (!irregular) {
      const int os = sst[S - 1];
      int err = ZB200_OK;
      if (os == ZB200_OK) {
        open_fin = sk[S - 1] != 0;
        open_n = sl[S - 1];
        open_stop = lim_bit;   // not final: the input is used up at a block boundary
        if (!open_fin && lim_last) err = ZB200_ERR_END_OF_BUFFER;   // the reference reads one more block header
      } else {
        open_n = res[1];
        open_stop = res[0];
        const bool ran_out = os == ZB200_ERR_DST_TOO_SMALL || (os == ZB200_ERR_END_OF_BUFFER && !lim_last) ||
                             (!lim_last && lim_bit - std::min(lim_bit, res[0]) < kDstreamHeaderBits);
        if (!ran_out) err = os;
      }
      if (err) {
        if (S == 1) return err;
        irregular = true;
      }
    }
    if (irregular) {
      if (S == 1) return ZB200_ERR_UNCOMPRESS;
      bits.resize(1);
      path = "fallback";
      continue;
    }
    if (S == 1 && !cut && open_n > kDstreamMaxOut && lim_bit > lo_bit + cut_bits) {
      cut = true;
      lim_bit = lo_bit + cut_bits;
      lim_last = false;
      continue;
    }
    if (S == 1 && cut && lim_bit != end_bit && open_stop == lo_bit && !open_fin) {   // one block longer than that
      lim_bit = end_bit;
      lim_last = last;
      continue;
    }
    // 3. what fits in one launch's output: whole segments, the first one always
    std::vector<uint64_t> size(S);
    for (size_t i = 0; i + 1 < S; i++) size[i] = sl[i];
    size[S - 1] = open_n;
    size_t T = 0;
    uint64_t tot = 0;
    while (T < S && (T == 0 || tot + size[T] <= kDstreamMaxOut)) tot += size[T++];
    const bool with_open = T == S;
    const uint64_t stop = with_open ? open_stop : bits[T];
    const bool fin = with_open && open_fin;
    // 4. marker decode of segments [0, T), all closed now, into [32768 markers | output] each
    std::vector<ZbMarkSegHost> segs;
    uint32_t max_n = 0;
    const uint64_t W = st->base_out > 0 ? 32768 : 0;
    rc = mark_segments(ctx, size.data(), T, W, segs, max_n);
    if (rc) return rc;
    ctx->timing.kernel_launches += 1;
    rc = pass(T, false, fin ? lim_bit : stop);
    if (rc) return rc;
    for (size_t i = 0; i < T && !irregular; i++)
      irregular = sst[i] != ZB200_OK || sl[i] != size[i] || (sk[i] != 0) != (fin && i + 1 == T);
    if (irregular) {
      if (S == 1) return ZB200_ERR_UNCOMPRESS;
      bits.resize(1);
      path = "fallback";
      continue;
    }
    uint64_t total = 0;
    for (size_t i = 0; i < T; i++) total += segs[i].n;
    // 5. resolve against the carried window in front of the output
    ENSURE(ctx->out_stage, W + total + 64);
    uint8_t *d_out = (uint8_t *)ctx->out_stage.p;
    if (W) CK(cudaMemcpyAsync(d_out, st->win.data(), W, cudaMemcpyHostToDevice, s));
    CK(cudaMemsetAsync(&counters(ctx)->bad, 0, 4, s));
    int bad = 0;
    rc = resolve_window(ctx, T, max_n, 0, W, d_out, &bad);
    if (rc) return rc;
    ctx->timing.kernel_launches += 4;
    if (bad) {
      if (S == 1) return ZB200_ERR_UNCOMPRESS;
      bits.resize(1);
      path = "fallback";
      continue;
    }
    // 6. emit what was not emitted before, fold its checksum in, carry the window and the resume point
    const uint64_t skip = st->out_total - st->base_out;
    const uint64_t fresh = total > skip ? total - skip : 0;
    uint32_t check = st->check;
    if (fresh && st->fmt != ZB200_DF_DEFLATE) {
      const uint64_t offs[2] = {0, fresh};
      ZbChecksumWork cw;
      memset(&cw, 0, sizeof(cw));
      rc = upload_pieces(ctx, offs, 1, cw);
      if (rc) return rc;
      ENSURE(ctx->src_off, 16);
      ENSURE(ctx->ck_out, 4);
      CK(cudaMemcpyAsync(ctx->src_off.p, offs, 16, cudaMemcpyHostToDevice, s));
      cw.src = d_out + W + skip;
      cw.off = (const uint64_t *)ctx->src_off.p;
      cw.out = (uint32_t *)ctx->ck_out.p;
      cw.kind = st->fmt == ZB200_DF_ZLIB ? 1 : 0;
      CK(zb_launch_checksum(cw, s));
      uint32_t c = 0;
      CK(cudaMemcpyAsync(&c, ctx->ck_out.p, 4, cudaMemcpyDeviceToHost, s));
      CK(cudaStreamSynchronize(s));
      ctx->timing.kernel_launches += 2;
      check = st->fmt == ZB200_DF_ZLIB ? zb_adler32_combine(check, c, fresh) : zb_crc32_combine(check, c, fresh);
    }
    const uint64_t new_base = st->base_out + total;
    const bool advance = fin || new_base >= 32768;
    std::vector<uint8_t> nwin;
    if (advance && !fin) nwin.resize(std::min<uint64_t>(32768, W + total));
    const size_t q0 = st->q.size();
    if (fresh) {
      if (st->q_head && st->q_head * 2 >= q0) {   // drop what was read
        st->q.erase(st->q.begin(), st->q.begin() + (ptrdiff_t)st->q_head);
        st->q_head = 0;
      }
      st->q.resize(st->q.size() + fresh);   // (a failure from here on is the stream's error: the bytes are never read)
      rc = d2h_copy(ctx, st->q.data() + (st->q.size() - fresh), d_out + W + skip, fresh, s, true);
      if (rc) return rc;
    }
    if (!nwin.empty())
      CK(cudaMemcpyAsync(nwin.data(), d_out + W + total - nwin.size(), nwin.size(), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    rc = d2h_flush(ctx);
    if (rc) return rc;
    // nothing can fail from here on: commit the launch
    ctx->timing.d2h_bytes += fresh;
    if (st->log)
      fprintf(stderr, "zb200 dstream: path=%s segs=%zu taken=%zu out=%llu final=%d\n", path, S, T,
              (unsigned long long)total, (int)fin);
    progress = fresh > 0 || (advance && stop > lo_bit) || fin;
    if (capped && !progress) return dstream_run(st, last_in, progress, drain, true);   // no complete block in the slice
    st->check = check;
    st->out_total = std::max(st->out_total, new_base);
    if (fin) {
      st->done = true;
      std::vector<uint8_t>().swap(st->in);
      std::vector<uint8_t>().swap(st->win);
      st->in_head = 0;
      st->in_off = st->total_in;
      st->bit0 = 0;
      st->base_out = new_base;
    } else if (advance) {
      st->in_head += stop / 8;
      if (st->in_head * 2 >= st->in.size()) {   // drop the decoded input: amortised, one large write is not moved per launch
        st->in.erase(st->in.begin(), st->in.begin() + (ptrdiff_t)st->in_head);
        st->in_head = 0;
      }
      st->in_off += stop / 8;
      st->bit0 = (uint32_t)(stop & 7);
      st->base_out = new_base;
      st->win.swap(nwin);
    }
    return ZB200_OK;
  }
}

// Work-queue order of one inflate launch: a member is decoded by one 8-lane group from start to end,
// so a long member that is fetched late finishes long after everything else (the tail of the launch).
// Members much longer than the average go first, longest first; the rest keep their order.
// Returns false when no member stands out (then the launch uses index order and nothing is uploaded).
bool longest_first_order(const uint64_t *src_offsets, size_t n, std::vector<uint32_t> &order) {
  if (n < 64) return false;
  const uint64_t total = src_offsets[n] - src_offsets[0];
  const uint64_t thr = std::max<uint64_t>(4 * (total / n), 32768);
  std::vector<uint32_t> big;
  for (size_t i = 0; i < n; i++)
    if (src_offsets[i + 1] - src_offsets[i] >= thr) big.push_back((uint32_t)i);
  if (big.empty() || big.size() > n / 2) return false;
  std::sort(big.begin(), big.end(), [&](uint32_t a, uint32_t b) {
    const uint64_t la = src_offsets[a + 1] - src_offsets[a], lb = src_offsets[b + 1] - src_offsets[b];
    return la != lb ? la > lb : a < b;
  });
  order.resize(n);
  size_t k = 0;
  for (uint32_t i : big) order[k++] = i;
  for (size_t i = 0; i < n; i++)
    if (src_offsets[i + 1] - src_offsets[i] < thr) order[k++] = (uint32_t)i;
  return true;
}

// The checksum pass behind an inflate launch over w's outputs (the piece table is already in cw).  Without d_crcs it
// verifies every gzip / zlib trailer, checksum then size (gzip.nim:80-88 / zippy.nim:154-162), and skips raw deflate.
// With d_crcs it is the plain crc32 configuration instead (no kinds, no expected values): d_crcs[i] gets the CRC-32 of
// every output that inflated, raw deflate included, and nothing is compared -- a ZIP entry's CRC lives in the
// archive's headers, not behind the stream.
// the dictionaries of the *_dict / *_dicts call in progress, if any, for a whole-member inflate launch over the
// call's members from m0 on
void set_dict(const zb200_ctx *ctx, ZbInflateWork &w, size_t m0) {
  if (!ctx->dict_on) return;
  w.mdict = (const ZbMemberDict *)ctx->dict_md.p + m0;
}

void set_check_pass(ZbChecksumWork &cw, const ZbInflateWork &w, uint32_t *d_crcs) {
  cw.src = w.dst;
  cw.off = w.dst_off;
  cw.lens = w.out_len;
  cw.status = w.status;
  if (d_crcs) {
    cw.out = d_crcs;
    cw.kind = 0;
    return;
  }
  cw.expect = w.expect;
  cw.kinds = w.kind;
  cw.isize_src = w.src;
  cw.isize_off = w.src_off;
}

// ---- uncompress, device-resident ----
// crcs (host, may be null): the CRC-32 of every output that inflated, computed on the device (set_check_pass)
int uncompress_device_locked(zb200_ctx *ctx, const uint8_t *d_src, const uint64_t *src_offsets, size_t n,
                             int data_format, uint64_t raw_pos, uint8_t *d_dst, const uint64_t *dst_offsets,
                             uint64_t *dst_lens, int *statuses, bool count_only,
                             const std::function<int()> *after_launch = nullptr, uint32_t *crcs = nullptr,
                             size_t dict_m0 = 0) {
  if (data_format < ZB200_DF_DETECT || data_format > ZB200_DF_DEFLATE) return ZB200_ERR_INVALID_FORMAT;
  if (n == 0) return ZB200_OK;
  ENSURE(ctx->src_off, (n + 1) * sizeof(uint64_t));
  ENSURE(ctx->dst_off, (n + 1) * sizeof(uint64_t));
  ENSURE(ctx->out_len, n * sizeof(uint64_t));
  ENSURE(ctx->status, n * sizeof(int));
  ENSURE(ctx->expect, n * sizeof(uint32_t));
  ENSURE(ctx->kind, n * sizeof(uint32_t));
  if (crcs) ENSURE(ctx->ck_out, n * sizeof(uint32_t));
  cudaStream_t s = ctx->stream;
  CK(cudaMemcpyAsync(ctx->src_off.p, src_offsets, (n + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, s));
  if (!count_only)
    CK(cudaMemcpyAsync(ctx->dst_off.p, dst_offsets, (n + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, s));
  ZbInflateWork w;
  memset(&w, 0, sizeof(w));
  w.src = d_src;
  w.src_off = (const uint64_t *)ctx->src_off.p;
  w.dst = d_dst;
  w.dst_off = (const uint64_t *)ctx->dst_off.p;
  w.out_len = (uint64_t *)ctx->out_len.p;
  w.status = (int *)ctx->status.p;
  w.expect = (uint32_t *)ctx->expect.p;
  w.kind = (uint32_t *)ctx->kind.p;
  w.counter = &counters(ctx)->member;
  w.tabs = ctx->d_tabs;
  w.n = (uint32_t)n;
  w.data_format = data_format;
  w.pos = raw_pos;
  w.count_only = count_only ? 1 : 0;
  w.skip = nullptr;
  w.seg_mode = 0;
  w.order = nullptr;
  set_dict(ctx, w, dict_m0);   // (with dictionaries: a group of uncompress_sizes_host, its first member)
  {
    std::vector<uint32_t> order;
    if (longest_first_order(src_offsets, n, order)) {
      ENSURE(ctx->order, n * sizeof(uint32_t));
      CK(cudaMemcpyAsync(ctx->order.p, order.data(), n * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
      CK(cudaStreamSynchronize(s));  // `order` goes out of scope
      w.order = (const uint32_t *)ctx->order.p;
    }
  }
  ZbChecksumWork cw;
  memset(&cw, 0, sizeof(cw));
  if (!count_only) {  // piece table for the verification pass, uploaded before anything is launched
    int rc = upload_pieces(ctx, dst_offsets, n, cw);
    if (rc) return rc;
  }
  CK(cudaEventRecord(ctx->ev[0], s));
  // large members first, as parallel segments where their streams allow it; the rest (and every
  // large member that did not work out) goes through the ordinary launch below
  std::vector<BigResult> big;
  std::vector<uint8_t> skip_host;
  if (!ctx->dict_on) {  // with a dictionary every member is decoded whole, by k_inflate's dictionary instantiation
    int rc = inflate_big_members(ctx, d_src, src_offsets, n, data_format, raw_pos, d_dst, dst_offsets, count_only, big);
    if (rc) return rc;
    if (!big.empty()) {
      skip_host.assign(n, 0);
      ENSURE(ctx->skip_mask, n);
      for (const BigResult &r : big) {
        skip_host[r.member] = 1;
        CK(cudaMemcpyAsync((int *)ctx->status.p + r.member, &r.status, 4, cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync((uint64_t *)ctx->out_len.p + r.member, &r.out_len, 8, cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync((uint32_t *)ctx->kind.p + r.member, &r.kind, 4, cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync((uint32_t *)ctx->expect.p + r.member, &r.expect, 4, cudaMemcpyHostToDevice, s));
      }
      CK(cudaMemcpyAsync(ctx->skip_mask.p, skip_host.data(), n, cudaMemcpyHostToDevice, s));
      CK(cudaStreamSynchronize(s));
      w.skip = (const uint8_t *)ctx->skip_mask.p;
    }
  }
  CK(zb_launch_inflate(w, s));
  CK(cudaEventRecord(ctx->ev[1], s));
  if (!count_only) {
    set_check_pass(cw, w, crcs ? (uint32_t *)ctx->ck_out.p : nullptr);
    CK(zb_launch_checksum(cw, s));
  }
  CK(cudaEventRecord(ctx->ev[2], s));
  if (after_launch) {  // work to queue behind the kernels (other streams) before this thread waits
    int rc = (*after_launch)();
    if (rc) return rc;
  }
  CK(cudaMemcpyAsync(dst_lens, ctx->out_len.p, n * sizeof(uint64_t), cudaMemcpyDeviceToHost, s));
  std::vector<int> st_tmp;
  int *st = statuses;
  if (!st) {
    st_tmp.resize(n);
    st = st_tmp.data();
  }
  CK(cudaMemcpyAsync(st, ctx->status.p, n * sizeof(int), cudaMemcpyDeviceToHost, s));
  if (crcs && !count_only) CK(cudaMemcpyAsync(crcs, ctx->ck_out.p, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  ctx->timing.inflate_ms += ev_ms(ctx->ev[0], ctx->ev[1]);
  ctx->timing.verify_ms += ev_ms(ctx->ev[1], ctx->ev[2]);
  ctx->timing.kernel_launches += count_only ? 1 : 3;
  for (size_t i = 0; i < n; i++)
    if (st[i] != ZB200_OK) {
      dst_lens[i] = 0;
      if (crcs) crcs[i] = 0;
    }
  return ZB200_OK;
}

// ---- uncompress, host buffers, fully asynchronous ----
// Everything the device needs for the WHOLE batch (offsets, verification pieces, work-queue orders) is
// built and uploaded once; then every member group is enqueued without a host wait in between:
//   H2D stream : copy-in of group 0, 1, 2, ... back to back
//   main stream: wait copy-in(g) -> inflate(g) -> verify(g)
//   D2H stream : wait verify(g) -> copy-out(g)
// and the host synchronises once at the end.  (The first version waited for every group's kernels on the
// host before it built and launched the next group, and each launch carried its own tail of long members.)
int uncompress_host_pipelined(zb200_ctx *ctx, const uint8_t *h_src, const std::vector<uint64_t> &reb, size_t n,
                              int data_format, uint8_t *h_dst, const std::vector<uint64_t> &dreb, uint64_t *dst_lens,
                              int *statuses, const std::vector<size_t> &gb, uint32_t *crcs) {
  const size_t ng = gb.size() - 1;
  // With dictionaries each group's windows go up with its input (DictWindows).  The gated launch keeps every group's
  // windows (no slot is reused: a reuse would have to wait for the kernel to finish a group, and the kernel's warps
  // can wait for a later group's gate, which would then wait for that copy), so it is used only while all of them
  // fit kDictSlots slots' worth; otherwise the launches go group by group and a slot is reused kDictSlots groups
  // later, once the launch that read it has finished.
  DictWindows dw;
  bool resident = true;
  if (ctx->dict_on) {
    dw.layout(ctx, gb, nullptr);
    resident = (uint64_t)ng * dw.slot_cap <= kDictSlots * kDictGroupWindowBytes;
  }
  // gated: ONE inflate launch walks the whole batch behind the copy-in (no per-group launch tails), the D2H
  // stream waits on the per-group done counts; otherwise one launch per group, chained with events
  const bool gated = ctx->memops.ok && ctx->gated_unc && n < 0xffffffffull && resident;
  if (ctx->dict_on) {
    if (int rc = dw.place(ctx, gated ? ng : kDictSlots)) return rc;
    ENSURE(ctx->dict_md, n * sizeof(ZbMemberDict));
    CK(cudaMemcpyAsync(ctx->dict_md.p, ctx->dict_member.data(), n * sizeof(ZbMemberDict), cudaMemcpyHostToDevice,
                       ctx->stream));
  }
  cudaStream_t s = ctx->stream, sh = ctx->h2d_stream, sd = ctx->d2h_stream;
  const uint8_t *d_src = (const uint8_t *)ctx->in_stage.p;
  uint8_t *d_dst = (uint8_t *)ctx->out_stage.p;
  // ---- plan (host) ----
  std::vector<ZbPiece> pieces;
  std::vector<uint32_t> first;          // per group: (members + 1) entries relative to the group's first piece
  std::vector<size_t> piece0(ng + 1), first0(ng + 1);
  std::vector<uint32_t> order(n);       // per group: entries relative to the group
  std::vector<uint8_t> has_order(ng, 0);
  for (size_t gi = 0; gi < ng; gi++) {
    const size_t m0 = gb[gi], m1 = gb[gi + 1];
    piece0[gi] = pieces.size();
    first0[gi] = first.size();
    for (size_t i = m0; i < m1; i++) {
      first.push_back((uint32_t)(pieces.size() - (gated ? 0 : piece0[gi])));
      const uint64_t cap = dreb[i + 1] - dreb[i];
      uint64_t rel = 0;
      do {
        ZbPiece pc;
        pc.rel = rel;
        pc.buf = (uint32_t)(i - (gated ? 0 : m0));
        pc.pad = 0;
        pieces.push_back(pc);
        rel += ZB_CK_PIECE_BYTES;
      } while (rel < cap);
    }
    if (!gated || gi + 1 == ng) first.push_back((uint32_t)(pieces.size() - (gated ? 0 : piece0[gi])));
    std::vector<uint32_t> o;
    if (longest_first_order(reb.data() + m0, m1 - m0, o)) {
      has_order[gi] = 1;
      std::copy(o.begin(), o.end(), order.begin() + m0);
      if (gated)
        for (size_t i = m0; i < m1; i++) order[i] += (uint32_t)m0;
    } else if (gated) {
      for (size_t i = m0; i < m1; i++) order[i] = (uint32_t)i;
    }
  }
  piece0[ng] = pieces.size();
  first0[ng] = first.size();
  // ---- device arrays for the whole batch ----
  ENSURE(ctx->src_off, (n + 1) * sizeof(uint64_t));
  ENSURE(ctx->dst_off, (n + 1) * sizeof(uint64_t));
  ENSURE(ctx->out_len, n * sizeof(uint64_t));
  ENSURE(ctx->status, n * sizeof(int));
  ENSURE(ctx->expect, n * sizeof(uint32_t));
  ENSURE(ctx->kind, n * sizeof(uint32_t));
  ENSURE(ctx->order, n * sizeof(uint32_t));
  ENSURE(ctx->counter, sizeof(ZbCounters) + ng * sizeof(uint32_t));
  uint32_t *group_counter = (uint32_t *)(counters(ctx) + 1);
  ENSURE(ctx->ck_pieces, pieces.size() * sizeof(ZbPiece));
  ENSURE(ctx->ck_first, first.size() * sizeof(uint32_t));
  ENSURE(ctx->ck_piece_out, pieces.size() * sizeof(ZbChunkCheck));
  ENSURE(ctx->ck_partials, pieces.size() * (size_t)ZB_CK_PARTIAL_BYTES);
  if (crcs) ENSURE(ctx->ck_out, n * sizeof(uint32_t));
  uint32_t *d_crcs = crcs ? (uint32_t *)ctx->ck_out.p : nullptr;
  {
    int rc = ensure_group_events(ctx, 2 * ng + 2);
    if (rc) return rc;
    rc = ensure_pinned(ctx, n * (sizeof(uint64_t) + sizeof(int) + sizeof(uint32_t)) + 64);
    if (rc) return rc;
  }
  CK(cudaMemcpyAsync(ctx->src_off.p, reb.data(), (n + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(ctx->dst_off.p, dreb.data(), (n + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(ctx->ck_pieces.p, pieces.data(), pieces.size() * sizeof(ZbPiece), cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(ctx->ck_first.p, first.data(), first.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(ctx->order.p, order.data(), n * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
  // the side streams start after whatever the caller's stream already holds (and after the tables above)
  CK(cudaEventRecord(ctx->gev[2 * ng], s));
  CK(cudaStreamWaitEvent(sh, ctx->gev[2 * ng], 0));
  CK(cudaStreamWaitEvent(sd, ctx->gev[2 * ng], 0));
  CK(cudaEventRecord(ctx->ev[6], sh));
  CK(cudaEventRecord(ctx->ev[8], sd));
  const bool src_pageable = is_pageable(h_src), dst_pageable = h_dst && is_pageable(h_dst);
  CK(cudaEventRecord(ctx->ev[0], s));
  if (gated) {
    // nothing that may synchronise the device (allocations, registrations) can happen while the gated kernel waits
    // for input: the staging rings of pageable callers are set up first
    if (src_pageable || ctx->dict_on) {   // (the windows always go through the staging ring)
      int rc = ring_ready(ctx, ctx->ring_in);
      if (rc) return rc;
    }
    if (dst_pageable) {
      int rc = ring_ready(ctx, ctx->ring_out);
      if (rc) return rc;
    }
    // gate words: [0] = groups copied in, [1 + g] = members of group g done, [1 + ng + g] = first queue position of group g
    std::vector<uint32_t> gate(2 * ng + 2, 0u);
    for (size_t gi = 0; gi <= ng; gi++) gate[1 + ng + gi] = (uint32_t)gb[gi];
    ENSURE(ctx->gate, gate.size() * sizeof(uint32_t));
    uint32_t *d_gate = (uint32_t *)ctx->gate.p;
    CK(cudaMemcpyAsync(d_gate, gate.data(), gate.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
    CK(cudaStreamSynchronize(s));  // `gate` is pageable: the copy has read it; and the zeroed words are in place before
                                   // the H2D stream's first write of d_gate[0]
    ZbInflateWork w;
    memset(&w, 0, sizeof(w));
    w.src = d_src;
    w.src_off = (const uint64_t *)ctx->src_off.p;
    w.dst = d_dst;
    w.dst_off = (const uint64_t *)ctx->dst_off.p;
    w.out_len = (uint64_t *)ctx->out_len.p;
    w.status = (int *)ctx->status.p;
    w.expect = (uint32_t *)ctx->expect.p;
    w.kind = (uint32_t *)ctx->kind.p;
    w.counter = group_counter;
    w.tabs = ctx->d_tabs;
    w.n = (uint32_t)n;
    w.data_format = data_format;
    w.order = (const uint32_t *)ctx->order.p;
    w.gate_ready = d_gate;
    w.gate_done = d_gate + 1;
    w.gate_first = d_gate + 1 + ng;
    w.n_gates = (uint32_t)ng;
    set_dict(ctx, w, 0);
    CK(zb_launch_inflate(w, s));
    // from here on the kernel may be waiting for copies: if this function leaves early (a failed copy, a failed
    // enqueue), open every gate so that the kernel drains instead of waiting out its timeout
    struct GateRelease {
      zb200_ctx *ctx;
      uint32_t *word;
      bool armed;
      ~GateRelease() {
        if (armed) ctx->memops.write32((CUstream)ctx->h2d_stream, (CUdeviceptr)(uintptr_t)word, 0xffffffffu, 0);
      }
    } gate_release{ctx, d_gate, true};
    // the checksum pass of every member that inflated (after the whole launch, under the last groups' copy-out)
    ZbChecksumWork cw;
    memset(&cw, 0, sizeof(cw));
    set_check_pass(cw, w, d_crcs);
    cw.pieces = (const ZbPiece *)ctx->ck_pieces.p;
    cw.first = (const uint32_t *)ctx->ck_first.p;
    cw.piece_out = (ZbChunkCheck *)ctx->ck_piece_out.p;
    cw.partials = (uint32_t *)ctx->ck_partials.p;
    cw.tabs = ctx->d_tabs;
    cw.n = (uint32_t)n;
    cw.n_pieces = (uint32_t)pieces.size();
    CK(zb_launch_checksum(cw, s));
    ctx->timing.kernel_launches += 3;
    auto copy_in = [&](size_t gi) -> int {
      const uint64_t b0 = reb[gb[gi]], b1 = reb[gb[gi + 1]];
      if (ctx->dict_on) {   // (one slot per group here: nothing waits for the kernel)
        if (int rc = dw.upload(ctx, gi, sh)) return rc;
      }
      int rc = h2d_copy(ctx, (uint8_t *)ctx->in_stage.p + b0, h_src + b0, (size_t)(b1 - b0), sh, src_pageable);
      if (rc) return rc;
      if (ctx->memops.write32((CUstream)sh, (CUdeviceptr)(uintptr_t)d_gate, (cuuint32_t)(gi + 1), 0) != CUDA_SUCCESS) return ZB200_ERR_CUDA;
      if (gi + 1 == ng) CK(cudaEventRecord(ctx->ev[7], sh));
      return ZB200_OK;
    };
    {
      int rc = copy_in(0);
      if (rc) return rc;
    }
    // ZB200_DEBUG_TIMELINE=1: per group, when its done count released the copy-out and when the copy ended (stderr)
    static const bool timeline = getenv("ZB200_DEBUG_TIMELINE") != nullptr;
    std::vector<cudaEvent_t> tl;
    if (timeline) {
      tl.resize(2 * ng + 1);
      for (auto &ev : tl) cudaEventCreate(&ev);
      cudaEventRecord(tl[2 * ng], sd);
    }
    for (size_t gi = 0; gi < ng; gi++) {
      if (gi + 1 < ng) {  // the next group's copy-in is queued before this thread may block on a pageable copy-out
        int rc = copy_in(gi + 1);
        if (rc) return rc;
      }
      const size_t m0 = gb[gi], m1 = gb[gi + 1];
      const uint64_t o0 = dreb[m0], o1 = dreb[m1];
      if (o1 > o0 && h_dst) {
        if (ctx->memops.wait32((CUstream)sd, (CUdeviceptr)(uintptr_t)(d_gate + 1 + gi), (cuuint32_t)(m1 - m0), CU_STREAM_WAIT_VALUE_GEQ) != CUDA_SUCCESS)
          return ZB200_ERR_CUDA;
        if (timeline) cudaEventRecord(tl[2 * gi], sd);
        int rc = d2h_copy(ctx, h_dst + o0, d_dst + o0, (size_t)(o1 - o0), sd, dst_pageable);
        if (rc) return rc;
        if (timeline) cudaEventRecord(tl[2 * gi + 1], sd);
      }
    }
    if (timeline) {
      cudaStreamSynchronize(sd);
      for (size_t gi = 0; gi < ng; gi++) {
        float a = 0, b = 0;
        cudaEventElapsedTime(&a, tl[2 * ng], tl[2 * gi]);
        cudaEventElapsedTime(&b, tl[2 * ng], tl[2 * gi + 1]);
        fprintf(stderr, "group %zu: members %zu, out %.1f MiB, released %.2f ms, copied %.2f ms\n", gi, gb[gi + 1] - gb[gi],
                (double)(dreb[gb[gi + 1]] - dreb[gb[gi]]) / 1048576.0, a, b);
      }
      for (auto &ev : tl) cudaEventDestroy(ev);
    }
    gate_release.armed = false;   // every group's copy-in (and its gate word) is queued
  }
  for (size_t gi = 0; gi < ng && !gated; gi++) {
    const size_t m0 = gb[gi], m1 = gb[gi + 1], nm = m1 - m0;
    if (ctx->dict_on) {   // the slot's previous group has been decoded and checked
      if (gi >= dw.slots) CK(cudaStreamWaitEvent(sh, ctx->gev[2 * (gi - dw.slots) + 1], 0));
      if (int rc = dw.upload(ctx, gi, sh)) return rc;
    }
    {
      const uint64_t b0 = reb[m0], b1 = reb[m1];
      int rc = h2d_copy(ctx, (uint8_t *)ctx->in_stage.p + b0, h_src + b0, (size_t)(b1 - b0), sh, src_pageable);
      if (rc) return rc;
      CK(cudaEventRecord(ctx->gev[2 * gi], sh));
      if (gi + 1 == ng) CK(cudaEventRecord(ctx->ev[7], sh));
    }
    CK(cudaStreamWaitEvent(s, ctx->gev[2 * gi], 0));
    ZbInflateWork w;
    memset(&w, 0, sizeof(w));
    w.src = d_src;
    w.src_off = (const uint64_t *)ctx->src_off.p + m0;
    w.dst = d_dst;
    w.dst_off = (const uint64_t *)ctx->dst_off.p + m0;
    w.out_len = (uint64_t *)ctx->out_len.p + m0;
    w.status = (int *)ctx->status.p + m0;
    w.expect = (uint32_t *)ctx->expect.p + m0;
    w.kind = (uint32_t *)ctx->kind.p + m0;
    w.counter = group_counter + gi;
    w.tabs = ctx->d_tabs;
    w.n = (uint32_t)nm;
    w.data_format = data_format;
    w.order = has_order[gi] ? (const uint32_t *)ctx->order.p + m0 : nullptr;
    set_dict(ctx, w, m0);
    CK(zb_launch_inflate(w, s));
    // the checksum pass of every member that inflated
    ZbChecksumWork cw;
    memset(&cw, 0, sizeof(cw));
    set_check_pass(cw, w, d_crcs ? d_crcs + m0 : nullptr);
    cw.pieces = (const ZbPiece *)ctx->ck_pieces.p + piece0[gi];
    cw.first = (const uint32_t *)ctx->ck_first.p + first0[gi];
    cw.piece_out = (ZbChunkCheck *)ctx->ck_piece_out.p + piece0[gi];
    cw.partials = (uint32_t *)ctx->ck_partials.p + piece0[gi] * (size_t)(ZB_CK_PARTIAL_BYTES / 4);
    cw.tabs = ctx->d_tabs;
    cw.n = (uint32_t)nm;
    cw.n_pieces = (uint32_t)(piece0[gi + 1] - piece0[gi]);
    CK(zb_launch_checksum(cw, s));
    CK(cudaEventRecord(ctx->gev[2 * gi + 1], s));
    CK(cudaStreamWaitEvent(sd, ctx->gev[2 * gi + 1], 0));
    const uint64_t o0 = dreb[m0], o1 = dreb[m1];
    if (o1 > o0 && h_dst) {
      int rc = d2h_copy(ctx, h_dst + o0, d_dst + o0, (size_t)(o1 - o0), sd, dst_pageable);
      if (rc) return rc;
    }
    ctx->timing.kernel_launches += 3;
  }
  CK(cudaEventRecord(ctx->ev[1], s));
  CK(cudaEventRecord(ctx->ev[9], sd));
  if (dst_pageable) {
    int rc = d2h_flush(ctx);
    if (rc) return rc;
  }
  uint64_t *pl = (uint64_t *)ctx->pin;
  int *ps = (int *)(pl + n);
  uint32_t *pc = (uint32_t *)(ps + n);
  CK(cudaMemcpyAsync(pl, ctx->out_len.p, n * sizeof(uint64_t), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(ps, ctx->status.p, n * sizeof(int), cudaMemcpyDeviceToHost, s));
  if (crcs) CK(cudaMemcpyAsync(pc, d_crcs, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
  // the caller's stream ends after the last copy out
  CK(cudaEventRecord(ctx->gev[2 * ng + 1], sd));
  CK(cudaStreamWaitEvent(s, ctx->gev[2 * ng + 1], 0));
  CK(cudaStreamSynchronize(s));  // also: the planning vectors above stay alive until their uploads are done
  CK(cudaStreamSynchronize(sh));
  for (size_t i = 0; i < n; i++) {
    dst_lens[i] = ps[i] == ZB200_OK ? pl[i] : 0;
    if (statuses) statuses[i] = ps[i];
    if (crcs) crcs[i] = ps[i] == ZB200_OK ? pc[i] : 0;
  }
  ctx->timing.inflate_ms = ev_ms(ctx->ev[0], ctx->ev[1]);  // inflate + verify of all groups (includes waits for copy-in)
  ctx->timing.verify_ms = 0.f;
  return ZB200_OK;
}

int checksum_device_locked(zb200_ctx *ctx, const uint8_t *d_src, const uint64_t *src_offsets, size_t n, int kind,
                           uint32_t *out) {
  if (kind != 0 && kind != 1) return ZB200_ERR_ARG;
  if (n == 0) return ZB200_OK;
  for (size_t i = 0; i < n; i++)
    if (src_offsets[i + 1] < src_offsets[i]) return ZB200_ERR_ARG;
  ENSURE(ctx->src_off, (n + 1) * sizeof(uint64_t));
  ENSURE(ctx->ck_out, n * sizeof(uint32_t));
  cudaStream_t s = ctx->stream;
  CK(cudaMemcpyAsync(ctx->src_off.p, src_offsets, (n + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, s));
  ZbChecksumWork w;
  memset(&w, 0, sizeof(w));
  int rc = upload_pieces(ctx, src_offsets, n, w);
  if (rc) return rc;
  w.src = d_src;
  w.off = (const uint64_t *)ctx->src_off.p;
  w.out = (uint32_t *)ctx->ck_out.p;
  w.kind = kind;
  CK(cudaEventRecord(ctx->ev[0], s));
  CK(zb_launch_checksum(w, s));
  CK(cudaEventRecord(ctx->ev[1], s));
  CK(cudaMemcpyAsync(out, ctx->ck_out.p, n * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  ctx->timing.checksum_ms = ev_ms(ctx->ev[0], ctx->ev[1]);
  ctx->timing.kernel_launches += 2;
  return ZB200_OK;
}

// copy host inputs [src_offsets[0], src_offsets[n]) into the ctx staging buffer, rebased to 0
int stage_in(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n,
             std::vector<uint64_t> &rebased) {
  uint64_t lo = src_offsets[0], hi = src_offsets[n];
  for (size_t i = 0; i < n; i++)
    if (src_offsets[i + 1] < src_offsets[i]) return ZB200_ERR_ARG;
  rebased.resize(n + 1);
  for (size_t i = 0; i <= n; i++) rebased[i] = src_offsets[i] - lo;
  ENSURE(ctx->in_stage, (size_t)(hi - lo) + 64);
  CK(cudaEventRecord(ctx->ev[6], ctx->stream));
  if (hi > lo)
    CK(cudaMemcpyAsync(ctx->in_stage.p, src_base + lo, (size_t)(hi - lo), cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaEventRecord(ctx->ev[7], ctx->stream));
  ctx->timing.h2d_bytes = hi - lo;
  return ZB200_OK;
}

// An error return must not leave copies that use the caller's buffers in flight.
void quiesce(zb200_ctx *ctx) {
  if (ctx->stream) cudaStreamSynchronize(ctx->stream);
  if (ctx->h2d_stream) cudaStreamSynchronize(ctx->h2d_stream);
  if (ctx->d2h_stream) cudaStreamSynchronize(ctx->d2h_stream);
  cudaGetLastError();
  // copies that were still waiting in the pinned ring belong to the failed call: their destinations are
  // the caller's buffers, which it may free now -- forget them
  for (int i = 0; i < kStageSlots; i++) ctx->ring_out.busy[i] = false;
}

// No C++ exception crosses the C ABI (std::vector growth on attacker-sized inputs, ...).
template <class F>
int guarded(zb200_ctx *ctx, F &&f) {
  int rc;
  try {
    rc = f();
  } catch (const std::bad_alloc &) {
    if (ctx) ctx->last_err = "host allocation failed";
    rc = ZB200_ERR_NOMEM;
  } catch (const std::exception &e) {
    if (ctx) ctx->last_err = e.what();
    rc = ZB200_ERR_ARG;
  }
  if (rc != ZB200_OK && ctx) quiesce(ctx);
  return rc;
}

}  // namespace

// =====================================================================================
extern "C" {

int zb200_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n;
}

static void zb_segv_handler(int sig) {
  void *frames[64];
  const int n = backtrace(frames, 64);
  const char msg[] = "zippy_b200: fatal signal, backtrace (resolve with addr2line -e libzippy_b200.so):\n";
  if (write(2, msg, sizeof(msg) - 1) < 0) _exit(128 + sig);
  backtrace_symbols_fd(frames, n, 2);
  _exit(128 + sig);
}

int zb200_init(int device, zb200_ctx **out) {
  if (!out) return ZB200_ERR_ARG;
  if (getenv("ZB200_DEBUG_SEGV")) signal(SIGSEGV, zb_segv_handler);  // debugging aid: where did a host fault happen
  *out = nullptr;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    return ZB200_ERR_CUDA;  // no CPU fallback
  }
  if (device < 0) {
    if (cudaGetDevice(&device) != cudaSuccess) return ZB200_ERR_CUDA;
  }
  if (device >= ndev) return ZB200_ERR_ARG;
  zb200_ctx *ctx = new zb200_ctx();
  ctx->device = device;
  memset(&ctx->timing, 0, sizeof(ctx->timing));
  if (const char *e = getenv("ZB200_GROUP_CHUNKS")) {  // test hook: force small launch groups
    long v = atol(e);
    if (v > 0) ctx->dev_group_chunks = ctx->host_group_chunks = (size_t)v;
  }
  if (const char *e = getenv("ZB200_STREAM_BATCH_BYTES")) {  // test hook: compress streams launch at this much pending input
    long long v = atoll(e);
    if (v > 0) ctx->stream_batch_bytes = (size_t)v;
  }
  if (const char *e = getenv("ZB200_DSTREAM_BATCH_BYTES")) {  // test hook: decompress streams launch at this much pending input
    long long v = atoll(e);
    if (v > 0) ctx->dstream_batch_bytes = (size_t)v;
  }
  if (const char *e = getenv("ZB200_DSTREAM_LOG")) ctx->dstream_log = atoi(e) != 0;  // test hook: the decode path of every launch
  if (const char *e = getenv("ZB200_BIG_MEMBER_BYTES")) {  // test hook: segment path for small members too
    long long v = atoll(e);
    if (v > 0) {
      ctx->big_member_bytes = (uint64_t)v;
      ctx->big_env = true;
    }
  }
  if (const char *e = getenv("ZB200_JOINT_MARKERS")) ctx->joint_markers = atoi(e) != 0;  // test hook: 0 = no marker segments at joints
  if (const char *e = getenv("ZB200_MARK_WINDOW_SEGS")) {  // test hook: small windows in the joint marker decode
    long v = atol(e);
    if (v > 0) ctx->mark_window_segs = (uint32_t)std::min<long>(v, 60000);
  }
  if (const char *e = getenv("ZB200_INDEX_GROUP_BYTES")) {  // test hook: small launch groups in index extraction
    long long v = atoll(e);
    if (v > 0) ctx->index_group_bytes = (uint64_t)v;
  }
  if (const char *e = getenv("ZB200_INDEX_LOG")) ctx->index_log = atoi(e) != 0;  // test hook: one line per extraction group
  ctx->memops = load_stream_memops();
  if (const char *e = getenv("ZB200_UNC_GATED")) ctx->gated_unc = atoi(e) != 0;  // test hook: 0 = one launch per group
  if (const char *e = getenv("ZB200_UNC_GROUP_BYTES")) {  // test hook: small pipelined groups in the host uncompress
    long long v = atoll(e);
    if (v > 0) ctx->unc_group_out_bytes = (uint64_t)v;
  }
  if (const char *e = getenv("ZB200_DEV_GROUP_CHUNKS")) {  // device-resident batches only (bench.py)
    long v = atol(e);
    if (v > 0) ctx->dev_group_chunks = (size_t)v;
  }
  DeviceGuard g(device);
  bool ok = cudaStreamCreateWithFlags(&ctx->own_stream, cudaStreamNonBlocking) == cudaSuccess;
  ctx->stream = ctx->own_stream;
  if (ok) ok = cudaStreamCreateWithFlags(&ctx->h2d_stream, cudaStreamNonBlocking) == cudaSuccess;
  if (ok) ok = cudaStreamCreateWithFlags(&ctx->d2h_stream, cudaStreamNonBlocking) == cudaSuccess;
  for (int i = 0; ok && i < 10; i++) ok = cudaEventCreate(&ctx->ev[i]) == cudaSuccess;
  if (ok) ok = cudaMalloc((void **)&ctx->d_tabs, sizeof(ZbCrcTables)) == cudaSuccess;
  if (ok) ok = ensure(ctx, ctx->counter, sizeof(ZbCounters)) == ZB200_OK;
  // kernel attributes are per device (and cheap to set again): every ctx sets them for its own
  if (ok) ok = zb_setup_deflate_attrs() == cudaSuccess && zb_setup_inflate_attrs() == cudaSuccess;
  if (ok) {
    ZbCrcTables t;
    zb_crc_build_tables(&t);
    ok = cudaMemcpy(ctx->d_tabs, &t, sizeof(t), cudaMemcpyHostToDevice) == cudaSuccess;
  }
  if (!ok) {
    cudaGetLastError();
    zb200_shutdown(ctx);  // releases whatever was created
    return ZB200_ERR_CUDA;
  }
  *out = ctx;
  return ZB200_OK;
}

void zb200_shutdown(zb200_ctx *ctx) {
  if (!ctx) return;
  DeviceGuard g(ctx->device);
  if (ctx->stream) cudaStreamSynchronize(ctx->stream);
  DevBuf *bufs[] = {&ctx->desc, &ctx->member_first, &ctx->fname, &ctx->masks, &ctx->recs, &ctx->hist, &ctx->chk,
                    &ctx->cb, &ctx->chunk_off, &ctx->member_off, &ctx->member_check, &ctx->member_isize,
                    &ctx->src_off, &ctx->dst_off, &ctx->out_len, &ctx->status, &ctx->expect, &ctx->kind,
                    &ctx->counter, &ctx->cix_rec, &ctx->cix_crc, &ctx->cix_first, &ctx->cix_out, &ctx->ck_out, &ctx->ck_pieces, &ctx->ck_first, &ctx->ck_piece_out, &ctx->ck_partials, &ctx->in_stage, &ctx->out_stage, &ctx->lz2_tables, &ctx->opt_scratch, &ctx->rs_meta, &ctx->rs_tiles, &ctx->rs_counts, &ctx->rs_starts, &ctx->carry,
                    &ctx->seg_src, &ctx->seg_dst, &ctx->seg_len, &ctx->seg_status, &ctx->seg_kind, &ctx->seg_expect, &ctx->seg_cand, &ctx->skip_mask, &ctx->order, &ctx->mark_scratch, &ctx->mark_segs, &ctx->seg_bits, &ctx->mark_win, &ctx->gate,
                    &ctx->idx_desc, &ctx->idx_out, &ctx->dict_win, &ctx->dict_md};
  for (DevBuf *b : bufs)
    if (b->p) cudaFree(b->p);
  if (ctx->d_tabs) cudaFree(ctx->d_tabs);
  for (int i = 0; i < 10; i++)
    if (ctx->ev[i]) cudaEventDestroy(ctx->ev[i]);
  for (cudaEvent_t e : ctx->gev) cudaEventDestroy(e);
  if (ctx->pin) cudaFreeHost(ctx->pin);
  ctx->pool.stop();
  for (StageRing *r : {&ctx->ring_in, &ctx->ring_out})
    for (int i = 0; i < kStageSlots; i++) {
      if (r->slot[i]) cudaFreeHost(r->slot[i]);
      if (r->ev[i]) cudaEventDestroy(r->ev[i]);
    }
  if (ctx->group_end.p) cudaFree(ctx->group_end.p);
  if (ctx->own_stream) cudaStreamDestroy(ctx->own_stream);
  if (ctx->h2d_stream) cudaStreamDestroy(ctx->h2d_stream);
  if (ctx->d2h_stream) cudaStreamDestroy(ctx->d2h_stream);
  cudaGetLastError();
  delete ctx;
}

int zb200_set_stream(zb200_ctx *ctx, void *cuda_stream) {
  if (!ctx) return ZB200_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  ctx->stream = cuda_stream ? (cudaStream_t)cuda_stream : ctx->own_stream;
  return ZB200_OK;
}

const char *zb200_last_cuda_error(zb200_ctx *ctx) { return ctx ? ctx->last_err.c_str() : ""; }

const char *zb200_strerror(int s) {
  switch (s) {
    case ZB200_OK: return "ok";
    case ZB200_ERR_INVALID_LEVEL: return "Invalid compression level";
    case ZB200_ERR_INVALID_FORMAT: return "Invalid data format";
    case ZB200_ERR_UNCOMPRESS: return "Invalid buffer, unable to uncompress";
    case ZB200_ERR_COMPRESS: return "Unexpected error while compressing";
    case ZB200_ERR_END_OF_BUFFER: return "Cannot read further, at end of buffer";
    case ZB200_ERR_BYTE_BOUNDARY: return "Must be at a byte boundary";
    case ZB200_ERR_BLOCK_HEADER: return "Invalid block header";
    case ZB200_ERR_INVALID_SYMBOL: return "Invalid symbol";
    case ZB200_ERR_DETECT: return "Unable to detect compressed data format";
    case ZB200_ERR_METHOD: return "Unsupported compression method";
    case ZB200_ERR_CINFO: return "Invalid compression info";
    case ZB200_ERR_HEADER: return "Invalid header";
    case ZB200_ERR_FDICT: return "Preset dictionary is not yet supported";
    case ZB200_ERR_CHECKSUM: return "Checksum verification failed";
    case ZB200_ERR_GZIP_ID: return "Failed gzip identification values check";
    case ZB200_ERR_GZIP_RESERVED: return "Reserved flag bits set";
    case ZB200_ERR_GZIP_FLAGS: return "Currently unsupported flags are set";
    case ZB200_ERR_SIZE: return "Size verification failed";
    case ZB200_ERR_DST_TOO_SMALL: return "Destination buffer too small";
    case ZB200_ERR_CUDA: return "CUDA error (no CPU fallback)";
    case ZB200_ERR_NOMEM: return "Out of device memory";
    case ZB200_ERR_ARG: return "Invalid argument";
    case ZB200_ERR_DICTIONARY: return "Dictionary does not match the member's DICTID";
    default: return "unknown status";
  }
}

size_t zb200_deflate_bound(size_t len) {
  size_t chunks = len == 0 ? 1 : (len + ZB_CHUNK_BYTES - 1) / ZB_CHUNK_BYTES;
  // per chunk: worst case is the stored path (two stored pieces for a full 64 KiB chunk);
  // a coded chunk is only chosen when it is smaller than that.
  return len + chunks * 10 + 8;
}
size_t zb200_compress_bound(size_t len, int data_format) {
  size_t frame = data_format == ZB200_DF_GZIP ? 36 + 8 : data_format == ZB200_DF_ZLIB ? 6 : 0;
  return zb200_deflate_bound(len) + frame;
}

int zb200_compress_batch_device_window(zb200_ctx *ctx, const uint8_t *d_src, const uint64_t *src_offsets, size_t n,
                                       int level, int strategy, int window_bits, int data_format,
                                       const uint8_t *fname_lens, uint8_t *d_dst, size_t dst_cap, uint64_t *dst_offsets,
                                       int *statuses) {
  return guarded(ctx, [&]() -> int {
  if (!ctx || !src_offsets || !dst_offsets || (n && (!d_src || !d_dst))) return ZB200_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  DeviceGuard g(ctx->device);
  ctx->timing.kernel_launches = 0;
  return compress_locked(ctx, d_src, nullptr, src_offsets, n, level, data_format, fname_lens, d_dst, dst_cap, nullptr,
                         0, dst_offsets, statuses, ctx->dev_group_chunks, nullptr, nullptr, strategy, window_bits);
  });
}

int zb200_compress_batch_device_optimal(zb200_ctx *ctx, const uint8_t *d_src, const uint64_t *src_offsets, size_t n,
                                        int window_bits, int data_format, const uint8_t *fname_lens, uint8_t *d_dst,
                                        size_t dst_cap, uint64_t *dst_offsets, int *statuses) {
  return guarded(ctx, [&]() -> int {
  if (!ctx || !src_offsets || !dst_offsets || (n && (!d_src || !d_dst))) return ZB200_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  DeviceGuard g(ctx->device);
  ctx->timing.kernel_launches = 0;
  return compress_locked(ctx, d_src, nullptr, src_offsets, n, 9, data_format, fname_lens, d_dst, dst_cap, nullptr, 0,
                         dst_offsets, statuses, ctx->dev_group_chunks, nullptr, nullptr, ZB_STRATEGY_DEFAULT, window_bits,
                         true);
  });
}

int zb200_compress_batch_device_strategy(zb200_ctx *ctx, const uint8_t *d_src, const uint64_t *src_offsets, size_t n,
                                         int level, int strategy, int data_format, const uint8_t *fname_lens,
                                         uint8_t *d_dst, size_t dst_cap, uint64_t *dst_offsets, int *statuses) {
  return zb200_compress_batch_device_window(ctx, d_src, src_offsets, n, level, strategy, 15, data_format, fname_lens,
                                            d_dst, dst_cap, dst_offsets, statuses);
}

int zb200_compress_batch_device(zb200_ctx *ctx, const uint8_t *d_src, const uint64_t *src_offsets, size_t n,
                                int level, int data_format, const uint8_t *fname_lens, uint8_t *d_dst,
                                size_t dst_cap, uint64_t *dst_offsets, int *statuses) {
  return zb200_compress_batch_device_strategy(ctx, d_src, src_offsets, n, level, ZB_STRATEGY_DEFAULT, data_format,
                                              fname_lens, d_dst, dst_cap, dst_offsets, statuses);
}

// zb200_compress_batch, and with a dictionary table zb200_compress_batch_dicts (dict_of: the member's entry; null:
// every member names entry 0, zb200_compress_batch_dict)
static int compress_batch_host(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n, int level,
                               int data_format, const uint8_t *dict_base, const uint64_t *dict_offsets, size_t k,
                               const int32_t *dict_of, const uint8_t *fname_lens, uint8_t *dst_base, size_t dst_cap,
                               uint64_t *dst_offsets, int *statuses, int strategy = ZB_STRATEGY_DEFAULT,
                               int window_bits = 15, bool optimal = false) {
  return guarded(ctx, [&]() -> int {
  if (!ctx || !src_offsets || !dst_offsets || (n && (!src_base || !dst_base))) return ZB200_ERR_ARG;
  if (zb_window_bits(window_bits, data_format)) return ZB200_ERR_ARG;
  const bool shared = k && !dict_of;   // zb200_compress_batch_dict: its checks apply even to an empty batch
  std::vector<int32_t> all0;
  if (shared) {
    all0.assign(n, 0);
    dict_of = all0.data();
  }
  bool any = false;
  if (int rc = check_dicts(dict_base, dict_offsets, k, dict_of, n, any)) return rc;
  if (any || (shared && dict_offsets[1] > dict_offsets[0])) {
    // zlib's deflateSetDictionary refuses gzip too: the format has no field for it
    if (level < -2 || level > 9) return ZB200_ERR_INVALID_LEVEL;
    if (data_format != ZB200_DF_ZLIB && data_format != ZB200_DF_DEFLATE) return ZB200_ERR_INVALID_FORMAT;
  }
  std::lock_guard<std::mutex> lk(ctx->mu);
  DeviceGuard g(ctx->device);
  memset(&ctx->timing, 0, sizeof(ctx->timing));
  DictScope ds(ctx);
  if (any) {
    if (int rc = ds.set(dict_base, dict_offsets, k, dict_of, n)) return rc;
  }
  if (n == 0) {
    dst_offsets[0] = 0;
    return ZB200_OK;
  }
  for (size_t i = 0; i < n; i++)
    if (src_offsets[i + 1] < src_offsets[i]) return ZB200_ERR_ARG;
  const uint64_t in_bytes = src_offsets[n] - src_offsets[0];
  uint64_t bound = 0;
  for (size_t i = 0; i < n; i++)
    bound += zb200_compress_bound((size_t)(src_offsets[i + 1] - src_offsets[i]), data_format) + 64;
  ENSURE(ctx->in_stage, (size_t)in_bytes + 64);
  ENSURE(ctx->out_stage, (size_t)bound + 64);
  int rc = compress_locked(ctx, (const uint8_t *)ctx->in_stage.p, src_base, src_offsets, n, level, data_format,
                           fname_lens, (uint8_t *)ctx->out_stage.p, ctx->out_stage.cap & ~(size_t)3, dst_base,
                           dst_cap, dst_offsets, statuses, ctx->host_group_chunks, nullptr, nullptr, strategy,
                           window_bits, optimal);
  if (rc) return rc;
  ctx->timing.h2d_ms = ev_ms(ctx->ev[6], ctx->ev[7]);
  ctx->timing.d2h_ms = ev_ms(ctx->ev[8], ctx->ev[9]);
  ctx->timing.h2d_bytes = in_bytes;
  ctx->timing.d2h_bytes = dst_offsets[n];
  return ZB200_OK;
  });
}

int zb200_compress_batch(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n, int level,
                         int data_format, const uint8_t *fname_lens, uint8_t *dst_base, size_t dst_cap,
                         uint64_t *dst_offsets, int *statuses) {
  return compress_batch_host(ctx, src_base, src_offsets, n, level, data_format, nullptr, nullptr, 0, nullptr, fname_lens,
                             dst_base, dst_cap, dst_offsets, statuses);
}

int zb200_compress_batch_strategy(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n,
                                  int level, int strategy, int data_format, const uint8_t *fname_lens,
                                  uint8_t *dst_base, size_t dst_cap, uint64_t *dst_offsets, int *statuses) {
  return zb200_compress_batch_window(ctx, src_base, src_offsets, n, level, strategy, 15, data_format, fname_lens,
                                     dst_base, dst_cap, dst_offsets, statuses);
}

int zb200_compress_batch_window(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n,
                                int level, int strategy, int window_bits, int data_format, const uint8_t *fname_lens,
                                uint8_t *dst_base, size_t dst_cap, uint64_t *dst_offsets, int *statuses) {
  return compress_batch_host(ctx, src_base, src_offsets, n, level, data_format, nullptr, nullptr, 0, nullptr, fname_lens,
                             dst_base, dst_cap, dst_offsets, statuses, strategy, window_bits);
}

int zb200_compress_batch_optimal(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n,
                                 int window_bits, int data_format, const uint8_t *fname_lens, uint8_t *dst_base,
                                 size_t dst_cap, uint64_t *dst_offsets, int *statuses) {
  return compress_batch_host(ctx, src_base, src_offsets, n, 9, data_format, nullptr, nullptr, 0, nullptr, fname_lens,
                             dst_base, dst_cap, dst_offsets, statuses, ZB_STRATEGY_DEFAULT, window_bits, true);
}

// ---- rsyncable compression (zb_rsync.cu; DESIGN.md section 5 "Rsyncable") ----
// The chunk map of the members d_src[src_offsets[i], src_offsets[i + 1]) (offsets checked by the caller: they do
// not decrease), on ctx->stream: the one path behind zb200_rsyncable_chunks and the _rsyncable compress calls.  Two
// launches, then one copy of the counts and starts back to the host.
static int rsync_chunks_locked(zb200_ctx *ctx, const uint8_t *d_src, const uint64_t *src_offsets, size_t n,
                               RsyncMap &map) {
  if (n > UINT32_MAX) return ZB200_ERR_ARG;
  std::vector<uint64_t> meta(3 * (n + 1), 0);   // src_off, tile_off, start_off: [n + 1] each
  uint64_t *src_off = meta.data(), *tile_off = src_off + (n + 1), *start_off = tile_off + (n + 1);
  for (size_t i = 0; i < n; i++) {
    const uint64_t len = src_offsets[i + 1] - src_offsets[i];
    src_off[i] = src_offsets[i];
    tile_off[i + 1] = tile_off[i] + (len + ZB_RSYNC_MIN - 1) / ZB_RSYNC_MIN;
    start_off[i + 1] = start_off[i] + zb_rsync_cap(len);
  }
  src_off[n] = src_offsets[n];
  ENSURE(ctx->rs_meta, meta.size() * sizeof(uint64_t));
  ENSURE(ctx->rs_tiles, (size_t)tile_off[n] * sizeof(uint32_t) + 4);
  ENSURE(ctx->rs_counts, n * sizeof(uint64_t));
  ENSURE(ctx->rs_starts, (size_t)start_off[n] * sizeof(uint64_t));
  cudaStream_t s = ctx->stream;
  CK(cudaMemcpyAsync(ctx->rs_meta.p, meta.data(), meta.size() * sizeof(uint64_t), cudaMemcpyHostToDevice, s));
  ZbRsyncWork w;
  w.src = d_src;
  w.src_off = (const uint64_t *)ctx->rs_meta.p;
  w.tile_off = w.src_off + (n + 1);
  w.start_off = w.tile_off + (n + 1);
  w.tile_cand = (uint32_t *)ctx->rs_tiles.p;
  w.counts = (uint64_t *)ctx->rs_counts.p;
  w.starts = (uint64_t *)ctx->rs_starts.p;
  w.n = (uint32_t)n;
  w.n_tiles = tile_off[n];
  CK(zb_launch_rsync(w, s));
  ctx->timing.kernel_launches += w.n_tiles ? 2 : 1;
  map.count.resize(n);
  map.off.assign(start_off, start_off + n + 1);
  map.starts.resize(start_off[n]);
  CK(cudaMemcpyAsync(map.count.data(), w.counts, n * sizeof(uint64_t), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(map.starts.data(), w.starts, map.starts.size() * sizeof(uint64_t), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  // the plan trusts the map with source ranges: check its shape before any descriptor is built from it
  for (size_t i = 0; i < n; i++) {
    const uint64_t len = src_offsets[i + 1] - src_offsets[i], c = map.count[i], *st = map.starts.data() + map.off[i];
    bool ok = c >= 1 && c <= map.off[i + 1] - map.off[i] && st[0] == 0;
    for (uint64_t k = 1; ok && k < c; k++) ok = st[k] > st[k - 1] && st[k] - st[k - 1] <= ZB_CHUNK_BYTES;
    ok = ok && (len == 0 ? c == 1 : st[c - 1] < len && len - st[c - 1] <= ZB_CHUNK_BYTES);
    if (!ok) {
      ctx->last_err = "rsyncable chunk map: malformed starts";
      return ZB200_ERR_CUDA;
    }
  }
  return ZB200_OK;
}

static int rsync_check_offsets(const uint64_t *src_offsets, size_t n) {
  for (size_t i = 0; i < n; i++)
    if (src_offsets[i + 1] < src_offsets[i]) return ZB200_ERR_ARG;
  return ZB200_OK;
}

// the batch src_base[src_offsets[0], src_offsets[n]) into in_stage, whole (no copy-in / compress overlap: the chunk
// map needs every byte first); offs receives the offsets rebased to in_stage
static int rsync_stage(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n,
                       std::vector<uint64_t> &offs) {
  const uint64_t in_bytes = src_offsets[n] - src_offsets[0];
  ENSURE(ctx->in_stage, (size_t)in_bytes + 64);
  offs.resize(n + 1);
  for (size_t i = 0; i <= n; i++) offs[i] = src_offsets[i] - src_offsets[0];
  const uint8_t *h = src_base + src_offsets[0];
  return h2d_copy(ctx, (uint8_t *)ctx->in_stage.p, h, (size_t)in_bytes, ctx->stream, is_pageable(h));
}

size_t zb200_rsyncable_chunks_bound(size_t len) { return (size_t)zb_rsync_cap(len); }

size_t zb200_compress_bound_rsyncable(size_t len, int data_format) {
  size_t frame = data_format == ZB200_DF_GZIP ? 36 + 8 : data_format == ZB200_DF_ZLIB ? 6 : 0;
  return len + (size_t)zb_rsync_cap(len) * 10 + 8 + frame;
}

int zb200_rsyncable_chunks(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n,
                           uint64_t *counts, uint64_t *starts, size_t starts_cap) {
  return guarded(ctx, [&]() -> int {
  if (!ctx || !src_offsets || (n && (!src_base || !counts))) return ZB200_ERR_ARG;
  if (int rc = rsync_check_offsets(src_offsets, n)) return rc;
  if (n == 0) return ZB200_OK;
  std::lock_guard<std::mutex> lk(ctx->mu);
  DeviceGuard g(ctx->device);
  ctx->timing.kernel_launches = 0;
  std::vector<uint64_t> offs;
  RsyncMap map;
  if (int rc = rsync_stage(ctx, src_base, src_offsets, n, offs)) return rc;
  if (int rc = rsync_chunks_locked(ctx, (const uint8_t *)ctx->in_stage.p, offs.data(), n, map)) return rc;
  uint64_t total = 0;
  for (size_t i = 0; i < n; i++) total += counts[i] = map.count[i];
  if (total > starts_cap || (total && !starts)) return ZB200_ERR_DST_TOO_SMALL;
  for (size_t i = 0; i < n; i++) {
    memcpy(starts, map.starts.data() + map.off[i], (size_t)map.count[i] * sizeof(uint64_t));
    starts += map.count[i];
  }
  return ZB200_OK;
  });
}

int zb200_compress_batch_rsyncable(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n,
                                   int level, int data_format, const uint8_t *fname_lens, uint8_t *dst_base,
                                   size_t dst_cap, uint64_t *dst_offsets, int *statuses) {
  return guarded(ctx, [&]() -> int {
  if (!ctx || !src_offsets || !dst_offsets || (n && (!src_base || !dst_base))) return ZB200_ERR_ARG;
  if (level < -2 || level > 9) return ZB200_ERR_INVALID_LEVEL;
  if (data_format != ZB200_DF_GZIP && data_format != ZB200_DF_ZLIB && data_format != ZB200_DF_DEFLATE)
    return ZB200_ERR_INVALID_FORMAT;
  if (int rc = rsync_check_offsets(src_offsets, n)) return rc;
  std::lock_guard<std::mutex> lk(ctx->mu);
  DeviceGuard g(ctx->device);
  memset(&ctx->timing, 0, sizeof(ctx->timing));
  dst_offsets[0] = 0;
  if (n == 0) return ZB200_OK;
  uint64_t bound = 0;
  for (size_t i = 0; i < n; i++)
    bound += zb200_compress_bound_rsyncable((size_t)(src_offsets[i + 1] - src_offsets[i]), data_format) + 64;
  ENSURE(ctx->out_stage, (size_t)bound + 64);
  std::vector<uint64_t> offs;
  RsyncMap map;
  if (int rc = rsync_stage(ctx, src_base, src_offsets, n, offs)) return rc;
  if (int rc = rsync_chunks_locked(ctx, (const uint8_t *)ctx->in_stage.p, offs.data(), n, map)) return rc;
  // the input is on the device already: the plan runs as for device input, with the output copied back per group
  int rc = compress_locked(ctx, (const uint8_t *)ctx->in_stage.p, nullptr, offs.data(), n, level, data_format,
                           fname_lens, (uint8_t *)ctx->out_stage.p, ctx->out_stage.cap & ~(size_t)3, dst_base,
                           dst_cap, dst_offsets, statuses, ctx->host_group_chunks, nullptr, nullptr,
                           ZB_STRATEGY_DEFAULT, 15, false, &map);
  if (rc) return rc;
  ctx->timing.d2h_ms = ev_ms(ctx->ev[8], ctx->ev[9]);
  ctx->timing.h2d_bytes = src_offsets[n] - src_offsets[0];
  ctx->timing.d2h_bytes = dst_offsets[n];
  return ZB200_OK;
  });
}

int zb200_compress_batch_device_rsyncable(zb200_ctx *ctx, const uint8_t *d_src, const uint64_t *src_offsets, size_t n,
                                          int level, int data_format, const uint8_t *fname_lens, uint8_t *d_dst,
                                          size_t dst_cap, uint64_t *dst_offsets, int *statuses) {
  return guarded(ctx, [&]() -> int {
  if (!ctx || !src_offsets || !dst_offsets || (n && (!d_src || !d_dst))) return ZB200_ERR_ARG;
  if (level < -2 || level > 9) return ZB200_ERR_INVALID_LEVEL;
  if (data_format != ZB200_DF_GZIP && data_format != ZB200_DF_ZLIB && data_format != ZB200_DF_DEFLATE)
    return ZB200_ERR_INVALID_FORMAT;
  if (int rc = rsync_check_offsets(src_offsets, n)) return rc;
  std::lock_guard<std::mutex> lk(ctx->mu);
  DeviceGuard g(ctx->device);
  ctx->timing.kernel_launches = 0;
  dst_offsets[0] = 0;
  if (n == 0) return ZB200_OK;
  RsyncMap map;
  if (int rc = rsync_chunks_locked(ctx, d_src, src_offsets, n, map)) return rc;
  return compress_locked(ctx, d_src, nullptr, src_offsets, n, level, data_format, fname_lens, d_dst, dst_cap, nullptr,
                         0, dst_offsets, statuses, ctx->dev_group_chunks, nullptr, nullptr, ZB_STRATEGY_DEFAULT, 15,
                         false, &map);
  });
}

int zb200_compress_batch_dict(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n, int level,
                              int data_format, const uint8_t *dict, size_t dict_len, uint8_t *dst_base, size_t dst_cap,
                              uint64_t *dst_offsets, int *statuses) {
  if (dict_len && !dict) return ZB200_ERR_ARG;
  const uint64_t offs[2] = {0, dict_len};
  return compress_batch_host(ctx, src_base, src_offsets, n, level, data_format, dict, offs, 1, nullptr, nullptr,
                             dst_base, dst_cap, dst_offsets, statuses);
}

int zb200_compress_batch_dicts(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n,
                               int level, int data_format, int window_bits, const uint8_t *dict_base,
                               const uint64_t *dict_offsets, size_t k, const int32_t *dict_of, uint8_t *dst_base,
                               size_t dst_cap, uint64_t *dst_offsets, int *statuses) {
  static const int32_t kNoMembers = -1;   // an empty batch may pass no dict_of (null means "shared" below)
  if (!dict_of) {
    if (n) return ZB200_ERR_ARG;
    dict_of = &kNoMembers;
  }
  return compress_batch_host(ctx, src_base, src_offsets, n, level, data_format, dict_base, dict_offsets, k, dict_of,
                             nullptr, dst_base, dst_cap, dst_offsets, statuses, ZB_STRATEGY_DEFAULT, window_bits);
}

// host inputs (pipelined H2D over launch groups) -> members left in device memory: the sharded
// multi-GPU path compresses this way, exchanges the sizes, and only then knows where each shard's
// bytes go in the concatenated host stream
int zb200_compress_batch_h2d(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n, int level,
                             int data_format, const uint8_t *fname_lens, uint8_t *d_dst, size_t dst_cap,
                             uint64_t *dst_offsets, int *statuses) {
  return guarded(ctx, [&]() -> int {
    if (!ctx || !src_offsets || !dst_offsets || (n && (!src_base || !d_dst))) return ZB200_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    DeviceGuard g(ctx->device);
    memset(&ctx->timing, 0, sizeof(ctx->timing));
    if (n == 0) {
      dst_offsets[0] = 0;
      return ZB200_OK;
    }
    for (size_t i = 0; i < n; i++)
      if (src_offsets[i + 1] < src_offsets[i]) return ZB200_ERR_ARG;
    const uint64_t in_bytes = src_offsets[n] - src_offsets[0];
    ENSURE(ctx->in_stage, (size_t)in_bytes + 64);
    int rc = compress_locked(ctx, (const uint8_t *)ctx->in_stage.p, src_base, src_offsets, n, level, data_format,
                             fname_lens, d_dst, dst_cap, nullptr, 0, dst_offsets, statuses, ctx->host_group_chunks);
    if (rc) return rc;
    ctx->timing.h2d_ms = ev_ms(ctx->ev[6], ctx->ev[7]);
    ctx->timing.h2d_bytes = in_bytes;
    return ZB200_OK;
  });
}

// ---- compress streams ----
// zb200_compress_stream_begin, and with a non-empty dictionary zb200_compress_stream_begin_dict: the window is the
// history in front of the first chunk (LZ levels), exactly as after a sync flush of it, and zlib's header carries it
static int compress_stream_begin(zb200_ctx *ctx, int level, int data_format, int fname_len, const uint8_t *dict,
                                 size_t dict_len, zb200_compress_stream **out, int strategy = ZB_STRATEGY_DEFAULT,
                                 int window_bits = 15, bool optimal = false) {
  return guarded(ctx, [&]() -> int {
    if (!ctx || !out || (dict_len && !dict)) return ZB200_ERR_ARG;
    *out = nullptr;
    // the stream keeps the folded pair: its history rules are those of the level the strategy leaves
    if (int rc = zb_strategy_level(level, strategy)) return rc;
    if (data_format != ZB200_DF_GZIP && data_format != ZB200_DF_ZLIB && data_format != ZB200_DF_DEFLATE)
      return ZB200_ERR_INVALID_FORMAT;
    if (dict_len && data_format == ZB200_DF_GZIP) return ZB200_ERR_INVALID_FORMAT;
    if (fname_len < 0 || fname_len > 25) return ZB200_ERR_ARG;
    if (int rc = zb_window_bits(window_bits, data_format)) return rc;
    zb200_compress_stream *st = new zb200_compress_stream();
    st->ctx = ctx;
    st->level = level;
    st->strategy = strategy;
    st->optimal = optimal;
    st->window_bits = window_bits;
    st->data_format = data_format;
    st->fname_len = (uint8_t)fname_len;
    {
      std::lock_guard<std::mutex> lk(ctx->mu);
      st->batch_bytes = ctx->stream_batch_bytes;
    }
    st->buf.reserve(65536);  // a non-null source even for an empty member
    if (dict_len) {
      st->has_dict = true;
      st->dict_id = host_adler32(dict, dict_len);
      if (level == -1 || level >= 2) {
        st->hist = std::min<size_t>(dict_len, 32768);
        st->buf.assign(dict + (dict_len - st->hist), dict + dict_len);
      }
    }
    *out = st;
    return ZB200_OK;
  });
}

int zb200_compress_stream_begin(zb200_ctx *ctx, int level, int data_format, int fname_len, zb200_compress_stream **out) {
  return compress_stream_begin(ctx, level, data_format, fname_len, nullptr, 0, out);
}

int zb200_compress_stream_begin_strategy(zb200_ctx *ctx, int level, int strategy, int data_format, int fname_len,
                                         zb200_compress_stream **out) {
  return zb200_compress_stream_begin_window(ctx, level, strategy, 15, data_format, fname_len, out);
}

int zb200_compress_stream_begin_window(zb200_ctx *ctx, int level, int strategy, int window_bits, int data_format,
                                       int fname_len, zb200_compress_stream **out) {
  return compress_stream_begin(ctx, level, data_format, fname_len, nullptr, 0, out, strategy, window_bits);
}

int zb200_compress_stream_begin_optimal(zb200_ctx *ctx, int window_bits, int data_format, int fname_len,
                                        zb200_compress_stream **out) {
  return compress_stream_begin(ctx, 9, data_format, fname_len, nullptr, 0, out, ZB_STRATEGY_DEFAULT, window_bits, true);
}

int zb200_compress_stream_begin_dict(zb200_ctx *ctx, int level, int data_format, const uint8_t *dict, size_t dict_len,
                                     zb200_compress_stream **out) {
  return compress_stream_begin(ctx, level, data_format, 0, dict, dict_len, out);
}

size_t zb200_compress_stream_bound(const zb200_compress_stream *st, size_t len) {
  return st ? zb200_compress_bound(st->buf.size() - st->hist + len, st->data_format) + (st->has_dict ? 4 : 0) : 0;
}

int zb200_compress_stream_write(zb200_compress_stream *st, const uint8_t *src, size_t len, uint8_t *dst, size_t dst_cap,
                                size_t *dst_len) {
  if (!st) return ZB200_ERR_ARG;
  zb200_ctx *ctx = st->ctx;
  return guarded(ctx, [&]() -> int {
    if (!dst_len || (len && !src)) return ZB200_ERR_ARG;
    *dst_len = 0;
    if (st->err) return st->err;
    if (st->finished) return ZB200_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    DeviceGuard g(ctx->device);
    memset(&ctx->timing, 0, sizeof(ctx->timing));
    const size_t old = st->buf.size(), pending = old - st->hist + len;
    st->buf.insert(st->buf.end(), src, src + len);
    // launch with enough input gathered, holding back 1..65536 bytes: the chunk that may turn out to be the last
    if (pending < st->batch_bytes || pending <= ZB_CHUNK_BYTES) return ZB200_OK;
    const int rc = stream_run(st, (pending - 1) / ZB_CHUNK_BYTES * ZB_CHUNK_BYTES, false, dst, dst_cap, dst_len);
    if (rc) {
      st->buf.resize(old);  // nothing consumed
      if (rc == ZB200_ERR_CUDA) st->err = rc;
    }
    return rc;
  });
}

int zb200_compress_stream_flush(zb200_compress_stream *st, int mode, uint8_t *dst, size_t dst_cap, size_t *dst_len) {
  if (!st) return ZB200_ERR_ARG;
  zb200_ctx *ctx = st->ctx;
  return guarded(ctx, [&]() -> int {
    if (!dst_len) return ZB200_ERR_ARG;
    *dst_len = 0;
    if (st->err) return st->err;
    if (st->finished || (mode != ZB200_SYNC_FLUSH && mode != ZB200_FULL_FLUSH)) return ZB200_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    DeviceGuard g(ctx->device);
    memset(&ctx->timing, 0, sizeof(ctx->timing));
    // a write always holds input back, so nothing pending means nothing written since the last flush (or begin)
    const size_t pending = st->buf.size() - st->hist;
    if (pending == 0) return ZB200_OK;
    // the flush segment ends here: its last chunk may be short, and the next segment's chunks start after it
    const int rc = stream_run(st, pending, false, dst, dst_cap, dst_len, mode == ZB200_FULL_FLUSH);
    if (rc == ZB200_ERR_CUDA) st->err = rc;
    return rc;
  });
}

int zb200_compress_stream_finish(zb200_compress_stream *st, uint8_t *dst, size_t dst_cap, size_t *dst_len) {
  if (!st) return ZB200_ERR_ARG;
  zb200_ctx *ctx = st->ctx;
  return guarded(ctx, [&]() -> int {
    if (!dst_len) return ZB200_ERR_ARG;
    *dst_len = 0;
    if (st->err) return st->err;
    if (st->finished) return ZB200_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    DeviceGuard g(ctx->device);
    memset(&ctx->timing, 0, sizeof(ctx->timing));
    const int rc = stream_run(st, st->buf.size() - st->hist, true, dst, dst_cap, dst_len);
    if (rc == ZB200_ERR_CUDA) st->err = rc;
    if (rc) return rc;
    st->finished = true;
    std::vector<uint8_t>().swap(st->buf);
    st->hist = 0;
    return ZB200_OK;
  });
}

void zb200_compress_stream_free(zb200_compress_stream *st) { delete st; }

// ---- decompress streams ----
static int decompress_stream_begin(zb200_ctx *ctx, int data_format, const uint8_t *dict, size_t dict_len,
                                   zb200_decompress_stream **out) {
  return guarded(ctx, [&]() -> int {
    if (!ctx || !out || (dict_len && !dict)) return ZB200_ERR_ARG;
    *out = nullptr;
    if (data_format < ZB200_DF_DETECT || data_format > ZB200_DF_DEFLATE) return ZB200_ERR_INVALID_FORMAT;
    zb200_decompress_stream *st = new zb200_decompress_stream();
    st->ctx = ctx;
    st->data_format = data_format;
    if (dict_len) {
      st->has_dict = true;
      st->dict_id = host_adler32(dict, dict_len);
      const size_t wl = std::min<size_t>(dict_len, 32768);
      st->dict_win.assign(dict + (dict_len - wl), dict + dict_len);
    }
    {
      std::lock_guard<std::mutex> lk(ctx->mu);
      st->batch_bytes = ctx->dstream_batch_bytes;
      st->log = ctx->dstream_log;
    }
    if (data_format == ZB200_DF_DEFLATE) dstream_header(st, false);
    *out = st;
    return ZB200_OK;
  });
}

int zb200_decompress_stream_begin(zb200_ctx *ctx, int data_format, zb200_decompress_stream **out) {
  return decompress_stream_begin(ctx, data_format, nullptr, 0, out);
}

int zb200_decompress_stream_begin_dict(zb200_ctx *ctx, int data_format, const uint8_t *dict, size_t dict_len,
                                       zb200_decompress_stream **out) {
  return decompress_stream_begin(ctx, data_format, dict, dict_len, out);
}

static size_t dstream_avail(const zb200_decompress_stream *st) { return st->q.size() - st->q_head; }

int zb200_decompress_stream_write(zb200_decompress_stream *st, const uint8_t *src, size_t len, size_t *avail) {
  if (!st) return ZB200_ERR_ARG;
  zb200_ctx *ctx = st->ctx;
  bool entered = false;   // past the argument checks: any failure (a host allocation too) is the stream's error
  const int rc = guarded(ctx, [&]() -> int {
    if (len && !src) return ZB200_ERR_ARG;
    if (avail) *avail = 0;
    if (st->err) return st->err;
    if (st->finished) return ZB200_ERR_ARG;
    entered = true;
    std::lock_guard<std::mutex> lk(ctx->mu);
    DeviceGuard g(ctx->device);
    memset(&ctx->timing, 0, sizeof(ctx->timing));
    // the member's last 8 bytes (its trailer, if this is the end), then the input itself unless the payload is over
    for (size_t i = len > 8 ? len - 8 : 0; i < len; i++) {
      memmove(st->tail, st->tail + 1, 7);
      st->tail[7] = src[i];
    }
    st->total_in += len;
    if (!st->done) st->in.insert(st->in.end(), src, src + len);
    int rc = ZB200_OK;
    if (st->fmt < 0) rc = dstream_header(st, false);
    while (!rc && st->fmt >= 0 && !st->done) {
      const uint64_t resv = dstream_reserve(st), held = st->in_off + resv;
      const uint64_t pending = st->total_in > held ? st->total_in - held : 0;
      if (pending < st->batch_bytes || pending * 8 <= st->bit0) break;
      bool progress = false;
      rc = dstream_run(st, false, progress);
      if (!progress) break;
    }
    if (!rc && avail) *avail = dstream_avail(st);
    return rc;
  });
  if (rc && entered) {
    st->err = rc;
    if (avail) *avail = 0;
  }
  return rc;
}

int zb200_decompress_stream_drain(zb200_decompress_stream *st, size_t *avail) {
  if (!st) return ZB200_ERR_ARG;
  zb200_ctx *ctx = st->ctx;
  bool entered = false;   // as in zb200_decompress_stream_write
  const int rc = guarded(ctx, [&]() -> int {
    if (avail) *avail = 0;
    if (st->err) return st->err;
    if (st->finished) return ZB200_ERR_ARG;
    entered = true;
    std::lock_guard<std::mutex> lk(ctx->mu);
    DeviceGuard g(ctx->device);
    memset(&ctx->timing, 0, sizeof(ctx->timing));
    int rc = st->fmt < 0 ? dstream_header(st, false) : ZB200_OK;
    // every complete block of what has arrived, whatever the batching threshold, the held-back tail included
    while (!rc && st->fmt >= 0 && !st->done && (st->in.size() - st->in_head) * 8 > st->bit0) {
      bool progress = false;
      rc = dstream_run(st, false, progress, true);
      if (!progress) break;
    }
    if (!rc && avail) *avail = dstream_avail(st);
    return rc;
  });
  if (rc && entered) {
    st->err = rc;
    if (avail) *avail = 0;
  }
  return rc;
}

int zb200_decompress_stream_finish(zb200_decompress_stream *st, size_t *avail) {
  if (!st) return ZB200_ERR_ARG;
  zb200_ctx *ctx = st->ctx;
  bool entered = false;   // as in zb200_decompress_stream_write
  const int rc = guarded(ctx, [&]() -> int {
    if (avail) *avail = 0;
    if (st->err) return st->err;
    if (st->finished) return ZB200_ERR_ARG;
    entered = true;
    std::lock_guard<std::mutex> lk(ctx->mu);
    DeviceGuard g(ctx->device);
    memset(&ctx->timing, 0, sizeof(ctx->timing));
    int rc = st->fmt < 0 ? dstream_header(st, true) : ZB200_OK;
    while (!rc && !st->done) {
      bool progress = false;
      rc = dstream_run(st, true, progress);
      if (!rc && !progress && !st->done) rc = ZB200_ERR_UNCOMPRESS;
    }
    // the trailer, checksum then size (gzip.nim:80-88, zippy.nim:154-162)
    if (!rc && st->fmt == ZB200_DF_GZIP) {
      if (zb_ld_le32(st->tail) != st->check) rc = ZB200_ERR_CHECKSUM;
      else if (zb_ld_le32(st->tail + 4) != (uint32_t)st->out_total) rc = ZB200_ERR_SIZE;
    } else if (!rc && st->fmt == ZB200_DF_ZLIB) {
      const uint8_t *t = st->tail + 4;
      const uint32_t expect = ((uint32_t)t[0] << 24) | ((uint32_t)t[1] << 16) | ((uint32_t)t[2] << 8) | t[3];
      if (expect != st->check) rc = ZB200_ERR_CHECKSUM;
    }
    if (rc) return rc;
    st->finished = true;
    std::vector<uint8_t>().swap(st->in);
    std::vector<uint8_t>().swap(st->win);
    st->in_head = 0;
    if (avail) *avail = dstream_avail(st);
    return ZB200_OK;
  });
  if (rc && entered) {
    st->err = rc;
    if (avail) *avail = 0;
  }
  return rc;
}

int zb200_decompress_stream_read(zb200_decompress_stream *st, uint8_t *dst, size_t dst_cap, size_t *dst_len) {
  if (!st || !dst_len) return ZB200_ERR_ARG;
  *dst_len = 0;
  if (st->err) return st->err;
  const size_t n = std::min(dst_cap, dstream_avail(st));
  if (n && !dst) return ZB200_ERR_ARG;
  if (n) memcpy(dst, st->q.data() + st->q_head, n);
  st->q_head += n;
  if (st->q_head == st->q.size()) {
    st->q.clear();
    st->q_head = 0;
  }
  *dst_len = n;
  return ZB200_OK;
}

void zb200_decompress_stream_free(zb200_decompress_stream *st) { delete st; }

// second half of the sharded path: once the size exchange has told a rank where its shard lands in
// the concatenated stream, its device-resident members go straight to that place in host memory
int zb200_download(zb200_ctx *ctx, const uint8_t *d_src, uint8_t *h_dst, size_t bytes) {
  return guarded(ctx, [&]() -> int {
    if (!ctx || (bytes && (!d_src || !h_dst))) return ZB200_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    DeviceGuard g(ctx->device);
    if (bytes) CK(cudaMemcpyAsync(h_dst, d_src, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return ZB200_OK;
  });
}

// page-lock a caller-owned host range so that the host-buffer calls can overlap their copies with
// the kernels (cudaHostRegister; a Nim string / malloc'd buffer is pageable otherwise)
int zb200_host_register(void *ptr, size_t bytes) {
  if (!ptr || !bytes) return ZB200_ERR_ARG;
  if (cudaHostRegister(ptr, bytes, cudaHostRegisterPortable) != cudaSuccess) {
    cudaGetLastError();
    return ZB200_ERR_CUDA;
  }
  return ZB200_OK;
}
int zb200_host_unregister(void *ptr) {
  if (!ptr) return ZB200_ERR_ARG;
  if (cudaHostUnregister(ptr) != cudaSuccess) {
    cudaGetLastError();
    return ZB200_ERR_CUDA;
  }
  return ZB200_OK;
}

int zb200_uncompress_batch_device(zb200_ctx *ctx, const uint8_t *d_src, const uint64_t *src_offsets, size_t n,
                                  int data_format, uint8_t *d_dst, const uint64_t *dst_offsets, uint64_t *dst_lens,
                                  int *statuses) {
  return guarded(ctx, [&]() -> int {
  if (!ctx || !src_offsets || !dst_offsets || !dst_lens || (n && !d_src)) return ZB200_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  DeviceGuard g(ctx->device);
  ctx->timing.kernel_launches = 0;
  ctx->timing.inflate_ms = ctx->timing.verify_ms = 0.f;
  return uncompress_device_locked(ctx, d_src, src_offsets, n, data_format, 0, d_dst, dst_offsets, dst_lens, statuses,
                                  false);
  });
}

int zb200_uncompress_sizes_device(zb200_ctx *ctx, const uint8_t *d_src, const uint64_t *src_offsets, size_t n,
                                  int data_format, uint64_t *sizes, int *statuses) {
  return guarded(ctx, [&]() -> int {
  if (!ctx || !src_offsets || !sizes || (n && !d_src)) return ZB200_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  DeviceGuard g(ctx->device);
  ctx->timing.kernel_launches = 0;
  ctx->timing.inflate_ms = ctx->timing.verify_ms = 0.f;
  return uncompress_device_locked(ctx, d_src, src_offsets, n, data_format, 0, nullptr, nullptr, sizes, statuses,
                                  true);
  });
}

// The decode calls' dictionary table (check_dicts, then DictScope::set): of == null means every member names entry 0
// (the *_dict calls).  Nothing happens without a member that names a non-empty entry.
static int set_decode_dicts(zb200_ctx *ctx, DictScope &ds, const uint8_t *base, const uint64_t *offs, size_t k,
                            const int32_t *of, size_t n) {
  std::vector<int32_t> all0;
  if (!of && k) {
    all0.assign(n, 0);
    of = all0.data();
  }
  bool any = false;
  if (int rc = check_dicts(base, offs, k, of, n, any)) return rc;
  return any ? ds.set(base, offs, k, of, n) : ZB200_OK;
}

// Group cuts for the decode calls' windows: gb (0, ..., n) with further cuts wherever a group's distinct windows
// (DictWindows with class 0) would pass kDictGroupWindowBytes.
static std::vector<size_t> dict_cut(const zb200_ctx *ctx, const std::vector<size_t> &gb) {
  std::vector<size_t> out(1, 0), stamp(ctx->dict_k, SIZE_MAX);
  uint64_t b = 0;
  for (size_t g = 0; g + 1 < gb.size(); g++) {
    for (size_t i = gb[g]; i < gb[g + 1]; i++) {
      const int32_t j = ctx->dict_entry[i];
      if (j < 0 || stamp[j] == out.size()) continue;
      const uint64_t st = zb_win_stride(ctx->dict_member[i].win_len);
      if (b + st > kDictGroupWindowBytes && i > out.back()) {
        out.push_back(i);
        b = 0;
      }
      stamp[j] = out.size();
      b += st;
    }
    if (gb[g + 1] > out.back()) out.push_back(gb[g + 1]);
    b = 0;
  }
  return out;
}

// zb200_uncompress_sizes, and with a dictionary table zb200_uncompress_sizes_dicts (dict_of null: every member names
// entry 0, zb200_uncompress_sizes_dict)
static int uncompress_sizes_host(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n,
                                 int data_format, const uint8_t *dict_base, const uint64_t *dict_offsets, size_t k,
                                 const int32_t *dict_of, uint64_t *sizes, int *statuses) {
  return guarded(ctx, [&]() -> int {
  if (!ctx || !src_offsets || !sizes || (n && !src_base)) return ZB200_ERR_ARG;
  if (data_format < ZB200_DF_DETECT || data_format > ZB200_DF_DEFLATE) return ZB200_ERR_INVALID_FORMAT;
  std::lock_guard<std::mutex> lk(ctx->mu);
  DeviceGuard g(ctx->device);
  memset(&ctx->timing, 0, sizeof(ctx->timing));
  DictScope ds(ctx);
  if (int rc = set_decode_dicts(ctx, ds, dict_base, dict_offsets, k, dict_of, n)) return rc;
  for (size_t i = 0; i < n; i++)
    if (src_offsets[i + 1] < src_offsets[i]) return ZB200_ERR_ARG;
  // gzip members answer from their trailer (gzip.nim:66) after the same wrapper checks the device decoder
  // makes: nothing is copied to the device for them.  Only a batch that holds zlib / raw members needs the
  // counting pass.
  bool need_device = false;
  for (size_t i = 0; i < n && !need_device; i++) {
    uint64_t payload = 0;
    uint32_t kind = 0, expect = 0, isize = 0;
    const ZbMemberDict *md = ctx->dict_on && ctx->dict_member[i].win_len ? &ctx->dict_member[i] : nullptr;
    const int st = zb_parse_wrapper(src_base + src_offsets[i], src_offsets[i + 1] - src_offsets[i], data_format, 0, payload,
                                    kind, expect, isize, md ? &md->dict_id : nullptr);
    if (st == ZB200_OK && kind != ZB200_DF_GZIP) need_device = true;
    sizes[i] = st == ZB200_OK ? isize : 0;
    if (statuses) statuses[i] = st;
  }
  if (!need_device) return ZB200_OK;
  std::vector<uint64_t> reb;
  int rc = stage_in(ctx, src_base, src_offsets, n, reb);
  if (rc) return rc;
  if (!ctx->dict_on)
    return uncompress_device_locked(ctx, (const uint8_t *)ctx->in_stage.p, reb.data(), n, data_format, 0, nullptr,
                                    nullptr, sizes, statuses, true);
  // with dictionaries: one counting launch per group of members whose windows fit one slot
  DictWindows dw;
  if (int rc2 = dw.plan(ctx, dict_cut(ctx, {0, n}), nullptr, 1)) return rc2;
  ENSURE(ctx->dict_md, n * sizeof(ZbMemberDict));
  CK(cudaMemcpyAsync(ctx->dict_md.p, ctx->dict_member.data(), n * sizeof(ZbMemberDict), cudaMemcpyHostToDevice,
                     ctx->stream));
  for (size_t g = 0; g + 1 < dw.gb.size(); g++) {
    const size_t m0 = dw.gb[g], m1 = dw.gb[g + 1];
    if (int rc2 = dw.upload(ctx, g, ctx->stream)) return rc2;
    rc = uncompress_device_locked(ctx, (const uint8_t *)ctx->in_stage.p, reb.data() + m0, m1 - m0, data_format, 0,
                                  nullptr, nullptr, sizes + m0, statuses ? statuses + m0 : nullptr, true,
                                  nullptr, nullptr, m0);
    if (rc) return rc;   // (it ends with the stream synchronised: the slot is free again)
  }
  return ZB200_OK;
  });
}

int zb200_uncompress_sizes(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n,
                           int data_format, uint64_t *sizes, int *statuses) {
  return uncompress_sizes_host(ctx, src_base, src_offsets, n, data_format, nullptr, nullptr, 0, nullptr, sizes, statuses);
}

int zb200_uncompress_sizes_dict(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n,
                                int data_format, const uint8_t *dict, size_t dict_len, uint64_t *sizes, int *statuses) {
  if (dict_len && !dict) return ZB200_ERR_ARG;
  const uint64_t offs[2] = {0, dict_len};
  return uncompress_sizes_host(ctx, src_base, src_offsets, n, data_format, dict, offs, 1, nullptr, sizes, statuses);
}

int zb200_uncompress_sizes_dicts(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n,
                                 int data_format, const uint8_t *dict_base, const uint64_t *dict_offsets, size_t k,
                                 const int32_t *dict_of, uint64_t *sizes, int *statuses) {
  if (n && !dict_of) return ZB200_ERR_ARG;
  return uncompress_sizes_host(ctx, src_base, src_offsets, n, data_format, dict_base, dict_offsets, k, dict_of, sizes,
                               statuses);
}

// zb200_uncompress_batch, with crcs (host, may be null) zb200_inflate_batch_crc32, with a dictionary table
// zb200_uncompress_batch_dicts (dict_of null: every member names entry 0, zb200_uncompress_batch_dict)
static int uncompress_batch_host(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n,
                                 int data_format, uint8_t *dst_base, const uint64_t *dst_offsets, uint64_t *dst_lens,
                                 int *statuses, uint32_t *crcs, const uint8_t *dict_base = nullptr,
                                 const uint64_t *dict_offsets = nullptr, size_t k = 0, const int32_t *dict_of = nullptr) {
  return guarded(ctx, [&]() -> int {
  if (!ctx || !src_offsets || !dst_offsets || !dst_lens || (n && !src_base)) return ZB200_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  DeviceGuard g(ctx->device);
  memset(&ctx->timing, 0, sizeof(ctx->timing));
  for (size_t i = 0; i < n; i++)
    if (src_offsets[i + 1] < src_offsets[i] || dst_offsets[i + 1] < dst_offsets[i]) return ZB200_ERR_ARG;
  DictScope ds(ctx);
  if (int rc = set_decode_dicts(ctx, ds, dict_base, dict_offsets, k, dict_of, n)) return rc;
  if (n == 0) return ZB200_OK;
  const uint64_t slo = src_offsets[0], shi = src_offsets[n], lo = dst_offsets[0], hi = dst_offsets[n];
  std::vector<uint64_t> reb(n + 1), dreb(n + 1);
  for (size_t i = 0; i <= n; i++) {
    reb[i] = src_offsets[i] - slo;
    dreb[i] = dst_offsets[i] - lo;
  }
  ENSURE(ctx->in_stage, (size_t)(shi - slo) + 64);
  ENSURE(ctx->out_stage, (size_t)(hi - lo) + 64);
  // Member groups: group g inflates while group g + 1 is copied in on the H2D stream and group
  // g - 1 is copied out on the D2H stream.  A launch wants ~7000 members to fill the GPU, so the
  // groups are big: an eighth of the batch, between 64 MiB and 1 GiB of output.  (The copies only
  // run asynchronously for page-locked host buffers; with pageable memory the same code is
  // correct but the copies block this thread.)
  std::vector<size_t> gb(1, 0);
  {
    uint64_t out_cap = ctx->unc_group_out_bytes;
    if (!out_cap) {
      // a member is decoded by ONE 8-lane group at ~9 MB/s, so every group's launch ends with the tail of its
      // longest member: a group must be worth several such tails (8192 x the largest output slot matches the
      // measured optimum of 512 MiB groups for 64 KiB members); otherwise an eighth of the batch
      uint64_t max_out = 0;
      for (size_t i = 0; i < n; i++) max_out = std::max<uint64_t>(max_out, dreb[i + 1] - dreb[i]);
      out_cap = std::max<uint64_t>(std::max<uint64_t>((hi - lo) / 8, 8192ull * max_out), 64ull << 20);
      // one gated launch for the whole batch has no per-group tail: the groups only set the granularity of the
      // overlap (what is exposed is the first group's copy-in and the last group's copy-out)
      if (ctx->memops.ok && ctx->gated_unc)
        out_cap = std::min<uint64_t>(std::max<uint64_t>((hi - lo) / 32, 32ull << 20), 256ull << 20);
    }
    const uint64_t in_cap = out_cap;
    size_t a = 0;
    for (size_t i = 1; i <= n; i++)
      if (i == n || dreb[i + 1] - dreb[a] > out_cap || reb[i + 1] - reb[a] > in_cap) {
        gb.push_back(i);
        a = i;
      }
    if (ctx->dict_on) gb = dict_cut(ctx, gb);
  }
  const size_t ng = gb.size() - 1;
  {
    bool any_big = false;
    uint64_t big_thr = (n == 1 && !ctx->big_env) ? ctx->single_member_bytes : ctx->big_member_bytes;
    {
      // the same rule as inflate_big_members: with hundreds of large members the batch fills the GPU by itself
      size_t count = 0;
      for (size_t i = 0; i < n; i++) count += reb[i + 1] - reb[i] >= big_thr;
      if (count > 256) big_thr = std::max<uint64_t>(big_thr, 64ull << 20);
    }
    for (size_t i = 0; i < n && !any_big && !ctx->dict_on; i++) any_big = reb[i + 1] - reb[i] >= big_thr;
    if (!any_big) {
      int rc = uncompress_host_pipelined(ctx, src_base + slo, reb, n, data_format, dst_base ? dst_base + lo : nullptr, dreb,
                                         dst_lens, statuses, gb, crcs);
      if (rc) return rc;
      ctx->timing.h2d_ms = ev_ms(ctx->ev[6], ctx->ev[7]);
      ctx->timing.d2h_ms = ev_ms(ctx->ev[8], ctx->ev[9]);
      ctx->timing.h2d_bytes = shi - slo;
      ctx->timing.d2h_bytes = hi - lo;
      return ZB200_OK;
    }
  }
  // a batch with large members takes the group-by-group path: those members are planned on the host
  int rc = ensure_group_events(ctx, 2 * ng + 2);
  if (rc) return rc;
  cudaStream_t s = ctx->stream, sh = ctx->h2d_stream, sd = ctx->d2h_stream;
  // the side streams start after whatever the caller's stream already holds
  CK(cudaEventRecord(ctx->gev[2 * ng], s));
  CK(cudaStreamWaitEvent(sh, ctx->gev[2 * ng], 0));
  CK(cudaStreamWaitEvent(sd, ctx->gev[2 * ng], 0));
  CK(cudaEventRecord(ctx->ev[6], sh));
  CK(cudaEventRecord(ctx->ev[8], sd));
  auto copy_in = [&](size_t gi) -> int {
    const uint64_t b0 = reb[gb[gi]], b1 = reb[gb[gi + 1]];
    if (b1 > b0)
      CK(cudaMemcpyAsync((uint8_t *)ctx->in_stage.p + b0, src_base + slo + b0, (size_t)(b1 - b0), cudaMemcpyHostToDevice, sh));
    CK(cudaEventRecord(ctx->gev[2 * gi], sh));
    return ZB200_OK;
  };
  rc = copy_in(0);
  if (rc) return rc;
  for (size_t gi = 0; gi < ng; gi++) {
    if (gi + 1 < ng) {
      rc = copy_in(gi + 1);
      if (rc) return rc;
    }
    CK(cudaStreamWaitEvent(s, ctx->gev[2 * gi], 0));
    const size_t m0 = gb[gi], m1 = gb[gi + 1];
    const std::function<int()> copy_out = [&]() -> int {
      CK(cudaEventRecord(ctx->gev[2 * gi + 1], s));
      CK(cudaStreamWaitEvent(sd, ctx->gev[2 * gi + 1], 0));
      const uint64_t b0 = dreb[m0], b1 = dreb[m1];
      if (b1 > b0 && dst_base)
        CK(cudaMemcpyAsync(dst_base + lo + b0, (uint8_t *)ctx->out_stage.p + b0, (size_t)(b1 - b0), cudaMemcpyDeviceToHost, sd));
      return ZB200_OK;
    };
    rc = uncompress_device_locked(ctx, (const uint8_t *)ctx->in_stage.p, reb.data() + m0, m1 - m0, data_format, 0,
                                  (uint8_t *)ctx->out_stage.p, dreb.data() + m0, dst_lens + m0,
                                  statuses ? statuses + m0 : nullptr, false, &copy_out, crcs ? crcs + m0 : nullptr);
    if (rc) return rc;
  }
  CK(cudaEventRecord(ctx->ev[7], sh));
  CK(cudaEventRecord(ctx->ev[9], sd));
  // the caller's stream ends after the last copy out
  CK(cudaEventRecord(ctx->gev[2 * ng + 1], sd));
  CK(cudaStreamWaitEvent(s, ctx->gev[2 * ng + 1], 0));
  CK(cudaStreamSynchronize(sd));
  CK(cudaStreamSynchronize(sh));
  ctx->timing.h2d_ms = ev_ms(ctx->ev[6], ctx->ev[7]);
  ctx->timing.d2h_ms = ev_ms(ctx->ev[8], ctx->ev[9]);
  ctx->timing.h2d_bytes = shi - slo;
  ctx->timing.d2h_bytes = hi - lo;
  return ZB200_OK;
  });
}

int zb200_uncompress_batch(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n,
                           int data_format, uint8_t *dst_base, const uint64_t *dst_offsets, uint64_t *dst_lens,
                           int *statuses) {
  return uncompress_batch_host(ctx, src_base, src_offsets, n, data_format, dst_base, dst_offsets, dst_lens, statuses,
                               nullptr);
}

int zb200_uncompress_batch_dict(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n,
                                int data_format, const uint8_t *dict, size_t dict_len, uint8_t *dst_base,
                                const uint64_t *dst_offsets, uint64_t *dst_lens, int *statuses) {
  if (dict_len && !dict) return ZB200_ERR_ARG;
  const uint64_t offs[2] = {0, dict_len};
  return uncompress_batch_host(ctx, src_base, src_offsets, n, data_format, dst_base, dst_offsets, dst_lens, statuses,
                               nullptr, dict, offs, 1, nullptr);
}

int zb200_uncompress_batch_dicts(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n,
                                 int data_format, const uint8_t *dict_base, const uint64_t *dict_offsets, size_t k,
                                 const int32_t *dict_of, uint8_t *dst_base, const uint64_t *dst_offsets,
                                 uint64_t *dst_lens, int *statuses) {
  if (n && !dict_of) return ZB200_ERR_ARG;
  return uncompress_batch_host(ctx, src_base, src_offsets, n, data_format, dst_base, dst_offsets, dst_lens, statuses,
                               nullptr, dict_base, dict_offsets, k, dict_of);
}

int zb200_inflate_batch_crc32(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n,
                              uint8_t *dst_base, const uint64_t *dst_offsets, uint64_t *dst_lens, uint32_t *crcs,
                              int *statuses) {
  if (!crcs) return ZB200_ERR_ARG;
  return uncompress_batch_host(ctx, src_base, src_offsets, n, ZB200_DF_DEFLATE, dst_base, dst_offsets, dst_lens,
                               statuses, crcs);
}

int zb200_checksum_batch_device(zb200_ctx *ctx, const uint8_t *d_src, const uint64_t *src_offsets, size_t n, int kind,
                                uint32_t *out) {
  return guarded(ctx, [&]() -> int {
  if (!ctx || !src_offsets || !out || (n && !d_src)) return ZB200_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  DeviceGuard g(ctx->device);
  ctx->timing.kernel_launches = 0;
  return checksum_device_locked(ctx, d_src, src_offsets, n, kind, out);
  });
}

int zb200_checksum_batch(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n, int kind,
                         uint32_t *out) {
  return guarded(ctx, [&]() -> int {
  if (!ctx || !src_offsets || !out || (n && !src_base)) return ZB200_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  DeviceGuard g(ctx->device);
  memset(&ctx->timing, 0, sizeof(ctx->timing));
  std::vector<uint64_t> reb;
  int rc = stage_in(ctx, src_base, src_offsets, n, reb);
  if (rc) return rc;
  return checksum_device_locked(ctx, (const uint8_t *)ctx->in_stage.p, reb.data(), n, kind, out);
  });
}

// ---- one input of unknown size, decoded ONCE ----
// The reference's inflate appends to a string that grows as it goes (inflate.nim:268-291); a fixed-capacity
// ABI would otherwise need a counting pass before the real one.  decode_begin inflates into library-owned
// device memory (capacity from the gzip trailer, else a guess that a counting pass corrects only when it
// was too small) and reports the size; decode_finish copies the bytes to the caller.  Also what gives the
// reference's answer for a gzip member whose ISIZE understates its content: the data is produced, the CRC
// is checked, then the size check fails (gzip.nim:80-88), instead of "destination too small".
// decode_begin with the ctx locked: the member staged in in_stage, its output in out_stage (ctx->pending)
// pre (pre_len bytes, raw members only): the member decoded is pre || src, staged in place (zb200_decode_begin_dict)
static int decode_begin_locked(zb200_ctx *ctx, const uint8_t *src, size_t len, int data_format, size_t pos, size_t *out_len,
                               const uint8_t *pre = nullptr, size_t pre_len = 0) {
    ctx->pending = false;
    ctx->pending_skip = 0;
    uint8_t dummy = 0;
    const uint8_t *sp = src ? src : &dummy;
    uint64_t payload = 0;
    uint32_t kind = 0, expect = 0, isize = 0;
    int st = zb_parse_wrapper(sp, len, data_format, pos, payload, kind, expect, isize);
    if (st != ZB200_OK) return st;
    uint64_t cap = kind == ZB200_DF_GZIP ? std::min<uint64_t>(isize, (uint64_t)len * 1032ull + 1024ull)
                                         : std::min<uint64_t>(std::max<uint64_t>((uint64_t)len * 8ull, 256ull << 10), 1ull << 30);
    std::vector<uint64_t> reb;
    int rc;
    if (pre_len) {
      len += pre_len;
      cap = std::min<uint64_t>(cap + pre_len, (1ull << 30) + pre_len);
      ENSURE(ctx->in_stage, len + 64);
      CK(cudaMemcpyAsync(ctx->in_stage.p, pre, pre_len, cudaMemcpyHostToDevice, ctx->stream));
      if (len > pre_len)
        CK(cudaMemcpyAsync((uint8_t *)ctx->in_stage.p + pre_len, sp, len - pre_len, cudaMemcpyHostToDevice, ctx->stream));
      ctx->timing.h2d_bytes = len;
      reb = {0, (uint64_t)len};
    } else {
      uint64_t so[2] = {0, len};
      rc = stage_in(ctx, sp, so, 1, reb);
      if (rc) return rc;
    }
    for (int attempt = 0; attempt < 2; attempt++) {
      ENSURE(ctx->out_stage, (size_t)cap + 64);
      uint64_t dof[2] = {0, cap}, dl = 0;
      rc = uncompress_device_locked(ctx, (const uint8_t *)ctx->in_stage.p, reb.data(), 1, data_format, pos,
                                    (uint8_t *)ctx->out_stage.p, dof, &dl, &st, false);
      if (rc) return rc;
      if (st != ZB200_ERR_DST_TOO_SMALL || attempt == 1) {
        if (st != ZB200_OK) return st;
        ctx->pending = true;
        ctx->pending_len = dl;
        *out_len = (size_t)dl;
        return ZB200_OK;
      }
      // too small: count the raw stream from the payload start (a gzip ISIZE is a claim, not a fact)
      int cst = ZB200_OK;
      uint64_t real = 0;
      rc = uncompress_device_locked(ctx, (const uint8_t *)ctx->in_stage.p, reb.data(), 1, ZB200_DF_DEFLATE, payload, nullptr,
                                    nullptr, &real, &cst, true);
      if (rc) return rc;
      if (cst != ZB200_OK) return cst;
      cap = real;
    }
    return ZB200_ERR_UNCOMPRESS;
}

int zb200_decode_begin(zb200_ctx *ctx, const uint8_t *src, size_t len, int data_format, size_t pos, size_t *out_len) {
  return guarded(ctx, [&]() -> int {
    if (!ctx || !out_len || (len && !src)) return ZB200_ERR_ARG;
    if (data_format < ZB200_DF_DETECT || data_format > ZB200_DF_DEFLATE) return ZB200_ERR_INVALID_FORMAT;
    std::lock_guard<std::mutex> lk(ctx->mu);
    DeviceGuard g(ctx->device);
    memset(&ctx->timing, 0, sizeof(ctx->timing));
    return decode_begin_locked(ctx, src, len, data_format, pos, out_len);
  });
}

// decode_begin against a dictionary D (ctx locked).  A raw member S, or the payload of a zlib member whose FDICT
// carries D's DICTID, is decoded as the raw member stored(W) || S through decode_begin_locked -- so every
// single-member path (joints, speculative segments, serial) and its verdicts apply -- and the first |W| output bytes
// are skipped.  A zlib member's trailer is then checked against the Adler-32 of the rest.  gzip members and zlib
// members without FDICT ignore the dictionary.
static int decode_begin_dict_locked(zb200_ctx *ctx, const uint8_t *src, size_t len, int data_format, const uint8_t *dict,
                                    size_t dict_len, size_t *out_len) {
  if (!dict_len) return decode_begin_locked(ctx, src, len, data_format, 0, out_len);
  ctx->pending = false;
  uint8_t dummy = 0;
  const uint8_t *sp = src ? src : &dummy;
  const uint32_t id = host_adler32(dict, dict_len);
  uint64_t payload = 0;
  uint32_t kind = 0, expect = 0, isize = 0;
  int st = zb_parse_wrapper(sp, len, data_format, 0, payload, kind, expect, isize, &id);
  if (st != ZB200_OK) return st;
  if (kind == ZB200_DF_GZIP || (kind == ZB200_DF_ZLIB && payload == 2))
    return decode_begin_locked(ctx, src, len, data_format, 0, out_len);
  const size_t wl = std::min<size_t>(dict_len, 32768);
  std::vector<uint8_t> pre(5 + wl);   // stored(W): one non-final stored block, staged in front of the payload
  pre[0] = 0;
  pre[1] = (uint8_t)wl;
  pre[2] = (uint8_t)(wl >> 8);
  pre[3] = (uint8_t)~wl;
  pre[4] = (uint8_t)(~wl >> 8);
  memcpy(pre.data() + 5, dict + (dict_len - wl), wl);
  size_t n = 0;
  st = decode_begin_locked(ctx, sp + payload, len - payload, ZB200_DF_DEFLATE, 0, &n, pre.data(), pre.size());
  if (st != ZB200_OK) return st;
  ctx->pending_skip = wl;
  ctx->pending_len = n - wl;
  if (kind == ZB200_DF_ZLIB) {
    const uint64_t offs[2] = {0, ctx->pending_len};
    uint32_t v = 0;
    int rc = checksum_device_locked(ctx, (const uint8_t *)ctx->out_stage.p + wl, offs, 1, 1, &v);
    if (rc) return rc;
    if (v != expect) {
      ctx->pending = false;
      return ZB200_ERR_CHECKSUM;
    }
  }
  *out_len = (size_t)ctx->pending_len;
  return ZB200_OK;
}

int zb200_decode_begin_dict(zb200_ctx *ctx, const uint8_t *src, size_t len, int data_format, const uint8_t *dict,
                            size_t dict_len, size_t *out_len) {
  return guarded(ctx, [&]() -> int {
    if (!ctx || !out_len || (len && !src) || (dict_len && !dict)) return ZB200_ERR_ARG;
    if (data_format < ZB200_DF_DETECT || data_format > ZB200_DF_DEFLATE) return ZB200_ERR_INVALID_FORMAT;
    std::lock_guard<std::mutex> lk(ctx->mu);
    DeviceGuard g(ctx->device);
    memset(&ctx->timing, 0, sizeof(ctx->timing));
    return decode_begin_dict_locked(ctx, src, len, data_format, dict, dict_len, out_len);
  });
}

int zb200_decode_finish(zb200_ctx *ctx, uint8_t *dst, size_t dst_cap, size_t *dst_len) {
  return guarded(ctx, [&]() -> int {
    if (!ctx || !dst_len) return ZB200_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    DeviceGuard g(ctx->device);
    if (!ctx->pending) return ZB200_ERR_ARG;
    if (ctx->pending_len > dst_cap) return ZB200_ERR_DST_TOO_SMALL;
    if (ctx->pending_len && !dst) return ZB200_ERR_ARG;
    if (ctx->pending_len) {
      CK(cudaMemcpyAsync(dst, (const uint8_t *)ctx->out_stage.p + ctx->pending_skip, (size_t)ctx->pending_len,
                         cudaMemcpyDeviceToHost, ctx->stream));
      CK(cudaStreamSynchronize(ctx->stream));
    }
    *dst_len = (size_t)ctx->pending_len;
    ctx->pending = false;
    return ZB200_OK;
  });
}

// ---- the single-input seam ----
int zb200_deflate(zb200_ctx *ctx, const uint8_t *src, size_t len, int level, uint8_t *dst, size_t dst_cap,
                  size_t *dst_len) {
  if (!dst_len) return ZB200_ERR_ARG;
  uint64_t so[2] = {0, len}, dof[2] = {0, 0};
  int st = 0;
  uint8_t dummy = 0;
  int rc = zb200_compress_batch(ctx, src ? src : &dummy, so, 1, level, ZB200_DF_DEFLATE, nullptr, dst, dst_cap, dof,
                                &st);
  if (rc) return rc;
  *dst_len = (size_t)dof[1];
  return st;
}

static int inflate_one(zb200_ctx *ctx, const uint8_t *src, size_t len, size_t pos, uint8_t *dst, size_t dst_cap,
                       size_t *dst_len, bool count_only) {
  return guarded(ctx, [&]() -> int {
  if (!ctx || !dst_len || (len && !src)) return ZB200_ERR_ARG;
  std::lock_guard<std::mutex> lk(ctx->mu);
  DeviceGuard g(ctx->device);
  memset(&ctx->timing, 0, sizeof(ctx->timing));
  uint64_t so[2] = {0, len};
  std::vector<uint64_t> reb;
  uint8_t dummy = 0;
  int rc = stage_in(ctx, src ? src : &dummy, so, 1, reb);
  if (rc) return rc;
  uint64_t dof[2] = {0, dst_cap}, dl = 0;
  int st = 0;
  if (!count_only) ENSURE(ctx->out_stage, dst_cap + 64);
  rc = uncompress_device_locked(ctx, (const uint8_t *)ctx->in_stage.p, reb.data(), 1, ZB200_DF_DEFLATE, pos,
                                count_only ? nullptr : (uint8_t *)ctx->out_stage.p, dof, &dl, &st, count_only);
  if (rc) return rc;
  if (st) return st;
  if (!count_only && dl) {
    CK(cudaMemcpyAsync(dst, ctx->out_stage.p, (size_t)dl, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  }
  *dst_len = (size_t)dl;
  return ZB200_OK;
  });
}

int zb200_inflate(zb200_ctx *ctx, const uint8_t *src, size_t len, size_t pos, uint8_t *dst, size_t dst_cap,
                  size_t *dst_len) {
  if (dst_cap && !dst) return ZB200_ERR_ARG;
  return inflate_one(ctx, src, len, pos, dst, dst_cap, dst_len, false);
}
int zb200_inflate_size(zb200_ctx *ctx, const uint8_t *src, size_t len, size_t pos, size_t *out_len) {
  return inflate_one(ctx, src, len, pos, nullptr, 0, out_len, true);
}

int zb200_crc32(zb200_ctx *ctx, const void *src, size_t len, uint32_t *out) {
  uint64_t so[2] = {0, len};
  uint8_t dummy = 0;
  return zb200_checksum_batch(ctx, src ? (const uint8_t *)src : &dummy, so, 1, 0, out);
}
int zb200_adler32(zb200_ctx *ctx, const void *src, size_t len, uint32_t *out) {
  uint64_t so[2] = {0, len};
  uint8_t dummy = 0;
  return zb200_checksum_batch(ctx, src ? (const uint8_t *)src : &dummy, so, 1, 1, out);
}

}  // extern "C"

// ---- random access (zb200_index_*) ----
namespace {

void index_edges(const uint8_t *src, uint64_t len, uint8_t *head, uint8_t *tail) {
  const size_t k = (size_t)std::min<uint64_t>(len, 32);
  memset(head, 0, 32);
  memset(tail, 0, 32);
  if (k) {
    memcpy(head, src, k);
    memcpy(tail, src + len - k, k);
  }
}

// gather byte ranges (src offset, dst offset, length) of a device buffer into dst, in pieces of ZB_GATHER_BYTES
int index_gather(zb200_ctx *ctx, const uint8_t *d_src, const std::vector<uint64_t> &ranges, bool wide, void *d_dst) {
  std::vector<ZbGather> g;
  for (size_t i = 0; i + 3 <= ranges.size(); i += 3)
    for (uint64_t r = 0; r < ranges[i + 2]; r += ZB_GATHER_BYTES) {
      ZbGather e;
      e.src = ranges[i] + r;
      e.dst = ranges[i + 1] + r;
      e.n = (uint32_t)std::min<uint64_t>(ZB_GATHER_BYTES, ranges[i + 2] - r);
      e.wide = wide ? 1u : 0u;
      g.push_back(e);
    }
  if (g.empty()) return ZB200_OK;
  ENSURE(ctx->idx_desc, g.size() * sizeof(ZbGather));
  CK(cudaMemcpyAsync(ctx->idx_desc.p, g.data(), g.size() * sizeof(ZbGather), cudaMemcpyHostToDevice, ctx->stream));
  CK(zb_launch_gather(d_src, (const ZbGather *)ctx->idx_desc.p, (uint32_t)g.size(), d_dst, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));   // `g` goes out of scope
  ctx->timing.kernel_launches += 1;
  ctx->timing.h2d_bytes += g.size() * sizeof(ZbGather);
  return ZB200_OK;
}

int index_build_locked(zb200_ctx *ctx, const uint8_t *src, size_t len, int data_format, uint64_t span, zb200_index **out) {
  cudaStream_t s = ctx->stream;
  uint64_t size = 0;
  {
    size_t n = 0;
    const int st = decode_begin_locked(ctx, src, len, data_format, 0, &n);
    ctx->pending = false;
    if (st) return st;
    size = n;
  }
  uint64_t payload = 0;
  uint32_t kind = 0, expect = 0, isize = 0;
  if (zb_parse_wrapper(src, len, data_format, 0, payload, kind, expect, isize) != ZB200_OK) return ZB200_ERR_UNCOMPRESS;
  const uint64_t trailer = kind == ZB200_DF_GZIP ? 8 : kind == ZB200_DF_ZLIB ? 4 : 0;
  // 1. block starts: closed segments at the boundaries the decompress streams use, else one serial segment
  std::vector<uint64_t> bits;
  const char *path = "serial";
  int rc = find_segment_bits(ctx, (const uint8_t *)ctx->in_stage.p, payload * 8ull, len - trailer, bits, path);
  if (rc) return rc;
  const uint32_t nrec = (uint32_t)(size / 32768ull + 1ull);
  ENSURE(ctx->idx_out, (size_t)nrec * 16);
  uint64_t *d_rec = (uint64_t *)ctx->idx_out.p;
  std::vector<uint64_t> sl, base;
  std::vector<int> sst;
  std::vector<uint32_t> sk;
  auto regular = [&]() {
    uint64_t t = 0;
    for (size_t i = 0; i < bits.size(); i++) {
      // (several segments: each one's output must fit the marker decode's 32-bit positions; one serial segment
      // has the limit uncompress has)
      if (sst[i] != ZB200_OK || (sk[i] != 0) != (i + 1 == bits.size()) || (bits.size() > 1 && sl[i] > 0xf0000000ull))
        return false;
      t += sl[i];
    }
    return t == size;
  };
  // counting passes over the segments bits[i] .. bits[i + 1] (the last one to the member's end) staged in in_stage
  ZbInflateWork w;
  memset(&w, 0, sizeof(w));
  w.src = (const uint8_t *)ctx->in_stage.p;
  w.seg_limit = len;
  w.count_only = 1;
  for (;;) {
    const size_t S = bits.size();
    base.assign(S + 1, 0);
    rc = seg_bounds_upload(ctx, bits.data(), S, len * 8ull, w);
    if (rc) return rc;
    if (S > 1) {   // the sizes first: every segment's output offset
      rc = seg_pass(ctx, w, S, sl, sst, sk);
      if (rc) return rc;
      ctx->timing.kernel_launches += 1;
      if (!regular()) {
        bits.resize(1);
        continue;
      }
      for (size_t i = 0; i < S; i++) base[i + 1] = base[i] + sl[i];
    } else {
      base[1] = size;
    }
    // then the recorder, with every segment's output offset in the member as rec_base
    ENSURE(ctx->seg_dst, (S + 1) * 8);
    CK(cudaMemcpyAsync(ctx->seg_dst.p, base.data(), (S + 1) * 8, cudaMemcpyHostToDevice, s));
    CK(cudaMemsetAsync(d_rec, 0xff, (size_t)nrec * 16, s));
    ZbInflateWork r = w;
    r.rec = d_rec;
    r.rec_base = (const uint64_t *)ctx->seg_dst.p;
    r.nrec = nrec;
    rc = seg_pass(ctx, r, S, sl, sst, sk);
    if (rc) return rc;
    ctx->timing.kernel_launches += 1;
    if (regular()) break;
    if (S == 1) return ZB200_ERR_UNCOMPRESS;   // a member uncompress accepts counts the same
    bits.resize(1);
  }
  std::vector<uint64_t> rec((size_t)nrec * 2);
  CK(cudaMemcpyAsync(rec.data(), d_rec, (size_t)nrec * 16, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  std::unique_ptr<zb200_index> idx(new zb200_index());
  idx->span = span;
  uint64_t next = 0;
  for (uint32_t k = 0; k < nrec; k++) {
    uint64_t b = rec[2 * k], o = rec[2 * k + 1];
    if (b == ~0ull) {   // no block start of its segment reaches the multiple: the next segment's start
      size_t j = 1;
      while (j < bits.size() && base[j] < (uint64_t)k * 32768ull) j++;
      if (j >= bits.size()) continue;
      b = bits[j];
      o = base[j];
    }
    if (index_add_point(idx.get(), b, o, next) < 0) return ZB200_ERR_UNCOMPRESS;
  }
  const size_t np = idx->bit.size();
  if (np == 0 || idx->out[0] != 0) return ZB200_ERR_UNCOMPRESS;
  // 2. windows and interval CRCs, from the decoded output in out_stage
  std::vector<uint64_t> ranges;
  for (size_t p = 0; p < np; p++)
    if (idx->win_at[p] != ~0ull) {
      ranges.push_back(idx->out[p] - 32768ull);
      ranges.push_back(idx->win_at[p]);
      ranges.push_back(32768ull);
    }
  const uint64_t wbytes = idx->windows.size();
  idx->crc.assign(np, 0);
  std::vector<uint64_t> offs(idx->out);
  offs.push_back(size);
  rc = checksum_device_locked(ctx, (const uint8_t *)ctx->out_stage.p, offs.data(), np, 0, idx->crc.data());
  if (rc) return rc;
  if (wbytes) {
    ENSURE(ctx->idx_out, wbytes);
    rc = index_gather(ctx, (const uint8_t *)ctx->out_stage.p, ranges, false, ctx->idx_out.p);
    if (rc) return rc;
    CK(cudaMemcpyAsync(idx->windows.data(), ctx->idx_out.p, wbytes, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    ctx->timing.d2h_bytes += wbytes;
  }
  idx->fmt = (int)kind;
  idx->payload = payload;
  idx->len = len;
  idx->size = size;
  index_edges(src, len, idx->head, idx->tail);
  *out = idx.release();
  return ZB200_OK;
}

// A chain decodes the segment intervals [p0, p1) of an index, starting at window point p0 (its window in front).
struct IndexChain {
  size_t p0, p1;
};

// One launch group of an extraction: the chains [c0, c1), then the pieces that they serve.  `piece` holds, per
// piece: chain, output offset, length, destination (host pointer).  chain_st receives each chain's status.
int index_extract_group(zb200_ctx *ctx, const zb200_index *idx, const uint8_t *src, const std::vector<IndexChain> &ch,
                        size_t c0, size_t c1, std::vector<int> &chain_st) {
  cudaStream_t s = ctx->stream;
  const size_t np = idx->bit.size();
  const uint64_t end_bit = idx->len * 8ull;
  // 1. the host staging: every chain's window, then its compressed slice
  std::vector<uint8_t> stage;
  std::vector<uint64_t> sb, dof, wranges;
  std::vector<ZbMarkSegHost> segs;
  std::vector<size_t> seg_chain, seg_point;   // per inflate segment: its chain and point
  std::vector<size_t> rseg_of_point;          // per inflate segment: its index in `segs`
  uint64_t se = 0, de = 0;
  uint32_t max_n = 0;
  for (size_t c = c0; c < c1; c++) {
    const IndexChain &k = ch[c];
    if (k.p0 > 0) {
      const uint64_t at = stage.size();
      stage.insert(stage.end(), idx->windows.begin() + (ptrdiff_t)idx->win_at[k.p0],
                   idx->windows.begin() + (ptrdiff_t)idx->win_at[k.p0] + 32768);
      se += 32768ull;
      ZbMarkSegHost m = {se, de, 32768u, 0u};
      segs.push_back(m);
      wranges.push_back(at);
      wranges.push_back(se);
      wranges.push_back(32768ull);
      se += 32768ull;
      de += 32768ull;
      max_n = std::max<uint32_t>(max_n, 32768u);
    }
    const uint64_t b0 = idx->bit[k.p0] / 8ull;
    const uint64_t b1 = k.p1 < np ? (idx->bit[k.p1] + 7ull) / 8ull : idx->len;
    const uint64_t at = stage.size();
    stage.insert(stage.end(), src + b0, src + b1);
    for (size_t p = k.p0; p < k.p1; p++) {
      const uint64_t n = (p + 1 < np ? idx->out[p + 1] : idx->size) - idx->out[p];
      const uint64_t eb = p + 1 < np ? idx->bit[p + 1] : end_bit;
      // the segment, then an empty one that starts where it must end: it owns the gap up to the next segment, so
      // every segment's capacity is exactly its interval and a corrupt one cannot write into its neighbours
      sb.push_back(at * 8ull + idx->bit[p] - b0 * 8ull);
      sb.push_back(at * 8ull + eb - b0 * 8ull);
      sb.push_back(at * 8ull + eb - b0 * 8ull);
      sb.push_back(at * 8ull + eb - b0 * 8ull);
      se += 32768ull;
      dof.push_back(se);
      dof.push_back(se + n);
      rseg_of_point.push_back(segs.size());
      ZbMarkSegHost m = {se, de, (uint32_t)n, 0u};
      segs.push_back(m);
      seg_chain.push_back(c);
      seg_point.push_back(p);
      se += n;
      de += n;
      max_n = std::max<uint32_t>(max_n, (uint32_t)n);
    }
  }
  dof.push_back(se);
  const size_t T = seg_chain.size(), R = segs.size();
  ENSURE(ctx->in_stage, stage.size() + 64);
  int rc = h2d_copy(ctx, (uint8_t *)ctx->in_stage.p, stage.data(), stage.size(), s, true);
  if (rc) return rc;
  ctx->timing.h2d_bytes += stage.size();
  const size_t T2 = 2 * T;   // every segment is followed by its empty gap segment
  ENSURE(ctx->out_stage, (size_t)de + 64);
  ZbInflateWork w;
  memset(&w, 0, sizeof(w));
  w.src = (const uint8_t *)ctx->in_stage.p;
  w.seg_limit = stage.size();
  w.seg_win0 = ch[c0].p0 > 0;   // a chain from point 0 has no window: a distance before the member start is an error
  rc = seg_bits_upload(ctx, sb, w);
  if (rc) return rc;
  // 2. markers, then the windows as byte symbols, then one marker decode of every segment of every chain
  rc = mark_upload(ctx, segs, dof);
  if (rc) return rc;
  ctx->timing.h2d_bytes += R * sizeof(ZbMarkSegHost) + T2 * 24 + 8;
  ctx->timing.kernel_launches += 1;
  rc = index_gather(ctx, (const uint8_t *)ctx->in_stage.p, wranges, true, ctx->mark_scratch.p);
  if (rc) return rc;
  w.dst = (uint8_t *)ctx->mark_scratch.p;
  w.mark = 1;
  std::vector<uint64_t> sl;
  std::vector<int> sst;
  std::vector<uint32_t> sk;
  rc = seg_pass(ctx, w, T2, sl, sst, sk);
  if (rc) return rc;
  ctx->timing.kernel_launches += 1;
  for (size_t c = c0; c < c1; c++) chain_st[c] = ZB200_OK;
  bool any_failed = false;
  for (size_t t = 0; t < T; t++) {
    const size_t c = seg_chain[t], p = seg_point[t];
    const bool last = p + 1 == np;
    if (sst[2 * t] != ZB200_OK || sl[2 * t] != segs[rseg_of_point[t]].n || (sk[2 * t] != 0) != last) {
      // a failed segment's symbols are not all written: resolve none of them (its chain has failed, and the next
      // chain starts from its own window, so nothing else reads them)
      chain_st[c] = ZB200_ERR_UNCOMPRESS;
      segs[rseg_of_point[t]].n = 0;
      any_failed = true;
    }
  }
  if (any_failed)
    CK(cudaMemcpyAsync(ctx->mark_segs.p, segs.data(), R * sizeof(ZbMarkSegHost), cudaMemcpyHostToDevice, s));
  // 3. one resolve over [window, chain segments, window, chain segments, ...]: the windows hold no markers, so
  // every chain resolves against its own window.  Only the first chain of a group can reach before the member
  // start, and only the chain from point 0 starts a group without a window; it decodes without one, so a marker
  // before the start (`bad`) cannot be produced by a segment that decoded.
  CK(cudaMemsetAsync(&counters(ctx)->bad, 0, 4, s));
  int bad = 0;
  rc = resolve_window(ctx, R, max_n, 0, 0, (uint8_t *)ctx->out_stage.p, &bad);
  if (rc) return rc;
  ctx->timing.kernel_launches += 4;
  // 4. every decoded interval against its CRC-32
  std::vector<uint64_t> coff(R + 1);
  for (size_t r = 0; r < R; r++) coff[r] = segs[r].dst;
  coff[R] = de;
  std::vector<uint32_t> crc(R);
  rc = checksum_device_locked(ctx, (const uint8_t *)ctx->out_stage.p, coff.data(), R, 0, crc.data());
  if (rc) return rc;
  if (bad) chain_st[c0] = ZB200_ERR_UNCOMPRESS;
  for (size_t t = 0; t < T; t++) {
    const size_t c = seg_chain[t], p = seg_point[t];
    if (chain_st[c] == ZB200_OK && crc[rseg_of_point[t]] != idx->crc[p]) chain_st[c] = ZB200_ERR_CHECKSUM;
  }
  if (ctx->index_log)
    fprintf(stderr, "zb200 index: group of %zu chains, %zu segments, %zu bytes uploaded\n", c1 - c0, T, stage.size());
  return ZB200_OK;
}

int index_extract_locked(zb200_ctx *ctx, const zb200_index *idx, const uint8_t *src, size_t len, const uint64_t *offsets,
                         const uint64_t *lens, size_t n, uint8_t *dst, const uint64_t *dst_offsets, int *statuses) {
  cudaStream_t s = ctx->stream;
  uint8_t head[32], tail[32];
  index_edges(src, len, head, tail);
  if (len != idx->len || memcmp(head, idx->head, 32) || memcmp(tail, idx->tail, 32)) return ZB200_ERR_ARG;
  for (size_t i = 0; i < n; i++) {
    if (offsets[i] > idx->size || lens[i] > idx->size - offsets[i]) return ZB200_ERR_ARG;
    if (dst_offsets[i + 1] < dst_offsets[i] || dst_offsets[i + 1] - dst_offsets[i] < lens[i]) return ZB200_ERR_ARG;
  }
  const size_t np = idx->bit.size();
  std::vector<size_t> wpts;   // window point indices
  for (size_t p = 0; p < np; p++)
    if (idx->win[p]) wpts.push_back(p);
  // every range cut at window points: piece (range, window point slot, start, end)
  struct Piece {
    size_t range, slot;
    uint64_t a, b;
  };
  std::vector<Piece> pieces;
  std::vector<size_t> reach(wpts.size(), 0);   // per window point: the chain's end point (exclusive), 0 = unused
  for (size_t i = 0; i < n; i++) {
    statuses[i] = ZB200_OK;
    uint64_t a = offsets[i];
    const uint64_t e = offsets[i] + lens[i];
    while (a < e) {
      // the last window point at or before a
      size_t j = (size_t)(std::upper_bound(wpts.begin(), wpts.end(), a, [&](uint64_t v, size_t p) { return v < idx->out[p]; }) -
                          wpts.begin()) - 1;
      const uint64_t b = j + 1 < wpts.size() ? std::min<uint64_t>(e, idx->out[wpts[j + 1]]) : e;
      // the first segment point at or past b, or the member's end
      const size_t p1 = (size_t)(std::lower_bound(idx->out.begin(), idx->out.end(), b) - idx->out.begin());
      reach[j] = std::max(reach[j], std::max(p1, wpts[j] + 1));
      pieces.push_back(Piece{i, j, a, b});
      a = b;
    }
  }
  std::vector<IndexChain> ch;
  std::vector<size_t> chain_of(wpts.size(), 0);
  for (size_t j = 0; j < wpts.size(); j++)
    if (reach[j]) {
      chain_of[j] = ch.size();
      ch.push_back(IndexChain{wpts[j], std::min(reach[j], np)});
    }
  std::vector<int> chain_st(ch.size(), ZB200_OK);
  std::vector<uint64_t> chain_dst(ch.size(), 0);   // output offset in out_stage of the chain's first interval
  // launch groups of chains under the output budget; a chain larger than it has a group of its own
  std::vector<uint8_t> host;
  for (size_t c0 = 0; c0 < ch.size();) {
    size_t c1 = c0;
    uint64_t bytes = 0;
    while (c1 < ch.size()) {
      const uint64_t o0 = idx->out[ch[c1].p0], o1 = ch[c1].p1 < np ? idx->out[ch[c1].p1] : idx->size;
      const uint64_t cb = (o1 - o0) + (ch[c1].p0 > 0 ? 32768ull : 0ull);
      if (c1 > c0 && bytes + cb > ctx->index_group_bytes) break;
      bytes += cb;
      chain_dst[c1] = bytes - (o1 - o0);
      c1++;
    }
    int rc = index_extract_group(ctx, idx, src, ch, c0, c1, chain_st);
    if (rc) return rc;
    // 5. the pieces this group serves, gathered into one packed buffer, one copy out
    std::vector<uint64_t> ranges;
    std::vector<size_t> which;
    uint64_t packed = 0;
    for (size_t k = 0; k < pieces.size(); k++) {
      const size_t c = chain_of[pieces[k].slot];
      if (c < c0 || c >= c1 || chain_st[c] != ZB200_OK) continue;
      ranges.push_back(chain_dst[c] + (pieces[k].a - idx->out[ch[c].p0]));
      ranges.push_back(packed);
      ranges.push_back(pieces[k].b - pieces[k].a);
      which.push_back(k);
      packed += pieces[k].b - pieces[k].a;
    }
    if (packed) {
      ENSURE(ctx->idx_out, packed);
      rc = index_gather(ctx, (const uint8_t *)ctx->out_stage.p, ranges, false, ctx->idx_out.p);
      if (rc) return rc;
      host.resize(packed);
      CK(cudaMemcpyAsync(host.data(), ctx->idx_out.p, packed, cudaMemcpyDeviceToHost, s));
      CK(cudaStreamSynchronize(s));
      ctx->timing.d2h_bytes += packed;
      uint64_t at = 0;
      for (size_t k : which) {
        const Piece &pc = pieces[k];
        memcpy(dst + dst_offsets[pc.range] + (pc.a - offsets[pc.range]), host.data() + at, pc.b - pc.a);
        at += pc.b - pc.a;
      }
    }
    c0 = c1;
  }
  // per range: the worst of its chains (a decode failure before a CRC mismatch)
  for (const Piece &pc : pieces) {
    const int cs = chain_st[chain_of[pc.slot]];
    int &st = statuses[pc.range];
    if (cs == ZB200_ERR_UNCOMPRESS || (cs != ZB200_OK && st == ZB200_OK)) st = cs;
  }
  return ZB200_OK;
}

// zb200_compress_batch_index (h_src / h_dst: d_src is in_stage, rebased to src_offsets[0]) and
// zb200_compress_batch_device_index (device buffers): the call without an index, with k_index_rec's records, then
// one index per member.  Windows are copied from the input, head and tail from the output.
int compress_index_locked(zb200_ctx *ctx, const uint8_t *d_src, const uint8_t *h_src, const uint64_t *src_offsets,
                          size_t n, int level, int data_format, const uint8_t *fname_lens, uint8_t *d_dst,
                          size_t dst_cap, uint8_t *h_dst, size_t h_dst_cap, uint64_t *dst_offsets, int *statuses,
                          size_t max_group_chunks, uint64_t span, zb200_index **indexes) {
  std::vector<uint64_t> rec_first(n + 1, 0);
  for (size_t i = 0; i < n; i++) {
    if (src_offsets[i + 1] < src_offsets[i]) return ZB200_ERR_ARG;
    rec_first[i + 1] = rec_first[i] + (src_offsets[i + 1] - src_offsets[i]) / 32768ull + 1ull;
  }
  const size_t nrec = (size_t)rec_first[n];
  ZbIndexWork x;
  int rc = index_rec_prepare(ctx, rec_first, nrec, x);
  if (rc) return rc;
  rc = compress_locked(ctx, d_src, h_src, src_offsets, n, level, data_format, fname_lens, d_dst, dst_cap, h_dst,
                       h_dst_cap, dst_offsets, statuses, max_group_chunks, nullptr, &x);
  if (rc) return rc;
  std::vector<uint64_t> rec;
  std::vector<uint32_t> crc;
  uint64_t lout[2];
  rc = index_rec_fetch(ctx, nrec, rec, crc, lout);
  if (rc) return rc;
  std::vector<std::unique_ptr<zb200_index>> out(n);
  std::vector<uint64_t> wranges, eranges;   // device buffers: (source offset, destination offset, length) to gather
  std::vector<uint64_t> wfirst(n + 1, 0);
  for (size_t m = 0; m < n; m++) {
    std::unique_ptr<zb200_index> idx(new zb200_index());
    idx->fmt = data_format;
    idx->payload = frame_head(data_format, fname_lens && data_format == ZB200_DF_GZIP ? fname_lens[m] : 0);
    idx->len = dst_offsets[m + 1] - dst_offsets[m];
    idx->size = src_offsets[m + 1] - src_offsets[m];
    idx->span = span;
    // every window point but the first at output 0 takes 32 KiB: reserve them at once rather than grow the vector
    idx->windows.reserve((size_t)std::min<uint64_t>(idx->size / span, rec_first[m + 1] - rec_first[m]) * 32768);
    uint64_t next = 0;
    for (uint64_t r = rec_first[m]; r < rec_first[m + 1]; r++) {
      if (rec[2 * r] == ~0ull) continue;   // past the member's last block start
      const int a = index_add_point(idx.get(), rec[2 * r], rec[2 * r + 1], next);
      if (a < 0) {
        ctx->last_err = "compress-time index: records out of order";
        return ZB200_ERR_CUDA;
      }
      if (a) idx->crc.push_back(crc[r]);
    }
    for (size_t p = 0; p < idx->bit.size(); p++) {
      if (idx->win_at[p] == ~0ull) continue;
      const uint64_t from = src_offsets[m] + idx->out[p] - 32768ull;
      if (h_src) {
        memcpy(idx->windows.data() + idx->win_at[p], h_src + from, 32768);
      } else {
        wranges.push_back(from);
        wranges.push_back(wfirst[m] + idx->win_at[p]);
        wranges.push_back(32768ull);
      }
    }
    wfirst[m + 1] = wfirst[m] + (h_src ? 0 : idx->windows.size());
    if (h_dst) {
      index_edges(h_dst + dst_offsets[m], idx->len, idx->head, idx->tail);
    } else {
      const uint64_t k = std::min<uint64_t>(idx->len, 32);
      eranges.insert(eranges.end(), {dst_offsets[m], 64ull * m, k, dst_offsets[m] + idx->len - k, 64ull * m + 32, k});
    }
    out[m] = std::move(idx);
  }
  cudaStream_t s = ctx->stream;
  if (wfirst[n]) {
    ENSURE(ctx->idx_out, (size_t)wfirst[n]);
    rc = index_gather(ctx, d_src, wranges, false, ctx->idx_out.p);
    if (rc) return rc;
    for (size_t m = 0; m < n; m++)   // straight into each index: the windows are most of its bytes
      if (!out[m]->windows.empty())
        CK(cudaMemcpyAsync(out[m]->windows.data(), (const uint8_t *)ctx->idx_out.p + wfirst[m], out[m]->windows.size(),
                           cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
  }
  if (!h_dst && n) {
    ENSURE(ctx->idx_out, 64 * n);
    CK(cudaMemsetAsync(ctx->idx_out.p, 0, 64 * n, s));
    rc = index_gather(ctx, d_dst, eranges, false, ctx->idx_out.p);
    if (rc) return rc;
    std::vector<uint8_t> eb(64 * n);
    CK(cudaMemcpyAsync(eb.data(), ctx->idx_out.p, eb.size(), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    for (size_t m = 0; m < n; m++) {
      memcpy(out[m]->head, eb.data() + 64 * m, 32);
      memcpy(out[m]->tail, eb.data() + 64 * m + 32, 32);
    }
  }
  for (size_t m = 0; m < n; m++) indexes[m] = out[m].release();
  return ZB200_OK;
}

// a compress-time index's span: the build's rule
bool index_span_ok(uint64_t span) { return span >= 32768 && span % 32768 == 0; }

}  // namespace

extern "C" {

int zb200_compress_batch_index(zb200_ctx *ctx, const uint8_t *src_base, const uint64_t *src_offsets, size_t n, int level,
                               int data_format, const uint8_t *fname_lens, uint8_t *dst_base, size_t dst_cap,
                               uint64_t *dst_offsets, int *statuses, uint64_t span, zb200_index **indexes) {
  return guarded(ctx, [&]() -> int {
    if (!ctx || !src_offsets || !dst_offsets || !indexes || (n && (!src_base || !dst_base))) return ZB200_ERR_ARG;
    for (size_t i = 0; i < n; i++) indexes[i] = nullptr;
    if (level < -2 || level > 9) return ZB200_ERR_INVALID_LEVEL;
    if (data_format != ZB200_DF_GZIP && data_format != ZB200_DF_ZLIB && data_format != ZB200_DF_DEFLATE)
      return ZB200_ERR_INVALID_FORMAT;
    if (!index_span_ok(span)) return ZB200_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    DeviceGuard g(ctx->device);
    memset(&ctx->timing, 0, sizeof(ctx->timing));
    if (n == 0) {
      dst_offsets[0] = 0;
      return ZB200_OK;
    }
    for (size_t i = 0; i < n; i++)
      if (src_offsets[i + 1] < src_offsets[i]) return ZB200_ERR_ARG;
    const uint64_t in_bytes = src_offsets[n] - src_offsets[0];
    uint64_t bound = 0;
    for (size_t i = 0; i < n; i++)
      bound += zb200_compress_bound((size_t)(src_offsets[i + 1] - src_offsets[i]), data_format) + 64;
    ENSURE(ctx->in_stage, (size_t)in_bytes + 64);
    ENSURE(ctx->out_stage, (size_t)bound + 64);
    return compress_index_locked(ctx, (const uint8_t *)ctx->in_stage.p, src_base, src_offsets, n, level, data_format,
                                 fname_lens, (uint8_t *)ctx->out_stage.p, ctx->out_stage.cap & ~(size_t)3, dst_base,
                                 dst_cap, dst_offsets, statuses, ctx->host_group_chunks, span, indexes);
  });
}

int zb200_compress_batch_device_index(zb200_ctx *ctx, const uint8_t *d_src, const uint64_t *src_offsets, size_t n,
                                      int level, int data_format, const uint8_t *fname_lens, uint8_t *d_dst,
                                      size_t dst_cap, uint64_t *dst_offsets, int *statuses, uint64_t span,
                                      zb200_index **indexes) {
  return guarded(ctx, [&]() -> int {
    if (!ctx || !src_offsets || !dst_offsets || !indexes || (n && (!d_src || !d_dst))) return ZB200_ERR_ARG;
    for (size_t i = 0; i < n; i++) indexes[i] = nullptr;
    if (level < -2 || level > 9) return ZB200_ERR_INVALID_LEVEL;
    if (data_format != ZB200_DF_GZIP && data_format != ZB200_DF_ZLIB && data_format != ZB200_DF_DEFLATE)
      return ZB200_ERR_INVALID_FORMAT;
    if (!index_span_ok(span)) return ZB200_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    DeviceGuard g(ctx->device);
    ctx->timing.kernel_launches = 0;
    if (n == 0) {
      dst_offsets[0] = 0;
      return ZB200_OK;
    }
    return compress_index_locked(ctx, d_src, nullptr, src_offsets, n, level, data_format, fname_lens, d_dst, dst_cap,
                                 nullptr, 0, dst_offsets, statuses, ctx->dev_group_chunks, span, indexes);
  });
}

int zb200_compress_stream_begin_index(zb200_ctx *ctx, int level, int data_format, int fname_len, uint64_t span,
                                      zb200_compress_stream **out) {
  if (ctx && out && level >= -2 && level <= 9 &&
      (data_format == ZB200_DF_GZIP || data_format == ZB200_DF_ZLIB || data_format == ZB200_DF_DEFLATE) &&
      !index_span_ok(span)) {
    *out = nullptr;
    return ZB200_ERR_ARG;
  }
  const int rc = zb200_compress_stream_begin(ctx, level, data_format, fname_len, out);
  if (rc) return rc;
  zb200_compress_stream *st = *out;
  st->ix.reset(new zb200_index());
  st->ix->fmt = data_format;
  st->ix->payload = frame_head(data_format, st->fname_len);
  st->ix->span = span;
  return ZB200_OK;
}

int zb200_compress_stream_index(zb200_compress_stream *st, zb200_index **out) {
  if (!st || !out) return ZB200_ERR_ARG;
  *out = nullptr;
  if (!st->ix || !st->finished) return ZB200_ERR_ARG;
  *out = new zb200_index(*st->ix);
  return ZB200_OK;
}

int zb200_index_build(zb200_ctx *ctx, const uint8_t *src, size_t len, int data_format, uint64_t span, zb200_index **out) {
  return guarded(ctx, [&]() -> int {
    if (!ctx || !out || (len && !src)) return ZB200_ERR_ARG;
    *out = nullptr;
    if (data_format < ZB200_DF_DETECT || data_format > ZB200_DF_DEFLATE) return ZB200_ERR_INVALID_FORMAT;
    if (span < 32768 || span % 32768) return ZB200_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    DeviceGuard g(ctx->device);
    memset(&ctx->timing, 0, sizeof(ctx->timing));
    uint8_t dummy = 0;
    return index_build_locked(ctx, src ? src : &dummy, len, data_format, span, out);
  });
}

int zb200_index_extract_batch(zb200_ctx *ctx, const zb200_index *idx, const uint8_t *src, size_t len,
                              const uint64_t *offsets, const uint64_t *lens, size_t n, uint8_t *dst,
                              const uint64_t *dst_offsets, int *statuses) {
  return guarded(ctx, [&]() -> int {
    if (!ctx || !idx || (len && !src) || (n && (!offsets || !lens || !dst_offsets || !statuses))) return ZB200_ERR_ARG;
    if (n && dst_offsets[n] > dst_offsets[0] && !dst) return ZB200_ERR_ARG;
    std::lock_guard<std::mutex> lk(ctx->mu);
    DeviceGuard g(ctx->device);
    memset(&ctx->timing, 0, sizeof(ctx->timing));
    uint8_t dummy = 0;
    return index_extract_locked(ctx, idx, src ? src : &dummy, len, offsets, lens, n, dst, dst_offsets, statuses);
  });
}

void zb200_index_free(zb200_index *idx) { delete idx; }

uint64_t zb200_index_size(const zb200_index *idx) { return idx ? idx->size : 0; }

size_t zb200_index_points(const zb200_index *idx, uint64_t *bits, uint64_t *outs, uint32_t *crcs, uint8_t *window,
                          size_t cap) {
  if (!idx) return 0;
  const size_t np = idx->bit.size();
  for (size_t p = 0; p < np && p < cap; p++) {
    if (bits) bits[p] = idx->bit[p];
    if (outs) outs[p] = idx->out[p];
    if (crcs) crcs[p] = idx->crc[p];
    if (window) window[p] = idx->win[p];
  }
  return np;
}

// ---- index serialisation (format: include/zippy_b200.h) ----
static const uint8_t kIndexMagic[8] = {'Z', 'B', '2', '0', '0', 'I', 'D', 'X'};
static constexpr uint32_t kIndexVersion = 1;
static constexpr size_t kIndexHeader = 8 + 4 + 4 + 8 * 5 + 32 + 32 + 8 + 8;   // through the two counts
static constexpr size_t kIndexPoint = 8 + 8 + 4 + 4;

static uint32_t host_crc32(const uint8_t *p, size_t n) {
  static uint32_t tab[256];
  static std::once_flag once;
  std::call_once(once, [] {
    for (uint32_t i = 0; i < 256; i++) {
      uint32_t c = i;
      for (int k = 0; k < 8; k++) c = (c >> 1) ^ ((0u - (c & 1u)) & 0xedb88320u);
      tab[i] = c;
    }
  });
  uint32_t c = 0xffffffffu;
  for (size_t i = 0; i < n; i++) c = tab[(c ^ p[i]) & 255u] ^ (c >> 8);
  return ~c;
}
static void put_le(std::vector<uint8_t> &b, uint64_t v, int n) {
  for (int i = 0; i < n; i++) b.push_back((uint8_t)(v >> (8 * i)));
}
static uint64_t get_le(const uint8_t *p, int n) {
  uint64_t v = 0;
  for (int i = 0; i < n; i++) v |= (uint64_t)p[i] << (8 * i);
  return v;
}

int zb200_index_export(zb200_ctx *ctx, const zb200_index *idx, uint8_t *dst, size_t cap, size_t *len) {
  if (!ctx || !idx || !len) return ZB200_ERR_ARG;
  const size_t np = idx->bit.size(), nw = idx->windows.size() / 32768;
  // the windows as raw DEFLATE at level 1, one compress_batch
  std::vector<uint64_t> so(nw + 1), doff(nw + 1, 0);
  for (size_t i = 0; i <= nw; i++) so[i] = 32768ull * i;
  std::vector<uint8_t> comp(nw * (zb200_compress_bound(32768, ZB200_DF_DEFLATE) + 64) + 64);
  std::vector<int> cst(nw + 1, 0);
  if (nw) {
    const int rc = zb200_compress_batch(ctx, idx->windows.data(), so.data(), nw, 1, ZB200_DF_DEFLATE, nullptr, comp.data(),
                                        comp.size(), doff.data(), cst.data());
    if (rc) return rc;
    for (size_t i = 0; i < nw; i++)
      if (cst[i]) return cst[i];
  }
  return guarded(ctx, [&]() -> int {
    std::vector<uint8_t> b;
    b.insert(b.end(), kIndexMagic, kIndexMagic + 8);
    put_le(b, kIndexVersion, 4);
    put_le(b, (uint64_t)idx->fmt, 4);
    put_le(b, idx->payload, 8);
    put_le(b, idx->len, 8);
    put_le(b, idx->size, 8);
    put_le(b, idx->span, 8);
    put_le(b, 0, 8);
    b.insert(b.end(), idx->head, idx->head + 32);
    b.insert(b.end(), idx->tail, idx->tail + 32);
    put_le(b, np, 8);
    put_le(b, nw, 8);
    for (size_t p = 0; p < np; p++) {
      put_le(b, idx->bit[p], 8);
      put_le(b, idx->out[p], 8);
      put_le(b, idx->crc[p], 4);
      put_le(b, idx->win[p], 4);
    }
    for (size_t i = 0; i < nw; i++) put_le(b, doff[i + 1] - doff[i], 8);
    b.insert(b.end(), comp.begin(), comp.begin() + (ptrdiff_t)doff[nw]);
    put_le(b, host_crc32(b.data(), b.size()), 4);
    *len = b.size();
    if (!dst) return ZB200_OK;
    if (cap < b.size()) return ZB200_ERR_DST_TOO_SMALL;
    memcpy(dst, b.data(), b.size());
    return ZB200_OK;
  });
}

static int index_import(zb200_ctx *ctx, const uint8_t *src, size_t len, zb200_index **out) {
  std::unique_ptr<zb200_index> idx(new zb200_index());
  std::vector<uint64_t> clen;
  size_t pos = 0;
  // everything but the windows' contents, checked on the host
  {
    if (len < kIndexHeader + 4 || memcmp(src, kIndexMagic, 8) || get_le(src + 8, 4) != kIndexVersion) return ZB200_ERR_ARG;
    if (host_crc32(src, len - 4) != (uint32_t)get_le(src + len - 4, 4)) return ZB200_ERR_ARG;
    const uint8_t *h = src + 12;
    const uint64_t fmt = get_le(h, 4);
    idx->payload = get_le(h + 4, 8);
    idx->len = get_le(h + 12, 8);
    idx->size = get_le(h + 20, 8);
    idx->span = get_le(h + 28, 8);
    const uint64_t reserved = get_le(h + 36, 8);
    memcpy(idx->head, h + 44, 32);
    memcpy(idx->tail, h + 76, 32);
    const uint64_t np = get_le(h + 108, 8), nw = get_le(h + 116, 8);
    if (fmt < ZB200_DF_ZLIB || fmt > ZB200_DF_DEFLATE || reserved || idx->span < 32768 || idx->span % 32768 ||
        idx->payload > idx->len || idx->len > (1ull << 62) || idx->size > (1ull << 62))
      return ZB200_ERR_ARG;
    idx->fmt = (int)fmt;
    const uint64_t body = len - 4 - kIndexHeader;
    if (np == 0 || np > idx->size / 32768 + 1 || np > body / kIndexPoint || nw > np || nw > (body - np * kIndexPoint) / 8)
      return ZB200_ERR_ARG;
    pos = kIndexHeader;
    idx->bit.resize(np);
    idx->out.resize(np);
    idx->crc.resize(np);
    idx->win.resize(np);
    idx->win_at.assign(np, ~0ull);
    uint64_t next = 0, w = 0;
    for (size_t p = 0; p < np; p++, pos += kIndexPoint) {
      idx->bit[p] = get_le(src + pos, 8);
      idx->out[p] = get_le(src + pos + 8, 8);
      idx->crc[p] = (uint32_t)get_le(src + pos + 16, 4);
      const uint64_t flag = get_le(src + pos + 20, 4);
      if (p == 0 ? idx->out[0] != 0 || idx->bit[0] != idx->payload * 8ull
                 : idx->bit[p] <= idx->bit[p - 1] || idx->out[p] <= idx->out[p - 1])
        return ZB200_ERR_ARG;
      if (idx->bit[p] >= idx->len * 8ull || idx->out[p] > idx->size) return ZB200_ERR_ARG;
      const bool is_win = idx->out[p] >= next;
      if (flag != (is_win ? 1u : 0u)) return ZB200_ERR_ARG;
      idx->win[p] = (uint8_t)flag;
      if (is_win) {
        next = (idx->out[p] / idx->span + 1) * idx->span;
        if (idx->out[p] > 0) idx->win_at[p] = 32768ull * w++;
      }
    }
    if (w != nw) return ZB200_ERR_ARG;
    clen.resize(nw);
    uint64_t total = 0;
    for (size_t i = 0; i < nw; i++, pos += 8) {
      clen[i] = get_le(src + pos, 8);
      if (clen[i] == 0 || clen[i] > len) return ZB200_ERR_ARG;
      total += clen[i];
    }
    if (total != len - 4 - pos) return ZB200_ERR_ARG;
  }
  // the windows: one uncompress_batch, each exactly 32768 bytes (every window point past 0 is at >= span >= 32768)
  const size_t nw = clen.size();
  idx->windows.resize(nw * 32768);
  if (nw) {
    std::vector<uint64_t> so(nw + 1), doff(nw + 1), dl(nw);
    std::vector<int> st(nw);
    so[0] = pos;
    for (size_t i = 0; i < nw; i++) {
      so[i + 1] = so[i] + clen[i];
      doff[i] = 32768ull * i;
    }
    doff[nw] = 32768ull * nw;
    const int rc = zb200_uncompress_batch(ctx, src, so.data(), nw, ZB200_DF_DEFLATE, idx->windows.data(), doff.data(),
                                          dl.data(), st.data());
    if (rc) return rc;
    for (size_t i = 0; i < nw; i++)
      if (st[i] != ZB200_OK || dl[i] != 32768) return ZB200_ERR_ARG;
  }
  *out = idx.release();
  return ZB200_OK;
}

int zb200_index_import(zb200_ctx *ctx, const uint8_t *src, size_t len, zb200_index **out) {
  if (!ctx || !out || (len && !src)) return ZB200_ERR_ARG;
  *out = nullptr;
  try {
    return index_import(ctx, src, len, out);
  } catch (const std::bad_alloc &) {
    return ZB200_ERR_NOMEM;
  }
}

int zb200_last_timing(zb200_ctx *ctx, zb200_timing *out) {
  if (!ctx || !out) return ZB200_ERR_ARG;
  *out = ctx->timing;
  return ZB200_OK;
}

}  // extern "C"
