// host_util.h -- host-side helpers for api.cu: the owners of every CUDA resource a handle holds (device buffers, pinned host
// buffers, streams, events, the block and event pools and what is borrowed from them), and the Arrow C Data / Device Interface structs (restated from the Arrow ABI
// specification, identical in layout to arrow/c/abi.h).
//
// This file is the only place that calls the raw allocate / free / create / destroy functions of the CUDA runtime.  Each
// owner frees what it holds in its destructor, without waiting: a handle synchronises its streams before its members go (a
// pending copy may still use a pinned mirror).  No owner may live in static storage, where its destructor would run after
// the CUDA runtime has shut down at exit.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <memory>
#include <utility>
#include <vector>

// a block of device memory (cudaMalloc) or of pinned host memory (cudaHostAlloc)
template <bool Pinned>
struct MemBlock {
  void* p = nullptr;
  size_t cap = 0;
  MemBlock() = default;
  MemBlock(MemBlock&& o) noexcept : p(std::exchange(o.p, nullptr)), cap(std::exchange(o.cap, 0)) {}
  MemBlock& operator=(MemBlock&& o) noexcept { std::swap(p, o.p); std::swap(cap, o.cap); return *this; }
  ~MemBlock() { reset(); }
  // replaces the block by one of exactly `bytes`; contents are NOT preserved, empty on failure
  cudaError_t alloc(size_t bytes) {
    reset();
    cudaError_t e = Pinned ? cudaHostAlloc(&p, bytes, cudaHostAllocDefault) : cudaMalloc(&p, bytes);
    if (e == cudaSuccess) cap = bytes; else p = nullptr;
    return e;
  }
 private:
  void reset() { if (p) { if (Pinned) cudaFreeHost(p); else cudaFree(p); } p = nullptr; cap = 0; }
};

// pinned host memory.  The caller decides when it grows and to what size (each use has its own rounding).
using PinnedBuf = MemBlock<true>;

// device memory
struct DevBuf : MemBlock<false> {
  // grows (never shrinks) to at least `bytes`, with a quarter of head-room when that fits; contents are NOT preserved
  cudaError_t ensure_raw(size_t bytes) {
    if (bytes <= cap) return cudaSuccess;
    cudaError_t e = alloc(bytes + bytes / 4 + 256);
    return e == cudaSuccess ? e : alloc(bytes);
  }
  int32_t ensure(size_t bytes);          // ensure_raw; a failure is reported through tfr_last_error (api.cu)
  int32_t ensure_exact(size_t bytes);    // grows (never shrinks) to exactly `bytes`; a failure is reported as ensure's
};

// a non-blocking stream; null until created
class Stream {
  cudaStream_t s_ = nullptr;
 public:
  Stream() = default;
  Stream(Stream&& o) noexcept : s_(std::exchange(o.s_, nullptr)) {}
  Stream& operator=(Stream&& o) noexcept { std::swap(s_, o.s_); return *this; }
  ~Stream() { if (s_) cudaStreamDestroy(s_); }
  cudaError_t create() { return cudaStreamCreateWithFlags(&s_, cudaStreamNonBlocking); }
  cudaError_t create(int priority) { return cudaStreamCreateWithPriority(&s_, cudaStreamNonBlocking, priority); }
  // waits for the stream's work.  A stream never created is skipped: synchronising the null stream would wait for the legacy
  // default stream, and so for other threads' work.
  void sync() const { if (s_) cudaStreamSynchronize(s_); }
  operator cudaStream_t() const { return s_; }
};

// an event without timing; null until created
class Event {
  cudaEvent_t e_ = nullptr;
 public:
  Event() = default;
  Event(Event&& o) noexcept : e_(std::exchange(o.e_, nullptr)) {}
  Event& operator=(Event&& o) noexcept { std::swap(e_, o.e_); return *this; }
  ~Event() { if (e_) cudaEventDestroy(e_); }
  cudaError_t create() { return cudaEventCreateWithFlags(&e_, cudaEventDisableTiming); }
  operator cudaEvent_t() const { return e_; }
};

// An event borrowed from an EventPool is held by a PoolEvent, null until taken.  Like a PoolBlock, its destructor and
// reset() give it back through this deleter, and nothing else does.  The pool must outlive it, and whoever resets it holds
// the pool's lock.
class EventPool;
struct EventGiver {
  EventPool* pool = nullptr;
  inline void operator()(cudaEvent_t e) const;
};
using PoolEvent = std::unique_ptr<CUevent_st, EventGiver>;

// Events lent out and taken back (a batch's completion, a profiling span's ends).  The pool owns every event it ever
// created; borrowers hold them in PoolEvents and never destroy them.
class EventPool {
  unsigned flags_;
  std::vector<cudaEvent_t> all_, free_;
  friend struct EventGiver;
  void give(cudaEvent_t e) { free_.push_back(e); }
 public:
  explicit EventPool(unsigned flags) : flags_(flags) {}
  EventPool(const EventPool&) = delete;
  EventPool& operator=(const EventPool&) = delete;
  ~EventPool() { for (cudaEvent_t e : all_) cudaEventDestroy(e); }
  // `out` is empty; it stays empty when no event can be created
  cudaError_t take(PoolEvent& out) {
    cudaEvent_t e = nullptr;
    if (!free_.empty()) { e = free_.back(); free_.pop_back(); }
    else {
      const cudaError_t err = cudaEventCreateWithFlags(&e, flags_);
      if (err != cudaSuccess) return err;
      all_.push_back(e);
    }
    out = PoolEvent(e, EventGiver{this});
    return cudaSuccess;
  }
};
inline void EventGiver::operator()(cudaEvent_t e) const { pool->give(e); }

// A block borrowed from a PinnedPool or a DevPool (`bytes` of it asked for) is held by a PoolBlock, empty when the pool could
// not provide one.  Its destructor and reset() give it back through this deleter, a device block on `st`, the stream whose
// queued work may still touch it; nothing else does.  The pool must outlive it, and whoever resets it holds the pool's lock.
template <class Pool>
struct PoolGiver {
  Pool* pool = nullptr;
  cudaStream_t st = nullptr;
  size_t bytes = 0;
  void operator()(void* p) const { pool->give_back(p, st); }
};
template <class Pool>
using PoolBlock = std::unique_ptr<void, PoolGiver<Pool>>;
template <class Pool>
size_t block_bytes(const PoolBlock<Pool>& b) { return b ? b.get_deleter().bytes : 0; }

struct PinnedPool {
  struct Block { void* p; size_t cap; bool used; };
  std::vector<Block> blocks;
  PinnedPool() = default;
  PinnedPool(const PinnedPool&) = delete;
  PinnedPool& operator=(const PinnedPool&) = delete;
  ~PinnedPool() { for (auto& b : blocks) cudaFreeHost(b.p); }
  PoolBlock<PinnedPool> acquire(size_t bytes) {
    int best = -1;
    for (size_t i = 0; i < blocks.size(); ++i)
      if (!blocks[i].used && blocks[i].cap >= bytes && (best < 0 || blocks[i].cap < blocks[best].cap)) best = (int)i;
    if (best >= 0) { blocks[best].used = true; return PoolBlock<PinnedPool>(blocks[best].p, {this, nullptr, bytes}); }
    // drop free blocks that are too small so the pool does not grow without bound
    for (size_t i = 0; i < blocks.size();) {
      if (!blocks[i].used) { cudaFreeHost(blocks[i].p); blocks.erase(blocks.begin() + i); } else ++i;
    }
    void* p = nullptr;
    size_t cap = bytes + bytes / 8 + 4096;
    if (cudaHostAlloc(&p, cap, cudaHostAllocDefault) != cudaSuccess) return {};
    blocks.push_back({p, cap, true});
    return PoolBlock<PinnedPool>(p, {this, nullptr, bytes});
  }
 private:
  friend struct PoolGiver<PinnedPool>;
  void give_back(void* p, cudaStream_t) { for (auto& b : blocks) if (b.p == p) b.used = false; }
};

// device blocks reused across batches.  A block goes back to the pool when its batch is released, possibly while kernels that
// write it are still queued on the decode stream: `ready` is recorded there at that moment, and whoever takes the block for
// work on ANOTHER stream waits for it.  Free blocks are handed out oldest-release-first, so that in a steady pipeline the
// block a new batch gets was released two or three batches ago and its event has long fired.
struct DevPool {
  struct Block { void* p; size_t cap; bool used; cudaEvent_t ready; unsigned long long stamp; };
  std::vector<Block> blocks;
  unsigned long long clock = 0;
  DevPool() = default;
  DevPool(const DevPool&) = delete;
  DevPool& operator=(const DevPool&) = delete;
  ~DevPool() { for (auto& b : blocks) { cudaFree(b.p); if (b.ready) cudaEventDestroy(b.ready); } }
  // `st`: the stream the block goes back on (give_back)
  PoolBlock<DevPool> acquire(size_t bytes, cudaStream_t st, cudaEvent_t* ready_out = nullptr) {
    int best = -1;
    for (size_t i = 0; i < blocks.size(); ++i) {
      const Block& b = blocks[i];
      if (b.used || b.cap < bytes) continue;
      if (best < 0) { best = (int)i; continue; }
      const Block& c = blocks[best];
      // a block up to 1/8 larger than the smallest fit counts as the same size class: among those, the oldest release wins
      const bool same_class = b.cap <= c.cap + c.cap / 8 && c.cap <= b.cap + b.cap / 8;
      if (same_class ? b.stamp < c.stamp : b.cap < c.cap) best = (int)i;
    }
    if (best >= 0) { blocks[best].used = true; if (ready_out) *ready_out = blocks[best].stamp ? blocks[best].ready : nullptr; return PoolBlock<DevPool>(blocks[best].p, {this, st, bytes}); }
    for (size_t i = 0; i < blocks.size();) {
      if (!blocks[i].used && blocks.size() > 8) { cudaFree(blocks[i].p); if (blocks[i].ready) cudaEventDestroy(blocks[i].ready); blocks.erase(blocks.begin() + i); } else ++i;
    }
    void* p = nullptr;
    size_t cap = bytes + bytes / 8 + 4096;
    if (cudaMalloc(&p, cap) != cudaSuccess) { cap = bytes; if (cudaMalloc(&p, cap) != cudaSuccess) return {}; }
    blocks.push_back({p, cap, true, nullptr, 0});
    if (ready_out) *ready_out = nullptr;
    return PoolBlock<DevPool>(p, {this, st, bytes});
  }
 private:
  friend struct PoolGiver<DevPool>;
  // `st`: the stream whose queued work may still touch the block
  void give_back(void* p, cudaStream_t st) {
    for (auto& b : blocks)
      if (b.p == p) {
        b.used = false;
        b.stamp = ++clock;
        if (!b.ready) cudaEventCreateWithFlags(&b.ready, cudaEventDisableTiming);
        if (b.ready) cudaEventRecord(b.ready, st);
      }
  }
};

extern "C" {
struct ArrowSchema {
  const char* format; const char* name; const char* metadata; int64_t flags; int64_t n_children;
  struct ArrowSchema** children; struct ArrowSchema* dictionary;
  void (*release)(struct ArrowSchema*); void* private_data;
};
struct ArrowArray {
  int64_t length; int64_t null_count; int64_t offset; int64_t n_buffers; int64_t n_children;
  const void** buffers; struct ArrowArray** children; struct ArrowArray* dictionary;
  void (*release)(struct ArrowArray*); void* private_data;
};
struct ArrowDeviceArray {
  struct ArrowArray array; int64_t device_id; int32_t device_type; void* sync_event; int64_t reserved[3];
};
}
