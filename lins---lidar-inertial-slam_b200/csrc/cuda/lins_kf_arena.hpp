// lins_kf_arena.hpp — the host store of the key frames of mapping-node slots with loop closure: a run-level arena of
// pinned slabs, carved into fixed-size chunks that the slots take as their stores grow.  The slabs grow with the run:
// the first holds first_chunks chunks, each later one as many as the run holds already (the total doubles), up to
// max_chunks per slab, so a small run pins little and a large one allocates rarely.  Plain C++ with no CUDA,
// so the CPU suite compiles it with g++ (tests/test_kf_arena_cpu.py); the library hands it cudaHostAlloc (pinned and
// mapped) through Allocator.
//
// A slot places each key frame's records at the end of its last chunk, or at the start of a chunk it takes next (the
// unused tail of the one before stays unused until the slot gives its chunks back).  A key frame larger than a chunk
// gets a large block of its own; a block given back is kept for a later key frame of at most its size.  Nothing is
// freed before release(): a chunk or block given back while a queued kernel may still write to it is only ever
// written again by later work on the same stream, or by host code that synchronised the stream first.
#pragma once
#include <algorithm>
#include <cstddef>
#include <cstdint>
#include <vector>

namespace lins_arena {

// the memory the arena draws on: alloc returns nullptr on failure
struct Allocator {
  void* (*alloc)(size_t bytes, void* user);
  void (*release)(void* p, void* user);
  void* user;
};

// what one slot holds of its run's arena
struct Holding {
  std::vector<int> chunks;  // chunk ids, in the order taken
  size_t tail = 0;          // bytes used in the last chunk
  std::vector<int> large;   // large blocks held
  uint64_t bytes = 0;       // bytes placed (the key frames' records)
};

class Arena {
 public:
  Arena(size_t chunk_bytes, int first_chunks, int max_chunks, Allocator a)
      : chunk_(chunk_bytes), first_(first_chunks), max_(max_chunks), a_(a) {}
  Arena(const Arena&) = delete;
  Arena& operator=(const Arena&) = delete;
  ~Arena() { release(); }

  // room for `bytes` of one key frame of the slot holding h, at *out (nullptr for 0 bytes).  False when the allocator
  // fails (h is then unchanged).
  bool take(Holding& h, size_t bytes, void** out) {
    *out = nullptr;
    if (bytes == 0) return true;
    if (bytes > chunk_) return take_large(h, bytes, out);
    if (h.chunks.empty() || chunk_ - h.tail < bytes) {
      if (free_.empty() && !add_slab()) return false;
      h.chunks.push_back(free_.back());
      free_.pop_back();
      h.tail = 0;
    }
    *out = chunk_ptr(h.chunks.back()) + h.tail;
    h.tail += bytes;
    h.bytes += bytes;
    return true;
  }

  // the slot's chunks and large blocks back to the run (nothing is freed)
  void give_back(Holding& h) {
    for (auto it = h.chunks.rbegin(); it != h.chunks.rend(); ++it) free_.push_back(*it);
    for (int b : h.large) large_[b].used = false;
    h = Holding();
  }

  // every slab and large block freed; the holdings of the run are void after it
  void release() {
    for (void* p : slabs_) a_.release(p, a_.user);
    for (const Large& b : large_) a_.release(b.p, a_.user);
    slabs_.clear();
    chunk_at_.clear();
    large_.clear();
    free_.clear();
    reserved_ = 0;
  }

  uint64_t reserved() const { return reserved_; }  // bytes of the slabs and large blocks
  size_t chunk_bytes() const { return chunk_; }
  size_t free_chunks() const { return free_.size(); }
  size_t slabs() const { return slabs_.size(); }
  size_t chunks() const { return chunk_at_.size(); }  // chunks in all slabs

 private:
  struct Large { void* p; size_t bytes; bool used; };

  char* chunk_ptr(int id) const { return chunk_at_[id]; }

  bool add_slab() {
    const int n = (int)std::min<size_t>((size_t)max_, std::max<size_t>((size_t)first_, chunk_at_.size()));
    void* p = a_.alloc(chunk_ * n, a_.user);
    if (!p) return false;
    slabs_.push_back(p);
    reserved_ += chunk_ * n;
    const int first = (int)chunk_at_.size();
    for (int i = 0; i < n; ++i) chunk_at_.push_back(static_cast<char*>(p) + (size_t)i * chunk_);
    for (int i = n - 1; i >= 0; --i) free_.push_back(first + i);  // (the lowest id on top)
    return true;
  }

  // the smallest free large block that fits, else a new one
  bool take_large(Holding& h, size_t bytes, void** out) {
    int best = -1;
    for (int i = 0; i < (int)large_.size(); ++i)
      if (!large_[i].used && large_[i].bytes >= bytes && (best < 0 || large_[i].bytes < large_[best].bytes)) best = i;
    if (best < 0) {
      void* p = a_.alloc(bytes, a_.user);
      if (!p) return false;
      large_.push_back(Large{p, bytes, false});
      reserved_ += bytes;
      best = (int)large_.size() - 1;
    }
    large_[best].used = true;
    h.large.push_back(best);
    h.bytes += bytes;
    *out = large_[best].p;
    return true;
  }

  size_t chunk_;
  int first_, max_;
  Allocator a_;
  std::vector<void*> slabs_;
  std::vector<char*> chunk_at_;  // each chunk's address, by id
  std::vector<int> free_;    // free chunk ids, taken from the back
  std::vector<Large> large_;
  uint64_t reserved_ = 0;
};

}  // namespace lins_arena
