"""CPU checks of the host key-frame store's arena (csrc/cuda/lins_kf_arena.hpp), compiled with g++ next to a driver that
hands it a counting malloc allocator: key frames placed across chunks, slabs that grow with the run, a key frame larger
than a chunk, reuse of the chunks and large blocks a slot gives back, release, and byte accounting that matches the
records placed."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUDA_DIR = os.path.join(ROOT, "lins---lidar-inertial-slam_b200", "csrc", "cuda")

DRIVER = r"""
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <vector>
#include "lins_kf_arena.hpp"

using namespace lins_arena;

struct Count { int64_t allocs = 0, frees = 0, live = 0; };
static Count g_count;
static void* count_alloc(size_t bytes, void* user) {
  Count* c = static_cast<Count*>(user);
  if (bytes > (size_t(1) << 32)) return nullptr;  // (a refused allocation)
  c->allocs += 1; c->live += 1;
  return std::malloc(bytes);
}
static void count_free(void* p, void* user) { Count* c = static_cast<Count*>(user); c->frees += 1; c->live -= 1; std::free(p); }

static std::unique_ptr<Arena> g_arena;
static std::vector<Holding> g_hold;

extern "C" {

// a run of n_slots slots on an arena of chunk_bytes chunks, slabs of first_chunks growing to max_chunks
void arena_open(uint64_t chunk_bytes, int first_chunks, int max_chunks, int n_slots) {
  g_arena.reset();
  g_count = Count();
  g_arena.reset(new Arena(chunk_bytes, first_chunks, max_chunks, Allocator{count_alloc, count_free, &g_count}));
  g_hold.assign(n_slots, Holding());
}
// one key frame of `bytes` for slot s: its address (0 for none), -1 on failure; fills it with the byte `fill`
int64_t arena_take(int s, uint64_t bytes, int fill) {
  void* p = nullptr;
  if (!g_arena->take(g_hold[s], bytes, &p)) return -1;
  if (p) std::memset(p, fill, bytes);
  return (int64_t)(intptr_t)p;
}
// 1 when the `bytes` at address p all hold `fill`
int arena_holds(int64_t p, uint64_t bytes, int fill) {
  const unsigned char* q = reinterpret_cast<const unsigned char*>((intptr_t)p);
  for (uint64_t i = 0; i < bytes; ++i) if (q[i] != (unsigned char)fill) return 0;
  return 1;
}
void arena_give_back(int s) { g_arena->give_back(g_hold[s]); }
void arena_release() { g_arena->release(); g_hold.assign(g_hold.size(), Holding()); }
// reserved bytes, slabs, free chunks, allocations, frees, live allocations, slot s's bytes / chunks / large blocks, and
// the chunks of all slabs
void arena_stats(int s, int64_t* out) {
  out[9] = (int64_t)g_arena->chunks();
  out[0] = (int64_t)g_arena->reserved(); out[1] = (int64_t)g_arena->slabs(); out[2] = (int64_t)g_arena->free_chunks();
  out[3] = g_count.allocs; out[4] = g_count.frees; out[5] = g_count.live;
  out[6] = (int64_t)g_hold[s].bytes; out[7] = (int64_t)g_hold[s].chunks.size(); out[8] = (int64_t)g_hold[s].large.size();
}
void arena_close() { g_arena.reset(); }
int64_t arena_live() { return g_count.live; }
}
"""

CHUNK = 1024
FIRST, MAX = 2, 4  # chunks of the first slab, and of any slab


def slab_sizes(chunks):
    """the arena's slabs (in chunks) once a run holds `chunks` chunks: the first FIRST, each later one as many as the
    run holds, at most MAX"""
    sizes = []
    while sum(sizes) < chunks:
        sizes.append(min(MAX, max(FIRST, sum(sizes))))
    return sizes


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("g++ is not available")
    d = tmp_path_factory.mktemp("arena")
    src, so = d / "arena_driver.cpp", d / "arena_driver.so"
    src.write_text(DRIVER)
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-shared", "-fPIC", "-I", CUDA_DIR, "-o", str(so), str(src)])
    L = C.CDLL(str(so))
    L.arena_open.argtypes = [C.c_uint64, C.c_int, C.c_int, C.c_int]
    L.arena_take.argtypes = [C.c_int, C.c_uint64, C.c_int]
    L.arena_take.restype = C.c_int64
    L.arena_holds.argtypes = [C.c_int64, C.c_uint64, C.c_int]
    L.arena_give_back.argtypes = [C.c_int]
    L.arena_stats.argtypes = [C.c_int, C.c_void_p]
    L.arena_live.restype = C.c_int64
    return L


def stats(L, s=0):
    out = np.zeros(10, np.int64)
    L.arena_stats(s, out.ctypes.data_as(C.c_void_p))
    keys = ["reserved", "slabs", "free", "allocs", "frees", "live", "bytes", "chunks", "large", "run_chunks"]
    return dict(zip(keys, (int(v) for v in out)))


def test_keyframes_fill_chunks_in_order_and_span_slabs(lib):
    lib.arena_open(CHUNK, FIRST, MAX, 1)
    sizes = [16 * k for k in (20, 30, 13, 64, 1, 40, 50, 7, 64, 33, 60, 2)]
    placed = []
    for i, b in enumerate(sizes):
        p = lib.arena_take(0, b, i + 1)
        assert p > 0
        placed.append((p, b, i + 1))
    # every key frame keeps its bytes: no two overlap
    for p, b, f in placed:
        assert lib.arena_holds(p, b, f)
    # a key frame that fits the rest of the slot's last chunk goes right behind the one before
    assert placed[1][0] == placed[0][0] + sizes[0]
    # the chunks a slot uses: a new one whenever the next key frame does not fit the last one's rest
    used, chunks = 0, 1
    for b in sizes:
        if used + b > CHUNK:
            chunks, used = chunks + 1, 0
        used += b
    st = stats(lib)
    assert st["chunks"] == chunks and chunks > FIRST + MAX  # (more than two slabs)
    slabs = slab_sizes(chunks)
    assert st["slabs"] == len(slabs) and st["run_chunks"] == sum(slabs)
    assert st["reserved"] == sum(slabs) * CHUNK
    assert st["bytes"] == sum(sizes)
    assert st["large"] == 0
    lib.arena_close()
    assert lib.arena_live() == 0


def test_keyframe_larger_than_a_chunk_gets_a_block_of_its_own(lib):
    lib.arena_open(CHUNK, FIRST, MAX, 2)
    a = lib.arena_take(0, 16 * 10, 1)
    big = lib.arena_take(0, 3 * CHUNK + 16, 2)
    c = lib.arena_take(0, 16 * 5, 3)
    assert min(a, big, c) > 0
    assert lib.arena_holds(a, 160, 1) and lib.arena_holds(big, 3 * CHUNK + 16, 2) and lib.arena_holds(c, 80, 3)
    assert c == a + 160  # (the large block does not end the slot's chunk)
    st = stats(lib)
    assert st["large"] == 1 and st["chunks"] == 1
    assert st["reserved"] == FIRST * CHUNK + 3 * CHUNK + 16
    assert st["bytes"] == 160 + 3 * CHUNK + 16 + 80
    # a key frame of exactly a chunk stays in the chunks
    assert lib.arena_take(1, CHUNK, 4) > 0
    assert stats(lib, 1)["large"] == 0 and stats(lib, 1)["chunks"] == 1
    # no bytes: no room taken
    assert lib.arena_take(1, 0, 5) == 0
    assert stats(lib, 1)["bytes"] == CHUNK
    lib.arena_close()


def test_reset_slots_reuse_their_chunks_and_blocks(lib):
    lib.arena_open(CHUNK, FIRST, MAX, 3)
    drive = [16 * k for k in (30, 50, 64, 70, 12, 64)]

    def fill(s, seed):
        for i, b in enumerate(drive):
            assert lib.arena_take(s, b, (seed + i) % 250 + 1) > 0

    for s in range(3):
        fill(s, 10 * s)
    before = stats(lib)
    for rnd in range(3):  # slots reset and refilled with the same drives: nothing new is allocated
        for s in range(3):
            lib.arena_give_back(s)
            assert stats(lib, s)["bytes"] == 0
        for s in (2, 0, 1):
            fill(s, 7 * rnd + s)
        st = stats(lib)
        assert st["reserved"] == before["reserved"] and st["allocs"] == before["allocs"] and st["frees"] == 0
        assert all(stats(lib, s)["bytes"] == 16 * sum(k // 16 for k in drive) for s in range(3))
    lib.arena_close()


def test_large_blocks_are_reused_by_size(lib):
    lib.arena_open(CHUNK, FIRST, MAX, 2)
    assert lib.arena_take(0, 2 * CHUNK, 1) > 0
    assert lib.arena_take(0, 5 * CHUNK, 2) > 0
    lib.arena_give_back(0)
    allocs = stats(lib)["allocs"]
    b = lib.arena_take(1, 3 * CHUNK, 3)  # the smallest free block that fits: the 5-chunk one
    assert b > 0 and stats(lib)["allocs"] == allocs
    c = lib.arena_take(1, 4 * CHUNK, 4)  # the 2-chunk block is too small: a new one
    assert c > 0 and stats(lib)["allocs"] == allocs + 1
    assert lib.arena_holds(b, 3 * CHUNK, 3) and lib.arena_holds(c, 4 * CHUNK, 4)
    lib.arena_close()


def test_release_frees_every_slab_and_block(lib):
    lib.arena_open(CHUNK, FIRST, MAX, 2)
    for i in range(12):
        assert lib.arena_take(i % 2, 16 * (40 + i), i + 1) > 0
    assert lib.arena_take(1, 2 * CHUNK, 99) > 0
    st = stats(lib)
    assert st["live"] == st["slabs"] + 1 and st["reserved"] > 0
    lib.arena_release()  # what opening a new run does
    st = stats(lib)
    assert st["live"] == 0 and st["reserved"] == 0 and st["slabs"] == 0 and st["free"] == 0
    assert st["frees"] == st["allocs"]
    # the arena serves a new run afterwards
    assert lib.arena_take(0, 160, 7) > 0 and stats(lib)["slabs"] == 1
    lib.arena_close()  # (the destructor frees the rest)
    assert lib.arena_live() == 0


def test_failed_allocation_leaves_the_slot_unchanged(lib):
    lib.arena_open(CHUNK, FIRST, MAX, 1)
    assert lib.arena_take(0, 160, 1) > 0
    before = stats(lib)
    assert lib.arena_take(0, (1 << 33), 2) == -1  # (the driver's allocator refuses it)
    assert stats(lib) == before
    lib.arena_close()


def test_slabs_grow_with_the_run(lib):
    """a one-chunk run pins the first slab only; each later slab doubles the run up to the largest slab size"""
    lib.arena_open(CHUNK, FIRST, MAX, 1)
    assert lib.arena_take(0, CHUNK, 1) > 0
    assert stats(lib)["reserved"] == FIRST * CHUNK and stats(lib)["slabs"] == 1
    for n in range(2, 15):
        assert lib.arena_take(0, CHUNK, n) > 0  # (a chunk per key frame)
        st = stats(lib)
        assert st["run_chunks"] == sum(slab_sizes(n)) and st["slabs"] == len(slab_sizes(n)), n
    assert slab_sizes(14) == [2, 2, 4, 4, 4]
    lib.arena_close()
    assert lib.arena_live() == 0
