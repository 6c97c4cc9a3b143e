"""malio_buffer.h without a GPU: the owning buffer types compiled by g++ against a fake CUDA runtime (malloc underneath) that
counts live allocations, frees, stream drains and copies, and can fail the next allocation.  cudart is not linked.

Checked: replacement growth drains only when it replaces a live buffer, and before the free; a failed replacement leaves
an empty buffer; keeping growth copies the first elements and leaves everything as it was when it fails, for a single buffer
and for a group; a replacement group reads as empty after a failed member; move, swap and destruction free each allocation
exactly once, for device and pinned buffers; CUB's temporary storage grows to the largest size its calls ask for plus headroom,
only when it holds less, drains before a replacement, hands a run all its bytes, and is left as it was by a failed query."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "ma-lio_b200", "csrc")

FAKE_RUNTIME = r"""
#include <cuda_runtime.h>
#include <cstdlib>
#include <cstring>
#include <set>
#include <string>

// the fake runtime's log: every event appended as one letter (m malloc, f free, s drain, c copy, h host alloc, H host free)
std::string g_log;
std::set<void*> g_live;
int g_fail_next = 0;        // fail this many of the next allocations, after g_skip successful ones
int g_skip = 0;
int g_double_free = 0;

static bool fail_now() {
  if (g_fail_next && g_skip == 0) { --g_fail_next; return true; }
  if (g_skip) --g_skip;
  return false;
}
extern "C" {
cudaError_t cudaMalloc(void** p, size_t n) {
  if (fail_now()) { *p = nullptr; g_log += 'x'; return cudaErrorMemoryAllocation; }
  *p = std::malloc(n ? n : 1); g_live.insert(*p); g_log += 'm'; return cudaSuccess;
}
cudaError_t cudaFree(void* p) {
  if (!p) return cudaSuccess;
  if (!g_live.erase(p)) { ++g_double_free; return cudaErrorInvalidValue; }
  std::free(p); g_log += 'f'; return cudaSuccess;
}
cudaError_t cudaHostAlloc(void** p, size_t n, unsigned int) {
  if (fail_now()) { *p = nullptr; g_log += 'x'; return cudaErrorMemoryAllocation; }
  *p = std::malloc(n ? n : 1); g_live.insert(*p); g_log += 'h'; return cudaSuccess;
}
cudaError_t cudaFreeHost(void* p) {
  if (!p) return cudaSuccess;
  if (!g_live.erase(p)) { ++g_double_free; return cudaErrorInvalidValue; }
  std::free(p); g_log += 'H'; return cudaSuccess;
}
cudaError_t cudaStreamSynchronize(cudaStream_t) { g_log += 's'; return cudaSuccess; }
cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, enum cudaMemcpyKind, cudaStream_t) {
  std::memcpy(d, s, n); g_log += 'c'; return cudaSuccess;
}
cudaError_t cudaGetLastError(void) { return cudaSuccess; }
const char* cudaGetErrorString(cudaError_t e) { return e == cudaErrorMemoryAllocation ? "out of memory" : "error"; }
}
"""

CHECKS = r"""
#include <cstdio>
#include <set>
#include <utility>
#include "malio_buffer.h"

extern std::string g_log;
extern std::set<void*> g_live;
extern int g_fail_next, g_skip, g_double_free;

using malio_buf::DeviceBuffer;
using malio_buf::PinnedBuffer;
static int g_failures = 0;
#define CHECK(c) do { if (!(c)) { std::printf("FAIL %s:%d %s\n", __FILE__, __LINE__, #c); ++g_failures; } } while (0)
static cudaStream_t const ST = reinterpret_cast<cudaStream_t>(0x10);

static void replace_growth(malio_handle* h) {
  DeviceBuffer<int> b;
  CHECK(b.data() == nullptr && b.size() == 0);
  g_log.clear();
  CHECK(b.allocate(h, ST, 10) == MALIO_OK);
  CHECK(g_log == "m");                       // the first allocation does not drain
  CHECK(b.size() == 10 && b.data() != nullptr);
  g_log.clear();
  CHECK(b.allocate(h, ST, 20) == MALIO_OK);
  CHECK(g_log == "sfm");                     // one drain, before the free, then the new allocation
  CHECK(b.size() == 20);
  g_log.clear();
  g_fail_next = 1;
  CHECK(b.allocate(h, ST, 40) == MALIO_ERR_CUDA);
  CHECK(g_log == "sfx");
  CHECK(b.data() == nullptr && b.size() == 0);
  CHECK(h->err == "cudaMalloc((void**)&ptr, count * sizeof(T)): out of memory");
  g_log.clear();
  CHECK(b.allocate(h, ST, 40) == MALIO_OK);  // the next growth allocates again, with nothing to drain
  CHECK(g_log == "m" && b.size() == 40);
}

static void keep_growth(malio_handle* h) {
  DeviceBuffer<int> b;
  CHECK(b.allocate(h, ST, 8) == MALIO_OK);
  for (int i = 0; i < 8; ++i) b.data()[i] = 100 + i;
  int* old = b.data();
  g_log.clear();
  CHECK(malio_buf::grow_keep(ST, {{b, 16, 5}}) == cudaSuccess);
  CHECK(g_log == "mcsf");                    // allocate, copy, drain, free the old one
  CHECK(b.size() == 16 && b.data() != old);
  for (int i = 0; i < 5; ++i) CHECK(b.data()[i] == 100 + i);
  old = b.data();
  g_log.clear();
  g_fail_next = 1;
  CHECK(malio_buf::grow_keep(ST, {{b, 64, 5}}) == cudaErrorMemoryAllocation);
  CHECK(g_log == "x");                       // nothing drained, copied or freed
  CHECK(b.data() == old && b.size() == 16);
  for (int i = 0; i < 5; ++i) CHECK(b.data()[i] == 100 + i);
  DeviceBuffer<int> e;                       // an empty buffer grows without a drain
  g_log.clear();
  CHECK(malio_buf::grow_keep(ST, {{e, 4, 4}}) == cudaSuccess);
  CHECK(g_log == "m" && e.size() == 4);
}

static void keep_group(malio_handle* h) {
  DeviceBuffer<float> a; DeviceBuffer<double> b; DeviceBuffer<char> c;
  CHECK(a.allocate(h, ST, 4) == MALIO_OK && b.allocate(h, ST, 4) == MALIO_OK && c.allocate(h, ST, 4) == MALIO_OK);
  for (int i = 0; i < 4; ++i) { a.data()[i] = 1.5f * i; b.data()[i] = 2.5 * i; c.data()[i] = (char)('a' + i); }
  for (int failing = 0; failing < 3; ++failing) {
    float* pa = a.data(); double* pb = b.data(); char* pc = c.data();
    const size_t live = g_live.size();
    g_skip = failing; g_fail_next = 1;
    CHECK(malio_buf::grow_keep(ST, {{a, 32, 3}, {b, 32, 3}, {c, 32, 3}}) == cudaErrorMemoryAllocation);
    CHECK(a.data() == pa && b.data() == pb && c.data() == pc);
    CHECK(a.size() == 4 && b.size() == 4 && c.size() == 4);
    CHECK(g_live.size() == live);            // the new buffers that were allocated went back
    for (int i = 0; i < 4; ++i) CHECK(a.data()[i] == 1.5f * i && b.data()[i] == 2.5 * i && c.data()[i] == (char)('a' + i));
  }
  g_log.clear();
  CHECK(malio_buf::grow_keep(ST, {{a, 32, 3}, {b, 32, 3}, {c, 32, 3}}) == cudaSuccess);
  CHECK(g_log == "mmmcccsfff");              // one drain for the group
  CHECK(a.size() == 32 && b.size() == 32 && c.size() == 32);
  for (int i = 0; i < 3; ++i) CHECK(a.data()[i] == 1.5f * i && b.data()[i] == 2.5 * i && c.data()[i] == (char)('a' + i));
}

static void replace_group(malio_handle* h) {
  DeviceBuffer<int> first; DeviceBuffer<double> second; DeviceBuffer<char> third;
  CHECK(malio_buf::allocate_group(h, ST, {{first, 10}, {second, 20}, {third, 30}}) == MALIO_OK);
  CHECK(first.size() == 10 && second.size() == 20 && third.size() == 30);
  g_skip = 1; g_fail_next = 1;               // `first` grows, `second` fails
  CHECK(malio_buf::allocate_group(h, ST, {{first, 100}, {second, 200}, {third, 300}}) == MALIO_ERR_CUDA);
  CHECK(first.data() == nullptr && first.size() == 0);   // the group's capacity reads 0: the next call grows it again
  CHECK(second.data() == nullptr && second.size() == 0);
  CHECK(malio_buf::allocate_group(h, ST, {{first, 100}, {second, 200}, {third, 300}}) == MALIO_OK);
  CHECK(first.size() == 100 && second.size() == 200 && third.size() == 300);
}

static void ownership(malio_handle* h) {
  const size_t live0 = g_live.size();
  {
    DeviceBuffer<int> a, b;
    CHECK(a.allocate(h, ST, 3) == MALIO_OK && b.allocate(h, ST, 7) == MALIO_OK);
    int* pa = a.data(); int* pb = b.data();
    std::swap(a, b);                         // pointers and sizes change places
    CHECK(a.data() == pb && a.size() == 7 && b.data() == pa && b.size() == 3);
    DeviceBuffer<int> c(std::move(a));
    CHECK(c.data() == pb && c.size() == 7 && a.data() == nullptr && a.size() == 0);
    c = std::move(b);                        // c's old buffer is freed, b's moves in
    CHECK(c.data() == pa && c.size() == 3 && b.data() == nullptr);
    CHECK(g_live.size() == live0 + 1);
    c.release();
    CHECK(c.data() == nullptr && c.size() == 0);
    CHECK(a.allocate(h, ST, 5) == MALIO_OK);
  }
  CHECK(g_live.size() == live0);
  {
    PinnedBuffer<double> p, q;
    CHECK(p.allocate(h, 4) == MALIO_OK && q.allocate(h, 6, cudaHostAllocMapped) == MALIO_OK);
    double* pp = p.data();
    std::swap(p, q);
    CHECK(q.data() == pp && q.size() == 4 && p.size() == 6);
    PinnedBuffer<double> r(std::move(p));
    CHECK(p.data() == nullptr && p.size() == 0 && r.size() == 6);
    r = std::move(q);
    CHECK(r.data() == pp && g_live.size() == live0 + 1);
    g_fail_next = 1;
    PinnedBuffer<double> s;
    CHECK(s.allocate(h, 2) == MALIO_ERR_CUDA && s.data() == nullptr && s.size() == 0);
  }
  CHECK(g_live.size() == live0);
}

static void cub_temp(malio_handle* h) {
  malio_buf::CubTemp t;
  void* ran = nullptr;
  size_t ran_bytes = 0;
  // a call that asks for `need` bytes and records what a run is handed
  auto call = [&](size_t need) {
    return [&, need](void* p, size_t& b) {
      if (!p) b = need; else { ran = p; ran_bytes = b; }
      return cudaSuccess;
    };
  };
  auto failing = [](void*, size_t& b) { b = 1u << 30; return cudaErrorInvalidValue; };
  g_log.clear();
  CHECK(t.reserve(h, ST, call(1000), call(8000), call(50)) == MALIO_OK);
  CHECK(g_log == "m");                       // the largest size plus t/8 + 4096, without a drain for the first allocation
  CHECK(t.bytes() == 8000 + 1000 + 4096);
  CHECK(t.reserve(h, ST, call(13096)) == MALIO_OK && g_log == "m");   // it fits: nothing happens
  CHECK(t.run(h, call(1)) == MALIO_OK && ran != nullptr && ran_bytes == 13096);
  g_log.clear();
  CHECK(t.reserve(h, ST, call(20000)) == MALIO_OK);
  CHECK(g_log == "sfm" && t.bytes() == 20000 + 2500 + 4096);   // one drain, before the free
  g_log.clear();
  CHECK(t.reserve(h, ST, call(10), failing, call(1u << 20)) == MALIO_ERR_CUDA);
  CHECK(g_log.empty() && t.bytes() == 26596);
  CHECK(h->err == "CUB temporary storage query: error");
  CHECK(t.run(h, failing) == MALIO_ERR_CUDA && h->err == "CUB device-wide algorithm: error");
  t.release();
  CHECK(t.bytes() == 0);
}

int main() {
  malio_handle h;
  replace_growth(&h);
  keep_growth(&h);
  keep_group(&h);
  replace_group(&h);
  ownership(&h);
  cub_temp(&h);
  CHECK(g_live.empty());
  CHECK(g_double_free == 0);
  std::printf("%s %d\n", g_failures ? "FAILED" : "OK", g_failures);
  return g_failures ? 1 : 0;
}
"""


@pytest.fixture(scope="module")
def checks(tmp_path_factory):
    d = tmp_path_factory.mktemp("device_buffer")
    (d / "fake_cudart.cpp").write_text(FAKE_RUNTIME)
    (d / "checks.cpp").write_text(CHECKS)
    exe = d / "checks"
    subprocess.run(["/usr/bin/g++", "-O1", "-std=c++17", "-Wall", "-I/usr/local/cuda/include", "-I" + os.path.join(ROOT, "include"),
                    "-I" + CSRC, str(d / "checks.cpp"), str(d / "fake_cudart.cpp"), "-o", str(exe)], check=True)
    return exe


def test_device_buffer_semantics(checks):
    r = subprocess.run([str(checks)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.strip().endswith("OK 0"), r.stdout
