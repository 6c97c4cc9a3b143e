"""malio_buffer.h's acquire / release of a handle's feature states without a GPU: compiled by g++ against the fake CUDA
runtime of test_device_buffer_cpu.py, with a test state whose init allocates several device and pinned buffers and enqueues
a memset, as the handle's states do.

Checked: an init that fails at its k-th allocation, for every k, leaves the slot empty and returns init's status and error,
after one drain of the stream and before any free, and frees each allocation it made exactly once; the next acquire runs
init from scratch and succeeds; a held state is handed back without a second init; release drains once and then frees each
allocation once; releasing an empty slot does nothing; the read-only lookup (the owner's get()) never creates a state."""
import os
import subprocess

import pytest

from test_device_buffer_cpu import CSRC, FAKE_RUNTIME, ROOT

# what the fake runtime lacks for the state code: device selection (logged as 'd') and memsets ('z')
FAKE_EXTRA = r"""
#include <cuda_runtime.h>
#include <cstring>
#include <string>

extern std::string g_log;
int g_fail_set_device = 0;
extern "C" {
cudaError_t cudaSetDevice(int) {
  if (g_fail_set_device) { g_log += 'D'; return cudaErrorInvalidDevice; }
  g_log += 'd'; return cudaSuccess;
}
cudaError_t cudaMemsetAsync(void* p, int v, size_t n, cudaStream_t) { std::memset(p, v, n); g_log += 'z'; return cudaSuccess; }
}
"""

CHECKS = r"""
#include <algorithm>
#include <cstdio>
#include <set>
#include <string>
#include "malio_buffer.h"

extern std::string g_log;
extern std::set<void*> g_live;
extern int g_fail_next, g_skip, g_double_free, g_fail_set_device;

static int g_failures = 0;
#define CHECK(c) do { if (!(c)) { std::printf("FAIL %s:%d %s  (log %s)\n", __FILE__, __LINE__, #c, g_log.c_str()); ++g_failures; } } while (0)

namespace malio_devstate {
struct DeviceState {
  int device = 2;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(0x10);
};
}  // namespace malio_devstate
using malio_devstate::DeviceState;

// four allocations (three device, one pinned) and a memset between the first two
struct TestState {
  static int inits;
  malio_buf::DeviceBuffer<int> a;
  malio_buf::DeviceBuffer<double> b;
  malio_buf::PinnedBuffer<unsigned> c;
  malio_buf::DeviceBuffer<char> d;
  int init(malio_handle* h, DeviceState* D, size_t n) {
    ++inits;
    if (int rc = a.allocate(h, D->stream, n)) return rc;
    if (cudaMemsetAsync(a, 0, n * sizeof(int), D->stream)) return MALIO_ERR_CUDA;
    if (int rc = b.allocate(h, D->stream, n)) return rc;
    if (int rc = c.allocate(h, n)) return rc;
    return d.allocate(h, D->stream, n);
  }
};
int TestState::inits = 0;
constexpr int ALLOCATIONS = 4;

static int count(char c) { return (int)std::count(g_log.begin(), g_log.end(), c); }
static int frees() { return count('f') + count('H'); }

static void failed_init(malio_handle* h, malio_owner<TestState>& slot) {
  for (int k = 0; k < ALLOCATIONS; ++k) {
    const size_t live = g_live.size();
    const int inits = TestState::inits;
    h->err.clear();
    g_log.clear();
    g_skip = k; g_fail_next = 1;
    TestState* s = nullptr;
    DeviceState* D = nullptr;
    CHECK(malio_buf::acquire(h, slot, s, D, 8) == MALIO_ERR_CUDA);
    CHECK(!slot && slot.get() == nullptr);
    CHECK(TestState::inits == inits + 1);
    CHECK(g_live.size() == live);                      // everything init allocated went back ...
    CHECK(frees() == k && count('m') + count('h') == k);   // ... each allocation once
    CHECK(count('s') == 1);                            // one drain, ahead of every free
    CHECK(g_log.find('s') < g_log.find_first_of("fH"));
    CHECK(g_log.find('s') > g_log.find('x'));
    CHECK(h->err == (k == 2 ? "cudaHostAlloc: out of memory" : "cudaMalloc((void**)&ptr, count * sizeof(T)): out of memory"));
  }
}

static void acquire_and_release(malio_handle* h, malio_owner<TestState>& slot) {
  const size_t live = g_live.size();
  const int inits = TestState::inits;
  TestState* s = nullptr;
  DeviceState* D = nullptr;
  g_log.clear();
  CHECK(malio_buf::acquire(h, slot, s, D, 8) == MALIO_OK);   // init from scratch after the failures
  CHECK(g_log == "dmzmhm");                          // device selected first; no drain, nothing freed
  CHECK(TestState::inits == inits + 1);
  CHECK(s == slot.get() && s != nullptr && D == h->dev.get());
  CHECK(s->a.size() == 8 && s->b.size() == 8 && s->c.size() == 8 && s->d.size() == 8);
  CHECK(g_live.size() == live + ALLOCATIONS);
  TestState* s2 = nullptr;
  D = nullptr;
  g_log.clear();
  CHECK(malio_buf::acquire(h, slot, s2, D, 8) == MALIO_OK);   // a held state: the device is selected, nothing else
  CHECK(g_log == "d" && s2 == s && D == h->dev.get() && TestState::inits == inits + 1);

  g_log.clear();
  CHECK(malio_buf::release(slot, h->dev->stream) == cudaSuccess);
  CHECK(!slot);
  CHECK(g_log.size() == 1 + ALLOCATIONS && g_log[0] == 's' && count('s') == 1 && frees() == ALLOCATIONS);
  CHECK(g_live.size() == live);

  g_log.clear();
  CHECK(malio_buf::release(slot, h->dev->stream) == cudaSuccess);   // an empty slot: no drain, no free
  CHECK(g_log.empty() && !slot);
}

static void lookup_never_creates(malio_handle* h, malio_owner<TestState>& slot) {
  const int inits = TestState::inits;
  g_log.clear();
  const TestState* s = slot.get();
  CHECK(s == nullptr && !slot && g_log.empty() && TestState::inits == inits);
  CHECK(!h->pre && !h->mapst && !h->voxmap && !h->prior && !h->place);   // nothing here created the handle's own states
}

static void device_not_selected(malio_handle* h, malio_owner<TestState>& slot) {
  const int inits = TestState::inits;
  TestState* s = nullptr;
  DeviceState* D = nullptr;
  g_log.clear();
  g_fail_set_device = 1;
  CHECK(malio_buf::acquire(h, slot, s, D, 8) == MALIO_ERR_CUDA);
  g_fail_set_device = 0;
  CHECK(g_log == "D" && !slot && TestState::inits == inits);
  CHECK(h->err == "cudaSetDevice(D->device): error");
}

int main() {
  {
    malio_handle h;
    h.dev = malio_owner<DeviceState>(new DeviceState);
    malio_owner<TestState> slot;
    failed_init(&h, slot);
    acquire_and_release(&h, slot);
    lookup_never_creates(&h, slot);
    device_not_selected(&h, slot);
    TestState* s = nullptr;
    DeviceState* D = nullptr;
    CHECK(malio_buf::acquire(&h, slot, s, D, 8) == MALIO_OK);   // a state still held goes back with its owner
  }
  CHECK(g_live.empty());
  CHECK(g_double_free == 0);
  std::printf("%s %d\n", g_failures ? "FAILED" : "OK", g_failures);
  return g_failures ? 1 : 0;
}
"""


@pytest.fixture(scope="module")
def checks(tmp_path_factory):
    d = tmp_path_factory.mktemp("handle_state")
    (d / "fake_cudart.cpp").write_text(FAKE_RUNTIME)
    (d / "fake_extra.cpp").write_text(FAKE_EXTRA)
    (d / "checks.cpp").write_text(CHECKS)
    exe = d / "checks"
    subprocess.run(["/usr/bin/g++", "-O1", "-std=c++17", "-Wall", "-I/usr/local/cuda/include", "-I" + os.path.join(ROOT, "include"),
                    "-I" + CSRC, str(d / "checks.cpp"), str(d / "fake_cudart.cpp"), str(d / "fake_extra.cpp"), "-o", str(exe)],
                   check=True)
    return exe


def test_handle_state_lifecycle(checks):
    r = subprocess.run([str(checks)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.strip().endswith("OK 0"), r.stdout
