// malio_buffer.h — the owning types of a handle's device and pinned host buffers.  A buffer is its pointer and its size in
// one object: the size is 0 whenever the pointer is NULL, it moves (and std::swap's) with the pointer, and the memory goes
// back when the owner is destroyed.  Kernels and copies take the raw pointer (implicit conversion, or data()).
//
// Growth.  A call that returned after enqueueing (the *_device calls) may still read or write a buffer on the handle's
// stream, so a live buffer is freed only after that stream is drained:
//   allocate()   grow by replacement, the old contents dropped: drain (only when a buffer is held), free, allocate.  A failed
//                allocation leaves the buffer empty.
//   grow_keep()  grow keeping the first elements: allocate every new buffer of the group, copy device to device, drain,
//                then free the old ones.  A failed allocation or copy leaves every buffer of the group as it was.
// Destruction frees without a drain (the stream may be gone already): the owner drains first when work may be in flight.
//
// States.  The buffers belong to the handle's states (malio_handle's owners, malio_internal.h): the device state and one
// state per feature.  A feature state is created whole on first use by acquire() and freed by release(), which drains the
// handle's stream first; teardown that is not a buffer is the state type's destructor.
#ifndef MALIO_BUFFER_H_
#define MALIO_BUFFER_H_

#include <cuda_runtime.h>

#include <cstddef>
#include <initializer_list>
#include <string>
#include <utility>
#include <vector>

#include "malio_internal.h"

namespace malio_buf {

inline int cuda_fail(malio_handle* h, const char* what, cudaError_t e) { h->err = std::string(what) + ": " + cudaGetErrorString(e); return MALIO_ERR_CUDA; }

// untyped cudaMalloc'ed memory, move-only; DeviceBuffer<T> gives it its element type
class DeviceMemory {
 public:
  DeviceMemory() = default;
  DeviceMemory(DeviceMemory&& o) noexcept : p_(std::exchange(o.p_, nullptr)), bytes_(std::exchange(o.bytes_, 0)) {}
  DeviceMemory& operator=(DeviceMemory&& o) noexcept {
    if (this != &o) { release(); p_ = std::exchange(o.p_, nullptr); bytes_ = std::exchange(o.bytes_, 0); }
    return *this;
  }
  ~DeviceMemory() { release(); }

  void* raw() const { return p_; }
  size_t bytes() const { return bytes_; }
  // frees without a drain: at destruction, or for a buffer the stream has been drained for
  void release() { if (p_) cudaFree(p_); p_ = nullptr; bytes_ = 0; }
  // grow by replacement to `bytes`; MALIO_ERR_CUDA with h->err set when the drain or the allocation fails
  int allocate_bytes(malio_handle* h, cudaStream_t st, size_t bytes) {
    if (p_) {
      if (cudaError_t e = cudaStreamSynchronize(st)) return cuda_fail(h, "cudaStreamSynchronize(D->stream)", e);
      release();
    }
    if (cudaError_t e = allocate_empty(bytes)) return cuda_fail(h, "cudaMalloc((void**)&ptr, count * sizeof(T))", e);
    return MALIO_OK;
  }
  // `bytes` into an empty buffer; it stays empty on failure
  cudaError_t allocate_empty(size_t bytes) {
    const cudaError_t e = cudaMalloc(&p_, bytes);
    if (e == cudaSuccess) bytes_ = bytes; else p_ = nullptr;
    return e;
  }

 protected:
  void* p_ = nullptr;
  size_t bytes_ = 0;
};

template <class T>
class DeviceBuffer : public DeviceMemory {
 public:
  T* data() const { return static_cast<T*>(p_); }
  operator T*() const { return data(); }
  size_t size() const { return bytes_ / sizeof(T); }   // capacity in elements
  int allocate(malio_handle* h, cudaStream_t st, size_t n) { return allocate_bytes(h, st, n * sizeof(T)); }
};

// one buffer of a group and what it grows to: n elements, keeping the first `keep` (grow_keep; at most what it holds)
struct Resize {
  DeviceMemory& buf;
  size_t bytes, keep_bytes;
  template <class T>
  Resize(DeviceBuffer<T>& b, size_t n, size_t keep = 0) : buf(b), bytes(n * sizeof(T)), keep_bytes(keep * sizeof(T)) {}
};

// A group of buffers whose sizes follow one capacity, read from the group's first buffer: each grows by replacement, in list
// order.  When an allocation fails the first buffer is released as well (this call allocated it: nothing is enqueued on it),
// so that the capacity reads 0 and the next call grows the whole group again.
inline int allocate_group(malio_handle* h, cudaStream_t st, std::initializer_list<Resize> group) {
  for (const Resize& r : group)
    if (int rc = r.buf.allocate_bytes(h, st, r.bytes)) { group.begin()->buf.release(); return rc; }
  return MALIO_OK;
}

// Grow a group of buffers keeping their first elements: all or nothing.  The error is returned (and cleared), the caller words it.
inline cudaError_t grow_keep(cudaStream_t st, std::initializer_list<Resize> group) {
  std::vector<DeviceMemory> fresh(group.size());
  cudaError_t e = cudaSuccess;
  bool live = false;
  size_t i = 0;
  for (const Resize& r : group)
    if (e == cudaSuccess) e = fresh[i++].allocate_empty(r.bytes);
  i = 0;
  for (const Resize& r : group) {
    const size_t k = r.keep_bytes < r.buf.bytes() ? r.keep_bytes : r.buf.bytes();
    if (e == cudaSuccess && k) e = cudaMemcpyAsync(fresh[i].raw(), r.buf.raw(), k, cudaMemcpyDeviceToDevice, st);
    live = live || r.buf.raw();
    ++i;
  }
  if (e == cudaSuccess && live) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return e;   // `fresh` goes back, the group is untouched
  }
  i = 0;
  for (const Resize& r : group) r.buf = std::move(fresh[i++]);
  return cudaSuccess;
}

// cudaHostAlloc'ed host memory, move-only (flags: cudaHostAllocMapped for a buffer the device writes into).  Pinned buffers
// are allocated once, on first use, and never grow.
template <class T>
class PinnedBuffer {
 public:
  PinnedBuffer() = default;
  PinnedBuffer(PinnedBuffer&& o) noexcept : p_(std::exchange(o.p_, nullptr)), n_(std::exchange(o.n_, 0)) {}
  PinnedBuffer& operator=(PinnedBuffer&& o) noexcept {
    if (this != &o) { release(); p_ = std::exchange(o.p_, nullptr); n_ = std::exchange(o.n_, 0); }
    return *this;
  }
  ~PinnedBuffer() { release(); }

  T* data() const { return p_; }
  operator T*() const { return p_; }
  size_t size() const { return n_; }
  void release() { if (p_) cudaFreeHost(p_); p_ = nullptr; n_ = 0; }
  // n elements into an empty buffer
  int allocate(malio_handle* h, size_t n, unsigned flags = cudaHostAllocDefault) {
    release();
    if (cudaError_t e = cudaHostAlloc((void**)&p_, n * sizeof(T), flags)) { p_ = nullptr; return cuda_fail(h, "cudaHostAlloc", e); }
    n_ = n;
    return MALIO_OK;
  }

 private:
  T* p_ = nullptr;
  size_t n_ = 0;
};

// Frees the state in `slot`, if any, after one drain of `st` (work enqueued on its buffers may be in flight; NULL: nothing
// was ever enqueued).  The state is freed whatever the drain returns, and the drain's error is returned.
template <class S>
cudaError_t release(malio_owner<S>& slot, cudaStream_t st) {
  if (!slot) return cudaSuccess;
  const cudaError_t e = st ? cudaStreamSynchronize(st) : cudaSuccess;
  slot.reset();
  return e;
}

// Selects the handle's device and hands back its device state D and the feature state in `slot`, creating it on first use:
// s.init(h, D, args...) allocates the state's fixed buffers.  The state goes into the slot only once init has succeeded;
// after a failure (init's status and h->err are returned) the partial state is released, so the next call starts afresh.
template <class S, class Dev, class... Args>
int acquire(malio_handle* h, malio_owner<S>& slot, S*& s, Dev*& D, Args&&... args) {
  D = h->dev.get();
  if (cudaError_t e = cudaSetDevice(D->device)) return cuda_fail(h, "cudaSetDevice(D->device)", e);
  if (!slot) {
    malio_owner<S> fresh(new S);
    if (int rc = fresh->init(h, D, std::forward<Args>(args)...)) {
      release(fresh, D->stream);
      return rc;
    }
    slot = std::move(fresh);
  }
  s = slot.get();
  return MALIO_OK;
}

}  // namespace malio_buf

#endif  // MALIO_BUFFER_H_
