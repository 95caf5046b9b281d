// context.h -- host-side runtime shared by all C-ABI entry points: the device
// pool (the GPU-native stand-in for arrow::cuda::CudaContext::Allocate,
// cpp/src/arrow/gpu/cuda_context.cc:110-121, which is a bare cuMemAlloc per buffer),
// error plumbing, scalar read-back slots and the launch counter.
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <map>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/arrow_b200.h"

namespace b2 {

extern std::atomic<int64_t> g_launches;
int set_error(int code, const char* fmt, ...);

#define B2_CUDA(expr)                                                              \
  do {                                                                             \
    cudaError_t _e = (expr);                                                       \
    if (_e != cudaSuccess)                                                         \
      return ::b2::set_error(_e == cudaErrorMemoryAllocation ? B2_OUT_OF_MEMORY    \
                                                             : B2_CUDA_ERROR,      \
                             "CUDA error %s at %s:%d: %s", cudaGetErrorName(_e),   \
                             __FILE__, __LINE__, cudaGetErrorString(_e));          \
  } while (0)

#define B2_RETURN_NOT_OK(expr) \
  do {                         \
    int _s = (expr);           \
    if (_s != B2_OK) return _s; \
  } while (0)

// count + check a kernel launch
#define B2_LAUNCHED()                                   \
  do {                                                  \
    ::b2::g_launches.fetch_add(1, std::memory_order_relaxed); \
    B2_CUDA(cudaGetLastError());                        \
  } while (0)

struct ScalarSlot;

}  // namespace b2

// The opaque context.  One per device (and per host thread group that wants its own
// default stream); entry points are re-entrant for distinct streams.
struct B2Context {
  int device = 0;
  cudaStream_t stream = nullptr;
  int sm_count = 132;

  // ---- pool ----
  std::mutex mu;
  struct Block {
    size_t size;
    cudaStream_t last_stream;
  };
  std::multimap<size_t, void*> free_blocks;          // size -> ptr
  std::unordered_map<void*, Block> blocks;            // all live + cached blocks
  std::unordered_map<void*, size_t> in_use;           // ptr -> rounded size
  int64_t bytes_in_use = 0, bytes_reserved = 0, max_in_use = 0;
  B2AllocFn user_alloc = nullptr;
  B2FreeFn user_free = nullptr;
  void* user_data = nullptr;
  std::unordered_map<void*, size_t> user_sizes;

  // ---- scalar read-back slots: 64-byte device cell + pinned host mirror ----
  static constexpr int kSlots = 64;
  static constexpr int kSlotBytes = 256;
  char* slot_dev = nullptr;
  char* slot_host = nullptr;
  std::vector<int> free_slots;

  int alloc(size_t nbytes, void** out, cudaStream_t s);
  int free(void* ptr, cudaStream_t s);
  int trim();
  cudaStream_t pick(void* s) const { return s ? static_cast<cudaStream_t>(s) : stream; }
};

namespace b2 {

// RAII device temporary from the context pool
struct Temp {
  B2Context* ctx;
  cudaStream_t s;
  void* ptr = nullptr;
  Temp(B2Context* c, cudaStream_t st) : ctx(c), s(st) {}
  ~Temp() {
    if (ptr) ctx->free(ptr, s);
  }
  int alloc(size_t n) { return ctx->alloc(n ? n : 1, &ptr, s); }
  template <typename T>
  T* as() const {
    return static_cast<T*>(ptr);
  }
  void* release() {
    void* p = ptr;
    ptr = nullptr;
    return p;
  }
};

// RAII array whose validity / data / data2 buffers go back to the context pool unless handed over
struct PoolArray {
  B2Context* ctx;
  cudaStream_t s;
  B2Array a{};
  PoolArray(B2Context* c, cudaStream_t st) : ctx(c), s(st) {}
  PoolArray(const PoolArray&) = delete;
  PoolArray& operator=(const PoolArray&) = delete;
  ~PoolArray() { reset(); }
  void reset() {
    if (a.validity) ctx->free(const_cast<void*>(a.validity), s);
    if (a.data) ctx->free(const_cast<void*>(a.data), s);
    if (a.data2) ctx->free(const_cast<void*>(a.data2), s);
    a = B2Array{};
  }
  // *out takes the buffers; this holder forgets them
  void give(B2Array* out) {
    *out = a;
    a = B2Array{};
  }
  // frees what this holder owns and takes o's buffers
  void take_from(PoolArray& o) {
    reset();
    o.give(&a);
  }
};

// RAII scalar slot: kernels write up to 32 int64 into dev(); fetch() copies them
// to the pinned mirror and synchronises the stream (the single read-back per call).
struct ScalarSlot {
  B2Context* ctx;
  int idx = -1;
  explicit ScalarSlot(B2Context* c);
  ~ScalarSlot();
  bool ok() const { return idx >= 0; }
  int64_t* dev() const {
    return reinterpret_cast<int64_t*>(ctx->slot_dev + idx * B2Context::kSlotBytes);
  }
  volatile int64_t* host() const {
    return reinterpret_cast<volatile int64_t*>(ctx->slot_host + idx * B2Context::kSlotBytes);
  }
  int zero(cudaStream_t s);
  int fetch(cudaStream_t s);  // D2H + stream sync
};

inline void fill_out(B2Array* out, int type, int64_t length, int64_t null_count,
                     const void* validity, const void* data, const void* data2 = nullptr) {
  out->validity = validity;
  out->data = data;
  out->data2 = data2;
  out->length = length;
  out->offset = 0;
  out->null_count = null_count;
  out->type = type;
  out->byte_width = 0;
}

}  // namespace b2
