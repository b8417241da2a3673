// amgpu — H100-native bulk change-replay engine: common device/host plumbing.
//
// Every per-item kernel of the engine is a functor with `void operator()(size_t i) const`, launched
// through foreach<F>() as a grid-stride CUDA kernel (k_foreach<F>; the functor name shows up in ncu).
// Grids are sized in multiples of the SM count (132 on H100) times resident CTAs per SM.
//
// AMG_EMU: a *development and host-logic test aid only*. In this build container there is no GPU, so
// the same functors can be compiled with g++ (-DAMG_EMU) and run as a serial loop to debug the
// pipeline's logic before spending GPU time. The emulation library is built under tests/_emu/, is
// only loaded by explicitly named "emu" tests, and is never built into or reachable from the
// product library (libamgpu.so), which is always compiled by nvcc and fails loudly without a GPU.
#pragma once
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>
#include <unordered_map>
#include <mutex>
#include <map>

#ifdef AMG_EMU
#define HD inline
#define DEV inline
#else
#include <cuda_runtime.h>
#define HD __host__ __device__ __forceinline__
#define DEV __device__ __forceinline__
#endif

namespace amg {

struct Error : std::runtime_error {
  int code;
  Error(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};

enum ErrCode {
  AMG_OK = 0, AMG_ERR_RANGE = 1, AMG_ERR_TYPE = 2, AMG_ERR_INTERNAL = 3, AMG_ERR_UNSUPPORTED = 4, AMG_ERR_CUDA = 5, AMG_ERR_FROZEN = 6
};

#ifndef AMG_EMU
#define CUDA_CHECK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) throw amg::Error(amg::AMG_ERR_CUDA, std::string("CUDA error: ") + cudaGetErrorString(e_) + " at " + __FILE__ + ":" + std::to_string(__LINE__)); } while (0)
#endif

struct Ctx {
#ifndef AMG_EMU
  cudaStream_t stream = nullptr;
  cudaStream_t side = nullptr;        // second stream: work that may overlap the main pipeline (joined through events)
  cudaEvent_t evFork = nullptr, evJoin = nullptr;
  cudaStream_t copy = nullptr;        // third stream: device -> host copy of the uploaded change bytes into the host mirror
  cudaEvent_t evUp = nullptr, evMirror = nullptr; bool copyPending = false; std::vector<cudaEvent_t> pieceEv; size_t pieceNext = 0;
  // small device -> host reads go through a kernel that stores into pinned (device-visible) host memory, not through the
  // copy engine: a read of 4 bytes must not queue behind a 100 MB transfer (see d2h / sync)
  struct Peek { void* dst; size_t off, bytes; };
  unsigned char* peekBuf = nullptr; size_t peekCap = 0, peekUsed = 0; std::vector<Peek> peeks;
  volatile unsigned long long* peekFlag = nullptr; unsigned long long peekSeq = 0; bool peekFlagArmed = false;   // completion flag of the last k_peek_words (pinned)
#endif
  int device = 0;
  int numSMs = 132;
  uint64_t launches = 0;   // kernels launched (gpu_launches in bench.py)
};

// ---------------------------------------------------------------- device buffers
#ifndef AMG_EMU
// Process-wide cache of freed device blocks, per device. cudaMalloc / cudaFree cost 0.1 - 1 ms each (they map and unmap
// memory); a fresh document allocates ~200 tables, so opening documents in a long-lived process was bound by them.
// A freed block is parked after a device synchronize (what cudaFree does implicitly: nothing in flight still uses it)
// and handed to the next request of about that size (at most 1.5x). Parked memory is capped, and given back to the
// driver when an allocation fails.
struct DevPool {
  typedef std::pair<int, size_t> Key;   // (device, block bytes)
  struct Block { Key key; bool fromSlab; };
  struct Slab { char* base; size_t used, size; };
  std::mutex m; std::multimap<Key, void*> parked; std::unordered_map<void*, Block> blocks; size_t parkedBytes = 0;
  std::map<int, Slab> slab;   // per device: the slab new blocks are carved from
  static const size_t kMaxParked = 16ull << 30;   // a fifth of an H100's 80 GB
  static const size_t kSlabBytes = 256ull << 20;   // a fresh document needs ~200 tables: carved from a few slabs instead of ~200 cudaMallocs (0.1 - 1 ms each)
  static DevPool& get() { static DevPool* p = new DevPool(); return *p; }   // never destroyed: must outlive every engine and the runtime's own teardown
  // gives parked blocks that own their allocation back to the driver (blocks carved from a slab stay parked: a slab is never freed)
  void trim() {
    for (auto it = parked.begin(); it != parked.end();) {
      auto b = blocks.find(it->second);
      if (b != blocks.end() && b->second.fromSlab) { ++it; continue; }
      parkedBytes -= it->first.second; if (b != blocks.end()) blocks.erase(b); cudaFree(it->second); it = parked.erase(it);
    }
  }
};
#endif
inline void* dev_alloc(size_t bytes) {
#ifdef AMG_EMU
  return malloc(bytes ? bytes : 1);
#else
  const size_t want = ((bytes ? bytes : 1) + 255) & ~(size_t)255;
  int dev = 0; CUDA_CHECK(cudaGetDevice(&dev));
  DevPool& pool = DevPool::get(); std::lock_guard<std::mutex> lock(pool.m);
  auto it = pool.parked.lower_bound(DevPool::Key(dev, want));
  if (it != pool.parked.end() && it->first.first == dev && it->first.second <= want + want / 2 + 4096) {
    void* p = it->second; pool.parkedBytes -= it->first.second; pool.parked.erase(it); return p;
  }
  if (want <= DevPool::kSlabBytes / 4) {   // small and medium tables: carved from the device's current slab
    DevPool::Slab& sl = pool.slab[dev];
    if (!sl.base || sl.used + want > sl.size) {
      void* base = nullptr; cudaError_t e = cudaMalloc(&base, DevPool::kSlabBytes);
      if (e == cudaErrorMemoryAllocation) { cudaGetLastError(); pool.trim(); e = cudaMalloc(&base, DevPool::kSlabBytes); }
      if (e == cudaSuccess) {
        if (sl.base && sl.size - sl.used >= 4096) {   // what is left of the old slab stays usable
          void* rest = sl.base + sl.used; const size_t restBytes = (sl.size - sl.used) & ~(size_t)255;
          pool.blocks[rest] = DevPool::Block{DevPool::Key(dev, restBytes), true}; pool.parked.emplace(DevPool::Key(dev, restBytes), rest); pool.parkedBytes += restBytes;
        }
        sl.base = (char*)base; sl.used = 0; sl.size = DevPool::kSlabBytes;
      } else cudaGetLastError();   // no room for a slab: fall through to a plain allocation
    }
    if (sl.base && sl.used + want <= sl.size) {
      void* p = sl.base + sl.used; sl.used += want;
      pool.blocks[p] = DevPool::Block{DevPool::Key(dev, want), true};
      return p;
    }
  }
  void* p = nullptr; cudaError_t e = cudaMalloc(&p, want);
  if (e == cudaErrorMemoryAllocation) { cudaGetLastError(); pool.trim(); e = cudaMalloc(&p, want); }
  CUDA_CHECK(e);
  pool.blocks[p] = DevPool::Block{DevPool::Key(dev, want), false};
  return p;
#endif
}
inline void dev_free(void* p) {
#ifdef AMG_EMU
  free(p);
#else
  if (!p) return;
  cudaDeviceSynchronize();
  DevPool& pool = DevPool::get(); std::lock_guard<std::mutex> lock(pool.m);
  auto it = pool.blocks.find(p);
  if (it == pool.blocks.end()) { cudaFree(p); return; }
  if (!it->second.fromSlab && pool.parkedBytes + it->second.key.second > DevPool::kMaxParked) { pool.blocks.erase(it); cudaFree(p); return; }
  pool.parked.emplace(it->second.key, p); pool.parkedBytes += it->second.key.second;
#endif
}
inline void dev_memset(Ctx& c, void* p, int v, size_t bytes) {
  if (!bytes) return;
#ifdef AMG_EMU
  memset(p, v, bytes);
#else
  CUDA_CHECK(cudaMemsetAsync(p, v, bytes, c.stream));
#endif
}
inline void h2d(Ctx& c, void* dst, const void* src, size_t bytes) {
  if (!bytes) return;
#ifdef AMG_EMU
  memcpy(dst, src, bytes);
#else
  CUDA_CHECK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, c.stream));
#endif
}
struct Ctx;
inline Ctx*& last_peek_ctx() { static thread_local Ctx* p = nullptr; return p; }   // for drop_pending_peeks() in the C ABI's catch handlers
#ifndef AMG_EMU
static __global__ void k_peek_bytes(unsigned char* dstPinned, const unsigned char* src, size_t bytes) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < bytes; i += (size_t)gridDim.x * blockDim.x) dstPinned[i] = src[i];
}
#endif
#ifndef AMG_EMU
struct PeekWords { const void* src[8]; unsigned bytes[8]; unsigned off[8]; int n; };
static __global__ void k_peek_words(PeekWords w, unsigned char* dstPinned, volatile unsigned long long* flag, unsigned long long seq) {   // a handful of 4- or 8-byte words in one launch
  const int k = threadIdx.x >> 3, b = threadIdx.x & 7;
  if (k < w.n && (unsigned)b < w.bytes[k]) dstPinned[w.off[k] + b] = ((const unsigned char*)w.src[k])[b];
  // completion flag in pinned host memory: the host spins on it instead of going through cudaStreamSynchronize (whose
  // wake-up costs more than the kernel); everything queued on the stream before this kernel has completed by then
  __threadfence_system(); __syncthreads();
  if (threadIdx.x == 0) { *flag = seq; __threadfence_system(); }
}
#endif
// dst is valid after the next sync(c). Up to 16 KB: read by a kernel into the pinned staging buffer (sync() moves it to
// dst); larger: an asynchronous copy.
inline void d2h(Ctx& c, void* dst, const void* src, size_t bytes) {
  if (!bytes) return;
#ifdef AMG_EMU
  memcpy(dst, src, bytes);
#else
  const size_t padded = (bytes + 15) & ~(size_t)15;
  if (bytes <= (16u << 10) && c.peekBuf && c.peekUsed + padded <= c.peekCap) {
    k_peek_bytes<<<(unsigned)((bytes + 255) / 256), 256, 0, c.stream>>>(c.peekBuf + c.peekUsed, (const unsigned char*)src, bytes);
    CUDA_CHECK(cudaGetLastError());
    c.peeks.push_back(Ctx::Peek{dst, c.peekUsed, bytes}); c.peekUsed += padded; last_peek_ctx() = &c; c.launches++;
    return;
  }
  CUDA_CHECK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, c.stream));
#endif
}
inline void d2h_side(Ctx& c, void* dst, const void* src, size_t bytes) {   // on the side stream (after side_fork): overlaps later kernels of the main one
  if (!bytes) return;
#ifdef AMG_EMU
  memcpy(dst, src, bytes);
#else
  CUDA_CHECK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, c.side));
#endif
}
inline void d2d(Ctx& c, void* dst, const void* src, size_t bytes) {
  if (!bytes) return;
#ifdef AMG_EMU
  memmove(dst, src, bytes);
#else
  CUDA_CHECK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, c.stream));
#endif
}
// up to 8 words of at most 8 bytes each, one kernel (readWords: the counts that size the next stage + the error word)
inline void d2h_words(Ctx& c, int n, const void* const* srcs, const size_t* sizes, void* const* dsts) {
#ifdef AMG_EMU
  for (int k = 0; k < n; k++) memcpy(dsts[k], srcs[k], sizes[k]);
#else
  bool small = n <= 8 && c.peekBuf && c.peekUsed + 16 * (size_t)n <= c.peekCap;
  for (int k = 0; k < n && small; k++) if (sizes[k] > 8) small = false;
  if (!small) { for (int k = 0; k < n; k++) d2h(c, dsts[k], srcs[k], sizes[k]); return; }
  PeekWords w; w.n = n;
  for (int k = 0; k < n; k++) { w.src[k] = srcs[k]; w.bytes[k] = (unsigned)sizes[k]; w.off[k] = (unsigned)(c.peekUsed + 16 * (size_t)k); c.peeks.push_back(Ctx::Peek{dsts[k], c.peekUsed + 16 * (size_t)k, sizes[k]}); }
  k_peek_words<<<1, 64, 0, c.stream>>>(w, c.peekBuf, c.peekFlag, ++c.peekSeq);
  CUDA_CHECK(cudaGetLastError());
  c.peekUsed += 16 * (size_t)n; last_peek_ctx() = &c; c.launches++; c.peekFlagArmed = true;
#endif
}
inline void drop_peeks(Ctx& c) {   // after an aborted call: whatever was pending must not be delivered into dead stack frames
#ifndef AMG_EMU
  c.peeks.clear(); c.peekUsed = 0;
#endif
}
inline void drop_pending_peeks() { if (last_peek_ctx()) drop_peeks(*last_peek_ctx()); }
inline void sync(Ctx& c, bool spinOnPeekFlag = false) {
  (void)spinOnPeekFlag;
#ifndef AMG_EMU
  cudaError_t e = cudaSuccess;
  if (spinOnPeekFlag && c.peekFlagArmed) {   // the LAST thing queued is a k_peek_words (readWords): spin on its flag (a failed launch / device error shows up in the stream query)
    c.peekFlagArmed = false; unsigned spins = 0;
    while (*c.peekFlag != c.peekSeq) {
      if ((++spins & 0xfff) == 0) { e = cudaStreamQuery(c.stream); if (e == cudaSuccess) continue; if (e != cudaErrorNotReady) break; e = cudaSuccess; }
#if defined(__x86_64__)
      __builtin_ia32_pause();
#endif
    }
    if (e == cudaSuccess && *c.peekFlag != c.peekSeq) e = cudaStreamSynchronize(c.stream);
  } else { c.peekFlagArmed = false; e = cudaStreamSynchronize(c.stream); }
  if (e != cudaSuccess) { drop_peeks(c); CUDA_CHECK(e); }
  for (const Ctx::Peek& p : c.peeks) memcpy(p.dst, c.peekBuf + p.off, p.bytes);
  c.peeks.clear(); c.peekUsed = 0;
#endif
}

// Growable device array. Growth keeps the old contents (needed for persistent state).
template <class T> struct DBuf {
  T* p = nullptr; size_t cap = 0;
  DBuf() {}
  DBuf(const DBuf&) = delete; DBuf& operator=(const DBuf&) = delete;
  ~DBuf() { dev_free(p); }
  void ensure(Ctx& c, size_t n, size_t keep = 0) {
    if (n <= cap) return;
    size_t ncap = n + n / 4 + 64;
    T* np_ = (T*)dev_alloc(ncap * sizeof(T));
    if (keep) { d2d(c, np_, p, keep * sizeof(T)); sync(c); }
    dev_free(p); p = np_; cap = ncap;
  }
  T* get() { return p; }
  void swap(DBuf& o) { std::swap(p, o.p); std::swap(cap, o.cap); }
};

// Pinned host staging buffer
template <class T> struct HBuf {
  T* p = nullptr; size_t cap = 0;
  HBuf() {}
  HBuf(const HBuf&) = delete; HBuf& operator=(const HBuf&) = delete;
  ~HBuf() { release(); }
  void release() {
#ifdef AMG_EMU
    free(p);
#else
    if (p) cudaFreeHost(p);
#endif
    p = nullptr; cap = 0;
  }
  void ensure(size_t n) {
    if (n <= cap) return;
    size_t ncap = n + n / 4 + 64; T* np_;
#ifdef AMG_EMU
    np_ = (T*)malloc(ncap * sizeof(T));
#else
    CUDA_CHECK(cudaMallocHost((void**)&np_, ncap * sizeof(T)));
#endif
    if (p && cap) memcpy(np_, p, cap * sizeof(T));
    release(); p = np_; cap = ncap;
  }
};

// ---------------------------------------------------------------- kernel launch
// minimum resident CTAs per SM a functor asks for (caps its registers): latency-bound byte parsers want more warps in flight
template <class F> struct LaunchTraits { static const int minBlocks = 1; };
#ifndef AMG_EMU
template <class F> __global__ void __launch_bounds__(256, LaunchTraits<F>::minBlocks) k_foreach(size_t n, F f) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) f(i);
}
#endif

template <class F> inline void foreach(Ctx& c, size_t n, const F& f, bool onSide = false) {
  if (n == 0) return;
#ifdef AMG_EMU
  for (size_t i = 0; i < n; i++) f(i);
#else
  const int block = 256;
  size_t want = (n + block - 1) / block;
  size_t maxGrid = (size_t)c.numSMs * 8;   // 8 resident CTAs of 256 threads per SM
  int grid = (int)(want < maxGrid ? want : maxGrid);
  k_foreach<F><<<grid, block, 0, onSide ? c.side : c.stream>>>(n, f);
  CUDA_CHECK(cudaGetLastError());
#endif
  c.launches++;
}
// One item per WARP (lane 0 works): for long serial state machines whose control flow differs from item to item
// (Huffman streams, RLE column walks). Packed 32 to a warp they would execute one after the other in lockstep.
#ifndef AMG_EMU
template <class F> __global__ void __launch_bounds__(256) k_foreach_warp(size_t n, F f) {
  if (threadIdx.x & 31) return;
  const size_t warps = (size_t)gridDim.x * (blockDim.x >> 5);
  for (size_t k = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); k < n; k += warps) f(k);
}
#endif
template <class F> inline void foreach_warp(Ctx& c, size_t n, const F& f) {
  if (n == 0) return;
#ifdef AMG_EMU
  for (size_t i = 0; i < n; i++) f(i);
#else
  size_t want = (n + 7) / 8, maxGrid = (size_t)c.numSMs * 8;
  int grid = (int)(want < maxGrid ? want : maxGrid);
  k_foreach_warp<F><<<grid, 256, 0, c.stream>>>(n, f);
  CUDA_CHECK(cudaGetLastError());
#endif
  c.launches++;
}
// side stream: fork() makes it wait for everything enqueued on the main stream so far, join() the reverse
inline void side_fork(Ctx& c) {
#ifndef AMG_EMU
  CUDA_CHECK(cudaEventRecord(c.evFork, c.stream)); CUDA_CHECK(cudaStreamWaitEvent(c.side, c.evFork, 0));
#endif
}
inline void side_join(Ctx& c) {
#ifndef AMG_EMU
  CUDA_CHECK(cudaEventRecord(c.evJoin, c.side)); CUDA_CHECK(cudaStreamWaitEvent(c.stream, c.evJoin, 0));
#endif
}

// Copy stream: uploads of a call's change bytes, piece by piece. copy_fork(): the copy stream starts behind what the main
// stream has queued so far. copy_piece_done(): main and side stream wait for everything queued on the copy stream so far
// (one event per piece, taken from a pool). copy_join(): host-side join at the end of the call (also on error paths).
inline void copy_fork(Ctx& c) {
#ifndef AMG_EMU
  CUDA_CHECK(cudaEventRecord(c.evUp, c.stream)); CUDA_CHECK(cudaStreamWaitEvent(c.copy, c.evUp, 0)); c.pieceNext = 0;
#endif
}
inline void h2d_copy(Ctx& c, void* dst, const void* src, size_t bytes) {
#ifdef AMG_EMU
  memcpy(dst, src, bytes);
#else
  CUDA_CHECK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, c.copy)); c.copyPending = true;
#endif
}
inline void d2d_copy(Ctx& c, void* dst, const void* src, size_t bytes) {
#ifdef AMG_EMU
  memmove(dst, src, bytes);
#else
  CUDA_CHECK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, c.copy)); c.copyPending = true;
#endif
}
inline size_t copy_piece_record(Ctx& c) {   // marks "everything queued on the copy stream so far"; returns the mark's number
#ifndef AMG_EMU
  if (c.pieceNext >= c.pieceEv.size()) { cudaEvent_t e; CUDA_CHECK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming)); c.pieceEv.push_back(e); }
  CUDA_CHECK(cudaEventRecord(c.pieceEv[c.pieceNext], c.copy));
  return c.pieceNext++;
#else
  return 0;
#endif
}
inline void copy_piece_wait(Ctx& c, size_t mark) {   // main and side stream wait for that mark
#ifndef AMG_EMU
  CUDA_CHECK(cudaStreamWaitEvent(c.stream, c.pieceEv[mark], 0)); CUDA_CHECK(cudaStreamWaitEvent(c.side, c.pieceEv[mark], 0));
#else
  (void)mark;
#endif
}
inline void copy_join(Ctx& c) noexcept {
#ifndef AMG_EMU
  if (c.copyPending) { cudaStreamSynchronize(c.copy); c.copyPending = false; }
#endif
}
inline void mirror_wait(Ctx&) noexcept {}

// ---------------------------------------------------------------- atomics (serial in EMU)
#ifdef AMG_EMU
template <class T> inline T atomic_add(T* p, T v) { T o = *p; *p = o + v; return o; }
template <class T> inline T atomic_min(T* p, T v) { T o = *p; if (v < o) *p = v; return o; }
template <class T> inline T atomic_max(T* p, T v) { T o = *p; if (v > o) *p = v; return o; }
template <class T> inline T atomic_or(T* p, T v) { T o = *p; *p = o | v; return o; }
template <class T> inline T atomic_cas(T* p, T cmp, T v) { T o = *p; if (o == cmp) *p = v; return o; }
#else
// host bodies exist only so that the functors can stay __host__ __device__; they are never executed in the CUDA build
#if defined(__CUDA_ARCH__)
#define AMG_ATOMIC(devexpr, hostexpr) return devexpr;
#else
#define AMG_ATOMIC(devexpr, hostexpr) hostexpr
#endif
HD uint32_t atomic_add(uint32_t* p, uint32_t v) { AMG_ATOMIC(atomicAdd(p, v), { uint32_t o = *p; *p = o + v; return o; }) }
HD unsigned long long atomic_add(unsigned long long* p, unsigned long long v) { AMG_ATOMIC(atomicAdd(p, v), { unsigned long long o = *p; *p = o + v; return o; }) }
HD uint32_t atomic_min(uint32_t* p, uint32_t v) { AMG_ATOMIC(atomicMin(p, v), { uint32_t o = *p; if (v < o) *p = v; return o; }) }
HD unsigned long long atomic_min(unsigned long long* p, unsigned long long v) { AMG_ATOMIC(atomicMin(p, v), { unsigned long long o = *p; if (v < o) *p = v; return o; }) }
HD uint32_t atomic_max(uint32_t* p, uint32_t v) { AMG_ATOMIC(atomicMax(p, v), { uint32_t o = *p; if (v > o) *p = v; return o; }) }
HD unsigned long long atomic_max(unsigned long long* p, unsigned long long v) { AMG_ATOMIC(atomicMax(p, v), { unsigned long long o = *p; if (v > o) *p = v; return o; }) }
HD uint32_t atomic_or(uint32_t* p, uint32_t v) { AMG_ATOMIC(atomicOr(p, v), { uint32_t o = *p; *p = o | v; return o; }) }
HD unsigned long long atomic_cas(unsigned long long* p, unsigned long long cmp, unsigned long long v) { AMG_ATOMIC(atomicCAS(p, cmp, v), { unsigned long long o = *p; if (o == cmp) *p = v; return o; }) }
HD uint32_t atomic_cas(uint32_t* p, uint32_t cmp, uint32_t v) { AMG_ATOMIC(atomicCAS(p, cmp, v), { uint32_t o = *p; if (o == cmp) *p = v; return o; }) }
#endif

// counter[index] += 1 with one atomic per distinct index per warp (consecutive items usually share the index)
HD void warp_agg_inc(uint32_t* counter, uint32_t index) {
#if defined(__CUDA_ARCH__)
  const unsigned active = __activemask();
  const unsigned peers = __match_any_sync(active, index);
  if ((int)(threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&counter[index], (uint32_t)__popc(peers));
#else
  counter[index] += 1;
#endif
}

typedef unsigned long long u64;
typedef uint32_t u32;
typedef uint8_t u8;

// *target = max(*target, v) / min with one atomic per warp: every lane calls it (inside divergent code is fine, the
// active lanes form the group)
HD void warp_agg_max(u64* target, u64 v) {
#if defined(__CUDA_ARCH__)
  const unsigned active = __activemask();
  const uint32_t hi = __reduce_max_sync(active, (uint32_t)(v >> 32));
  const uint32_t lo = __reduce_max_sync(active, (uint32_t)(v >> 32) == hi ? (uint32_t)v : 0u);
  if ((int)(threadIdx.x & 31) == __ffs(active) - 1) { const u64 m = ((u64)hi << 32) | lo; if (m > *target) atomicMax(target, m); }
#else
  if (v > *target) *target = v;
#endif
}
HD void warp_agg_max(uint32_t* target, uint32_t v) {
#if defined(__CUDA_ARCH__)
  const unsigned active = __activemask();
  const uint32_t m = __reduce_max_sync(active, v);
  if ((int)(threadIdx.x & 31) == __ffs(active) - 1 && m > *target) atomicMax(target, m);
#else
  if (v > *target) *target = v;
#endif
}
// base[index] = min(base[index], v) with one atomic per distinct index per warp
HD void warp_agg_min_at(uint32_t* base, uint32_t index, uint32_t v) {
#if defined(__CUDA_ARCH__)
  const unsigned active = __activemask();
  const unsigned peers = __match_any_sync(active, index);
  const uint32_t m = __reduce_min_sync(peers, v);
  if ((int)(threadIdx.x & 31) == __ffs(peers) - 1 && base[index] > m) atomicMin(&base[index], m);
#else
  if (v < base[index]) base[index] = v;
#endif
}
HD void warp_agg_add(uint32_t* target, uint32_t v) {
#if defined(__CUDA_ARCH__)
  const unsigned active = __activemask();
  const uint32_t sum = __reduce_add_sync(active, v);
  if ((int)(threadIdx.x & 31) == __ffs(active) - 1) atomicAdd(target, sum);
#else
  *target += v;
#endif
}

HD u64 mix64(u64 x) {   // splitmix64 finaliser: hash for open-addressing tables
  x ^= x >> 30; x *= 0xbf58476d1ce4e5b9ULL; x ^= x >> 27; x *= 0x94d049bb133111ebULL; x ^= x >> 31; return x;
}
HD int bits_for(u64 maxValue) { int b = 0; while (maxValue) { b++; maxValue >>= 1; } return b ? b : 1; }
inline size_t pow2_at_least(size_t n) { size_t p = 1; while (p < n) p <<= 1; return p; }

}  // namespace amg
