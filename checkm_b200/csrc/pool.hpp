// pool.hpp -- workspace buffers handed out from the engine's grow-only device cache, and the staging every entry point does
// around its kernels: typed copies, fills, timing events and the stream synchronise
#pragma once
#include <algorithm>
#include "engine.hpp"

namespace ckm {

inline int cuda_check(cudaError_t err, const char *what) { return err == cudaSuccess ? CKM_OK : cuda_fail(err, what); }

// Copies of n elements on a stream; a copy of no elements is not issued.
template <class T> int copy_in(T *dev, const T *host, size_t n, cudaStream_t st) {
  return n ? cuda_check(cudaMemcpyAsync(dev, host, sizeof(T) * n, cudaMemcpyHostToDevice, st), "cudaMemcpyAsync (upload)") : CKM_OK;
}
template <class T> int copy_out(T *host, const T *dev, size_t n, cudaStream_t st) {
  return n ? cuda_check(cudaMemcpyAsync(host, dev, sizeof(T) * n, cudaMemcpyDeviceToHost, st), "cudaMemcpyAsync (download)") : CKM_OK;
}
inline int set_bytes(void *dev, int byte, size_t bytes, cudaStream_t st) { return cuda_check(cudaMemsetAsync(dev, byte, bytes, st), "cudaMemsetAsync"); }
inline int stream_sync(cudaStream_t st) { return cuda_check(cudaStreamSynchronize(st), "cudaStreamSynchronize"); }
// kernel timing on the engine's events, on its stream; ev_elapsed does nothing when ms is null
inline int ev_record(ckm_engine *e, int k) { return cuda_check(cudaEventRecord(e->ev[k], e->stream), "cudaEventRecord"); }
inline int ev_elapsed(ckm_engine *e, float *ms, int k0, int k1) {
  return ms ? cuda_check(cudaEventElapsedTime(ms, e->ev[k0], e->ev[k1]), "cudaEventElapsedTime") : CKM_OK;
}

// ---- device buffers come from the engine's grow-only cache: no cudaMalloc/cudaFree in the steady state ----
extern thread_local ckm_engine *g_pool_engine;   // one search per host thread; engines are not shared between threads (defined in search.cu)
extern thread_local int g_pool_next;
// One entry point's device work: the engine's device, its stream, and its cache handed out from slot 0 again.
struct DeviceScope {
  cudaStream_t st;
  explicit DeviceScope(ckm_engine *e) : st(e->stream) { cudaSetDevice(e->device); g_pool_engine = e; g_pool_next = 0; }
  ~DeviceScope() { g_pool_engine = nullptr; }
};
struct DevBuf {
  void *p = nullptr; size_t bytes = 0; int slot = -1;
  int alloc(size_t n) {
    ckm_engine *e = g_pool_engine;
    if (e == nullptr) { set_error("internal: workspace requested outside a search"); return CKM_EINVAL; }
    if (slot < 0) { slot = g_pool_next++; if ((size_t)slot >= e->pool.size()) e->pool.resize(slot + 1, std::make_pair((void *)nullptr, (size_t)0)); }
    bytes = std::max<size_t>(n, 256);
    auto &ent = e->pool[slot];
    if (ent.second < bytes) {
      if (ent.first) cudaFree(ent.first);
      ent.first = nullptr; ent.second = 0;
      const size_t want = bytes + bytes / 4;
      cudaError_t err = cudaMalloc(&ent.first, want);
      if (err != cudaSuccess) {
        // out of memory: the blocks cached by earlier searches that this search has not handed out yet (slots past
        // g_pool_next) go back to the device, then the request is tried again at its exact size
        cudaGetLastError();
        for (size_t s = (size_t)g_pool_next; s < e->pool.size(); ++s)
          if (e->pool[s].first) { cudaFree(e->pool[s].first); e->pool[s] = std::make_pair((void *)nullptr, (size_t)0); }
        err = cudaMalloc(&ent.first, bytes);
        if (err != cudaSuccess) { cudaGetLastError(); ent.first = nullptr; p = nullptr; return cuda_fail(err, "cudaMalloc(workspace)"); }
        ent.second = bytes;
      }
      else ent.second = want;
    }
    p = ent.first;
    return CKM_OK;
  }
  template <class T> T *as() { return reinterpret_cast<T *>(p); }
  // allocates n elements and uploads them
  template <class T> int put(const T *host, size_t n, cudaStream_t st) { const int rc = alloc(sizeof(T) * n); return rc ? rc : copy_in(as<T>(), host, n, st); }
  // allocates nbytes and sets each of them to `byte`
  int fill(size_t nbytes, int byte, cudaStream_t st) { const int rc = alloc(nbytes); return rc ? rc : set_bytes(p, byte, nbytes, st); }
  // downloads elements [first, first + n)
  template <class T> int get(T *host, size_t n, cudaStream_t st, size_t first = 0) { return copy_out(host, as<T>() + first, n, st); }
};

}  // namespace ckm
