// cuda_runtime.h -- TEST INFRASTRUCTURE ONLY: host stand-in for the CUDA runtime calls multical_b200/csrc/solver.cu makes, used
// when tests/simt builds the kernels for the SIMT interpreter (simt.h).  "Device" memory is host memory, streams are
// synchronous, the one reported device calls itself sm_90 so that mcba_create accepts it.  Peer / IPC calls fail.
#pragma once
#include <chrono>
#include <condition_variable>
#include <dlfcn.h>
#include <map>
#include <mutex>
#include <string>
#include "simt.h"

#define MCBA_SIMT_BUILD 1      // solver.cu: plain launches instead of cooperative launches / CUDA graphs (host-driven loop)

typedef int cudaError_t;
enum { cudaSuccess = 0, cudaErrorMemoryAllocation = 2, cudaErrorNotSupported = 801 };
struct CUstream_st;
typedef CUstream_st* cudaStream_t;
struct SimtEvent { std::chrono::steady_clock::time_point t; };
typedef SimtEvent* cudaEvent_t;
typedef void* cudaGraph_t;
typedef void* cudaGraphExec_t;
typedef unsigned long long cudaGraphConditionalHandle;
static inline void cudaGraphSetConditional(cudaGraphConditionalHandle, unsigned) {}
enum cudaMemcpyKind { cudaMemcpyHostToHost = 0, cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3, cudaMemcpyDefault = 4 };
enum { cudaStreamNonBlocking = 1 };
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
enum { cudaIpcMemLazyEnablePeerAccess = 1 };
struct cudaIpcMemHandle_t { char reserved[64]; };
struct cudaDeviceProp {
  char name[256];
  int major, minor, multiProcessorCount;
  size_t sharedMemPerBlockOptin, totalGlobalMem;
};

static inline const char* cudaGetErrorString(cudaError_t e) {
  return e == cudaSuccess ? "no error" : e == cudaErrorMemoryAllocation ? "out of memory" : e == cudaErrorNotSupported ? "operation not supported (SIMT host build)" : "error";
}
static inline cudaError_t cudaGetLastError() { return cudaSuccess; }
static inline cudaError_t cudaGetDeviceCount(int* n) { *n = 1; return cudaSuccess; }
static inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
static inline cudaError_t cudaGetDeviceProperties(cudaDeviceProp* p, int) {
  memset(p, 0, sizeof(*p));
  snprintf(p->name, sizeof(p->name), "SIMT interpreter (host)");
  p->major = 9; p->minor = 0;
  const char* e = getenv("SIMT_SMS");
  p->multiProcessorCount = e ? std::max(1, atoi(e)) : 132;
  p->sharedMemPerBlockOptin = 227 * 1024;
  p->totalGlobalMem = (size_t)8 << 30;
  return cudaSuccess;
}
// device allocations are poisoned (0xFF bytes: NaN doubles, -1 integers) like uninitialised HBM may be, and fenced: 64 canary bytes on
// either side, checked when the buffer is freed -- a kernel writing just outside a buffer aborts the test instead of corrupting a neighbour
namespace simt_mem {
constexpr size_t GUARD = 64;
inline std::mutex m;
inline std::map<void*, size_t> sizes;
inline void check(void* user, size_t bytes) {
  const unsigned char* base = (const unsigned char*)user - GUARD;
  for (size_t i = 0; i < GUARD; i++)
    if (base[i] != 0xA5 || base[GUARD + bytes + i] != 0xA5) {
      fprintf(stderr, "[simt] out-of-bounds write %s a device buffer of %zu bytes (canary at offset %zd)\n", base[i] != 0xA5 ? "before" : "after", bytes,
              base[i] != 0xA5 ? (ssize_t)i - (ssize_t)GUARD : (ssize_t)(bytes + i));
      abort();
    }
}
}  // namespace simt_mem
template <class T>
static inline cudaError_t cudaMalloc(T** p, size_t bytes) {
  unsigned char* q = (unsigned char*)malloc(bytes + 2 * simt_mem::GUARD);
  if (!q) return cudaErrorMemoryAllocation;
  memset(q, 0xA5, simt_mem::GUARD);
  memset(q + simt_mem::GUARD, 0xFF, bytes);
  memset(q + simt_mem::GUARD + bytes, 0xA5, simt_mem::GUARD);
  { std::lock_guard<std::mutex> lk(simt_mem::m); simt_mem::sizes[q + simt_mem::GUARD] = bytes; }
  *p = (T*)(q + simt_mem::GUARD);
  return cudaSuccess;
}
static inline cudaError_t cudaFree(void* p) {
  if (!p) return cudaSuccess;
  size_t bytes;
  { std::lock_guard<std::mutex> lk(simt_mem::m); auto it = simt_mem::sizes.find(p); if (it == simt_mem::sizes.end()) { fprintf(stderr, "[simt] cudaFree of an unknown pointer\n"); abort(); }
    bytes = it->second; simt_mem::sizes.erase(it); }
  simt_mem::check(p, bytes);
  free((unsigned char*)p - simt_mem::GUARD);
  return cudaSuccess;
}
static inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { if (n) memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t = nullptr) { if (n) memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemset(void* d, int v, size_t n) { if (n) memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t = nullptr) { if (n) memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaStreamCreate(cudaStream_t* s) { *s = (cudaStream_t)malloc(8); return cudaSuccess; }
static inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { return cudaStreamCreate(s); }
static inline cudaError_t cudaStreamDestroy(cudaStream_t s) { free(s); return cudaSuccess; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
static inline cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = new SimtEvent(); return cudaSuccess; }
static inline cudaError_t cudaEventDestroy(cudaEvent_t e) { delete e; return cudaSuccess; }
enum { cudaEventDisableTiming = 2 };
static inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) { return cudaEventCreate(e); }
static inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned = 0) { return cudaSuccess; }      // everything runs synchronously, in issue order
static inline cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t = nullptr) { e->t = std::chrono::steady_clock::now(); return cudaSuccess; }
static inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
static inline cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t a, cudaEvent_t b) {
  *ms = std::chrono::duration<float, std::milli>(b->t - a->t).count();
  return cudaSuccess;
}
template <class F> static inline cudaError_t cudaFuncSetAttribute(F*, int, int) { return cudaSuccess; }
// "IPC": the ranks of a multi-rank interpreter test are host threads of one process, so a handle simply carries the pointer
static inline cudaError_t cudaIpcGetMemHandle(cudaIpcMemHandle_t* h, void* p) { memset(h, 0, sizeof(*h)); memcpy(h->reserved, &p, sizeof(p)); return cudaSuccess; }
static inline cudaError_t cudaIpcOpenMemHandle(void** p, cudaIpcMemHandle_t h, unsigned) { memcpy(p, h.reserved, sizeof(*p)); return cudaSuccess; }
static inline cudaError_t cudaIpcCloseMemHandle(void*) { return cudaSuccess; }

// ---------------------------------------------------------------------------------------------------------------------------
// In-process stand-in for the NCCL entry points solver.cu loads with dlopen/dlsym: ranks are host threads, a communicator is a
// rendezvous keyed by the unique id, an all-reduce reduces in rank order behind two barriers.  Same ABI as the real signatures
// (the 128-byte unique id travels by value).
namespace simt_nccl {
struct UniqueId { char internal[128]; };
struct Group {
  int world = 0, joined = 0, arrived = 0; unsigned gen = 0;
  std::mutex m; std::condition_variable cv;
  const void* send[16] = {nullptr};
  void barrier() {
    std::unique_lock<std::mutex> lk(m);
    const unsigned g = gen;
    if (++arrived == world) { arrived = 0; gen++; cv.notify_all(); } else cv.wait(lk, [&] { return gen != g; });
  }
};
struct Comm { Group* g; int rank; };
inline std::mutex reg_m;
inline std::map<std::string, Group*> registry;
inline int GetUniqueId(UniqueId* id) {
  static int counter = 0;
  std::lock_guard<std::mutex> lk(reg_m);
  memset(id, 0, sizeof(*id));
  snprintf(id->internal, sizeof(id->internal), "simt-nccl-%d", ++counter);
  return 0;
}
inline int CommInitRank(Comm** out, int world, UniqueId id, int rank) {
  if (world < 1 || world > 16 || rank < 0 || rank >= world) return 4;
  Group* g;
  { std::lock_guard<std::mutex> lk(reg_m); Group*& slot = registry[std::string(id.internal, 128)]; if (!slot) { slot = new Group(); slot->world = world; } g = slot; }
  { std::unique_lock<std::mutex> lk(g->m); g->joined++; g->cv.notify_all(); g->cv.wait(lk, [&] { return g->joined >= world; }); }
  *out = new Comm{g, rank};
  return 0;
}
inline int CommDestroy(Comm* c) { delete c; return 0; }
inline int AllReduce(const void* send, void* recv, size_t count, int dtype, int op, Comm* c, cudaStream_t) {
  if (dtype != 8) return 5;                                   // ncclFloat64 only
  Group* g = c->g;
  g->send[c->rank] = send;
  g->barrier();
  std::vector<double> acc(count);
  for (size_t i = 0; i < count; i++) {
    double a = ((const double*)g->send[0])[i];
    for (int r = 1; r < g->world; r++) { const double v = ((const double*)g->send[r])[i]; a = op == 0 ? a + v : (op == 2 ? fmax(a, v) : a); }
    acc[i] = a;
  }
  g->barrier();                                               // every rank has read every send buffer (in-place reductions)
  memcpy(recv, acc.data(), count * sizeof(double));
  g->barrier();
  return 0;
}
inline const char* GetErrorString(int) { return "simt-nccl error"; }
inline int GroupStart() { return 0; }
inline int GroupEnd() { return 0; }
}  // namespace simt_nccl
static inline void* simt_dlopen(const char* name, int flags) { return strstr(name, "nccl") ? (void*)&simt_nccl::registry : dlopen(name, flags); }
static inline void* simt_dlsym(void* h, const char* sym) {
  if (h != (void*)&simt_nccl::registry) return dlsym(h, sym);
  const std::string s(sym);
  if (s == "ncclGetUniqueId") return (void*)&simt_nccl::GetUniqueId;
  if (s == "ncclCommInitRank") return (void*)&simt_nccl::CommInitRank;
  if (s == "ncclCommDestroy") return (void*)&simt_nccl::CommDestroy;
  if (s == "ncclAllReduce") return (void*)&simt_nccl::AllReduce;
  if (s == "ncclGetErrorString") return (void*)&simt_nccl::GetErrorString;
  if (s == "ncclGroupStart") return (void*)&simt_nccl::GroupStart;
  if (s == "ncclGroupEnd") return (void*)&simt_nccl::GroupEnd;
  return nullptr;
}
#define dlopen simt_dlopen
#define dlsym simt_dlsym
