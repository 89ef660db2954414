// cuda_runtime.h for the HOST SIMT INTERPRETER build of the kernels (tests/simt) -- TEST
// INFRASTRUCTURE.  Found first on the include path of that build only: it supplies the CUDA
// vector types, qualifiers, built-ins and a trivial runtime (device memory = host memory, streams
// are immediate) so that torchmd_b200/csrc/tmd_b200.cu compiles with g++ and every kernel launch
// runs in the interpreter of simt.h.  Nothing of this is ever part of the product.
#pragma once
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

// ---- vector types ------------------------------------------------------------------------
struct float2 { float x, y; };
struct float3 { float x, y, z; };
struct alignas(16) float4 { float x, y, z, w; };
struct int2 { int x, y; };
struct alignas(16) int4 { int x, y, z, w; };
struct uint2 { unsigned x, y; };
struct alignas(16) uint4 { unsigned x, y, z, w; };
inline float2 make_float2(float x, float y) { return float2{x, y}; }
inline float4 make_float4(float x, float y, float z, float w) { return float4{x, y, z, w}; }
inline int4 make_int4(int x, int y, int z, int w) { return int4{x, y, z, w}; }
inline uint2 make_uint2(unsigned x, unsigned y) { return uint2{x, y}; }
inline int2 make_int2(int x, int y) { return int2{x, y}; }
inline uint4 make_uint4(unsigned x, unsigned y, unsigned z, unsigned w) { return uint4{x, y, z, w}; }
struct dim3 {
  unsigned x, y, z;
  dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};

// ---- qualifiers --------------------------------------------------------------------------
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __noinline__
#define __launch_bounds__(...)
#define __shared__ static
#define __cudart_builtin__

#include "../simt.h"  // threadIdx & co., warp / block collectives, run_grid

// ---- scalar built-ins -----------------------------------------------------------------------
inline int min(int a, int b) { return a < b ? a : b; }
inline int max(int a, int b) { return a > b ? a : b; }
inline unsigned min(unsigned a, unsigned b) { return a < b ? a : b; }
inline unsigned max(unsigned a, unsigned b) { return a > b ? a : b; }
inline long long min(long long a, long long b) { return a < b ? a : b; }
inline long long max(long long a, long long b) { return a > b ? a : b; }
inline int __float_as_int(float f) { int i; memcpy(&i, &f, 4); return i; }
inline float __int_as_float(int i) { float f; memcpy(&f, &i, 4); return f; }
inline unsigned __float_as_uint(float f) { unsigned i; memcpy(&i, &f, 4); return i; }
inline float __uint_as_float(unsigned i) { float f; memcpy(&f, &i, 4); return f; }
inline int __popc(unsigned v) { return __builtin_popcount(v); }
inline int __ffs(int v) { return __builtin_ffs(v); }
inline int __ffsll(long long v) { return __builtin_ffsll(v); }
inline unsigned __umulhi(unsigned a, unsigned b) { return (unsigned)(((unsigned long long)a * b) >> 32); }
template <typename T> inline T __ldg(const T* p) { return *p; }
template <typename T> inline T __ldcs(const T* p) { return *p; }
inline void __threadfence() {}
inline void __threadfence_block() {}
inline void __threadfence_system() {}
inline void __nanosleep(unsigned) { simt::yield(); }
inline long long clock64() { return simt::fake_clock(); }
template <typename T> inline T atomicAdd(T* p, T v) { T o = *p; *p = o + v; return o; }  // fibers of one OS thread: no races
inline int atomicMax(int* p, int v) { int o = *p; if (v > o) *p = v; return o; }
inline int atomicOr(int* p, int v) { int o = *p; *p = o | v; return o; }
inline int atomicMin(int* p, int v) { int o = *p; if (v < o) *p = v; return o; }

// ---- runtime: "device" memory is host memory, streams execute immediately ----------------------
typedef int cudaError_t;
enum { cudaSuccess = 0, cudaErrorNotSupported = 801, cudaErrorMemoryAllocation = 2 };
inline const char* cudaGetErrorString(cudaError_t e) { return e == cudaSuccess ? "no error" : (e == cudaErrorNotSupported ? "not supported by the SIMT interpreter" : "error"); }
inline cudaError_t cudaGetLastError() { return cudaSuccess; }
typedef struct simt_stream_* cudaStream_t;
typedef struct simt_event_* cudaEvent_t;
enum cudaMemcpyKind { cudaMemcpyHostToHost, cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice };
inline cudaError_t cudaMalloc(void** p, size_t n) { *p = aligned_alloc(256, (n + 255) / 256 * 256); return *p ? cudaSuccess : cudaErrorMemoryAllocation; }
template <typename T> inline cudaError_t cudaMalloc(T** p, size_t n) { return cudaMalloc((void**)p, n); }
inline cudaError_t cudaFree(void* p) { free(p); return cudaSuccess; }
inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { memmove(d, s, n); return cudaSuccess; }
inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t st = nullptr);  // (capture-aware: below)
inline cudaError_t cudaMemset(void* d, int v, size_t n) { memset(d, v, n); return cudaSuccess; }
inline cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t st = nullptr);
inline cudaError_t cudaGetDeviceCount(int* n) { *n = 1; return cudaSuccess; }
inline cudaError_t cudaGetDevice(int* d) { *d = 0; return cudaSuccess; }
inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
inline cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
enum cudaDeviceAttr { cudaDevAttrMultiProcessorCount };
inline cudaError_t cudaDeviceGetAttribute(int* v, cudaDeviceAttr a, int) { *v = (a == cudaDevAttrMultiProcessorCount) ? 4 : 0; return cudaSuccess; }
template <typename F> inline cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessor(int* n, F, int, size_t) { *n = 1; return cudaSuccess; }
enum { cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2 };
// (a created stream is a distinct non-null handle, as on the device: the library tests handles for "in use")
inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { static long n = 0; *s = reinterpret_cast<cudaStream_t>(++n); return cudaSuccess; }
inline cudaError_t cudaStreamDestroy(cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaStreamWaitEvent(cudaStream_t st, cudaEvent_t e, unsigned);  // (a captured event pulls the waiting stream into the capture: below)
inline cudaError_t cudaEventCreate(cudaEvent_t* e) { static long n = 0; *e = reinterpret_cast<cudaEvent_t>(++n); return cudaSuccess; }
inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) { return cudaEventCreate(e); }
inline cudaError_t cudaEventDestroy(cudaEvent_t) { return cudaSuccess; }
inline cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t st = nullptr);
inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
inline cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t, cudaEvent_t) { *ms = 0.f; return cudaSuccess; }
struct cudaIpcMemHandle_t { char reserved[64]; };
enum { cudaIpcMemLazyEnablePeerAccess = 1 };
// "inter-process" handles inside one process: the handle carries the pointer (several contexts = several ranks)
inline cudaError_t cudaIpcGetMemHandle(cudaIpcMemHandle_t* h, void* p) { memset(h, 0, sizeof(*h)); memcpy(h->reserved, &p, sizeof(p)); return cudaSuccess; }
inline cudaError_t cudaIpcOpenMemHandle(void** p, cudaIpcMemHandle_t h, unsigned) { memcpy(p, h.reserved, sizeof(*p)); return *p ? cudaSuccess : cudaErrorNotSupported; }
inline cudaError_t cudaIpcCloseMemHandle(void*) { return cudaSuccess; }
// ---- graphs: record and replay -------------------------------------------------------------------
// A capturing stream records its work (kernel launches through the library's launch() helper, async memsets and
// copies) as closures in program order -- a valid topological order of the real graph -- and cudaGraphLaunch runs them
// again.  A stream that waits on an event recorded in a capturing stream joins that capture, as in CUDA.  An IF node
// holds a body graph and runs it when its handle is non-zero; handles created with cudaGraphCondAssignDefault fall
// back to their default after every launch.  This models the CONTROL structure the library builds (what is captured
// where, what a replay executes); it says nothing about the real API's argument checking.
#include <functional>
#include <map>
#include <vector>
struct simt_graph_;
struct simt_graph_node_ {
  std::function<void()> run;                  // kernel / memset / memcpy
  unsigned long long handle = 0;              // IF node: its condition ...
  simt_graph_* body = nullptr;                // ... and body
  simt_graph_* body_out[1] = {nullptr};       // storage behind cudaConditionalNodeParams::phGraph_out
};
struct simt_graph_ { std::vector<simt_graph_node_*> nodes; };
typedef simt_graph_* cudaGraph_t;
typedef simt_graph_* cudaGraphExec_t;
typedef simt_graph_node_* cudaGraphNode_t;
typedef unsigned long long cudaGraphConditionalHandle;
enum cudaStreamCaptureStatus { cudaStreamCaptureStatusNone, cudaStreamCaptureStatusActive };
enum cudaStreamCaptureMode { cudaStreamCaptureModeGlobal, cudaStreamCaptureModeThreadLocal, cudaStreamCaptureModeRelaxed };
enum { cudaGraphCondAssignDefault = 1, cudaStreamSetCaptureDependencies = 1 };
enum cudaGraphNodeType { cudaGraphNodeTypeKernel, cudaGraphNodeTypeConditional = 13 };
enum cudaGraphConditionalNodeType { cudaGraphCondTypeIf };
struct cudaConditionalNodeParams { cudaGraphConditionalHandle handle; cudaGraphConditionalNodeType type; unsigned size; cudaGraph_t* phGraph_out; };
struct cudaGraphNodeParams { cudaGraphNodeType type; cudaConditionalNodeParams conditional; };
struct cudaGraphEdgeData;
namespace simt_stub {
struct Cond { unsigned value, def; bool reset; };
struct State {
  std::map<cudaStream_t, simt_graph_*> capture;   // streams that are capturing, and into which graph
  std::map<cudaStream_t, cudaStream_t> origin;    // a joined stream -> the stream whose capture it joined
  std::map<cudaEvent_t, cudaStream_t> event_in;   // events recorded in a capturing stream -> that stream
  std::vector<Cond> conds{Cond{0, 0, false}};     // handle = index (0 is "no handle")
  long long graph_launches = 0, bodies_run = 0, bodies_skipped = 0;  // what the replays did (simt_lib.cpp exports them)
};
inline State& state() { static State s; return s; }
inline bool capturing(cudaStream_t st) { return state().capture.count(st) != 0; }
inline void record(cudaStream_t st, std::function<void()> fn) {
  simt_graph_node_* n = new simt_graph_node_;
  n->run = std::move(fn);
  state().capture[st]->nodes.push_back(n);
}
inline void run_graph(simt_graph_* g) {
  for (simt_graph_node_* n : g->nodes) {
    if (n->body) {
      if (state().conds[n->handle].value) { state().bodies_run++; run_graph(n->body); }
      else state().bodies_skipped++;
    }
    else n->run();
  }
}
}  // namespace simt_stub
inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t st) {
  if (simt_stub::capturing(st)) simt_stub::record(st, [=]() { memmove(d, s, n); });
  else memmove(d, s, n);
  return cudaSuccess;
}
inline cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t st) {
  if (simt_stub::capturing(st)) simt_stub::record(st, [=]() { memset(d, v, n); });
  else memset(d, v, n);
  return cudaSuccess;
}
inline cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t st) {
  if (simt_stub::capturing(st)) simt_stub::state().event_in[e] = st;
  else simt_stub::state().event_in.erase(e);
  return cudaSuccess;
}
inline cudaError_t cudaStreamWaitEvent(cudaStream_t st, cudaEvent_t e, unsigned) {
  auto& S = simt_stub::state();
  auto it = S.event_in.find(e);
  if (it != S.event_in.end() && !simt_stub::capturing(st) && simt_stub::capturing(it->second)) {
    S.capture[st] = S.capture[it->second];  // fork: the waiting stream records into the same graph
    S.origin[st] = it->second;
  }
  return cudaSuccess;
}
inline cudaError_t cudaStreamIsCapturing(cudaStream_t st, cudaStreamCaptureStatus* s) {
  *s = simt_stub::capturing(st) ? cudaStreamCaptureStatusActive : cudaStreamCaptureStatusNone;
  return cudaSuccess;
}
inline cudaError_t cudaStreamGetCaptureInfo(cudaStream_t st, cudaStreamCaptureStatus* s, unsigned long long* = nullptr, cudaGraph_t* g = nullptr,
                                            const cudaGraphNode_t** deps = nullptr, size_t* ndeps = nullptr) {
  const bool on = simt_stub::capturing(st);
  *s = on ? cudaStreamCaptureStatusActive : cudaStreamCaptureStatusNone;
  if (g) *g = on ? simt_stub::state().capture[st] : nullptr;
  if (deps) *deps = nullptr;
  if (ndeps) *ndeps = 0;
  return cudaSuccess;
}
inline cudaError_t cudaStreamBeginCapture(cudaStream_t st, cudaStreamCaptureMode) {
  if (simt_stub::capturing(st)) return cudaErrorNotSupported;
  simt_stub::state().capture[st] = new simt_graph_;
  return cudaSuccess;
}
inline cudaError_t cudaStreamBeginCaptureToGraph(cudaStream_t st, cudaGraph_t g, const cudaGraphNode_t*, const cudaGraphEdgeData*, size_t, cudaStreamCaptureMode) {
  if (simt_stub::capturing(st) || !g) return cudaErrorNotSupported;
  simt_stub::state().capture[st] = g;
  return cudaSuccess;
}
inline cudaError_t cudaStreamEndCapture(cudaStream_t st, cudaGraph_t* g) {
  auto& S = simt_stub::state();
  if (!simt_stub::capturing(st)) return cudaErrorNotSupported;
  *g = S.capture[st];
  S.capture.erase(st);
  for (auto it = S.origin.begin(); it != S.origin.end();)  // streams that joined this capture leave it with it
    if (it->second == st) { S.capture.erase(it->first); it = S.origin.erase(it); } else ++it;
  return cudaSuccess;
}
inline cudaError_t cudaStreamUpdateCaptureDependencies(cudaStream_t st, cudaGraphNode_t*, size_t, unsigned) {
  return simt_stub::capturing(st) ? cudaSuccess : cudaErrorNotSupported;  // (program order already is the dependency order)
}
inline cudaError_t cudaGraphConditionalHandleCreate(cudaGraphConditionalHandle* h, cudaGraph_t, unsigned def, unsigned flags) {
  auto& c = simt_stub::state().conds;
  c.push_back(simt_stub::Cond{def, def, (flags & cudaGraphCondAssignDefault) != 0});
  *h = c.size() - 1;
  return cudaSuccess;
}
inline cudaError_t cudaGraphAddNode(cudaGraphNode_t* node, cudaGraph_t g, const cudaGraphNode_t*, size_t, cudaGraphNodeParams* p) {
  if (!g || p->type != cudaGraphNodeTypeConditional || p->conditional.type != cudaGraphCondTypeIf || p->conditional.size != 1 || !p->conditional.handle)
    return cudaErrorNotSupported;
  simt_graph_node_* n = new simt_graph_node_;
  n->handle = p->conditional.handle;
  n->body = n->body_out[0] = new simt_graph_;
  p->conditional.phGraph_out = n->body_out;
  g->nodes.push_back(n);
  *node = n;
  return cudaSuccess;
}
inline cudaError_t cudaGraphInstantiate(cudaGraphExec_t* e, cudaGraph_t g, unsigned long long) { *e = g; return g ? cudaSuccess : cudaErrorNotSupported; }
inline cudaError_t cudaGraphLaunch(cudaGraphExec_t e, cudaStream_t) {
  simt_stub::state().graph_launches++;
  simt_stub::run_graph(e);
  for (auto& c : simt_stub::state().conds) if (c.reset) c.value = c.def;
  return cudaSuccess;
}
inline cudaError_t cudaGraphDestroy(cudaGraph_t) { return cudaSuccess; }      // (leaked: test processes are short-lived)
inline cudaError_t cudaGraphExecDestroy(cudaGraphExec_t) { return cudaSuccess; }
inline void cudaGraphSetConditional(cudaGraphConditionalHandle h, unsigned v) { simt_stub::state().conds[h].value = v; }
