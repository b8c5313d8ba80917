// cuda_shim.h -- TEST-ONLY host emulation of the small CUDA subset used by
// jssenv_b200/csrc (see tests/emu/README.md).  Lets the kernels' logic run in this
// GPU-less container: every CUDA thread of a block is a ucontext fiber, warp
// collectives (__shfl_sync, __ballot_sync, __reduce_*_sync, __syncwarp) and
// __syncthreads are rendezvous points resolved by a scheduler, and the runtime API
// is mapped onto malloc/memcpy.  Collectives are checked strictly: all 32 lanes of
// a warp must arrive at the SAME kind of collective with a full mask, otherwise the
// emulator aborts -- this catches divergent-collective bugs before GPU time is spent.
//
// This is NOT a product backend: nothing in jssenv_b200/ references it, the built
// library (tests/emu/libjss_emu.so) is only loaded by tests that monkeypatch the
// loader, and it is ~1000x slower than one H100 SM.
#pragma once
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <cmath>

#define JSS_EMU 1
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __launch_bounds__(...)
#define __restrict__

using std::max;
using std::min;

struct int2 { int x, y; };
struct alignas(16) int4 { int x, y, z, w; };
struct float2 { float x, y; };
struct alignas(8) uint2 { unsigned x, y; };
static inline uint2 make_uint2(unsigned a, unsigned b) { return uint2{a, b}; }
struct alignas(16) float4 { float x, y, z, w; };
struct alignas(16) uint4 { unsigned x, y, z, w; };
struct dim3 { unsigned x = 1, y = 1, z = 1; dim3(unsigned a = 1, unsigned b = 1, unsigned c = 1) : x(a), y(b), z(c) {} };
static inline int2 make_int2(int a, int b) { return int2{a, b}; }
static inline int4 make_int4(int a, int b, int c, int d) { return int4{a, b, c, d}; }
static inline float2 make_float2(float a, float b) { return float2{a, b}; }
static inline float4 make_float4(float a, float b, float c, float d) { return float4{a, b, c, d}; }

namespace emu {
extern thread_local dim3 threadIdx_, blockIdx_, blockDim_, gridDim_;
extern void *smem_ptr;
extern int poison;   // -1, or the byte every block's dynamic shared memory and every cudaMalloc start as
enum Op { OP_SHFL = 1, OP_SHFL_XOR, OP_SHFL_UP, OP_BALLOT, OP_RED_MIN, OP_RED_MAX, OP_RED_ADD, OP_RED_OR, OP_SYNCWARP, OP_SYNCTHREADS };
uint64_t collective(int op, unsigned mask, uint64_t value, int arg);
void launch_impl(void (*entry)(void *), void *args, dim3 grid, dim3 block, size_t smem);
}  // namespace emu

#define threadIdx (emu::threadIdx_)
#define blockIdx (emu::blockIdx_)
#define blockDim (emu::blockDim_)
#define gridDim (emu::gridDim_)

template <typename T>
static inline uint64_t emu_pack(T v) { uint64_t u = 0; static_assert(sizeof(T) <= 8, ""); memcpy(&u, &v, sizeof(T)); return u; }
template <typename T>
static inline T emu_unpack(uint64_t u) { T v; memcpy(&v, &u, sizeof(T)); return v; }

template <typename T>
static inline T __shfl_sync(unsigned mask, T v, int src) { return emu_unpack<T>(emu::collective(emu::OP_SHFL, mask, emu_pack(v), src & 31)); }
template <typename T>
static inline T __shfl_xor_sync(unsigned mask, T v, int x) { return emu_unpack<T>(emu::collective(emu::OP_SHFL_XOR, mask, emu_pack(v), x)); }
template <typename T>
static inline T __shfl_up_sync(unsigned mask, T v, unsigned d) { return emu_unpack<T>(emu::collective(emu::OP_SHFL_UP, mask, emu_pack(v), (int)d)); }
static inline bool __any_sync(unsigned mask, bool pred) { return emu::collective(emu::OP_BALLOT, mask, pred ? 1 : 0, 0) != 0; }
static inline unsigned __ballot_sync(unsigned mask, bool pred) { return (unsigned)emu::collective(emu::OP_BALLOT, mask, pred ? 1 : 0, 0); }
static inline unsigned __reduce_min_sync(unsigned mask, unsigned v) { return (unsigned)emu::collective(emu::OP_RED_MIN, mask, v, 0); }
static inline unsigned __reduce_max_sync(unsigned mask, unsigned v) { return (unsigned)emu::collective(emu::OP_RED_MAX, mask, v, 0); }
static inline unsigned __reduce_add_sync(unsigned mask, unsigned v) { return (unsigned)emu::collective(emu::OP_RED_ADD, mask, v, 0); }
static inline unsigned __reduce_or_sync(unsigned mask, unsigned v) { return (unsigned)emu::collective(emu::OP_RED_OR, mask, v, 0); }
static inline void __syncwarp(unsigned mask = 0xffffffffu) { emu::collective(emu::OP_SYNCWARP, mask, 0, 0); }
static inline void __syncthreads() { emu::collective(emu::OP_SYNCTHREADS, 0xffffffffu, 0, 0); }

static inline int __float_as_int(float f) { int i; memcpy(&i, &f, 4); return i; }
static inline float __int_as_float(int i) { float f; memcpy(&f, &i, 4); return f; }
static inline int __popc(unsigned v) { return __builtin_popcount(v); }
static inline int __ffs(int v) { return __builtin_ffs(v); }
static inline float __fdiv_rn(float a, float b) { return a / b; }  // IEEE fp32 divide, round-to-nearest
static inline float __fmul_rn(float a, float b) { volatile float r = a * b; return r; }   // never contracted
static inline float __fmaf_rn(float a, float b, float c) { return fmaf(a, b, c); }       // single rounding
template <typename T>
static inline T atomicAdd(T *p, T v) { T o = *p; *p = o + v; return o; }
template <typename T>
static inline T atomicMin(T *p, T v) { T o = *p; *p = std::min(o, v); return o; }
template <typename T>
static inline T atomicMax(T *p, T v) { T o = *p; *p = std::max(o, v); return o; }

#define JSS_SMEM_DECL(name) uint4 *name = reinterpret_cast<uint4 *>(emu::smem_ptr)

// ---- kernel launch -------------------------------------------------------------------
namespace emu {
template <typename... Args>
struct Pack;
template <typename A, typename B, typename C>
struct Pack<A, B, C> { void (*k)(A, B, C); A a; B b; C c; static void run(void *s) { auto *q = (Pack *)s; q->k(q->a, q->b, q->c); } };
template <typename A, typename B>
struct Pack<A, B> { void (*k)(A, B); A a; B b; static void run(void *s) { auto *q = (Pack *)s; q->k(q->a, q->b); } };
template <typename A, typename B, typename C>
void launch(void (*k)(A, B, C), dim3 g, dim3 b, size_t smem, A a, B bb, C c) { Pack<A, B, C> p{k, a, bb, c}; launch_impl(&Pack<A, B, C>::run, &p, g, b, smem); }
template <typename A, typename B>
void launch(void (*k)(A, B), dim3 g, dim3 b, size_t smem, A a, B bb) { Pack<A, B> p{k, a, bb}; launch_impl(&Pack<A, B>::run, &p, g, b, smem); }
template <typename A, typename B, typename C, typename A2, typename B2, typename C2>
void launch(void (*k)(A, B, C), dim3 g, dim3 b, size_t smem, A2 a, B2 bb, C2 c) { Pack<A, B, C> p{k, (A)a, (B)bb, (C)c}; launch_impl(&Pack<A, B, C>::run, &p, g, b, smem); }
}  // namespace emu
#define JSS_LAUNCH(kern, grid, block, smem, stream, ...) emu::launch(kern, dim3(grid), dim3(block), smem, __VA_ARGS__)

// ---- runtime API subset ----------------------------------------------------------------
typedef int cudaError_t;
typedef void *cudaStream_t;
#define cudaSuccess 0
enum cudaMemcpyKind { cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3 };
struct cudaDeviceProp { int major, minor, multiProcessorCount; };
static inline const char *cudaGetErrorString(cudaError_t) { return "emu"; }
static inline cudaError_t cudaGetDeviceCount(int *n) { *n = 1; return 0; }
static inline cudaError_t cudaGetDeviceProperties(cudaDeviceProp *p, int) { p->major = 9; p->minor = 0; p->multiProcessorCount = 2; return 0; }
static inline cudaError_t cudaSetDevice(int) { return 0; }
static inline cudaError_t cudaMalloc(void **p, size_t n) {
    const size_t bytes = (n + 255) / 256 * 256;
    *p = aligned_alloc(256, bytes);
    if (*p && emu::poison >= 0) memset(*p, emu::poison, bytes);   // device memory is not zeroed on allocation
    return *p ? 0 : 2;
}
static inline cudaError_t cudaFree(void *p) { free(p); return 0; }
static inline cudaError_t cudaFreeHost(void *p) { free(p); return 0; }
enum { cudaHostAllocMapped = 2, cudaHostAllocPortable = 1 };
static inline cudaError_t cudaHostAlloc(void **p, size_t n, unsigned) { *p = aligned_alloc(256, (n + 255) / 256 * 256); return *p ? 0 : 2; }
static inline cudaError_t cudaMemset(void *p, int v, size_t n) { memset(p, v, n); return 0; }
static inline cudaError_t cudaMemcpy(void *d, const void *s, size_t n, cudaMemcpyKind) { memcpy(d, s, n); return 0; }
static inline cudaError_t cudaMemcpyAsync(void *d, const void *s, size_t n, cudaMemcpyKind, cudaStream_t) { memcpy(d, s, n); return 0; }
static inline cudaError_t cudaMemcpy2DAsync(void *d, size_t dp, const void *s, size_t sp, size_t w, size_t h, cudaMemcpyKind, cudaStream_t) {
    for (size_t r = 0; r < h; r++) memcpy((char *)d + r * dp, (const char *)s + r * sp, w);
    return 0;
}
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return 0; }
static inline cudaError_t cudaHostGetDevicePointer(void **d, void *h, unsigned) { *d = h; return 0; }
typedef void *cudaEvent_t;
enum { cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2 };
static inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t *s, unsigned) { *s = nullptr; return 0; }
static inline cudaError_t cudaStreamDestroy(cudaStream_t) { return 0; }
static inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t *e, unsigned) { *e = nullptr; return 0; }
static inline cudaError_t cudaEventDestroy(cudaEvent_t) { return 0; }
static inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t) { return 0; }
static inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return 0; }
static inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned) { return 0; }
static inline cudaError_t cudaGetLastError() { return 0; }
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
template <typename F>
static inline cudaError_t cudaFuncSetAttribute(F, cudaFuncAttribute, int) { return 0; }
template <typename F>
static inline cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessor(int *n, F, int, size_t) { *n = 1; return 0; }
