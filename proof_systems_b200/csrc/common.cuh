// common.cuh — error handling, the owners of device memory, streams and events, vectorised element access, library-wide ids.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <utility>

#include "../../include/zkb200.h"
#include "curve.cuh"

namespace zkb {

// error codes: the ZK_ERR_* macros of include/zkb200.h
void zk_set_error(const char* fmt, ...);

#define ZK_CUDA(call)                                                                      \
    do {                                                                                   \
        cudaError_t e__ = (call);                                                          \
        if (e__ != cudaSuccess) {                                                          \
            zkb::zk_set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__)); \
            return ZK_ERR_CUDA;                                                       \
        }                                                                                  \
    } while (0)

// The library's device memory, streams and events live in the owners below and are released with them; only zk_dev_alloc's memory
// belongs to the caller.  Whoever destroys an owner makes its device current first (zk_ctx_destroy and the handles' free functions).

// Memory that grows on demand (the contents are not kept): device memory, or page-locked host memory with PINNED.  Moving hands the
// buffer over, so a table built in a local owner is published to a cache only once it is complete.
template <bool PINNED> struct Scratch {
    void* p = nullptr;
    size_t cap = 0;
    Scratch() = default;
    Scratch(const Scratch&) = delete;
    Scratch& operator=(const Scratch&) = delete;
    Scratch(Scratch&& o) noexcept : p(std::exchange(o.p, nullptr)), cap(std::exchange(o.cap, 0)) {}
    Scratch& operator=(Scratch&& o) noexcept { std::swap(p, o.p), std::swap(cap, o.cap); return *this; }   // the old buffer leaves with o
    ~Scratch() { release(); }
    void release() {
        if (p) PINNED ? cudaFreeHost(p) : cudaFree(p);
        p = nullptr, cap = 0;
    }
    int ensure(size_t bytes) {
        if (cap >= bytes) return ZK_OK;
        release();
        ZK_CUDA(PINNED ? cudaMallocHost(&p, bytes) : cudaMalloc(&p, bytes));
        cap = bytes;
        return ZK_OK;
    }
    template <class T> T* at(size_t byte_off = 0) const { return (T*)((char*)p + byte_off); }
};
using DevScratch = Scratch<false>;
using PinnedScratch = Scratch<true>;

// sub-buffers of one scratch allocation: add() hands out 256-byte aligned offsets in order, total is the size to ensure
struct Layout {
    size_t total = 0;
    size_t add(size_t bytes) { const size_t off = (total + 255) & ~(size_t)255; total = off + bytes; return off; }
};

// A CUDA event, and a CUDA stream (the library's own are non-blocking).  create() makes the handle on its first call only, so a
// member created on first use is created once however often that use is reached, also after a failed attempt.
struct Event {
    cudaEvent_t e = nullptr;
    Event() = default;
    Event(const Event&) = delete;
    Event& operator=(const Event&) = delete;
    ~Event() { if (e) cudaEventDestroy(e); }
    cudaError_t create(unsigned flags) { return e ? cudaSuccess : cudaEventCreateWithFlags(&e, flags); }
};
struct Stream {
    cudaStream_t s = nullptr;
    Stream() = default;
    Stream(const Stream&) = delete;
    Stream& operator=(const Stream&) = delete;
    ~Stream() { if (s) cudaStreamDestroy(s); }
    cudaError_t create(unsigned flags) { return s ? cudaSuccess : cudaStreamCreateWithFlags(&s, flags); }
};

// 128-bit vector access: an fe is two uint4, an affine point four, an XYZZ point eight.
__device__ __forceinline__ fe load_fe(const fe* p) {
    const uint4* q = reinterpret_cast<const uint4*>(p);
    uint4 a = q[0], b = q[1];
    fe r;
    r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w;
    r.v[4] = b.x; r.v[5] = b.y; r.v[6] = b.z; r.v[7] = b.w;
    return r;
}
__device__ __forceinline__ fe load_fe_nc(const fe* p) {
    const uint4* q = reinterpret_cast<const uint4*>(p);
    uint4 a = __ldg(q), b = __ldg(q + 1);
    fe r;
    r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w;
    r.v[4] = b.x; r.v[5] = b.y; r.v[6] = b.z; r.v[7] = b.w;
    return r;
}
__device__ __forceinline__ void store_fe(fe* p, const fe& r) {
    uint4* q = reinterpret_cast<uint4*>(p);
    q[0] = make_uint4(r.v[0], r.v[1], r.v[2], r.v[3]);
    q[1] = make_uint4(r.v[4], r.v[5], r.v[6], r.v[7]);
}
__device__ __forceinline__ affine_t load_affine_nc(const affine_t* p) {
    affine_t r;
    r.x = load_fe_nc(&p->x);
    r.y = load_fe_nc(&p->y);
    return r;
}
__device__ __forceinline__ void store_affine(affine_t* p, const affine_t& r) {
    store_fe(&p->x, r.x);
    store_fe(&p->y, r.y);
}
__device__ __forceinline__ xyzz_t load_xyzz(const xyzz_t* p) {
    xyzz_t r;
    r.X = load_fe(&p->X); r.Y = load_fe(&p->Y); r.ZZ = load_fe(&p->ZZ); r.ZZZ = load_fe(&p->ZZZ);
    return r;
}
__device__ __forceinline__ void store_xyzz(xyzz_t* p, const xyzz_t& r) {
    store_fe(&p->X, r.X); store_fe(&p->Y, r.Y); store_fe(&p->ZZ, r.ZZ); store_fe(&p->ZZZ, r.ZZZ);
}

__device__ __forceinline__ fe shfl_fe(const fe& a, int src_lane) {
    fe r;
#pragma unroll
    for (int i = 0; i < 8; i++) r.v[i] = __shfl_sync(0xffffffffu, a.v[i], src_lane);
    return r;
}
__device__ __forceinline__ fe shfl_xor_fe(const fe& a, int m) {
    fe r;
#pragma unroll
    for (int i = 0; i < 8; i++) r.v[i] = __shfl_xor_sync(0xffffffffu, a.v[i], m);
    return r;
}
__device__ __forceinline__ fe shfl_up_fe(const fe& a, unsigned d) {
    fe r;
#pragma unroll
    for (int i = 0; i < 8; i++) r.v[i] = __shfl_up_sync(0xffffffffu, a.v[i], d);
    return r;
}
__device__ __forceinline__ fe shfl_down_fe(const fe& a, unsigned d) {
    fe r;
#pragma unroll
    for (int i = 0; i < 8; i++) r.v[i] = __shfl_down_sync(0xffffffffu, a.v[i], d);
    return r;
}
__device__ __forceinline__ xyzz_t shfl_up_xyzz(const xyzz_t& p, unsigned d) {
    xyzz_t r;
    r.X = shfl_up_fe(p.X, d); r.Y = shfl_up_fe(p.Y, d); r.ZZ = shfl_up_fe(p.ZZ, d); r.ZZZ = shfl_up_fe(p.ZZZ, d);
    return r;
}
__device__ __forceinline__ xyzz_t shfl_down_xyzz(const xyzz_t& p, unsigned d) {
    xyzz_t r;
    r.X = shfl_down_fe(p.X, d); r.Y = shfl_down_fe(p.Y, d); r.ZZ = shfl_down_fe(p.ZZ, d); r.ZZZ = shfl_down_fe(p.ZZZ, d);
    return r;
}

}  // namespace zkb
