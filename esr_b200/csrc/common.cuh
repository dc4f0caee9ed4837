// common.cuh -- shared host/device helpers of libesr_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <atomic>

#include "../../include/esr_b200.h"

namespace esr {

void set_error(const char *fmt, ...);
extern std::atomic<long long> g_launches;
inline void count_launch(int n = 1) { g_launches.fetch_add(n, std::memory_order_relaxed); }

#define ESR_CUDA_CHECK(expr)                                                                       \
    do {                                                                                           \
        cudaError_t _e = (expr);                                                                   \
        if (_e != cudaSuccess) {                                                                   \
            esr::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
            (void)cudaGetLastError();  /* a non-sticky error is reported once, not again by the next launch */ \
            return ESR_ECUDA;                                                                      \
        }                                                                                          \
    } while (0)

#define ESR_LAUNCH_CHECK()                                                                         \
    do {                                                                                           \
        cudaError_t _e = cudaGetLastError();                                                       \
        if (_e != cudaSuccess) {                                                                   \
            esr::set_error("kernel launch failed: %s (%s:%d)", cudaGetErrorString(_e), __FILE__, __LINE__); \
            return ESR_ECUDA;                                                                      \
        }                                                                                          \
        esr::count_launch();                                                                       \
    } while (0)

#define ESR_REQUIRE(cond, ...)                                                                     \
    do {                                                                                           \
        if (!(cond)) {                                                                             \
            esr::set_error(__VA_ARGS__);                                                           \
            return ESR_EINVAL;                                                                     \
        }                                                                                          \
    } while (0)

// ---------------------------------------------------------------------------------------------
// Programmatic dependent launch (PDL).  The network is ~50 dependent kernels of 20-200 us; a normal stream edge drains the GPU
// between two of them (tail of the last wave, launch latency, the next kernel's prologue: barrier init,
// descriptor fetch).  With the programmatic-serialization attribute the next grid is launched as soon as every CTA of the
// current one has executed `griddepcontrol.launch_dependents` (first instruction of our kernels): its CTAs take over SMs as
// they free up and run their prologue, then block in `griddepcontrol.wait` until the predecessor grid has COMPLETED and its
// memory is visible.  Rules kept by every kernel launched through launch_pdl(): no global-memory access of any kind before
// PDL_WAIT().  Works inside stream capture (the edge becomes a programmatic graph dependency).
// ---------------------------------------------------------------------------------------------
#ifdef __CUDACC__
#define PDL_LAUNCH_DEPENDENTS() asm volatile("griddepcontrol.launch_dependents;" ::: "memory")
#define PDL_WAIT() asm volatile("griddepcontrol.wait;" ::: "memory")
#endif
template <typename... KArgs, typename... Args>
static inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args &&...args)
{
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

static inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }
static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// bump allocator over a caller-provided workspace (base == nullptr: size query only)
struct Bump {
    uint8_t *base; size_t off, cap;
    void *take(size_t bytes) { void *p = base ? base + off : nullptr; off = align_up(off + bytes, 256); return p; }
};

// device properties cache (immutable after first use)
struct DevInfo { int sm_count; int max_smem_optin; };
const DevInfo &dev_info();

// ---------------------------------------------------------------------------------------------
// split-bf16 activation storage: value = float(hi) + float(lo).  hi = RN_bf16(v), lo = RN_bf16(v - hi).
// The two planes are what the wgmma kernels consume directly as MMA operands (3-pass product
// hi*hi + lo*hi + hi*lo, fp32 accumulate), giving ~2^-17 relative operand error.
// ---------------------------------------------------------------------------------------------
#ifdef __CUDACC__
__device__ __forceinline__ void split_bf16(float v, __nv_bfloat16 &hi, __nv_bfloat16 &lo)
{
    hi = __float2bfloat16_rn(v);
    lo = __float2bfloat16_rn(v - __bfloat162float(hi));
}
// Gate activations of the epilogues: MUFU-based (ex2 + rcp), ~1e-6 relative error -- three orders below the 1e-3 parity
// budget; the IEEE expf / division / tanhf versions cost ~40-60 instructions per element and made the ConvGRU gate epilogue
// (128 sigmoids or 64 tanh per pixel) the longest part of every serial phase (clock64 trace, profiles/r1_notes.md).
__device__ __forceinline__ float fast_sigmoid(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }
__device__ __forceinline__ float fast_tanh(float x) { return 1.0f - __fdividef(2.0f, 1.0f + __expf(2.0f * x)); }

// two values at once: one packed cvt.rn.bf16x2.f32 per plane (same roundings as split_bf16; a in the low half)
__device__ __forceinline__ void split_pack2(float a, float b, uint32_t &hi, uint32_t &lo)
{
    const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    hi = *reinterpret_cast<const uint32_t *>(&h);
    const __nv_bfloat162 l = __floats2bfloat162_rn(a - __uint_as_float(hi << 16), b - __uint_as_float(hi & 0xffff0000u));
    lo = *reinterpret_cast<const uint32_t *>(&l);
}
__device__ __forceinline__ float join_bf16(__nv_bfloat16 hi, __nv_bfloat16 lo)
{
    return __bfloat162float(hi) + __bfloat162float(lo);
}
#endif

} // namespace esr
