// tc_common.cuh -- device-side building blocks shared by the Hopper tensor-core kernels (tc_conv.cu, dcn_fused.cu, wgrad_tc.cu):
// PTX wrappers (mbarrier, TMA, wgmma), shared-memory matrix descriptors, the accumulator staging of the epilogues, split-bf16 vector
// I/O and the fused conv epilogue.
#pragma once
#include "tc_conv.cuh"

namespace esr {

constexpr int TC_BLOCK_M = 128;                       // output pixels per tile: two warpgroups x 64 rows
constexpr int TC_A_BYTES = TC_BLOCK_M * 128;          // one plane of one A tile: 128 rows x 64 bf16
constexpr int TC_STG_LD = 68;                         // row stride (floats) of an epilogue staging tile: 64 columns + 4 (bank spread)
// one warpgroup's staging tile: 64 rows x 64 fp32 columns (the last row needs no bank padding: with it, npad = 256 at two
// stages would exceed the 227 KB of shared memory an H100 block may use)
constexpr uint32_t TC_STG_BYTES = (63u * TC_STG_LD + 64u) * 4u;

// ------------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// One lane of a CONVERGED warp (the single-thread TMA issuers).
__device__ __forceinline__ bool elect_one_sync()
{
    uint32_t pred;
    asm volatile(
        "{\n\t"
        ".reg .pred P;\n\t"
        "elect.sync _|P, 0xffffffff;\n\t"
        "selp.u32 %0, 1, 0, P;\n\t"
        "}" : "=r"(pred));
    return pred != 0;
}

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity)
{
    asm volatile(
        "{\n\t"
        ".reg .pred P1;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
        "@P1 bra DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "DONE:\n\t"
        "}" ::"r"(bar), "r"(parity) : "memory");
}
// same, for waits that last microseconds (a producer thread idling while other warps of the CTA do the real work): back off
// between polls so the spin does not eat the issue slots of the warps it is waiting for
__device__ __forceinline__ void mbar_wait_backoff(uint32_t bar, uint32_t parity)
{
    uint32_t done;
    do {
        asm volatile(
            "{\n\t"
            ".reg .pred P1;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, P1;\n\t"
            "}" : "=r"(done) : "r"(bar), "r"(parity) : "memory");
        if (!done) __nanosleep(40);
    } while (!done);
}
__device__ __forceinline__ void tma_load_5d(const CUtensorMap *map, uint32_t bar, uint32_t dst, int c0, int c1, int c2,
                                            int c3, int c4)
{
    asm volatile("cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes"
                 " [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
                 ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4) : "memory");
}
__device__ __forceinline__ void tma_load_3d(const CUtensorMap *map, uint32_t bar, uint32_t dst, int c0, int c1, int c2)
{
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
                 " [%0], [%1, {%3, %4, %5}], [%2];"
                 ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
// named barrier over `count` threads (id 0 is __syncthreads)
__device__ __forceinline__ void named_sync(int id, int count)
{
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// ------------------------------------------------------------------------------------------------
// wgmma (sm_90a): D[64 rows, N] (+)= A[64 x 16, smem] * B[16 x N, smem], bf16 x bf16 -> fp32 registers of one warpgroup.
// Accumulator fragment of thread (warp w of the warpgroup, lane l), register i:
//   row = 16 w + l / 4 + 8 ((i / 2) % 2),   column = 8 (i / 4) + 2 (l % 4) + i % 2
// ------------------------------------------------------------------------------------------------
// 128B-swizzled operand tile: rows of 128 bytes, 8-row groups 1024 bytes apart (SBO).  K-major: LBO unused.  MN-major: LBO =
// distance between 64-element column blocks.  Bits: start>>4 [0,14) | LBO>>4 [16,30) | SBO>>4 [32,46) | SWIZZLE_128B (1) [62,64).
// Advancing the operand by n bytes (n a multiple of 16, the result below 256 KB) is desc + n / 16.
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t smem_addr, uint32_t lbo_bytes = 16u)
{
    return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16) |
           ((uint64_t)(1024u >> 4) << 32) | ((uint64_t)1 << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
template <int R> __device__ __forceinline__ void acc_fence(float *acc)
{
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(acc[i])::"memory");
}

// TNSP = 0: both operands K-major; 1: both MN-major
template <int TNSP> __device__ __forceinline__ void wgmma_n16(float *d, uint64_t da, uint64_t db)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, %10, %10;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(da), "l"(db), "n"(TNSP));
}
template <int TNSP> __device__ __forceinline__ void wgmma_n32(float *d, uint64_t da, uint64_t db)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %18, %18;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(da), "l"(db), "n"(TNSP));
}
template <int TNSP> __device__ __forceinline__ void wgmma_n64(float *d, uint64_t da, uint64_t db)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %34, %34;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "n"(TNSP));
}
template <int TNSP> __device__ __forceinline__ void wgmma_n128(float *d, uint64_t da, uint64_t db)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31,"
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47,"
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %66, %66;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "n"(TNSP));
}
template <int TNSP> __device__ __forceinline__ void wgmma_n256(float *d, uint64_t da, uint64_t db)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 {"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31,"
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47,"
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63,"
        "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79,"
        "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95,"
        "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111,"
        "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, %130, %130;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
          "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
          "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
          "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
          "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
          "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
          "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
          "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
          "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(da), "l"(db), "n"(TNSP));
}

// D[64, NP] (+)= A * B for any NP that is a multiple of 16 up to 256: one instruction per set bit of NP (the fragment layout above
// makes the concatenated accumulators one [NP / 2] array).  The B operand of columns [c, ...) starts c rows (K-major) or c
// elements (MN-major, c a multiple of 64: c / 64 column blocks) further on.
template <int NP, int TNSP>
__device__ __forceinline__ void wgmma_rows(float *acc, uint64_t da, uint64_t db, uint32_t b_block_bytes = 0)
{
    constexpr int C256 = NP & 256, C128 = NP & 128, C64 = NP & 64, C32 = NP & 32, C16 = NP & 16;
    auto boff = [&](int c) -> uint64_t { return TNSP ? (uint64_t)((c / 64) * b_block_bytes >> 4) : (uint64_t)(c * 128 >> 4); };
    if constexpr (C256 != 0) wgmma_n256<TNSP>(acc, da, db);
    if constexpr (C128 != 0) wgmma_n128<TNSP>(acc + C256 / 2, da, db + boff(C256));
    if constexpr (C64 != 0) wgmma_n64<TNSP>(acc + (C256 + C128) / 2, da, db + boff(C256 + C128));
    if constexpr (C32 != 0) wgmma_n32<TNSP>(acc + (C256 + C128 + C64) / 2, da, db + boff(C256 + C128 + C64));
    if constexpr (C16 != 0) wgmma_n16<TNSP>(acc + (C256 + C128 + C64 + C32) / 2, da, db + boff(C256 + C128 + C64 + C32));
}

// Epilogue staging: columns [64 p, 64 p + 64) of a warpgroup's accumulator -> its [64][TC_STG_LD] fp32 tile in shared memory
// (row = accumulator row), so that each thread can then read one row's 32 consecutive columns.
template <int NP>
__device__ __forceinline__ void stage_acc(const float *acc, int p, float *stg)
{
    const int w = (threadIdx.x >> 5) & 3, l = threadIdx.x & 31;
    const int r0 = 16 * w + (l >> 2), c0 = 2 * (l & 3);
#pragma unroll
    for (int i = 0; i < NP / 2; i += 2) {
        if (i / 32 != p) continue;
        const int row = r0 + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) + c0 - 64 * p;
        *reinterpret_cast<float2 *>(stg + row * TC_STG_LD + col) = make_float2(acc[i], acc[i + 1]);
    }
}
// 32 staged columns [32 h, 32 h + 32) of row r (16 valid ones when only 16 remain: zeros above)
__device__ __forceinline__ void staged_row32(const float *stg, int r, int h, int nvalid, uint32_t (&raw)[32])
{
    const float4 *sp = reinterpret_cast<const float4 *>(stg + r * TC_STG_LD + 32 * h);
#pragma unroll
    for (int q = 0; q < 8; ++q) {
        const float4 v = (q < 4 || nvalid >= 32) ? sp[q] : make_float4(0.f, 0.f, 0.f, 0.f);
        raw[4 * q] = __float_as_uint(v.x); raw[4 * q + 1] = __float_as_uint(v.y);
        raw[4 * q + 2] = __float_as_uint(v.z); raw[4 * q + 3] = __float_as_uint(v.w);
    }
}

__device__ __forceinline__ float apply_act(float x, int act)
{
    if (act == ACT_RELU) return fmaxf(x, 0.0f);
    if (act == ACT_SIGMOID) return fast_sigmoid(x);
    if (act == ACT_TANH) return fast_tanh(x);
    return x;
}

// 32 consecutive channels of one pixel of a split tensor -> fp32
__device__ __forceinline__ void load_split32(const __nv_bfloat16 *hi_ptr, size_t plane, float (&o)[32])
{
    const uint4 *ph = reinterpret_cast<const uint4 *>(hi_ptr);
    const uint4 *pl = reinterpret_cast<const uint4 *>(hi_ptr + plane);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const uint4 h = ph[q], l = pl[q];
        const uint32_t hw[4] = {h.x, h.y, h.z, h.w}, lw[4] = {l.x, l.y, l.z, l.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            o[q * 8 + e * 2 + 0] = __uint_as_float(hw[e] << 16) + __uint_as_float(lw[e] << 16);
            o[q * 8 + e * 2 + 1] = __uint_as_float(hw[e] & 0xffff0000u) + __uint_as_float(lw[e] & 0xffff0000u);
        }
    }
}
__device__ __forceinline__ void store_split32(__nv_bfloat16 *hi_ptr, size_t plane, const float (&x)[32])
{
    uint32_t hw[16], lw[16];
#pragma unroll
    for (int e = 0; e < 16; ++e) {
        split_pack2(x[2 * e], x[2 * e + 1], hw[e], lw[e]);
    }
    uint4 *ph = reinterpret_cast<uint4 *>(hi_ptr);
    uint4 *pl = reinterpret_cast<uint4 *>(hi_ptr + plane);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        ph[q] = make_uint4(hw[q * 4], hw[q * 4 + 1], hw[q * 4 + 2], hw[q * 4 + 3]);
        pl[q] = make_uint4(lw[q * 4], lw[q * 4 + 1], lw[q * 4 + 2], lw[q * 4 + 3]);
    }
}

// activation over 32 values with a warp-uniform selector (no per-element branching)
__device__ __forceinline__ void act32(float (&v)[32], int act)
{
    if (act == ACT_RELU) {
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.0f);
    } else if (act == ACT_SIGMOID) {
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = fast_sigmoid(v[j]);
    } else if (act == ACT_TANH) {
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = fast_tanh(v[j]);
    }
}

// One thread's 32 accumulator columns [n0, n0+32) of one valid output pixel -> global memory.
// residual / activation part of the standard epilogue on 32 biased accumulator values (in place)
__device__ __forceinline__ void epilogue_std_math(const ConvTCArgs &a, float (&v)[32], int n0, int img, int y, int x, bool valid)
{
    // activation selector for this chunk: uniform unless act_from falls inside it (conv_offset_mask: 144 = 4.5 chunks)
    const bool mixed = (a.act_from > n0) && (a.act_from < n0 + 32);
    const int act = (n0 >= a.act_from) ? a.act : ACT_NONE;
    float r[32];
    const bool has_res = valid && a.res_mode != RES_NONE && n0 < a.cout;
    if (has_res) {
        const size_t rpix = ((size_t)(a.res_img ? a.res_img[img] : img) * a.H + y) * a.W + x;
        load_split32(a.res + rpix * a.res_C + n0, a.res_plane, r);
        if (a.res_mode == RES_PRE_ACT) {
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] += r[j];
        }
    }
    if (!mixed) act32(v, act);
    else {
#pragma unroll
        for (int j = 0; j < 32; ++j)
            if (n0 + j >= a.act_from) v[j] = apply_act(v[j], a.act);
    }
    if (has_res && a.res_mode == RES_POST_ACT) {
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] += r[j];
    }
}
__device__ __forceinline__ void epilogue_chunk(const ConvTCArgs &a, const uint32_t (&raw)[32], int n0, size_t pix, int img,
                                               int y, int x)
{
    float v[32];
    {
        // bias: 16-byte broadcast loads (npad is a multiple of 16, the blob is 256-byte aligned)
        const float4 *bp = reinterpret_cast<const float4 *>(a.bias + n0);
        const int nq = (a.npad - n0 >= 32) ? 8 : 4;
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            float4 b = make_float4(0.f, 0.f, 0.f, 0.f);
            if (q < nq) b = bp[q];
            v[4 * q + 0] = __uint_as_float(raw[4 * q + 0]) + b.x;
            v[4 * q + 1] = __uint_as_float(raw[4 * q + 1]) + b.y;
            v[4 * q + 2] = __uint_as_float(raw[4 * q + 2]) + b.z;
            v[4 * q + 3] = __uint_as_float(raw[4 * q + 3]) + b.w;
        }
    }

    if (a.epi_mode == EPI_GRU_ZR) {
        // channels [0,64): update gate z -> fp32; [64,128): reset gate r -> rh = h * r (split)
        act32(v, ACT_SIGMOID);
        if (n0 < 64) {
            float4 *zp = reinterpret_cast<float4 *>(a.z_buf + pix * 64 + n0);
#pragma unroll
            for (int q = 0; q < 8; ++q) zp[q] = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
        } else {
            float h[32];
            load_split32(a.h_prev + pix * 64 + (n0 - 64), a.h_plane, h);
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] *= h[j];
            store_split32(a.out + pix * a.out_C + a.out_coff + (n0 - 64), a.out_plane, v);
        }
        return;
    }
    if (a.epi_mode == EPI_GRU_OUT) {
        // h' = h (1 - z) + tanh(.) z        (models/submodules.py:511-512)
        float h[32];
        load_split32(a.h_prev + pix * 64 + n0, a.h_plane, h);
        const float4 *zp = reinterpret_cast<const float4 *>(a.z_buf + pix * 64 + n0);
        float4 zq[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) zq[q] = zp[q];
        act32(v, ACT_TANH);
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            const float zz[4] = {zq[q].x, zq[q].y, zq[q].z, zq[q].w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int j = 4 * q + e;
                v[j] = h[j] * (1.0f - zz[e]) + v[j] * zz[e];
            }
        }
        store_split32(a.out + pix * a.out_C + a.out_coff + n0, a.out_plane, v);
        return;
    }
    // ---- standard epilogue: bias (+ residual before or after the activation)
    epilogue_std_math(a, v, n0, img, y, x, true);
    if (a.out && n0 + 32 <= a.cout) store_split32(a.out + pix * a.out_C + a.out_coff + n0, a.out_plane, v);
    if (a.out_f32 && a.out_f32_nchw) {
        // the autograd layout of the training operators: consecutive lanes = consecutive pixels of a tile row -> each of the
        // 32 per-channel stores of a warp is one or two contiguous segments
        float *op = a.out_f32 + (((size_t)img * a.out_f32_C + n0) * a.H + y) * a.W + x;
        const size_t cs = (size_t)a.H * a.W;
#pragma unroll
        for (int j = 0; j < 32; ++j)
            if (n0 + j < a.cout) op[j * cs] = v[j];
    } else if (a.out_f32) {
        float *op = a.out_f32 + pix * a.out_f32_C + n0;
        if ((a.out_f32_C & 3) == 0) {                 // 16-byte stores (conv_offset_mask: 216 channels)
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                if (n0 + 4 * q + 4 <= a.cout)
                    reinterpret_cast<float4 *>(op)[q] = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
                else                                  // a cout that is not a multiple of 4 ends inside this quad
                    for (int e = 0; e < 4; ++e)
                        if (n0 + 4 * q + e < a.cout) op[4 * q + e] = v[4 * q + e];
            }
        } else {
#pragma unroll
            for (int j = 0; j < 32; ++j)
                if (n0 + j < a.cout) op[j] = v[j];
        }
    }
}

} // namespace esr
