// dcn_fused.cu -- DCNv2 forward with the deformable sampling fused into the tensor-core contraction.
//
// Reference: modulated_deformable_im2col (models/DCNv2/src/cuda/dcn_v2_im2col_cuda.cu:125-195) writes columns[B, Ci*9, h*w]
// to HBM and dcn_v2_cuda.cu:90-92 multiplies them by W[Co, Ci*9].  Here the columns never exist in HBM: per CTA (128
// output pixels) and tap, the 256 threads of two warpgroups evaluate the bilinear sample x mask for the tile's 128 pixels x
// 64 channels and write it as split bf16 directly in the 128-byte-swizzled K-major shared-memory layout that wgmma reads
// (hi and lo planes, chunk = deformable group, chunk index XOR (row & 7)); after fence.proxy.async and a barrier each
// warpgroup multiplies its 64 rows by the tap's weight tile (TMA) into register accumulators, and samples the next tap
// while those MMAs run.  The same threads then run the epilogue (bias + ReLU of STFusion.fuse, models/model.py:217) and
// store split bf16.  Warps: 0-7 = samplers / MMA / epilogue, 8 = weight TMA.  Two A + two B stages (96 KB): 2 CTAs per SM.
#include "tc_common.cuh"
#include "net.cuh"

namespace esr {

constexpr int DF_THREADS = 288;
constexpr uint32_t DF_B_BYTES = 64u * 128u;                       // one plane of the 64 x 64 weight tile
constexpr uint32_t DF_A_STAGE = 2u * TC_A_BYTES, DF_B_STAGE = 2u * DF_B_BYTES;

struct DcnFusedArgs {
    CUtensorMap bmap;                          // packed DCN weight: (64, 64, 2*9), box (64, 64, 1)
    const __nv_bfloat16 *feat; size_t f_plane; // features to sample (split, 64 ch), indexed through feat_img
    const int *feat_img;
    const float *om;                           // [n_img, H, W, 216]: 144 offsets, 72 masks (sigmoid applied)
    const float *bias;
    __nv_bfloat16 *out; size_t out_plane;      // [n_img, H, W, 64] split
    int n_img, H, W, TW, TH, tiles_x, tiles_y, act;
};

__device__ __forceinline__ void df_ld8(const __nv_bfloat16 *hi, size_t plane, float (&o)[8])
{
    const uint4 h = *reinterpret_cast<const uint4 *>(hi);
    const uint4 l = *reinterpret_cast<const uint4 *>(hi + plane);
    const uint32_t hw[4] = {h.x, h.y, h.z, h.w}, lw[4] = {l.x, l.y, l.z, l.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        o[2 * e] = __uint_as_float(hw[e] << 16) + __uint_as_float(lw[e] << 16);
        o[2 * e + 1] = __uint_as_float(hw[e] & 0xffff0000u) + __uint_as_float(lw[e] & 0xffff0000u);
    }
}

__global__ void __launch_bounds__(DF_THREADS, 2) k_dcn_fused(const __grid_constant__ DcnFusedArgs a)
{
    PDL_LAUNCH_DEPENDENTS();
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t *smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));        // generic pointer to the aligned base
    const uint32_t a_ring = smem_base, b_ring = smem_base + 2u * DF_A_STAGE;
    const uint32_t bar_base = b_ring + 2u * DF_B_STAGE;
    const uint32_t bar_bfull = bar_base, bar_bempty = bar_base + 16u;
    const int warp = threadIdx.x >> 5;

    const int tiles_per_img = a.tiles_x * a.tiles_y;
    const int img = blockIdx.x / tiles_per_img;
    const int trem = blockIdx.x - img * tiles_per_img;
    const int y0 = (trem / a.tiles_x) * a.TH, x0 = (trem % a.tiles_x) * a.TW;

    if (threadIdx.x == 0) {
        for (int s = 0; s < 2; ++s) { mbar_init(bar_bfull + 8u * s, 1); mbar_init(bar_bempty + 8u * s, 1); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    PDL_WAIT();                      // everything above is CTA-local set-up; global memory only from here on

    if (warp == 8) {
        if (elect_one_sync()) {
            for (int t = 0; t < 9; ++t) {
                const uint32_t s = t & 1, ph = (t >> 1) & 1;
                mbar_wait_backoff(bar_bempty + 8u * s, ph ^ 1u);
                mbar_expect_tx(bar_bfull + 8u * s, DF_B_STAGE);
                tma_load_3d(&a.bmap, bar_bfull + 8u * s, b_ring + s * DF_B_STAGE, 0, 0, t);
                tma_load_3d(&a.bmap, bar_bfull + 8u * s, b_ring + s * DF_B_STAGE + DF_B_BYTES, 0, 0, 9 + t);
            }
        }
        return;                      // the named barriers below count the 256 sampler threads
    }

    // ===================== samplers: 256 threads, 4 (pixel, group) items each per tap =====================
    const int st = threadIdx.x;                             // 0..255
    const int wg = warp >> 2;
    const int g = st & 7;                                   // deformable group: the same for this thread's 4 items
    // everything that does not depend on the tap is computed once per item (integer divisions, 64-bit addressing)
    const __nv_bfloat16 *f0 = a.feat + (size_t)(a.feat_img ? a.feat_img[img] : img) * a.H * a.W * 64 + g * 8;
    int iy[4], ix[4];
    const float *omp[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int m = (j * 256 + st) >> 3;
        iy[j] = y0 + m / a.TW; ix[j] = x0 + m % a.TW;
        const bool inb = iy[j] < a.H && ix[j] < a.W;
        if (!inb) iy[j] = -1000000;                         // far outside: every tap fails the range test below
        omp[j] = a.om + (((size_t)img * a.H + (inb ? iy[j] : 0)) * a.W + (inb ? ix[j] : 0)) * 216 + g * 18;
    }
    float acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.0f;
    for (int t = 0; t < 9; ++t) {
        const uint32_t s = t & 1, ph = (t >> 1) & 1;
        // stage s is free: the MMAs of tap t - 2 retired in both warpgroups before the barrier that ended the previous tap
        uint8_t *stage = smem_gen + (size_t)s * DF_A_STAGE;
        const int ty_ = t / 3 - 1, tx_ = t % 3 - 1;
        // the offsets / masks of this thread's 4 items first: one L2 round trip instead of one per item
        float oh[4], ow[4], omk[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            oh[j] = __ldg(omp[j] + 2 * t); ow[j] = __ldg(omp[j] + 2 * t + 1); omk[j] = __ldg(omp[j] + 144 - g * 9 + t);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int m = (j * 256 + st) >> 3;              // tile row (pixel)
            float v[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) v[e] = 0.0f;
            {
                const float mk = omk[j];
                const float h_im = (float)(iy[j] + ty_) + oh[j];
                const float w_im = (float)(ix[j] + tx_) + ow[j];
                // branch-free: corners are clamped into the image and always loaded (8 independent 16-byte loads in flight);
                // a corner outside the image, or a sample outside (-1, H) x (-1, W), gets weight 0 instead
                const bool ok = h_im > -1.0f && w_im > -1.0f && h_im < (float)a.H && w_im < (float)a.W;
                const float hf = floorf(h_im), wf = floorf(w_im);
                const int h_low = ok ? (int)hf : 0, w_low = ok ? (int)wf : 0;
                const float lh = h_im - hf, lw = w_im - wf;
                const float hh = 1.0f - lh, hw = 1.0f - lw;
                const bool t_ok = ok && h_low >= 0, b_ok = ok && h_low + 1 <= a.H - 1, l_ok = w_low >= 0, r_ok = w_low + 1 <= a.W - 1;
                const float w1 = (t_ok && l_ok) ? hh * hw : 0.0f, w2 = (t_ok && r_ok) ? hh * lw : 0.0f;
                const float w3 = (b_ok && l_ok) ? lh * hw : 0.0f, w4 = (b_ok && r_ok) ? lh * lw : 0.0f;
                const int r0 = max(h_low, 0) * a.W, r1 = min(h_low + 1, a.H - 1) * a.W;
                const int q0 = max(w_low, 0), q1 = min(w_low + 1, a.W - 1);
                float c1[8], c2[8], c3[8], c4[8];
                df_ld8(f0 + (r0 + q0) * 64, a.f_plane, c1);
                df_ld8(f0 + (r0 + q1) * 64, a.f_plane, c2);
                df_ld8(f0 + (r1 + q0) * 64, a.f_plane, c3);
                df_ld8(f0 + (r1 + q1) * 64, a.f_plane, c4);
#pragma unroll
                for (int e = 0; e < 8; ++e) v[e] = (w1 * c1[e] + w2 * c2[e] + w3 * c3[e] + w4 * c4[e]) * mk;
            }
            uint32_t hw_[4], lw_[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                split_pack2(v[2 * e], v[2 * e + 1], hw_[e], lw_[e]);
            }
            // K-major SWIZZLE_128B: row m at m*128, 16-byte chunk g stored at chunk (g ^ (m & 7))
            const uint32_t off = (uint32_t)m * 128u + (uint32_t)((g ^ (m & 7)) << 4);
            *reinterpret_cast<uint4 *>(stage + off) = make_uint4(hw_[0], hw_[1], hw_[2], hw_[3]);
            *reinterpret_cast<uint4 *>(stage + TC_A_BYTES + off) = make_uint4(lw_[0], lw_[1], lw_[2], lw_[3]);
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy stores -> visible to the tensor core
        named_sync(1, 256);                                             // the whole A tile of tap t is written
        mbar_wait(bar_bfull + 8u * s, ph);
        const uint32_t a_hi = a_ring + s * DF_A_STAGE + (uint32_t)wg * 8192u, a_lo = a_hi + TC_A_BYTES;
        const uint32_t b_hi = b_ring + s * DF_B_STAGE, b_lo = b_hi + DF_B_BYTES;
        acc_fence<32>(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            wgmma_rows<64, 0>(acc, wgmma_desc(a_lo) + 2 * k, wgmma_desc(b_hi) + 2 * k);
            wgmma_rows<64, 0>(acc, wgmma_desc(a_hi) + 2 * k, wgmma_desc(b_lo) + 2 * k);
            wgmma_rows<64, 0>(acc, wgmma_desc(a_hi) + 2 * k, wgmma_desc(b_hi) + 2 * k);
        }
        wgmma_commit();
        wgmma_wait<1>();                                                // tap t - 1 retired in this warpgroup
        acc_fence<32>(acc);
        named_sync(1, 256);                                             // ... and in the other one: its A and B stages are free
        if (st == 0 && t > 0) mbar_arrive(bar_bempty + 8u * ((t - 1) & 1));
    }
    wgmma_wait<0>();
    acc_fence<32>(acc);
    named_sync(1, 256);

    // ===================== epilogue: thread = (tile row r, 32-column half h) =====================
    float *stg = reinterpret_cast<float *>(smem_gen) + wg * (TC_STG_BYTES / 4);
    stage_acc<64>(acc, 0, stg);
    named_sync(2 + wg, 128);
    const int r = st & 63, half = (st >> 6) & 1;
    const int m = wg * 64 + r;
    const int y = y0 + m / a.TW, x = x0 + m % a.TW;
    if ((y < a.H) && (x < a.W)) {
        uint32_t raw[32];
        staged_row32(stg, r, half, 32, raw);
        float v[32];
        const float4 *bp = reinterpret_cast<const float4 *>(a.bias + half * 32);
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            const float4 b = bp[q];
            v[4 * q + 0] = __uint_as_float(raw[4 * q + 0]) + b.x;
            v[4 * q + 1] = __uint_as_float(raw[4 * q + 1]) + b.y;
            v[4 * q + 2] = __uint_as_float(raw[4 * q + 2]) + b.z;
            v[4 * q + 3] = __uint_as_float(raw[4 * q + 3]) + b.w;
        }
        act32(v, a.act);
        const size_t pix = ((size_t)img * a.H + y) * a.W + x;
        store_split32(a.out + pix * 64 + half * 32, a.out_plane, v);
    }
}

struct DcnFusedPlan { DcnFusedArgs args; unsigned grid; size_t smem; };

int dcn_fused_prepare(const SplitTensor &feat, const int *feat_img, const float *om, const void *wpacked, const float *bias,
                      int n_img, int act, const SplitTensor &out, void **plan_out)
{
    ESR_REQUIRE(feat.C == 64 && out.C == 64 && out.H == feat.H && out.W == feat.W, "dcn_fused: bad shapes");
    DcnFusedPlan *p = new DcnFusedPlan();
    DcnFusedArgs &a = p->args;
    memset(&a, 0, sizeof(a));
    int rc = tc_make_bmap(wpacked, 64, 9, 64, &a.bmap);
    if (rc) { delete p; return rc; }
    const int H = feat.H, W = feat.W;
    a.feat = feat.base; a.f_plane = feat.plane(); a.feat_img = feat_img; a.om = om; a.bias = bias;
    a.out = out.base; a.out_plane = out.plane(); a.n_img = n_img; a.H = H; a.W = W; a.act = act;
    a.TW = W >= 12 ? 16 : 8; a.TH = TC_BLOCK_M / a.TW;
    a.tiles_x = (W + a.TW - 1) / a.TW; a.tiles_y = (H + a.TH - 1) / a.TH;
    p->grid = (unsigned)(n_img * a.tiles_x * a.tiles_y);
    p->smem = 1024 + 2 * DF_A_STAGE + 2 * DF_B_STAGE + 64;
    cudaError_t e = cudaFuncSetAttribute(k_dcn_fused, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p->smem);
    if (e != cudaSuccess) { set_error("dcn_fused: %s", cudaGetErrorString(e)); delete p; return ESR_ECUDA; }
    *plan_out = p;
    return ESR_OK;
}

int dcn_fused_launch(void *plan, cudaStream_t st)
{
    DcnFusedPlan *p = (DcnFusedPlan *)plan;
    ESR_CUDA_CHECK(launch_pdl(k_dcn_fused, dim3(p->grid), dim3(DF_THREADS), p->smem, st, p->args));
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}

void dcn_fused_destroy(void *plan) { delete (DcnFusedPlan *)plan; }

} // namespace esr
