// lpips.cu -- LPIPS (version 0.1, AlexNet backbone, linear heads) on the Hopper tensor cores, split-bf16 three-term precision.
//
// Reference: loss/restore.py:10-39 perceptual_loss -> loss/PerceptualSimilarity/models/__init__.py:19-46 PerceptualLoss
// (normalize: 2x - 1) -> networks_basic.py:32-101 PNetLin.forward: ScalingLayer (:103-110), pretrained_networks.py:57-95
// alexnet (torchvision alexnet().features sliced at relu1 .. relu5), normalize_tensor (__init__.py:48-50, eps 1e-10), the
// squared difference, NetLinLayer (1x1 conv, no bias; dropout is the identity in eval) and spatial_average, summed over the
// five layers.
//
//   conv1 (3 -> 64, 11x11 / 4, pad 2) + ReLU   k_lpips_conv1: the 128 output pixels x 363 (padded to 384) im2col operand is
//                                              built in shared memory per 64-wide K-block, input transform applied per channel
//   maxpool 3x3 / 2                            k_lpips_maxpool on split tensors (copies the (hi, lo) pair of the maximum: exact)
//   conv2 (64 -> 192, 5x5, pad 2) + ReLU       k_conv_tc<192, 5> (one A box per kernel column, reused by its five taps)
//   maxpool 3x3 / 2                            k_lpips_maxpool
//   conv3 (192 -> 384) + ReLU                  k_conv_tc<192>, twice (output channels 0-191 and 192-383 through out_coff)
//   conv4 (384 -> 256), conv5 (256 -> 256)     k_conv_tc<256>
//   heads                                      k_lpips_head: per (pair, layer, 64-pixel block) a partial sum in fp64;
//                                              k_lpips_finish: per pair, layers in order, blocks in order -> deterministic, and a
//                                              pair's value does not depend on what else is in the batch
#include "tc_common.cuh"
#include <algorithm>

namespace esr {

constexpr int LP_K1 = 363;                          // 3 x 11 x 11: conv1's reduction length
constexpr int LP_KB1 = 6;                           // 64-wide K-blocks after padding to 384
constexpr uint32_t LP_B1_BYTES = 64u * 128u;        // one plane of one conv1 K-block: 64 outputs x 64 K
constexpr uint32_t LP_A1_STAGE = 2u * TC_A_BYTES;   // hi + lo planes of one A K-block
constexpr int LP_HEAD_PIX = 64;                     // pixels per head block: 8 warps x 8 pixels
constexpr int LP_NLAYER = 5;
static const int LP_CH[LP_NLAYER] = {64, 192, 384, 256, 256};

// ------------------------------------------------------------------------------------------------
// conv1
// ------------------------------------------------------------------------------------------------
struct LpConv1Args {
    CUtensorMap bmap;                     // packed conv1 weight [2][6][64][64] bf16, box (64, 64, 1)
    const float *planes;                  // fp32 [*][H][W]
    const int *chan_src;                  // [n_img][3]: the plane of each input channel
    const float *bias;                    // [64]
    __nv_bfloat16 *out; size_t out_plane; // relu1, split [n_img][Ho][Wo][64]
    int H, W, Ho, Wo, TW, TH, tiles_x, tiles_y, normalize;
};

// normalize (PerceptualLoss.forward: 2x - 1), then ScalingLayer ((x - shift_c) / scale_c), in fp32 like torch
__device__ __forceinline__ float lp_scale(float x, int c, int normalize)
{
    const float shift = c == 0 ? -0.030f : c == 1 ? -0.088f : -0.188f;
    const float scale = c == 0 ? 0.458f : c == 1 ? 0.448f : 0.450f;
    if (normalize) x = 2.0f * x - 1.0f;
    return (x - shift) / scale;
}

__global__ void __launch_bounds__(256, 1) k_lpips_conv1(const __grid_constant__ LpConv1Args a)
{
    extern __shared__ uint8_t smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t *gen = smem_raw + (base - smem_u32(smem_raw));
    const uint32_t b_base = base + 2u * LP_A1_STAGE, bar = b_base + 2u * LP_KB1 * LP_B1_BYTES;
    const int tiles_per_img = a.tiles_x * a.tiles_y;
    const int img = blockIdx.x / tiles_per_img, trem = blockIdx.x - img * tiles_per_img;
    const int y0 = (trem / a.tiles_x) * a.TH, x0 = (trem % a.tiles_x) * a.TW;
    const int st = threadIdx.x, wg = st >> 7, g = st & 7;

    if (st == 0) {
        mbar_init(bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (st == 0) {                       // the whole weight (96 KB) once: 6 hi then 6 lo K-blocks
        mbar_expect_tx(bar, 2u * LP_KB1 * LP_B1_BYTES);
        for (int i = 0; i < 2 * LP_KB1; ++i) tma_load_3d(&a.bmap, bar, b_base + (uint32_t)i * LP_B1_BYTES, 0, 0, i);
    }

    // this thread's 4 tile rows (pixels) and 16-byte column chunk g (K values 8 g .. 8 g + 7 of each K-block)
    const size_t HW = (size_t)a.H * a.W;
    const float *p0 = a.planes + (size_t)a.chan_src[img * 3 + 0] * HW;
    const float *p1 = a.planes + (size_t)a.chan_src[img * 3 + 1] * HW;
    const float *p2 = a.planes + (size_t)a.chan_src[img * 3 + 2] * HW;
    int iy0[4], ix0[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int m = (j * 256 + st) >> 3;
        const int oy = y0 + m / a.TW, ox = x0 + m % a.TW;
        const bool inb = oy < a.Ho && ox < a.Wo;
        iy0[j] = inb ? oy * 4 - 2 : -1000000;          // far outside: every tap fails the range test
        ix0[j] = ox * 4 - 2;
    }
    float acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.0f;
    for (int kb = 0; kb < LP_KB1; ++kb) {
        const uint32_t s = kb & 1;
        uint8_t *stage = gen + s * LP_A1_STAGE;
        int kc[8], ky[8], kx[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            const int k = kb * 64 + g * 8 + e;                  // torch's flattening of [64, 3, 11, 11]: c * 121 + ky * 11 + kx
            const int c = k / 121, r = k - 121 * c;
            kc[e] = k < LP_K1 ? c : -1;
            ky[e] = r / 11; kx[e] = r - 11 * (r / 11);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int m = (j * 256 + st) >> 3;
            float v[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const int iy = iy0[j] + ky[e], ix = ix0[j] + kx[e];
                const bool ok = kc[e] >= 0 && iy >= 0 && iy < a.H && ix >= 0 && ix < a.W;
                const float *pc = kc[e] == 0 ? p0 : kc[e] == 1 ? p1 : p2;
                // zero padding is applied after the transform, as torch pads the transformed tensor
                v[e] = ok ? lp_scale(__ldg(pc + (size_t)iy * a.W + ix), kc[e], a.normalize) : 0.0f;
            }
            uint32_t hw_[4], lw_[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) split_pack2(v[2 * e], v[2 * e + 1], hw_[e], lw_[e]);
            // K-major SWIZZLE_128B: row m at m * 128, 16-byte chunk g stored at chunk (g ^ (m & 7))
            const uint32_t off = (uint32_t)m * 128u + (uint32_t)((g ^ (m & 7)) << 4);
            *reinterpret_cast<uint4 *>(stage + off) = make_uint4(hw_[0], hw_[1], hw_[2], hw_[3]);
            *reinterpret_cast<uint4 *>(stage + TC_A_BYTES + off) = make_uint4(lw_[0], lw_[1], lw_[2], lw_[3]);
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy stores -> visible to the tensor core
        __syncthreads();                                                // the whole A block kb is written
        if (kb == 0) mbar_wait(bar, 0);
        const uint32_t a_hi = base + s * LP_A1_STAGE + (uint32_t)wg * 8192u, a_lo = a_hi + TC_A_BYTES;
        const uint32_t b_hi = b_base + (uint32_t)kb * LP_B1_BYTES, b_lo = b_base + (uint32_t)(LP_KB1 + kb) * LP_B1_BYTES;
        acc_fence<32>(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            wgmma_rows<64, 0>(acc, wgmma_desc(a_lo) + 2 * k, wgmma_desc(b_hi) + 2 * k);   // small terms first
            wgmma_rows<64, 0>(acc, wgmma_desc(a_hi) + 2 * k, wgmma_desc(b_lo) + 2 * k);
            wgmma_rows<64, 0>(acc, wgmma_desc(a_hi) + 2 * k, wgmma_desc(b_hi) + 2 * k);
        }
        wgmma_commit();
        wgmma_wait<1>();                                                // block kb - 1 retired in this warpgroup
        acc_fence<32>(acc);
        __syncthreads();                                                // ... and in the other one: its A stage is free
    }
    wgmma_wait<0>();
    acc_fence<32>(acc);
    __syncthreads();                                                    // the A stages become the epilogue's staging

    // ===================== epilogue: thread = (tile row r, 32-column half h): bias, ReLU, split store =====================
    float *stg = reinterpret_cast<float *>(gen) + wg * (TC_STG_BYTES / 4);
    stage_acc<64>(acc, 0, stg);
    named_sync(2 + wg, 128);
    const int r = st & 63, half = (st >> 6) & 1;
    const int m = wg * 64 + r;
    const int y = y0 + m / a.TW, x = x0 + m % a.TW;
    if (y < a.Ho && x < a.Wo) {
        uint32_t raw[32];
        staged_row32(stg, r, half, 32, raw);
        float v[32];
#pragma unroll
        for (int q = 0; q < 32; ++q) v[q] = fmaxf(__uint_as_float(raw[q]) + a.bias[half * 32 + q], 0.0f);
        const size_t pix = ((size_t)img * a.Ho + y) * a.Wo + x;
        store_split32(a.out + pix * 64 + half * 32, a.out_plane, v);
    }
}

static size_t lp_conv1_smem() { return 1024 + 2 * LP_A1_STAGE + 2 * LP_KB1 * LP_B1_BYTES + 16; }

// w [64, 3, 11, 11] fp32 -> [2][6][64 outputs][64 K] split bf16, K = c * 121 + ky * 11 + kx, zero beyond 363
__global__ void k_lpips_pack_conv1(const float *__restrict__ w, __nv_bfloat16 *__restrict__ dst)
{
    constexpr int total = LP_KB1 * 64 * 64;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int c = i % 64, n = (i / 64) % 64, kb = i / 4096;
        const int k = kb * 64 + c;
        __nv_bfloat16 hi, lo;
        split_bf16(k < LP_K1 ? w[n * LP_K1 + k] : 0.0f, hi, lo);
        dst[i] = hi;
        dst[total + i] = lo;
    }
}

// ------------------------------------------------------------------------------------------------
// max pool 3x3 / 2 (no padding, floor) on split NHWC tensors: hi + lo is exact in fp32, so comparing the joined values and
// copying the winning pair keeps the pooled tensor bit-exact
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_lpips_maxpool(const __nv_bfloat16 *__restrict__ in, size_t in_plane, int Hi, int Wi, int C,
                                                       __nv_bfloat16 *__restrict__ out, size_t out_plane, int Ho, int Wo, int n_img)
{
    const size_t total = (size_t)n_img * Ho * Wo * C;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const size_t p = i / C;
        const int x = (int)(p % Wo), y = (int)((p / Wo) % Ho), n = (int)(p / ((size_t)Wo * Ho));
        const size_t s0 = (((size_t)n * Hi + 2 * y) * Wi + 2 * x) * C + c;
        __nv_bfloat16 bh = in[s0], bl = in[in_plane + s0];
        float best = join_bf16(bh, bl);
#pragma unroll
        for (int t = 1; t < 9; ++t) {
            const size_t s = s0 + ((size_t)(t / 3) * Wi + t % 3) * C;
            const __nv_bfloat16 h = in[s], l = in[in_plane + s];
            const float v = join_bf16(h, l);
            if (v > best) { best = v; bh = h; bl = l; }
        }
        out[i] = bh;
        out[out_plane + i] = bl;
    }
}

// ------------------------------------------------------------------------------------------------
// heads: grid (blocks of the largest layer, pairs, layers)
// ------------------------------------------------------------------------------------------------
struct LpHeadArgs {
    const __nv_bfloat16 *f[LP_NLAYER]; size_t plane[LP_NLAYER];
    const float *lin[LP_NLAYER];
    int C[LP_NLAYER], HW[LP_NLAYER];
};

__device__ __forceinline__ float warp_sum_to_all(float v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    return __shfl_sync(0xffffffffu, v, 0);           // lane 0's total, the same bits in every lane
}

__global__ void __launch_bounds__(256) k_lpips_head(const __grid_constant__ LpHeadArgs a, const int *__restrict__ pair_a,
                                                    const int *__restrict__ pair_b, int nblk, double *__restrict__ partial)
{
    __shared__ double wsum[8];
    const int l = blockIdx.z, pair = blockIdx.y, HW = a.HW[l], C = a.C[l];
    if (blockIdx.x * LP_HEAD_PIX >= HW) return;       // past this layer's last block (the finish reads only the real ones)
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const __nv_bfloat16 *fa = a.f[l] + (size_t)pair_a[pair] * HW * C, *fb = a.f[l] + (size_t)pair_b[pair] * HW * C;
    const size_t plane = a.plane[l];
    const float *w = a.lin[l];
    double acc = 0.0;
    for (int q = 0; q < LP_HEAD_PIX / 8; ++q) {
        const int p = blockIdx.x * LP_HEAD_PIX + warp * (LP_HEAD_PIX / 8) + q;
        if (p >= HW) break;
        const __nv_bfloat16 *pa = fa + (size_t)p * C, *pb = fb + (size_t)p * C;
        float sa = 0.0f, sb = 0.0f;
        for (int c = lane; c < C; c += 32) {
            const float va = join_bf16(pa[c], pa[plane + c]), vb = join_bf16(pb[c], pb[plane + c]);
            sa += va * va; sb += vb * vb;
        }
        const float na = sqrtf(warp_sum_to_all(sa)) + 1e-10f, nb = sqrtf(warp_sum_to_all(sb)) + 1e-10f;
        float d = 0.0f;
        for (int c = lane; c < C; c += 32) {
            const float va = join_bf16(pa[c], pa[plane + c]), vb = join_bf16(pb[c], pb[plane + c]);
            const float df = va / na - vb / nb;
            d += w[c] * (df * df);
        }
        d = warp_sum_to_all(d);
        acc += (double)d;
    }
    if (lane == 0) wsum[warp] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int i = 0; i < 8; ++i) s += wsum[i];
        partial[((size_t)pair * LP_NLAYER + l) * nblk + blockIdx.x] = s;
    }
}

__global__ void k_lpips_finish(const double *__restrict__ partial, int nblk, LpHeadArgs a, int n_pairs, double *__restrict__ out)
{
    const int pair = blockIdx.x * blockDim.x + threadIdx.x;
    if (pair >= n_pairs) return;
    double v = 0.0;
    for (int l = 0; l < LP_NLAYER; ++l) {
        const int nb = (a.HW[l] + LP_HEAD_PIX - 1) / LP_HEAD_PIX;
        double s = 0.0;
        for (int b = 0; b < nb; ++b) s += partial[((size_t)pair * LP_NLAYER + l) * nblk + b];
        v += s / (double)a.HW[l];
    }
    out[pair] = v;
}

// ------------------------------------------------------------------------------------------------
// host side: parameter blob, workspace, plan
// ------------------------------------------------------------------------------------------------
struct LpLayout {
    size_t w1, b1, w2, b2, w3[2], b3, w4, b4, w5, b5, lin[LP_NLAYER], total;
};
static LpLayout lp_layout()
{
    LpLayout L;
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t r = off; off = align_up(off + bytes, 1024); return r; };
    L.w1 = take((size_t)2 * LP_KB1 * 64 * 64 * sizeof(__nv_bfloat16)); L.b1 = take(64 * sizeof(float));
    L.w2 = take(tc_packed_weight_bytes(192, 64, 25)); L.b2 = take(192 * sizeof(float));
    L.w3[0] = take(tc_packed_weight_bytes(192, 192, 9)); L.w3[1] = take(tc_packed_weight_bytes(192, 192, 9));
    L.b3 = take(384 * sizeof(float));
    L.w4 = take(tc_packed_weight_bytes(256, 384, 9)); L.b4 = take(256 * sizeof(float));
    L.w5 = take(tc_packed_weight_bytes(256, 256, 9)); L.b5 = take(256 * sizeof(float));
    for (int l = 0; l < LP_NLAYER; ++l) L.lin[l] = take(LP_CH[l] * sizeof(float));
    L.total = off;
    return L;
}

struct LpGeo {
    int h[4], w[4];                 // [0] input, [1] conv1 / relu1, [2] pool1 / relu2, [3] pool2 / relu3-5
    int nblk;                       // head blocks of the largest layer (relu1)
};
static bool lp_geo(int H, int W, LpGeo *g)
{
    g->h[0] = H; g->w[0] = W;
    if (H < 7 || W < 7) return false;
    g->h[1] = (H - 7) / 4 + 1; g->w[1] = (W - 7) / 4 + 1;
    if (g->h[1] < 3 || g->w[1] < 3) return false;
    g->h[2] = (g->h[1] - 3) / 2 + 1; g->w[2] = (g->w[1] - 3) / 2 + 1;
    if (g->h[2] < 3 || g->w[2] < 3) return false;       // the second pool needs a 3 x 3 window: H, W >= 31
    g->h[3] = (g->h[2] - 3) / 2 + 1; g->w[3] = (g->w[2] - 3) / 2 + 1;
    g->nblk = (g->h[1] * g->w[1] + LP_HEAD_PIX - 1) / LP_HEAD_PIX;
    return true;
}

struct LpWs { size_t f1, p1, f2, p2, f3, f4, f5, partial, total; };
static LpWs lp_ws(int N, const LpGeo &g)
{
    LpWs s;
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t r = off; off = align_up(off + bytes, 1024); return r; };
    auto split = [&](int h, int w, int C) { return take((size_t)2 * N * h * w * C * sizeof(__nv_bfloat16)); };
    s.f1 = split(g.h[1], g.w[1], 64); s.p1 = split(g.h[2], g.w[2], 64); s.f2 = split(g.h[2], g.w[2], 192);
    s.p2 = split(g.h[3], g.w[3], 192); s.f3 = split(g.h[3], g.w[3], 384); s.f4 = split(g.h[3], g.w[3], 256);
    s.f5 = split(g.h[3], g.w[3], 256);
    s.partial = take((size_t)N * LP_NLAYER * g.nblk * sizeof(double));
    s.total = off;
    return s;
}

struct LpPlan {
    int N;
    LpGeo g;
    LpConv1Args c1;
    size_t c1_smem;
    SplitTensor f1, p1, f2, p2;
    ConvTCArgs c2, c3[2], c4, c5;
    LpHeadArgs head;
    double *partial;
};

static SplitTensor lp_split(uint8_t *base, int N, int h, int w, int C)
{
    SplitTensor t;
    t.base = (__nv_bfloat16 *)base; t.n_img = N; t.H = h; t.W = w; t.C = C;
    return t;
}

static int lp_conv(const SplitTensor &src, int ntaps, int cout, const uint8_t *wp, const float *bias, const SplitTensor &out,
                   int out_coff, ConvTCArgs *args)
{
    ConvTCDesc d;
    d.src[0] = src; d.n_src = 1; d.ntaps = ntaps; d.cout = cout; d.wpacked = wp; d.bias = bias; d.n_img = src.n_img;
    d.act = ACT_RELU; d.out = out; d.out_coff = out_coff;
    return conv_tc_prepare(d, args);
}

static int lp_maxpool(const SplitTensor &in, const SplitTensor &out, int n_img, cudaStream_t st)
{
    const size_t total = (size_t)n_img * out.H * out.W * out.C;
    const unsigned grid = (unsigned)std::min<int64_t>(ceil_div64((int64_t)total, 256), (int64_t)dev_info().sm_count * 16);
    k_lpips_maxpool<<<grid, 256, 0, st>>>(in.base, in.plane(), in.H, in.W, in.C, out.base, out.plane(), out.H, out.W, n_img);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}

} // namespace esr

using namespace esr;

extern "C" size_t esr_lpips_param_bytes(void) { return lp_layout().total; }

extern "C" int esr_lpips_pack_params(const float *const *params, void *blob, esr_stream_t stream)
{
    ESR_REQUIRE(params && blob, "esr_lpips_pack_params: null pointer");
    for (int i = 0; i < 15; ++i) ESR_REQUIRE(params[i], "esr_lpips_pack_params: parameter %d is null", i);
    cudaStream_t st = (cudaStream_t)stream;
    const LpLayout L = lp_layout();
    uint8_t *b = (uint8_t *)blob;
    k_lpips_pack_conv1<<<96, 256, 0, st>>>(params[0], (__nv_bfloat16 *)(b + L.w1));
    ESR_LAUNCH_CHECK();
    int rc;
    if ((rc = pack_conv_weight(params[2], 192, 64, 5, b + L.w2, st))) return rc;
    if ((rc = pack_conv_weight(params[4], 192, 192, 3, b + L.w3[0], st))) return rc;
    if ((rc = pack_conv_weight(params[4] + (size_t)192 * 192 * 9, 192, 192, 3, b + L.w3[1], st))) return rc;
    if ((rc = pack_conv_weight(params[6], 256, 384, 3, b + L.w4, st))) return rc;
    if ((rc = pack_conv_weight(params[8], 256, 256, 3, b + L.w5, st))) return rc;
    const size_t bias_off[5] = {L.b1, L.b2, L.b3, L.b4, L.b5};
    for (int l = 0; l < LP_NLAYER; ++l) {
        ESR_CUDA_CHECK(cudaMemcpyAsync(b + bias_off[l], params[2 * l + 1], LP_CH[l] * sizeof(float), cudaMemcpyDeviceToDevice, st));
        ESR_CUDA_CHECK(cudaMemcpyAsync(b + L.lin[l], params[10 + l], LP_CH[l] * sizeof(float), cudaMemcpyDeviceToDevice, st));
    }
    return ESR_OK;
}

extern "C" size_t esr_lpips_workspace_bytes(int n_img, int H, int W)
{
    LpGeo g;
    if (n_img < 1 || !lp_geo(H, W, &g)) return 0;
    return lp_ws(n_img, g).total;
}

extern "C" int esr_lpips_create(esr_lpips_t *plan_out, int n_img, int H, int W, const void *blob, void *workspace, size_t ws_bytes)
{
    ESR_REQUIRE(plan_out && blob && workspace, "esr_lpips_create: null pointer");
    *plan_out = nullptr;
    LpGeo g;
    ESR_REQUIRE(n_img >= 1 && n_img <= 65535, "esr_lpips_create: n_img %d", n_img);
    ESR_REQUIRE(lp_geo(H, W, &g), "esr_lpips_create: a %d x %d image is too small for AlexNet's second max-pool (LPIPS needs "
                "at least 31 x 31)", H, W);
    const LpWs s = lp_ws(n_img, g);
    if (ws_bytes < s.total) { set_error("esr_lpips_create: workspace %zu < %zu", ws_bytes, s.total); return ESR_EWORKSPACE; }
    const LpLayout L = lp_layout();
    const uint8_t *b = (const uint8_t *)blob;
    uint8_t *ws = (uint8_t *)workspace;
    LpPlan *p = new LpPlan();
    p->N = n_img; p->g = g;
    const int *h = g.h, *w = g.w;
    p->f1 = lp_split(ws + s.f1, n_img, h[1], w[1], 64);
    p->p1 = lp_split(ws + s.p1, n_img, h[2], w[2], 64);
    p->f2 = lp_split(ws + s.f2, n_img, h[2], w[2], 192);
    p->p2 = lp_split(ws + s.p2, n_img, h[3], w[3], 192);
    const SplitTensor f3 = lp_split(ws + s.f3, n_img, h[3], w[3], 384), f4 = lp_split(ws + s.f4, n_img, h[3], w[3], 256),
                      f5 = lp_split(ws + s.f5, n_img, h[3], w[3], 256);
    p->partial = (double *)(ws + s.partial);

    LpConv1Args &c1 = p->c1;
    memset(&c1, 0, sizeof(c1));
    int rc = tc_make_bmap(b + L.w1, 64, LP_KB1, 64, &c1.bmap);
    if (!rc) {
        c1.bias = (const float *)(b + L.b1);
        c1.out = p->f1.base; c1.out_plane = p->f1.plane();
        c1.H = H; c1.W = W; c1.Ho = h[1]; c1.Wo = w[1];
        c1.TW = w[1] >= 12 ? 16 : 8; c1.TH = TC_BLOCK_M / c1.TW;
        c1.tiles_x = (w[1] + c1.TW - 1) / c1.TW; c1.tiles_y = (h[1] + c1.TH - 1) / c1.TH;
        p->c1_smem = lp_conv1_smem();
        cudaError_t e = cudaFuncSetAttribute(k_lpips_conv1, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p->c1_smem);
        if (e != cudaSuccess) { set_error("esr_lpips_create: %s", cudaGetErrorString(e)); rc = ESR_ECUDA; }
    }
    const float *b3 = (const float *)(b + L.b3);
    if (!rc) rc = lp_conv(p->p1, 25, 192, b + L.w2, (const float *)(b + L.b2), p->f2, 0, &p->c2);
    if (!rc) rc = lp_conv(p->p2, 9, 192, b + L.w3[0], b3, f3, 0, &p->c3[0]);
    if (!rc) rc = lp_conv(p->p2, 9, 192, b + L.w3[1], b3 + 192, f3, 192, &p->c3[1]);
    if (!rc) rc = lp_conv(f3, 9, 256, b + L.w4, (const float *)(b + L.b4), f4, 0, &p->c4);
    if (!rc) rc = lp_conv(f4, 9, 256, b + L.w5, (const float *)(b + L.b5), f5, 0, &p->c5);
    if (rc) { delete p; return rc; }
    const SplitTensor feats[LP_NLAYER] = {p->f1, p->f2, f3, f4, f5};
    for (int l = 0; l < LP_NLAYER; ++l) {
        p->head.f[l] = feats[l].base; p->head.plane[l] = feats[l].plane();
        p->head.lin[l] = (const float *)(b + L.lin[l]);
        p->head.C[l] = LP_CH[l]; p->head.HW[l] = feats[l].H * feats[l].W;
    }
    *plan_out = p;
    return ESR_OK;
}

extern "C" int esr_lpips_destroy(esr_lpips_t plan)
{
    delete (LpPlan *)plan;
    return ESR_OK;
}

extern "C" int esr_lpips_forward(esr_lpips_t plan, const float *planes, const int32_t *channel_src, int n_img, int normalize,
                                 int n_pairs, const int32_t *pair_a, const int32_t *pair_b, double *out, esr_stream_t stream)
{
    LpPlan *p = (LpPlan *)plan;
    ESR_REQUIRE(p && planes && channel_src && pair_a && pair_b && out, "esr_lpips_forward: null pointer");
    ESR_REQUIRE(n_img >= 1 && n_img <= p->N, "esr_lpips_forward: n_img %d outside [1, %d]", n_img, p->N);
    ESR_REQUIRE(n_pairs >= 1 && n_pairs <= p->N, "esr_lpips_forward: n_pairs %d outside [1, %d]", n_pairs, p->N);
    cudaStream_t st = (cudaStream_t)stream;
    int rc;
    {
        LpConv1Args a = p->c1;
        a.planes = planes; a.chan_src = channel_src; a.normalize = normalize ? 1 : 0;
        k_lpips_conv1<<<(unsigned)(n_img * a.tiles_x * a.tiles_y), 256, p->c1_smem, st>>>(a);
        ESR_LAUNCH_CHECK();
    }
    if ((rc = lp_maxpool(p->f1, p->p1, n_img, st))) return rc;
    ConvTCArgs *convs[5] = {&p->c2, &p->c3[0], &p->c3[1], &p->c4, &p->c5};
    for (int i = 0; i < 5; ++i) {
        ConvTCArgs a = *convs[i];
        a.n_img = n_img;
        if ((rc = conv_tc_launch(a, st))) return rc;
        if (i == 0 && (rc = lp_maxpool(p->f2, p->p2, n_img, st))) return rc;
    }
    k_lpips_head<<<dim3((unsigned)p->g.nblk, (unsigned)n_pairs, LP_NLAYER), 256, 0, st>>>(p->head, pair_a, pair_b, p->g.nblk, p->partial);
    ESR_LAUNCH_CHECK();
    k_lpips_finish<<<(unsigned)((n_pairs + 127) / 128), 128, 0, st>>>(p->partial, p->g.nblk, p->head, n_pairs, out);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}
