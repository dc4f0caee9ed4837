// dcn_bwd.cu -- backward of the modulated deformable 3x3 convolution (the `_ext.dcn_v2_backward` operator).
// Reference: models/DCNv2/src/cuda/dcn_v2_cuda.cu:97-216 (per-sample loop: W^T.gO, col2im, coord kernel, gO.cols^T, gO.1)
// with kernels models/DCNv2/src/cuda/dcn_v2_im2col_cuda.cu:197-254 (col2im, atomicAdd) and :256-327 (offset / mask grads).
// Same analytic gradients, organised for the split-bf16 NHWC data layout:
//   1. gcols[p][tap*64+c] = sum_co gO[p][co] * W[co][c][tap]     wgmma GEMM (tc_conv.cu, 1x1 mode, 3 launches of N=192)
//   2. one thread per (pixel, tap, group) re-derives the bilinear corners and, for its 8 channels,
//        grad_mask   += gcols * sample                      grad_offset += gcols * mask * d(sample)/d(h,w)
//        grad_input  += corner weight * gcols * mask        (fp32 atomicAdd, like the reference's col2im)
//   3. grad_weight[co][c][tap] = sum_p gO[p][co] * cols[p][tap*64+c]   (cols re-sampled by dcn_columns; tiled fp32 GEMM
//      over pixel slices with atomicAdd of the partial tiles),  grad_bias[co] = sum_p gO[p][co].
// Configuration: the one ESR uses (64 -> 64, 3x3, stride 1, pad 1, dilation 1, 8 deformable groups).
// Deterministic mode (ESR_DETERMINISTIC, esr_dcn_v2_backward_ex): grad_input in int64 fixed point, grad_weight / grad_bias from
// per-slice partials added in slice order -- bitwise reproducible.
#include "net.cuh"

namespace esr {

__device__ __forceinline__ void bw_ld8(const __nv_bfloat16 *hi, size_t plane, float (&o)[8])
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

// W [co][c][tap] fp32 -> 1x1-conv weight [n = tap*64+c][k = co] fp32 (then packed by pack_conv_weight)
__global__ void k_dcn_wt(const float *__restrict__ w, float *__restrict__ wt)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= 576 * 64) return;
    const int co = i % 64, n = i / 64, c = n % 64, tap = n / 64;
    wt[i] = w[((size_t)co * 64 + c) * 9 + tap];
}

// ---- deterministic grad_input (ESR_DETERMINISTIC): the bilinear scatter's targets depend on the learned offsets, so instead of
// fp32 atomics it accumulates in int64 fixed point, whose atomics give the same sum in any order.  A pre-pass takes the largest
// |gcols * mask| over the batch (order-independent max); every scattered value is that product times a corner weight <= 1.
// The scale is the power of two that keeps the worst case -- all 72 (tap, group) x 4 corner values of every pixel of an image
// landing on one element, each rounded up by half a unit -- below 2^63: 288 * H * W * (max * scale + 1/2) <= 2^62 + 144 H W.
__device__ __forceinline__ double dcn_fixed_scale(unsigned max_bits, int H, int W)
{
    const float m = __uint_as_float(max_bits);
    if (!(m > 0.0f)) return 1.0;
    return exp2(floor(log2(0x1p62 / (288.0 * (double)H * (double)W * (double)m))));
}

// max over (p, tap, group, channel) of |gcols * mask|: thread per (p, tap, group), warp max, one atomicMax per warp on the bit
// pattern (the values are >= 0, so the unsigned order of the bits is the float order)
__global__ void __launch_bounds__(256)
k_dcn_gin_max(const float *__restrict__ om, const float *__restrict__ gcols, size_t total, unsigned *__restrict__ max_bits)
{
    unsigned mx = 0u;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int g = (int)(i % 8), k = (int)((i / 8) % 9);
        const size_t p = i / 72;
        const float m = om[p * 216 + 144 + g * 9 + k];
        const float4 *gp = reinterpret_cast<const float4 *>(gcols + p * 576 + k * 64 + g * 8);
        const float4 ga = gp[0], gb = gp[1];
        const float gc[8] = {ga.x, ga.y, ga.z, ga.w, gb.x, gb.y, gb.z, gb.w};
#pragma unroll
        for (int e = 0; e < 8; ++e) mx = max(mx, __float_as_uint(fabsf(gc[e] * m)));
    }
    mx = __reduce_max_sync(0xffffffffu, mx);
    if ((threadIdx.x & 31) == 0 && mx) atomicMax(max_bits, mx);
}

__device__ __forceinline__ unsigned long long to_fixed(float v, double scale) { return (unsigned long long)__double2ll_rn((double)v * scale); }

// offset/mask NCHW -> om NHWC [p][216] is k_om_from_nchw in dcn.cu; grads go back the other way
// DET: grad_input goes to gin_q (int64 fixed point at `scale`) instead of gin
template <bool DET>
__device__ __forceinline__ void dcn_bwd_sample_body(const __nv_bfloat16 *__restrict__ feat, size_t f_plane, const float *__restrict__ om,
                                                    const float *__restrict__ gcols, int n_img, int H, int W, float *__restrict__ gin,
                                                    unsigned long long *__restrict__ gin_q, double scale, float *__restrict__ gom)
{
    const size_t total = (size_t)n_img * H * W * 72;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int g = (int)(i % 8), k = (int)((i / 8) % 9);
        const size_t p = i / 72;
        const int x = (int)(p % W), y = (int)((p / W) % H), img = (int)(p / ((size_t)W * H));
        const float *o = om + p * 216;
        const float off_h = o[g * 18 + 2 * k], off_w = o[g * 18 + 2 * k + 1], m = o[144 + g * 9 + k];
        const float h_im = (float)(y - 1 + k / 3) + off_h;
        const float w_im = (float)(x - 1 + k % 3) + off_w;
        float g_off_h = 0.0f, g_off_w = 0.0f, g_mask = 0.0f;
        if (h_im > -1.0f && w_im > -1.0f && h_im < (float)H && w_im < (float)W) {
            const int h_low = (int)floorf(h_im), w_low = (int)floorf(w_im);
            const int h_high = h_low + 1, w_high = w_low + 1;
            const float lh = h_im - (float)h_low, lw = w_im - (float)w_low;
            const float hh = 1.0f - lh, hw = 1.0f - lw;
            const bool ok1 = h_low >= 0 && w_low >= 0, ok2 = h_low >= 0 && w_high <= W - 1;
            const bool ok3 = h_high <= H - 1 && w_low >= 0, ok4 = h_high <= H - 1 && w_high <= W - 1;
            const size_t base = (size_t)img * H * W;
            const size_t p1 = base + (size_t)h_low * W + w_low, p2 = p1 + 1, p3 = p1 + W, p4 = p3 + 1;
            float c1[8], c2[8], c3[8], c4[8], gc[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) c1[e] = c2[e] = c3[e] = c4[e] = 0.0f;
            if (ok1) bw_ld8(feat + p1 * 64 + g * 8, f_plane, c1);
            if (ok2) bw_ld8(feat + p2 * 64 + g * 8, f_plane, c2);
            if (ok3) bw_ld8(feat + p3 * 64 + g * 8, f_plane, c3);
            if (ok4) bw_ld8(feat + p4 * 64 + g * 8, f_plane, c4);
            const float4 *gp = reinterpret_cast<const float4 *>(gcols + p * 576 + k * 64 + g * 8);
            const float4 ga = gp[0], gb = gp[1];
            gc[0] = ga.x; gc[1] = ga.y; gc[2] = ga.z; gc[3] = ga.w; gc[4] = gb.x; gc[5] = gb.y; gc[6] = gb.z; gc[7] = gb.w;
            const float w1 = hh * hw, w2 = hh * lw, w3 = lh * hw, w4 = lh * lw;
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const float val = w1 * c1[e] + w2 * c2[e] + w3 * c3[e] + w4 * c4[e];
                g_mask += gc[e] * val;
                // d(sample)/dh = hw (v3 - v1) + lw (v4 - v2),  d/dw = hh (v2 - v1) + lh (v4 - v3)   (im2col_cuda.cu:82-121)
                g_off_h += gc[e] * m * (hw * (c3[e] - c1[e]) + lw * (c4[e] - c2[e]));
                g_off_w += gc[e] * m * (hh * (c2[e] - c1[e]) + lh * (c4[e] - c3[e]));
                const float t = gc[e] * m;
                if (DET) {
                    if (ok1) atomicAdd(gin_q + p1 * 64 + g * 8 + e, to_fixed(w1 * t, scale));
                    if (ok2) atomicAdd(gin_q + p2 * 64 + g * 8 + e, to_fixed(w2 * t, scale));
                    if (ok3) atomicAdd(gin_q + p3 * 64 + g * 8 + e, to_fixed(w3 * t, scale));
                    if (ok4) atomicAdd(gin_q + p4 * 64 + g * 8 + e, to_fixed(w4 * t, scale));
                } else {
                    if (ok1) atomicAdd(gin + p1 * 64 + g * 8 + e, w1 * t);
                    if (ok2) atomicAdd(gin + p2 * 64 + g * 8 + e, w2 * t);
                    if (ok3) atomicAdd(gin + p3 * 64 + g * 8 + e, w3 * t);
                    if (ok4) atomicAdd(gin + p4 * 64 + g * 8 + e, w4 * t);
                }
            }
        }
        float *go = gom + p * 216;
        go[g * 18 + 2 * k] = g_off_h;
        go[g * 18 + 2 * k + 1] = g_off_w;
        go[144 + g * 9 + k] = g_mask;
    }
}
__global__ void __launch_bounds__(256)
k_dcn_bwd_sample(const __nv_bfloat16 *__restrict__ feat, size_t f_plane, const float *__restrict__ om,
                 const float *__restrict__ gcols, int n_img, int H, int W, float *__restrict__ gin /*[p][64]*/,
                 float *__restrict__ gom /*[p][216]*/)
{
    dcn_bwd_sample_body<false>(feat, f_plane, om, gcols, n_img, H, W, gin, nullptr, 0.0, gom);
}
__global__ void __launch_bounds__(256)
k_dcn_bwd_sample_det(const __nv_bfloat16 *__restrict__ feat, size_t f_plane, const float *__restrict__ om,
                     const float *__restrict__ gcols, int n_img, int H, int W, const unsigned *__restrict__ max_bits,
                     unsigned long long *__restrict__ gin_q /*[p][64]*/, float *__restrict__ gom /*[p][216]*/)
{
    dcn_bwd_sample_body<true>(feat, f_plane, om, gcols, n_img, H, W, nullptr, gin_q, dcn_fixed_scale(*max_bits, H, W), gom);
}

// fixed-point grad_input [p][64] -> fp32 NCHW
__global__ void k_dcn_gin_from_fixed(const long long *__restrict__ q, const unsigned *__restrict__ max_bits, int n_img, int HW,
                                     float *__restrict__ dst)
{
    const double inv = 1.0 / dcn_fixed_scale(*max_bits, 1, HW);
    const size_t total = (size_t)n_img * 64 * HW;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int pix = (int)(i % HW), c = (int)((i / HW) % 64), n = (int)(i / ((size_t)HW * 64));
        dst[i] = (float)((double)q[((size_t)n * HW + pix) * 64 + c] * inv);
    }
}

// grad_weight partial tiles: block = 64 co x 64 columns (one tap), over a slice of PSL pixels.  DET: slice y -> gw[y][co][c][tap]
constexpr int WG_PSL = 512;
template <bool DET>
__device__ __forceinline__ void dcn_wgrad_body(const float *__restrict__ go, const __nv_bfloat16 *__restrict__ cols, size_t c_plane,
                                               size_t npix, float *__restrict__ gw)
{
    __shared__ float sA[32][65];   // gO[pix][co]
    __shared__ float sB[32][65];   // cols[pix][c] of this tap
    const int tap = blockIdx.x;
    const size_t p_beg = (size_t)blockIdx.y * WG_PSL, p_end = min(npix, p_beg + WG_PSL);
    const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;     // 16 x 16 threads, 4 x 4 outputs each
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.0f;
    for (size_t p0 = p_beg; p0 < p_end; p0 += 32) {
        for (int i = threadIdx.x; i < 32 * 64; i += 256) {
            const int pp = i / 64, ch = i % 64;
            const size_t p = p0 + pp;
            float a = 0.0f, b = 0.0f;
            if (p < p_end) {
                a = go[p * 64 + ch];
                const size_t o = p * 576 + tap * 64 + ch;
                b = join_bf16(cols[o], cols[c_plane + o]);
            }
            sA[pp][ch] = a;
            sB[pp][ch] = b;
        }
        __syncthreads();
#pragma unroll 8
        for (int pp = 0; pp < 32; ++pp) {
            float a[4], b[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) { a[i] = sA[pp][ty * 4 + i]; b[i] = sB[pp][tx * 4 + i]; }
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (DET) gw[(size_t)blockIdx.y * 64 * 64 * 9 + ((size_t)(ty * 4 + i) * 64 + tx * 4 + j) * 9 + tap] = acc[i][j];
            else atomicAdd(gw + ((size_t)(ty * 4 + i) * 64 + tx * 4 + j) * 9 + tap, acc[i][j]);
        }
}
__global__ void __launch_bounds__(256)
k_dcn_wgrad(const float *__restrict__ go /*[p][64] fp32 NHWC*/, const __nv_bfloat16 *__restrict__ cols, size_t c_plane,
            size_t npix, float *__restrict__ gw /*[co][c][tap]*/)
{
    dcn_wgrad_body<false>(go, cols, c_plane, npix, gw);
}
__global__ void __launch_bounds__(256)
k_dcn_wgrad_det(const float *__restrict__ go, const __nv_bfloat16 *__restrict__ cols, size_t c_plane, size_t npix, float *__restrict__ part)
{
    dcn_wgrad_body<true>(go, cols, c_plane, npix, part);
}

// DET: thread (block b, lane_p) -> gb[b * 4 + lane_p][co]
constexpr int BG_BLOCKS = 148;
template <bool DET>
__device__ __forceinline__ void dcn_bgrad_body(const float *__restrict__ go, size_t npix, float *__restrict__ gb)
{
    const int co = threadIdx.x % 64, lane_p = threadIdx.x / 64;
    float s = 0.0f;
    for (size_t p = (size_t)blockIdx.x * 4 + lane_p; p < npix; p += (size_t)gridDim.x * 4) s += go[p * 64 + co];
    if (DET) gb[((size_t)blockIdx.x * 4 + lane_p) * 64 + co] = s;
    else atomicAdd(gb + co, s);
}
__global__ void __launch_bounds__(256) k_dcn_bgrad(const float *__restrict__ go, size_t npix, float *__restrict__ gb)
{
    dcn_bgrad_body<false>(go, npix, gb);
}
__global__ void __launch_bounds__(256) k_dcn_bgrad_det(const float *__restrict__ go, size_t npix, float *__restrict__ part)
{
    dcn_bgrad_body<true>(go, npix, part);
}

// NCHW fp32 <-> NHWC fp32 helpers
__global__ void k_nchw_to_nhwc(const float *__restrict__ src, int n_img, int C, int HW, float *__restrict__ dst)
{
    const size_t total = (size_t)n_img * C * HW;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const size_t p = i / C;
        const int pix = (int)(p % HW), n = (int)(p / HW);
        dst[i] = src[((size_t)n * C + c) * HW + pix];
    }
}
__global__ void k_nhwc_to_nchw(const float *__restrict__ src, int n_img, int C, int c0, int Cs, int HW, float *__restrict__ dst)
{
    // dst [n][C][HW] <- src [n][HW][Cs] channels [c0, c0+C)
    const size_t total = (size_t)n_img * C * HW;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int pix = (int)(i % HW), c = (int)((i / HW) % C), n = (int)(i / ((size_t)HW * C));
        dst[i] = src[((size_t)n * HW + pix) * Cs + c0 + c];
    }
}

} // namespace esr

using namespace esr;

// det: grad_input in int64 fixed point (twice the bytes), then the partial buffers of grad_weight / grad_bias and the max word
struct DcnBwdWs { size_t feat, om, go_split, go_nhwc, gcols, cols, gin, gom, wt, wtp, bz, wpart, bpart, maxw, total; };
static DcnBwdWs dcn_bwd_layout(int B, int H, int W, bool det)
{
    DcnBwdWs l{};
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t r = off; off = align_up(off + bytes, 1024); return r; };
    const size_t px = (size_t)B * H * W;
    l.feat = take(px * 64 * 4); l.om = take(px * 216 * 4); l.go_split = take(px * 64 * 4); l.go_nhwc = take(px * 64 * 4);
    l.gcols = take(px * 576 * 4); l.cols = take(px * 576 * 4); l.gin = take(px * 64 * (det ? 8 : 4)); l.gom = take(px * 216 * 4);
    l.wt = take(576 * 64 * 4); l.wtp = take(3 * tc_packed_weight_bytes(192, 64, 1)); l.bz = take(256 * 4);
    if (det) {
        l.wpart = take((size_t)ceil_div64((int64_t)px, WG_PSL) * 64 * 64 * 9 * 4);
        l.bpart = take((size_t)BG_BLOCKS * 4 * 64 * 4);
        l.maxw = take(4);
    }
    l.total = off;
    return l;
}

extern "C" size_t esr_dcn_v2_backward_workspace_bytes(int B, int H, int W) { return dcn_bwd_layout(B, H, W, false).total; }

extern "C" size_t esr_dcn_v2_backward_workspace_bytes_ex(int B, int C, int H, int W, int Co, int kernel, int stride, int pad,
                                                         int dilation, int deformable_group, int flags)
{
    if (dcn_is_tuned(C, Co, kernel, stride, pad, dilation, deformable_group))
        return dcn_bwd_layout(B, H, W, (flags & ESR_DETERMINISTIC) != 0).total;
    return dcn_generic_ws_bytes(B, C, H, W, Co, kernel, stride, pad, dilation, deformable_group, 1);
}

extern "C" int esr_dcn_v2_backward(const float *input, const float *weight, const float *bias, const float *offset,
                                   const float *mask, const float *grad_output, int B, int C, int H, int W, int Co, int kernel,
                                   int stride, int pad, int dilation, int deformable_group, float *grad_input,
                                   float *grad_offset, float *grad_mask, float *grad_weight, float *grad_bias, void *workspace,
                                   size_t ws_bytes, esr_stream_t stream)
{
    return esr_dcn_v2_backward_ex(input, weight, bias, offset, mask, grad_output, B, C, H, W, Co, kernel, stride, pad, dilation,
                                  deformable_group, grad_input, grad_offset, grad_mask, grad_weight, grad_bias, 0, workspace, ws_bytes,
                                  stream);
}

extern "C" int esr_dcn_v2_backward_ex(const float *input, const float *weight, const float *bias, const float *offset,
                                      const float *mask, const float *grad_output, int B, int C, int H, int W, int Co, int kernel,
                                      int stride, int pad, int dilation, int deformable_group, float *grad_input,
                                      float *grad_offset, float *grad_mask, float *grad_weight, float *grad_bias, int flags,
                                      void *workspace, size_t ws_bytes, esr_stream_t stream)
{
    (void)bias;
    ESR_REQUIRE(input && weight && offset && mask && grad_output && grad_input && grad_offset && grad_mask && grad_weight &&
                grad_bias && workspace, "esr_dcn_v2_backward: null pointer");
    const bool det = (flags & ESR_DETERMINISTIC) != 0;
    if (!dcn_is_tuned(C, Co, kernel, stride, pad, dilation, deformable_group)) {    // any other configuration: dcn_generic.cu
        if (det) {
            set_error("esr_dcn_v2_backward: only the 64 -> 64, 3x3, stride 1, pad 1, dilation 1, 8-group configuration has a "
                      "deterministic backward (this is C=%d Co=%d k=%d s=%d p=%d d=%d dg=%d); leave deterministic mode for it",
                      C, Co, kernel, stride, pad, dilation, deformable_group);
            return ESR_EUNSUPPORTED;
        }
        return dcn_generic_backward(input, weight, offset, mask, grad_output, B, C, H, W, Co, kernel, stride, pad, dilation,
                                    deformable_group, grad_input, grad_offset, grad_mask, grad_weight, grad_bias, workspace, ws_bytes,
                                    (cudaStream_t)stream);
    }
    const DcnBwdWs L = dcn_bwd_layout(B, H, W, det);
    if (ws_bytes < L.total) { set_error("esr_dcn_v2_backward: workspace %zu < %zu", ws_bytes, L.total); return ESR_EWORKSPACE; }
    cudaStream_t st = (cudaStream_t)stream;
    char *ws = (char *)workspace;
    const size_t px = (size_t)B * H * W;
    const int HW = H * W;
    SplitTensor feat, gos, cols;
    feat.base = (__nv_bfloat16 *)(ws + L.feat); feat.n_img = B; feat.H = H; feat.W = W; feat.C = 64;
    gos = feat; gos.base = (__nv_bfloat16 *)(ws + L.go_split);
    cols = feat; cols.base = (__nv_bfloat16 *)(ws + L.cols); cols.C = 576;
    float *om = (float *)(ws + L.om), *go_nhwc = (float *)(ws + L.go_nhwc), *gcols = (float *)(ws + L.gcols);
    float *gin = (float *)(ws + L.gin), *gom = (float *)(ws + L.gom), *wt = (float *)(ws + L.wt), *bz = (float *)(ws + L.bz);
    int rc;
    // layouts
    if ((rc = split_from_nchw(input, B, 64, H, W, feat.base, st))) return rc;
    if ((rc = split_from_nchw(grad_output, B, 64, H, W, gos.base, st))) return rc;
    k_nchw_to_nhwc<<<(unsigned)ceil_div64((int64_t)px * 64, 256), 256, 0, st>>>(grad_output, B, 64, HW, go_nhwc);
    ESR_LAUNCH_CHECK();
    if ((rc = om_from_nchw(offset, mask, B, HW, om, st))) return rc;
    ESR_CUDA_CHECK(cudaMemsetAsync(bz, 0, 256 * 4, st));
    ESR_CUDA_CHECK(cudaMemsetAsync(gin, 0, px * 64 * (det ? 8 : 4), st));
    ESR_CUDA_CHECK(cudaMemsetAsync(grad_weight, 0, 64 * 64 * 9 * 4, st));
    ESR_CUDA_CHECK(cudaMemsetAsync(grad_bias, 0, 64 * 4, st));
    // 1. gcols = gO . W^T  (three N=192 slices of the 576 columns)
    k_dcn_wt<<<(576 * 64 + 255) / 256, 256, 0, st>>>(weight, wt);
    ESR_LAUNCH_CHECK();
    const size_t wslice = tc_packed_weight_bytes(192, 64, 1);
    for (int s = 0; s < 3; ++s) {
        if ((rc = pack_conv_weight(wt + (size_t)s * 192 * 64, 192, 64, 1, ws + L.wtp + s * wslice, st))) return rc;
        ConvTCDesc d;
        d.src[0] = gos; d.n_src = 1; d.ntaps = 1; d.cout = 192; d.wpacked = ws + L.wtp + s * wslice; d.bias = bz;
        d.n_img = B; d.act = ACT_NONE; d.out_f32 = gcols + s * 192; d.out_f32_C = 576;
        ConvTCArgs args;
        if ((rc = conv_tc_prepare(d, &args))) return rc;
        if ((rc = conv_tc_launch(args, st))) return rc;
    }
    // 2. sampling backward
    const unsigned wslices = (unsigned)ceil_div64((int64_t)px, WG_PSL);
    if (!det) {
        k_dcn_bwd_sample<<<(unsigned)ceil_div64((int64_t)px * 72, 256), 256, 0, st>>>(feat.base, feat.plane(), om, gcols, B, H, W, gin, gom);
        ESR_LAUNCH_CHECK();
    } else {
        unsigned *maxw = (unsigned *)(ws + L.maxw);
        unsigned long long *gin_q = (unsigned long long *)(ws + L.gin);
        ESR_CUDA_CHECK(cudaMemsetAsync(maxw, 0, 4, st));
        k_dcn_gin_max<<<(unsigned)min((int64_t)4096, ceil_div64((int64_t)px * 72, 256)), 256, 0, st>>>(om, gcols, px * 72, maxw);
        ESR_LAUNCH_CHECK();
        k_dcn_bwd_sample_det<<<(unsigned)ceil_div64((int64_t)px * 72, 256), 256, 0, st>>>(feat.base, feat.plane(), om, gcols, B, H, W,
                                                                                          maxw, gin_q, gom);
        ESR_LAUNCH_CHECK();
    }
    // 3. weight / bias gradients (forward columns re-sampled)
    if ((rc = dcn_columns(feat, nullptr, om, B, cols, st))) return rc;
    if (!det) {
        k_dcn_wgrad<<<dim3(9, wslices), 256, 0, st>>>(go_nhwc, cols.base, cols.plane(), px, grad_weight);
        ESR_LAUNCH_CHECK();
        k_dcn_bgrad<<<BG_BLOCKS, 256, 0, st>>>(go_nhwc, px, grad_bias);
        ESR_LAUNCH_CHECK();
    } else {
        float *wpart = (float *)(ws + L.wpart), *bpart = (float *)(ws + L.bpart);
        k_dcn_wgrad_det<<<dim3(9, wslices), 256, 0, st>>>(go_nhwc, cols.base, cols.plane(), px, wpart);
        ESR_LAUNCH_CHECK();
        if ((rc = sum_slices(wpart, (int)wslices, 64 * 64 * 9, grad_weight, st))) return rc;
        k_dcn_bgrad_det<<<BG_BLOCKS, 256, 0, st>>>(go_nhwc, px, bpart);
        ESR_LAUNCH_CHECK();
        if ((rc = sum_slices(bpart, BG_BLOCKS * 4, 64, grad_bias, st))) return rc;
    }
    // back to the reference layouts
    if (!det) {
        k_nhwc_to_nchw<<<(unsigned)ceil_div64((int64_t)px * 64, 256), 256, 0, st>>>(gin, B, 64, 0, 64, HW, grad_input);
    } else {
        k_dcn_gin_from_fixed<<<(unsigned)ceil_div64((int64_t)px * 64, 256), 256, 0, st>>>((const long long *)(ws + L.gin),
                                                                                          (const unsigned *)(ws + L.maxw), B, HW, grad_input);
    }
    ESR_LAUNCH_CHECK();
    k_nhwc_to_nchw<<<(unsigned)ceil_div64((int64_t)px * 144, 256), 256, 0, st>>>(gom, B, 144, 0, 216, HW, grad_offset);
    ESR_LAUNCH_CHECK();
    k_nhwc_to_nchw<<<(unsigned)ceil_div64((int64_t)px * 72, 256), 256, 0, st>>>(gom, B, 72, 144, 216, HW, grad_mask);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}
