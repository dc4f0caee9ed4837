// render.cu -- the event-count image of the evaluation script (myutils/vis_events/matplotlib_plot_events.py:125-248,
// event_visualisation.plot_event_cnt with is_save=False), for a batch of [2, H, W] count images in one call.
//
// Percentiles.  plot_event_cnt takes np.percentile(plane, 1) and (plane, 99) of both planes of a float32 image.  numpy 2.x
// (method 'linear') computes them in float32: q = float32(q) / float32(100); the virtual index v = float32(n - 1) * q; the
// order statistics k0 = floor(v) and k1 = k0 + 1 (both n - 1 when v >= n - 1); gamma = v - k0; and _lerp:
//   d = x[k1] - x[k0];  r = x[k0] + d * gamma;  if gamma >= 0.5: r = x[k1] - d * (1 - gamma)      (all float32 roundings)
// The host computes v, k0, k1 and gamma exactly as numpy does.  The four order statistics of every plane come from a radix
// select on order-preserving uint32 keys: four passes of 8 bits; each pass histograms, per target, the elements that share
// the target's resolved prefix (k_select_hist, many CTAs per plane) and then finds the digit holding the target's rank
// (k_select_scan, one CTA per plane).  All planes of the batch go through the same eight launches.
//
// Colour map (k_colour).  One thread per pixel follows numpy's dtypes step by step: float32 normalisation
// (pos - pos_min) / (max - pos_min) and clip; channel values pos, 1 - pos (float32) or constants, widened into the float64
// image; gray adds float32 pos * 0.5 + neg * -0.5 to 0.5 in float64; then * 255 in float64 and the truncating astype(uint8).
// Output is HWC uint8 in BGR order when `bgr` is set (use_opencv=True) and RGB otherwise (cv2.cvtColor(BGR2RGB)); the gray
// scheme writes one channel.
#include "common.cuh"

namespace esr {

constexpr int RS_TARGETS = 4;              // k0, k1 of the 1st percentile, k0, k1 of the 99th
constexpr int RS_BINS = 256;
constexpr int RS_CHUNK = 16384;            // elements per histogram CTA

struct RenderQ {
    int k[RS_TARGETS];                     // order statistics, 0-based ranks
    float gamma[2];                        // interpolation weight of q = 1 and q = 99
};

__device__ __forceinline__ uint32_t f2key(float f)
{
    const uint32_t u = __float_as_uint(f);
    return u ^ ((u & 0x80000000u) ? 0xffffffffu : 0x80000000u);
}
__device__ __forceinline__ float key2f(uint32_t k)
{
    return __uint_as_float(k ^ ((k & 0x80000000u) ? 0x80000000u : 0xffffffffu));
}

// hist [P][4][256] += counts of digit (key >> shift) & 255 among the elements whose higher bits equal prefix[p][t]
__global__ void __launch_bounds__(256) k_select_hist(const float *__restrict__ x, int n, int shift, const uint32_t *__restrict__ prefix,
                                                     uint32_t *__restrict__ hist)
{
    __shared__ uint32_t sh[RS_TARGETS][RS_BINS];
    const int p = blockIdx.y;
    for (int i = threadIdx.x; i < RS_TARGETS * RS_BINS; i += blockDim.x) (&sh[0][0])[i] = 0;
    uint32_t pre[RS_TARGETS];
    const uint32_t hmask = shift == 24 ? 0u : (0xffffffffu << (shift + 8));
#pragma unroll
    for (int t = 0; t < RS_TARGETS; ++t) pre[t] = shift == 24 ? 0u : prefix[p * RS_TARGETS + t];
    __syncthreads();
    const float *src = x + (size_t)p * n;
    const int lane = threadIdx.x & 31;
    const int begin = blockIdx.x * RS_CHUNK, end = min(n, begin + RS_CHUNK);
    // every warp runs the same number of iterations so that the whole warp takes part in __match_any_sync
    for (int base = begin + (threadIdx.x & ~31); base < end; base += blockDim.x) {
        const int i = base + lane;
        const bool ok = i < end;
        const uint32_t key = ok ? f2key(__ldg(src + i)) : 0u;
        const uint32_t upper = key >> shift;                  // resolved prefix and this pass's digit
        const uint32_t active = __ballot_sync(0xffffffffu, ok);
        const uint32_t group = __match_any_sync(0xffffffffu, ok ? upper : 0xffffffffu) & active;
        if (ok && lane == __ffs(group) - 1) {                 // one atomic per distinct (prefix, digit) in the warp
            const uint32_t cnt = __popc(group), d = upper & 255u;
#pragma unroll
            for (int t = 0; t < RS_TARGETS; ++t)
                if (((key ^ pre[t]) & hmask) == 0u) atomicAdd(&sh[t][d], cnt);
        }
    }
    __syncthreads();
    uint32_t *g = hist + (size_t)p * RS_TARGETS * RS_BINS;
    for (int i = threadIdx.x; i < RS_TARGETS * RS_BINS; i += blockDim.x) {
        const uint32_t v = (&sh[0][0])[i];
        if (v) atomicAdd(g + i, v);
    }
}

// one CTA (4 warps, one per target) per plane: pick the digit holding the target's rank, extend the prefix, clear the
// histogram for the next pass; after the last pass turn the four order statistics into the two percentiles
__global__ void __launch_bounds__(128) k_select_scan(int shift, RenderQ q, uint32_t *__restrict__ prefix, uint32_t *__restrict__ rank,
                                                     uint32_t *__restrict__ hist, float *__restrict__ pct)
{
    const int p = blockIdx.x, t = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint32_t *h = hist + ((size_t)p * RS_TARGETS + t) * RS_BINS;
    const uint32_t r = shift == 24 ? (uint32_t)q.k[t] : rank[p * RS_TARGETS + t];
    const uint32_t pre = shift == 24 ? 0u : prefix[p * RS_TARGETS + t];
    uint32_t c[8], s = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) { c[j] = h[lane * 8 + j]; s += c[j]; }
    uint32_t incl = s;                                        // inclusive scan of the lanes' sums
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
    }
    uint32_t before = incl - s;
    int digit = -1;
    uint32_t below = 0;
    if (r >= before && r < incl) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            if (digit < 0 && r < before + c[j]) { digit = lane * 8 + j; below = before; }
            before += c[j];
        }
    }
    const uint32_t owner = __ballot_sync(0xffffffffu, digit >= 0);
    const int src = __ffs(owner) - 1;
    digit = __shfl_sync(0xffffffffu, digit, src);
    below = __shfl_sync(0xffffffffu, below, src);
#pragma unroll
    for (int j = 0; j < 8; ++j) h[lane * 8 + j] = 0u;
    __syncwarp();                                             // every lane has read rank / prefix before lane 0 rewrites them
    __shared__ uint32_t keys[RS_TARGETS];
    if (lane == 0) {
        const uint32_t np = pre | ((uint32_t)digit << shift);
        prefix[p * RS_TARGETS + t] = np;
        rank[p * RS_TARGETS + t] = r - below;
        keys[t] = np;
    }
    if (shift != 0) return;
    __syncthreads();
    if (threadIdx.x < 2) {
        const int i = threadIdx.x;                            // 0: q = 1, 1: q = 99
        const float a = key2f(keys[2 * i]), b = key2f(keys[2 * i + 1]), g = q.gamma[i];
        const float d = __fsub_rn(b, a);
        float v = __fadd_rn(a, __fmul_rn(d, g));
        if (g >= 0.5f) v = __fsub_rn(b, __fmul_rn(d, __fsub_rn(1.0f, g)));
        pct[p * 2 + i] = v;
    }
}

__device__ __forceinline__ unsigned char to_u8(double v) { return (unsigned char)(int)__dmul_rn(v, 255.0); }

// pct [B][2 planes][2] = {p1, p99}; scheme 0 gray, 1 green_red, 2 blue_red
__global__ void __launch_bounds__(256) k_colour(const float *__restrict__ cnt, int HW, const float *__restrict__ pct, int scheme,
                                                int black, int norm, int bgr, unsigned char *__restrict__ out)
{
    const int b = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= HW) return;
    float pos = __ldg(cnt + (size_t)b * 2 * HW + i), neg = __ldg(cnt + (size_t)b * 2 * HW + HW + i);
    if (norm) {
        const float pos_min = pct[b * 4 + 0], pos_max = pct[b * 4 + 1], neg_min = pct[b * 4 + 2], neg_max = pct[b * 4 + 3];
        const float mx = pos_max > neg_max ? pos_max : neg_max;
        if (pos_min != mx) pos = __fdiv_rn(__fsub_rn(pos, pos_min), __fsub_rn(mx, pos_min));
        if (neg_min != mx) neg = __fdiv_rn(__fsub_rn(neg, neg_min), __fsub_rn(mx, neg_min));
    } else {
        const bool m_pos = pos >= neg && pos != 0.0f, m_neg = pos < neg && neg != 0.0f;
        if (m_pos) { pos = 1.0f; neg = 0.0f; }
        if (m_neg) { neg = 1.0f; pos = 0.0f; }
    }
    pos = fminf(fmaxf(pos, 0.0f), 1.0f);                      // np.clip(x, 0, 1)
    neg = fminf(fmaxf(neg, 0.0f), 1.0f);
    if (scheme == 0) {
        const float s = __fadd_rn(__fmul_rn(pos, 0.5f), __fmul_rn(neg, -0.5f));
        out[(size_t)b * HW + i] = to_u8(__dadd_rn(0.5, (double)s));
        return;
    }
    double c0, c1, c2;                                        // the float64 image, channels in plot_event_cnt's (BGR) order
    if (black) {
        c0 = 0.0; c1 = 0.0; c2 = 0.0;
        if (scheme == 1) { if (pos > 0.0f) c1 = pos; }
        else { if (pos > 0.0f) c0 = pos; }
        if (neg > 0.0f) c2 = neg;
    } else {
        c0 = 1.0; c1 = 1.0; c2 = 1.0;
        if (pos > 0.0f && pos >= neg) {                       // only pos, or both with pos >= neg
            const double v = (double)__fsub_rn(1.0f, pos);
            if (scheme == 1) { c0 = v; c2 = v; }
            else { c1 = v; c2 = v; }
        } else if (neg > 0.0f) {                              // only neg, or both with pos < neg
            const double v = (double)__fsub_rn(1.0f, neg);
            c0 = v; c1 = v;
        }
    }
    unsigned char *o = out + ((size_t)b * HW + i) * 3;
    const unsigned char u0 = to_u8(c0), u1 = to_u8(c1), u2 = to_u8(c2);
    o[0] = bgr ? u0 : u2;
    o[1] = u1;
    o[2] = bgr ? u2 : u0;
}

// numpy's linear-method indices for the q-th percentile of n float32 values (see the file comment)
static void percentile_index(int n, int q, int *k0, int *k1, float *gamma)
{
    const float qq = (float)q / 100.0f;
    const volatile float v = (float)(n - 1) * qq;              // volatile: one float32 rounding, as numpy
    if (v >= (float)(n - 1)) { *k0 = *k1 = n - 1; *gamma = (float)((double)v + 1.0); return; }
    *k0 = (int)floorf(v);
    *k1 = *k0 + 1;
    *gamma = (float)((double)v - (double)*k0);
}

} // namespace esr

using namespace esr;

static size_t render_ws_layout(int B, size_t *o_prefix, size_t *o_rank, size_t *o_pct)
{
    const size_t P = (size_t)2 * B;
    size_t off = align_up(P * RS_TARGETS * RS_BINS * sizeof(uint32_t), 256);
    *o_prefix = off; off += align_up(P * RS_TARGETS * sizeof(uint32_t), 256);
    *o_rank = off; off += align_up(P * RS_TARGETS * sizeof(uint32_t), 256);
    *o_pct = off; off += align_up(P * 2 * sizeof(float), 256);
    return off;
}

extern "C" size_t esr_render_workspace_bytes(int B, int H, int W)
{
    (void)H; (void)W;
    if (B <= 0) return 0;
    size_t a, b, c;
    return render_ws_layout(B, &a, &b, &c);
}

extern "C" int esr_render_event_cnt(const float *cnt, int B, int H, int W, int color_scheme, int black_background, int is_norm,
                                    int bgr, unsigned char *out, float *percentiles, void *workspace, size_t ws_bytes,
                                    esr_stream_t stream)
{
    ESR_REQUIRE(cnt && out && workspace, "esr_render_event_cnt: null pointer");
    ESR_REQUIRE(B > 0 && H > 0 && W > 0 && (long long)H * W < (1ll << 24),
                "esr_render_event_cnt: bad dims (H * W must be below 2^24, where numpy's float32 virtual index stays exact)");
    ESR_REQUIRE(B <= 32767, "esr_render_event_cnt: at most 32767 images per call");
    ESR_REQUIRE(color_scheme >= 0 && color_scheme <= 2, "esr_render_event_cnt: color_scheme must be 0 (gray), 1 (green_red) or 2 (blue_red)");
    size_t o_prefix, o_rank, o_pct;
    const size_t need = render_ws_layout(B, &o_prefix, &o_rank, &o_pct);
    if (ws_bytes < need) { set_error("esr_render_event_cnt: workspace %zu < %zu", ws_bytes, need); return ESR_EWORKSPACE; }
    cudaStream_t st = (cudaStream_t)stream;
    char *ws = (char *)workspace;
    uint32_t *hist = (uint32_t *)ws, *prefix = (uint32_t *)(ws + o_prefix), *rank = (uint32_t *)(ws + o_rank);
    float *pct = (float *)(ws + o_pct);
    const int HW = H * W, P = 2 * B;
    if (is_norm || percentiles) {
        RenderQ q;
        percentile_index(HW, 1, &q.k[0], &q.k[1], &q.gamma[0]);
        percentile_index(HW, 99, &q.k[2], &q.k[3], &q.gamma[1]);
        ESR_CUDA_CHECK(cudaMemsetAsync(hist, 0, (size_t)P * RS_TARGETS * RS_BINS * sizeof(uint32_t), st));
        const dim3 hgrid((unsigned)((HW + RS_CHUNK - 1) / RS_CHUNK), (unsigned)P);
        for (int shift = 24; shift >= 0; shift -= 8) {
            k_select_hist<<<hgrid, 256, 0, st>>>(cnt, HW, shift, prefix, hist);
            ESR_LAUNCH_CHECK();
            k_select_scan<<<P, 128, 0, st>>>(shift, q, prefix, rank, hist, pct);
            ESR_LAUNCH_CHECK();
        }
        if (percentiles)
            ESR_CUDA_CHECK(cudaMemcpyAsync(percentiles, pct, (size_t)P * 2 * sizeof(float), cudaMemcpyDeviceToDevice, st));
    }
    k_colour<<<dim3((unsigned)((HW + 255) / 256), (unsigned)B), 256, 0, st>>>(cnt, HW, pct, color_scheme, black_background, is_norm,
                                                                             bgr, out);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}
