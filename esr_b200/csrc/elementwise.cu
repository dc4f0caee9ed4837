// elementwise.cu -- the fused element-wise / reduction glue of DeepRecurrNet on split-bf16 NHWC tensors.
// All HBM-bound: 16-byte vector accesses, 8 channels per thread.
#include "net.cuh"

namespace esr {

__device__ __forceinline__ void load8(const __nv_bfloat16 *hi, size_t plane, float (&o)[8])
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
__device__ __forceinline__ void store8(__nv_bfloat16 *hi, size_t plane, const float (&x)[8])
{
    uint32_t hw[4], lw[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        split_pack2(x[2 * e], x[2 * e + 1], hw[e], lw[e]);
    }
    *reinterpret_cast<uint4 *>(hi) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
    *reinterpret_cast<uint4 *>(hi + plane) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
}

// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_ltc_cat(const __nv_bfloat16 *__restrict__ f, size_t f_plane, const float *__restrict__ maps, const int *__restrict__ idx,
          int n_img, int HW, __nv_bfloat16 *__restrict__ out, size_t out_plane)
{
    PDL_LAUNCH_DEPENDENTS();
    PDL_WAIT();
    const size_t total = (size_t)n_img * HW * 24;            // 24 groups of 8 channels = 192
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int g = (int)(i % 24);
        const size_t p = i / 24;
        const int pix = (int)(p % HW), img = (int)(p / HW);
        const int part = g / 8, c0 = (g % 8) * 8;            // part 0: f0*m0, 1: f1, 2: f2*m1
        const int *ix = idx + img * 5;
        const size_t src = ((size_t)ix[part] * HW + pix) * 64 + c0;
        float v[8];
        load8(f + src, f_plane, v);
        if (part != 1) {
            const float m = maps[(size_t)ix[part == 0 ? 3 : 4] * HW + pix];
#pragma unroll
            for (int e = 0; e < 8; ++e) v[e] *= m;
        }
        store8(out + p * 192 + part * 64 + c0, out_plane, v);
    }
}
int ltc_cat(const SplitTensor &f, const float *maps, const int *idx, int n_img, const SplitTensor &out, cudaStream_t st)
{
    const int HW = f.H * f.W;
    const size_t total = (size_t)n_img * HW * 24;
    ESR_CUDA_CHECK(launch_pdl(k_ltc_cat, dim3((unsigned)ceil_div64((int64_t)total, 256)), dim3(256), 0, st, f.base, f.plane(), maps, idx, n_img, HW, out.base,
                                                                         out.plane()));
    esr::count_launch();
    return ESR_OK;
}

// ---------------------------------------------------------------------------------------------
// per-image channel max: grid (slices, n_img); partial maxima merged with integer atomicMax on the ordered
// bit pattern (monotone map of fp32), out pre-filled with -inf by the launcher.
__device__ __forceinline__ int f2ord(float f) { int i = __float_as_int(f); return i >= 0 ? i : i ^ 0x7fffffff; }
__device__ __forceinline__ float ord2f(int i) { return __int_as_float(i >= 0 ? i : i ^ 0x7fffffff); }

__global__ void __launch_bounds__(256)
k_chan_max(const __nv_bfloat16 *__restrict__ t, size_t plane, int HW, int *__restrict__ out_ord)
{
    PDL_LAUNCH_DEPENDENTS();
    PDL_WAIT();
    const int img = blockIdx.y;
    const int c8 = threadIdx.x & 7;                      // 8 groups of 8 channels
    const int lane_pix = threadIdx.x >> 3;               // 32 pixels per pass
    float mx[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) mx[e] = -INFINITY;
    for (int pix = blockIdx.x * 32 + lane_pix; pix < HW; pix += gridDim.x * 32) {
        float v[8];
        load8(t + ((size_t)img * HW + pix) * 64 + c8 * 8, plane, v);
#pragma unroll
        for (int e = 0; e < 8; ++e) mx[e] = fmaxf(mx[e], v[e]);
    }
    __shared__ float sm[32][64];
#pragma unroll
    for (int e = 0; e < 8; ++e) sm[lane_pix][c8 * 8 + e] = mx[e];
    __syncthreads();
    if (threadIdx.x < 64) {
        float m = -INFINITY;
        for (int r = 0; r < 32; ++r) m = fmaxf(m, sm[r][threadIdx.x]);
        atomicMax(out_ord + img * 64 + threadIdx.x, f2ord(m));
    }
}
static int f2ord_host_neg_inf() { return (int)(0xFF800000u ^ 0x7FFFFFFFu); }
__global__ void k_fill_int(int *p, int n, int v)
{
    PDL_LAUNCH_DEPENDENTS();
    PDL_WAIT();
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}
int chan_max(const SplitTensor &t, int n_img, float *out, cudaStream_t st)
{
    const int HW = t.H * t.W;
    ESR_CUDA_CHECK(launch_pdl(k_fill_int, dim3((n_img * 64 + 255) / 256), dim3(256), 0, st, (int *)out, n_img * 64, f2ord_host_neg_inf()));
    esr::count_launch();
    int slices = (HW + 32 * 8 - 1) / (32 * 8);
    if (slices > 64) slices = 64;
    ESR_CUDA_CHECK(launch_pdl(k_chan_max, dim3(slices, n_img), dim3(256), 0, st, t.base, t.plane(), HW, (int *)out));
    esr::count_launch();
    return ESR_OK;
}

// channel attention: ck = sigmoid(W1 relu(W0 mx + b0) + b1); mx arrives as ordered ints from chan_max
__global__ void __launch_bounds__(128)
k_attn_mlp(const int *__restrict__ mx_ord, const float *__restrict__ w0, const float *__restrict__ b0,
           const float *__restrict__ w1, const float *__restrict__ b1, float *__restrict__ ck)
{
    PDL_LAUNCH_DEPENDENTS();
    PDL_WAIT();
    __shared__ float m[64], hdn[32];
    const int img = blockIdx.x, t = threadIdx.x;
    if (t < 64) m[t] = ord2f(mx_ord[img * 64 + t]);
    __syncthreads();
    if (t < 32) {
        float s = b0[t];
        for (int k = 0; k < 64; ++k) s = fmaf(w0[t * 64 + k], m[k], s);
        hdn[t] = fmaxf(s, 0.0f);
    }
    __syncthreads();
    float s = b1[t];
    for (int k = 0; k < 32; ++k) s = fmaf(w1[t * 32 + k], hdn[k], s);
    ck[img * 128 + t] = 1.0f / (1.0f + expf(-s));
}
int attn_mlp(const float *mx, int n_img, const float *w0, const float *b0, const float *w1, const float *b1, float *ck,
             cudaStream_t st)
{
    ESR_CUDA_CHECK(launch_pdl(k_attn_mlp, dim3(n_img), dim3(128), 0, st, (const int *)mx, w0, b0, w1, b1, ck));
    esr::count_launch();
    return ESR_OK;
}

// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_attn_apply(const __nv_bfloat16 *__restrict__ al, size_t al_plane, const __nv_bfloat16 *__restrict__ mid, size_t mid_plane,
             const int *__restrict__ mid_img, const float *__restrict__ sk, const float *__restrict__ ck, int n_img, int HW,
             __nv_bfloat16 *__restrict__ out, size_t out_plane)
{
    PDL_LAUNCH_DEPENDENTS();
    PDL_WAIT();
    const size_t total = (size_t)n_img * HW * 16;            // 16 groups of 8 channels = 128
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int g = (int)(i % 16);
        const size_t p = i / 16;
        const int pix = (int)(p % HW), img = (int)(p / HW);
        const int part = g / 8, c0 = (g % 8) * 8;
        float v[8];
        if (part == 0) load8(al + p * 64 + c0, al_plane, v);
        else load8(mid + ((size_t)(mid_img ? mid_img[img] : img) * HW + pix) * 64 + c0, mid_plane, v);
        const float s = sk[p * 2 + part];
        const float *c = ck + img * 128 + part * 64 + c0;
#pragma unroll
        for (int e = 0; e < 8; ++e) v[e] = (v[e] * s) * c[e];       // (feat * spatial) * channel, as model.py:224-227
        store8(out + p * 128 + part * 64 + c0, out_plane, v);
    }
}
int attn_apply(const SplitTensor &aligned, const SplitTensor &mid_src, const int *mid_img, const float *sk, const float *ck,
               int n_img, const SplitTensor &out, cudaStream_t st)
{
    const int HW = aligned.H * aligned.W;
    const size_t total = (size_t)n_img * HW * 16;
    ESR_CUDA_CHECK(launch_pdl(k_attn_apply, dim3((unsigned)ceil_div64((int64_t)total, 256)), dim3(256), 0, st, aligned.base, aligned.plane(), mid_src.base,
                                                                            mid_src.plane(), mid_img, sk, ck, n_img, HW,
                                                                            out.base, out.plane()));
    esr::count_launch();
    return ESR_OK;
}

// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_scale_aggregate(const __nv_bfloat16 *__restrict__ x, size_t x_plane, const __nv_bfloat16 *__restrict__ feats, size_t f_plane,
                  const float *__restrict__ att, const int *__restrict__ fidx, int B, int N, int HW, int C,
                  __nv_bfloat16 *__restrict__ out, size_t out_plane)
{
    PDL_LAUNCH_DEPENDENTS();
    PDL_WAIT();
    const int G = C / 8;
    const size_t total = (size_t)B * HW * G;
    const float inv = 1.0f / (float)N;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int g = (int)(i % G);
        const size_t p = i / G;
        const int pix = (int)(p % HW), b = (int)(p / HW);
        float acc[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] = 0.0f;
        for (int n = 0; n < N; ++n) {
            const size_t fp = (size_t)(fidx ? fidx[b * N + n] : b * N + n) * HW + pix;
            float v[8];
            load8(feats + fp * C + g * 8, f_plane, v);
            const float a = att[fp];
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[e] += v[e] * a;         // sum over frames in order, then / N (mean)
        }
        float xv[8];
        load8(x + p * C + g * 8, x_plane, xv);
#pragma unroll
        for (int e = 0; e < 8; ++e) xv[e] += acc[e] * inv;
        store8(out + p * C + g * 8, out_plane, xv);
    }
}
int scale_aggregate(const SplitTensor &x, const SplitTensor &feats, const float *att, const int *fidx, int B, int N,
                    const SplitTensor &out, cudaStream_t st)
{
    const int HW = x.H * x.W, C = x.C;
    const size_t total = (size_t)B * HW * (C / 8);
    ESR_CUDA_CHECK(launch_pdl(k_scale_aggregate, dim3((unsigned)ceil_div64((int64_t)total, 256)), dim3(256), 0, st, x.base, x.plane(), feats.base, feats.plane(),
                                                                                 att, fidx, B, N, HW, C, out.base, out.plane()));
    esr::count_launch();
    return ESR_OK;
}

// ---------------------------------------------------------------------------------------------
// F.interpolate(scale_factor=2, mode='bilinear', align_corners=False) (models/submodules.py:290) on a split tensor:
// src index = max(0, (dst + 0.5) / 2 - 0.5), neighbours clamped; same association as ATen's upsample_bilinear2d.
__global__ void __launch_bounds__(256)
k_upsample2x(const __nv_bfloat16 *__restrict__ src, size_t s_plane, int n_img, int H, int W, int C,
             __nv_bfloat16 *__restrict__ dst, size_t d_plane)
{
    PDL_LAUNCH_DEPENDENTS();
    PDL_WAIT();
    // grid = (chunks of an output row, output rows, images): no 64-bit index arithmetic per element (the flat-index form spent more
    // instructions on its divisions than on the interpolation: 29 us for 63 MB at cfg2)
    const int G = C / 8, W2 = 2 * W;
    const int y = blockIdx.y, img = blockIdx.z;
    const float fy = fmaxf(0.0f, ((float)y + 0.5f) * 0.5f - 0.5f);
    const int y0 = (int)fy, y1 = min(y0 + 1, H - 1);
    const float ly = fy - (float)y0;
    const __nv_bfloat16 *r0 = src + ((size_t)img * H + y0) * W * C, *r1 = src + ((size_t)img * H + y1) * W * C;
    __nv_bfloat16 *drow = dst + ((size_t)img * 2 * H + y) * W2 * C;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < W2 * G; i += gridDim.x * blockDim.x) {
        const int x = i / G, g = i - x * G;
        const float fx = fmaxf(0.0f, ((float)x + 0.5f) * 0.5f - 0.5f);
        const int x0 = (int)fx, x1 = min(x0 + 1, W - 1);
        const float lx = fx - (float)x0;
        float v00[8], v01[8], v10[8], v11[8], o[8];
        load8(r0 + x0 * C + g * 8, s_plane, v00);
        load8(r0 + x1 * C + g * 8, s_plane, v01);
        load8(r1 + x0 * C + g * 8, s_plane, v10);
        load8(r1 + x1 * C + g * 8, s_plane, v11);
#pragma unroll
        for (int e = 0; e < 8; ++e)
            o[e] = (1.0f - ly) * ((1.0f - lx) * v00[e] + lx * v01[e]) + ly * ((1.0f - lx) * v10[e] + lx * v11[e]);
        store8(drow + (size_t)i * 8, d_plane, o);
    }
}
int upsample2x(const SplitTensor &src, int n_img, const SplitTensor &dst, cudaStream_t st)
{
    ESR_REQUIRE(dst.H == 2 * src.H && dst.W == 2 * src.W && dst.C == src.C && src.C % 8 == 0, "upsample2x: bad shapes");
    ESR_REQUIRE(dst.H <= 65535 && n_img <= 65535, "upsample2x: grid too large");
    const int row_items = dst.W * (src.C / 8);
    ESR_CUDA_CHECK(launch_pdl(k_upsample2x, dim3((unsigned)((row_items + 255) / 256), (unsigned)dst.H, (unsigned)n_img), dim3(256), 0, st, src.base, src.plane(),
                              n_img, src.H, src.W, src.C, dst.base, dst.plane()));
    esr::count_launch();
    return ESR_OK;
}

// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_copy_split(const __nv_bfloat16 *__restrict__ src, size_t s_plane, const int *__restrict__ src_img, int n_img, size_t per_img8,
             __nv_bfloat16 *__restrict__ dst, size_t d_plane)
{
    PDL_LAUNCH_DEPENDENTS();
    PDL_WAIT();
    const size_t total = (size_t)n_img * per_img8;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t img = i / per_img8, r = i % per_img8;
        const size_t s = ((size_t)(src_img ? src_img[img] : (int)img) * per_img8 + r) * 8;
        const size_t d = i * 8;
        *reinterpret_cast<uint4 *>(dst + d) = *reinterpret_cast<const uint4 *>(src + s);
        *reinterpret_cast<uint4 *>(dst + d_plane + d) = *reinterpret_cast<const uint4 *>(src + s_plane + s);
    }
}
int copy_split(const SplitTensor &src, const int *src_img, int n_img, const SplitTensor &dst, cudaStream_t st)
{
    const size_t per_img8 = (size_t)src.H * src.W * src.C / 8;
    const size_t total = (size_t)n_img * per_img8;
    ESR_CUDA_CHECK(launch_pdl(k_copy_split, dim3((unsigned)ceil_div64((int64_t)total, 256)), dim3(256), 0, st, src.base, src.plane(), src_img, n_img, per_img8,
                                                                            dst.base, dst.plane()));
    esr::count_launch();
    return ESR_OK;
}

} // namespace esr

// ------------------------------------------------------------------------------------------------
// Narrow-output convolution of a 64-channel split tensor on CUDA cores: the spatial-attention kernel (models/model.py:183),
// 1x1, Cout = 2, sigmoid.  On the tensor cores it pads N to 16 and moves a full 128 x 64 A tile for 2 useful columns (19 us per
// cfg2 step, 1.2 TB/s); it is a read of an L2-resident tensor, so plain fp32 FMAs do: 8 lanes per pixel, 8 channels (16 B hi +
// 16 B lo) each, 3 shuffles to reduce.  fp32 products of the exact hi + lo values (no operand split needed).
// ------------------------------------------------------------------------------------------------
namespace esr {

template <int CIN, int COUT, int TAPS>
__global__ void __launch_bounds__(256)
k_conv_narrow(const __nv_bfloat16 *__restrict__ x, size_t plane, const int *__restrict__ src_img, const float *__restrict__ w /*[TAPS][CIN][COUT]*/,
              const float *__restrict__ bias, int n_img, int H, int W, float *__restrict__ out)
{
    PDL_LAUNCH_DEPENDENTS();
    PDL_WAIT();
    constexpr int LPP = CIN / 8;                          // lanes per pixel: 8 channels (16 B hi + 16 B lo) each
    constexpr int PPB = 256 / LPP, TH = PPB / 8;          // pixels per block: 8 wide x TH tall
    __shared__ float sw[TAPS * CIN * COUT];
    for (int i = threadIdx.x; i < TAPS * CIN * COUT; i += 256) sw[i] = w[i];
    __syncthreads();
    const int lc = threadIdx.x % LPP;                     // channels [8 lc, 8 lc + 8)
    const int px_in_blk = threadIdx.x / LPP;
    const int tiles_x = (W + 7) / 8, tiles_y = (H + TH - 1) / TH;
    const int tile = blockIdx.x % (tiles_x * tiles_y), img = blockIdx.x / (tiles_x * tiles_y);
    const int y = (tile / tiles_x) * TH + (px_in_blk >> 3), xx = (tile % tiles_x) * 8 + (px_in_blk & 7);
    const bool valid = y < H && xx < W;
    const size_t ibase = (size_t)(src_img ? src_img[img] : img) * H * W;
    float acc[COUT];
#pragma unroll
    for (int c = 0; c < COUT; ++c) acc[c] = 0.0f;
    // branch-free taps: out-of-image neighbours read a clamped (valid) address and are zeroed, so all 2 x TAPS loads of a thread are
    // independent and issue back to back
    uint4 hv[TAPS], lv[TAPS];
#pragma unroll
    for (int t = 0; t < TAPS; ++t) {
        const int yy = y + (TAPS == 9 ? t / 3 - 1 : 0), xs = xx + (TAPS == 9 ? t % 3 - 1 : 0);
        const bool ok = valid && yy >= 0 && yy < H && xs >= 0 && xs < W;
        const int yc = min(max(yy, 0), H - 1), xc = min(max(xs, 0), W - 1);
        const __nv_bfloat16 *p = x + ((ibase + (size_t)yc * W + xc) * CIN + lc * 8);
        hv[t] = *reinterpret_cast<const uint4 *>(p);
        lv[t] = *reinterpret_cast<const uint4 *>(p + plane);
        if (!ok) { hv[t] = make_uint4(0u, 0u, 0u, 0u); lv[t] = make_uint4(0u, 0u, 0u, 0u); }
    }
#pragma unroll
    for (int t = 0; t < TAPS; ++t) {
        const uint32_t hw[4] = {hv[t].x, hv[t].y, hv[t].z, hv[t].w}, lw[4] = {lv[t].x, lv[t].y, lv[t].z, lv[t].w};
        const float *wt = sw + (t * CIN + lc * 8) * COUT;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float v0 = __uint_as_float(hw[e] << 16) + __uint_as_float(lw[e] << 16);
            const float v1 = __uint_as_float(hw[e] & 0xffff0000u) + __uint_as_float(lw[e] & 0xffff0000u);
#pragma unroll
            for (int c = 0; c < COUT; ++c) {
                acc[c] = fmaf(v0, wt[(2 * e) * COUT + c], acc[c]);
                acc[c] = fmaf(v1, wt[(2 * e + 1) * COUT + c], acc[c]);
            }
        }
    }
#pragma unroll
    for (int c = 0; c < COUT; ++c) {
#pragma unroll
        for (int o = 1; o < LPP; o <<= 1) acc[c] += __shfl_xor_sync(0xffffffffu, acc[c], o);
    }
    if (valid && lc == 0) {
#pragma unroll
        for (int c = 0; c < COUT; ++c) out[(((size_t)img * H + y) * W + xx) * COUT + c] = fast_sigmoid(acc[c] + bias[c]);
    }
}

template <int CIN, int COUT, int TAPS>
static int launch_narrow(const SplitTensor &x, const int *src_img, const float *w, const float *bias, int n_img, float *out, cudaStream_t st)
{
    constexpr int TH = (256 / (CIN / 8)) / 8;
    const dim3 grid((unsigned)(n_img * ((x.W + 7) / 8) * ((x.H + TH - 1) / TH)));
    ESR_CUDA_CHECK(launch_pdl(k_conv_narrow<CIN, COUT, TAPS>, grid, dim3(256), 0, st, x.base, x.plane(), src_img, w, bias, n_img, x.H,
                              x.W, out));
    esr::count_launch();
    return ESR_OK;
}

int conv_narrow(const SplitTensor &x, const int *src_img, const float *w, const float *bias, int cout, int ntaps, int n_img, float *out,
                cudaStream_t st)
{
    if (x.C == 64 && cout == 2 && ntaps == 1) return launch_narrow<64, 2, 1>(x, src_img, w, bias, n_img, out, st);
    set_error("conv_narrow: C=%d cout=%d taps=%d has no instantiation", x.C, cout, ntaps);
    return ESR_EINVAL;
}

// fp32 [Cout, 64, k, k] -> [tap][ci][co]
__global__ void k_pack_narrow_weight(const float *__restrict__ w, int cout, int ntaps, float *__restrict__ dst)
{
    const int total = ntaps * 64 * cout;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int co = i % cout, ci = (i / cout) % 64, tap = i / (cout * 64);
        dst[i] = w[((size_t)co * 64 + ci) * ntaps + tap];
    }
}
int pack_narrow_weight(const float *w, int cout, int ntaps, float *dst, cudaStream_t st)
{
    k_pack_narrow_weight<<<(ntaps * 64 * cout + 255) / 256, 256, 0, st>>>(w, cout, ntaps, dst);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}

} // namespace esr

// ---- esr_glue: one launcher of the element-wise glue, as esr_net_forward calls it
using namespace esr;

static SplitTensor glue_split(const void *p, int n_img, int H, int W, int C)
{
    SplitTensor t;
    t.base = (__nv_bfloat16 *)p; t.n_img = n_img; t.H = H; t.W = W; t.C = C;
    return t;
}

extern "C" int esr_glue(const esr_glue_desc *d, esr_stream_t stream)
{
    ESR_REQUIRE(d, "esr_glue: null descriptor");
    const int op = d->op;
    ESR_REQUIRE(op >= ESR_GLUE_LTC_CAT && op <= ESR_GLUE_COPY_SPLIT, "esr_glue: op %d", op);
    ESR_REQUIRE(d->n_img > 0 && d->H > 0 && d->W > 0, "esr_glue: n_img=%d H=%d W=%d", d->n_img, d->H, d->W);
    const bool c64 = op <= ESR_GLUE_ATTN_APPLY;
    ESR_REQUIRE(c64 ? d->C == 64 : d->C > 0 && d->C % 8 == 0, "esr_glue: op %d has no kernel for C=%d (%s)", op, d->C,
                c64 ? "64 only" : "a multiple of 8");
    const int n = d->n_img, N = d->N;
    const bool needs_in = op != ESR_GLUE_ATTN_MLP, needs_in2 = op == ESR_GLUE_ATTN_APPLY || op == ESR_GLUE_SCALE_AGGREGATE;
    ESR_REQUIRE(!needs_in || (d->in && d->in_n_img > 0), "esr_glue: op %d: missing input", op);
    ESR_REQUIRE(!needs_in2 || (d->in2 && d->in2_n_img > 0), "esr_glue: op %d: missing second input", op);
    ESR_REQUIRE(op != ESR_GLUE_LTC_CAT || (d->idx && d->maps), "esr_glue: ltc_cat needs idx and maps");
    ESR_REQUIRE(op != ESR_GLUE_ATTN_MLP || (d->mx && d->w0 && d->b0 && d->w1 && d->b1 && d->ck), "esr_glue: attn_mlp: missing mx, weights or ck");
    ESR_REQUIRE(op != ESR_GLUE_CHAN_MAX || d->mx, "esr_glue: chan_max: missing mx");
    ESR_REQUIRE(op != ESR_GLUE_ATTN_APPLY || (d->sk && d->ck_in), "esr_glue: attn_apply: missing sk or ck_in");
    ESR_REQUIRE(op != ESR_GLUE_SCALE_AGGREGATE || (d->att && N > 0), "esr_glue: scale_aggregate: missing att or N=%d", N);
    const bool split_out = op != ESR_GLUE_CHAN_MAX && op != ESR_GLUE_ATTN_MLP;
    ESR_REQUIRE(!split_out || d->out, "esr_glue: op %d: missing output", op);
    ESR_REQUIRE(d->out_n_img >= n, "esr_glue: op %d: %d output images for n_img=%d", op, d->out_n_img, n);
    // inputs read at the output's own image (no table): they must hold n_img images (n_img * N frames for the aggregation)
    ESR_REQUIRE(!(op == ESR_GLUE_CHAN_MAX || op == ESR_GLUE_ATTN_APPLY || op == ESR_GLUE_SCALE_AGGREGATE || op == ESR_GLUE_UPSAMPLE2X ||
                  (op == ESR_GLUE_COPY_SPLIT && !d->idx)) || d->in_n_img >= n,
                "esr_glue: op %d: input holds %d images for n_img=%d", op, d->in_n_img, n);
    ESR_REQUIRE(!(op == ESR_GLUE_SCALE_AGGREGATE && !d->idx) || (long long)d->in2_n_img >= (long long)n * N,
                "esr_glue: scale_aggregate: %d frames for n_img=%d x N=%d", d->in2_n_img, n, N);
    ESR_REQUIRE(!(op == ESR_GLUE_ATTN_APPLY && !d->idx) || d->in2_n_img >= n, "esr_glue: attn_apply: second input holds %d images for n_img=%d",
                d->in2_n_img, n);
    // grid limits: chan_max puts images on grid y, upsample2x output rows on y and images on z
    ESR_REQUIRE(op != ESR_GLUE_CHAN_MAX || n <= 65535, "esr_glue: chan_max: n_img=%d > 65535", n);
    ESR_REQUIRE(op != ESR_GLUE_UPSAMPLE2X || (2 * (long long)d->H <= 65535 && n <= 65535), "esr_glue: upsample2x: 2H=%lld or n_img=%d > 65535",
                2 * (long long)d->H, n);

    cudaStream_t st = (cudaStream_t)stream;
    const int H = d->H, W = d->W, C = d->C;
    const SplitTensor in = glue_split(d->in, d->in_n_img, H, W, C), in2 = glue_split(d->in2, d->in2_n_img, H, W, C);
    switch (op) {
    case ESR_GLUE_LTC_CAT: return ltc_cat(in, d->maps, d->idx, n, glue_split(d->out, d->out_n_img, H, W, 192), st);
    case ESR_GLUE_CHAN_MAX: return chan_max(in, n, (float *)d->mx, st);
    case ESR_GLUE_ATTN_MLP: return attn_mlp((const float *)d->mx, n, d->w0, d->b0, d->w1, d->b1, d->ck, st);
    case ESR_GLUE_ATTN_APPLY: return attn_apply(in, in2, d->idx, d->sk, d->ck_in, n, glue_split(d->out, d->out_n_img, H, W, 128), st);
    case ESR_GLUE_SCALE_AGGREGATE: return scale_aggregate(in, in2, d->att, d->idx, n, N, glue_split(d->out, d->out_n_img, H, W, C), st);
    case ESR_GLUE_UPSAMPLE2X: return upsample2x(in, n, glue_split(d->out, d->out_n_img, 2 * H, 2 * W, C), st);
    default: return copy_split(in, d->idx, n, glue_split(d->out, d->out_n_img, H, W, C), st);
    }
}
