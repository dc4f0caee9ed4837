// dcn_generic.cu -- the `_ext.dcn_v2_forward` / `_ext.dcn_v2_backward` operators for ANY configuration the reference's
// operator accepts (channels, groups, kernel size, stride, padding, dilation): the shapes other than the one ESR's network
// uses (64 -> 64, 3x3, 8 groups, which runs on the wgmma path of dcn.cu / dcn_fused.cu / dcn_bwd.cu).  The reference's own
// tests and examples call the operator with 2 -> 2 channels on 4x4 maps and with deformable_groups = 2
// (models/DCNv2/testcuda.py:14-17, 169-180), so a drop-in has to serve them.
//
// Semantics restated from models/DCNv2/src/cuda/dcn_v2_cuda.cu:20-216 and dcn_v2_im2col_cuda.cu:25-327:
//   columns[b][(c*kh + i)*kw + j][p] = bilinear(in[b][c], y*s - pad + i*dil + off_h, x*s - pad + j*dil + off_w) * mask
//     with off_h / off_w = offset[b][g*2*K + 2*(i*kw+j) (+1)][p], mask[b][g*K + i*kw + j][p], g = c / (C/G), K = kh*kw;
//     a sample contributes only if it lies in (-1, H) x (-1, W); corners outside the image read as zero.
//   out[b][co][p] = bias[co] + sum_r W[co][r] * columns[b][r][p]
//   backward: grad_columns = W^T . grad_out; grad_weight = grad_out . columns^T; grad_bias = sum grad_out;
//             grad_mask, grad_offset and grad_input from grad_columns through the bilinear weights (atomics on grad_input,
//             as in the reference's col2im kernel).
// Plain fp32 CUDA-core kernels (FFMA, shared-memory tiled GEMMs): generality first, this is not the hot path.
#include "net.cuh"

namespace esr {

struct DcnGeo {
    int B, C, H, W, Co, kh, kw, stride, pad, dil, G, Ho, Wo;
    __host__ __device__ int K() const { return kh * kw; }
    __host__ __device__ int cpg() const { return C / G; }
};

__device__ __forceinline__ float bilinear_zero(const float *__restrict__ im, int H, int W, float h, float w)
{
    const int h_low = (int)floorf(h), w_low = (int)floorf(w);
    const int h_high = h_low + 1, w_high = w_low + 1;
    const float lh = h - (float)h_low, lw = w - (float)w_low, hh = 1.0f - lh, hw = 1.0f - lw;
    float v1 = 0.f, v2 = 0.f, v3 = 0.f, v4 = 0.f;
    if (h_low >= 0 && w_low >= 0) v1 = im[h_low * W + w_low];
    if (h_low >= 0 && w_high <= W - 1) v2 = im[h_low * W + w_high];
    if (h_high <= H - 1 && w_low >= 0) v3 = im[h_high * W + w_low];
    if (h_high <= H - 1 && w_high <= W - 1) v4 = im[h_high * W + w_high];
    return hh * hw * v1 + hh * lw * v2 + lh * hw * v3 + lh * lw * v4;
}

// one thread per (b, c, output pixel): all K taps of one channel
__global__ void __launch_bounds__(256)
k_dcng_columns(DcnGeo g, const float *__restrict__ input, const float *__restrict__ offset, const float *__restrict__ mask,
               float *__restrict__ cols)
{
    const int K = g.K(), P = g.Ho * g.Wo;
    const size_t total = (size_t)g.B * g.C * P;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int p = (int)(i % P), c = (int)((i / P) % g.C), b = (int)(i / ((size_t)P * g.C));
        const int y = p / g.Wo, x = p % g.Wo, grp = c / g.cpg();
        const float *im = input + ((size_t)b * g.C + c) * g.H * g.W;
        const float *off = offset + ((size_t)b * g.G + grp) * 2 * K * P;
        const float *msk = mask + ((size_t)b * g.G + grp) * K * P;
        float *dst = cols + ((size_t)b * g.C + c) * K * P + p;
        for (int k = 0; k < K; ++k) {
            const int ki = k / g.kw, kj = k % g.kw;
            const float h_im = (float)(y * g.stride - g.pad + ki * g.dil) + off[(size_t)(2 * k) * P + p];
            const float w_im = (float)(x * g.stride - g.pad + kj * g.dil) + off[(size_t)(2 * k + 1) * P + p];
            float v = 0.0f;
            if (h_im > -1.0f && w_im > -1.0f && h_im < (float)g.H && w_im < (float)g.W) v = bilinear_zero(im, g.H, g.W, h_im, w_im);
            dst[(size_t)k * P] = v * msk[(size_t)k * P + p];
        }
    }
}

// C[M x N] (+)= op(A) . B per batch; 32 x 32 tiles, K in steps of 32.
//   TA = 0: A is [M x Kd] row-major;  TA = 1: A is [Kd x M] row-major (A^T used).
//   TB = 0: B is [Kd x N] row-major;  TB = 1: B is [N x Kd] row-major (B^T used).
// batch strides sA / sB / sC (0 = shared operand); `reduce_batches` sums all batches into ONE C with atomics.
template <int TA, int TB>
__global__ void __launch_bounds__(256)
k_dcng_gemm(const float *__restrict__ A, const float *__restrict__ Bm, float *__restrict__ Cm, const float *__restrict__ bias,
            int M, int N, int Kd, size_t sA, size_t sB, size_t sC, int reduce_batches)
{
    __shared__ float As[32][33], Bs[32][33];
    const int b = blockIdx.z;
    const float *Ab = A + (size_t)b * sA;
    const float *Bb = Bm + (size_t)b * sB;
    float *Cb = Cm + (reduce_batches ? 0 : (size_t)b * sC);
    const int m0 = blockIdx.y * 32, n0 = blockIdx.x * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;            // 32 x 8 threads, 4 rows each
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int k0 = 0; k0 < Kd; k0 += 32) {
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const int row = ty * 4 + r;
            {   // As[m][k]
                const int m = m0 + row, k = k0 + tx;
                float v = 0.f;
                if (TA == 0) { if (m < M && k < Kd) v = Ab[(size_t)m * Kd + k]; As[row][tx] = v; }
                else { const int kk = k0 + row, mm = m0 + tx; if (mm < M && kk < Kd) v = Ab[(size_t)kk * M + mm]; As[tx][row] = v; }
            }
            {   // Bs[k][n]
                float v = 0.f;
                if (TB == 0) { const int k = k0 + row, n = n0 + tx; if (k < Kd && n < N) v = Bb[(size_t)k * N + n]; Bs[row][tx] = v; }
                else { const int n = n0 + row, k = k0 + tx; if (n < N && k < Kd) v = Bb[(size_t)n * Kd + k]; Bs[tx][row] = v; }
            }
        }
        __syncthreads();
#pragma unroll 8
        for (int k = 0; k < 32; ++k) {
            const float bv = Bs[k][tx];
#pragma unroll
            for (int r = 0; r < 4; ++r) acc[r] += As[ty * 4 + r][k] * bv;
        }
        __syncthreads();
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        const int m = m0 + ty * 4 + r, n = n0 + tx;
        if (m < M && n < N) {
            if (reduce_batches) atomicAdd(&Cb[(size_t)m * N + n], acc[r]);
            else Cb[(size_t)m * N + n] = acc[r] + (bias ? bias[m] : 0.0f);
        }
    }
}

// grad_bias[co] = sum over b, p
__global__ void __launch_bounds__(256) k_dcng_bias_grad(const float *__restrict__ go, int B, int Co, int P, float *__restrict__ gb)
{
    const int co = blockIdx.x;
    float s = 0.f;
    for (int i = threadIdx.x; i < B * P; i += 256) s += go[((size_t)(i / P) * Co + co) * P + i % P];
    __shared__ float red[256];
    red[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) { if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o]; __syncthreads(); }
    if (threadIdx.x == 0) gb[co] = red[0];
}

// one thread per (b, group, tap, output pixel): loops over the group's channels; grad_mask / grad_offset are owned by the
// thread (plain stores), grad_input takes atomics (different taps / pixels hit the same input pixel)
__global__ void __launch_bounds__(256)
k_dcng_bwd_sample(DcnGeo g, const float *__restrict__ input, const float *__restrict__ offset, const float *__restrict__ mask,
                  const float *__restrict__ gcols, float *__restrict__ gin, float *__restrict__ goff, float *__restrict__ gmask)
{
    const int K = g.K(), P = g.Ho * g.Wo, cpg = g.cpg();
    const size_t total = (size_t)g.B * g.G * K * P;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int p = (int)(i % P), k = (int)((i / P) % K), grp = (int)((i / ((size_t)P * K)) % g.G), b = (int)(i / ((size_t)P * K * g.G));
        const int y = p / g.Wo, x = p % g.Wo, ki = k / g.kw, kj = k % g.kw;
        const size_t o_idx = (((size_t)b * g.G + grp) * 2 * K + 2 * k) * P + p;
        const size_t m_idx = (((size_t)b * g.G + grp) * K + k) * P + p;
        const float h_im = (float)(y * g.stride - g.pad + ki * g.dil) + offset[o_idx];
        const float w_im = (float)(x * g.stride - g.pad + kj * g.dil) + offset[o_idx + P];
        const float m = mask[m_idx];
        float gm = 0.f, gh = 0.f, gw = 0.f;
        if (h_im > -1.0f && w_im > -1.0f && h_im < (float)g.H && w_im < (float)g.W) {
            const int h_low = (int)floorf(h_im), w_low = (int)floorf(w_im), h_high = h_low + 1, w_high = w_low + 1;
            const float lh = h_im - (float)h_low, lw = w_im - (float)w_low, hh = 1.0f - lh, hw = 1.0f - lw;
            const bool ok1 = h_low >= 0 && w_low >= 0, ok2 = h_low >= 0 && w_high <= g.W - 1;
            const bool ok3 = h_high <= g.H - 1 && w_low >= 0, ok4 = h_high <= g.H - 1 && w_high <= g.W - 1;
            for (int cc = 0; cc < cpg; ++cc) {
                const int c = grp * cpg + cc;
                const float *im = input + ((size_t)b * g.C + c) * g.H * g.W;
                float *gi = gin + ((size_t)b * g.C + c) * g.H * g.W;
                const float gc = gcols[(((size_t)b * g.C + c) * K + k) * P + p];
                const float v1 = ok1 ? im[h_low * g.W + w_low] : 0.f, v2 = ok2 ? im[h_low * g.W + w_high] : 0.f;
                const float v3 = ok3 ? im[h_high * g.W + w_low] : 0.f, v4 = ok4 ? im[h_high * g.W + w_high] : 0.f;
                gm += gc * (hh * hw * v1 + hh * lw * v2 + lh * hw * v3 + lh * lw * v4);
                gh += gc * m * (-hw * v1 - lw * v2 + hw * v3 + lw * v4);
                gw += gc * m * (-hh * v1 + hh * v2 - lh * v3 + lh * v4);
                const float t = gc * m;
                if (ok1) atomicAdd(&gi[h_low * g.W + w_low], t * hh * hw);
                if (ok2) atomicAdd(&gi[h_low * g.W + w_high], t * hh * lw);
                if (ok3) atomicAdd(&gi[h_high * g.W + w_low], t * lh * hw);
                if (ok4) atomicAdd(&gi[h_high * g.W + w_high], t * lh * lw);
            }
        }
        gmask[m_idx] = gm;
        goff[o_idx] = gh;
        goff[o_idx + P] = gw;
    }
}

static bool geo_ok(const DcnGeo &g)
{
    return g.B > 0 && g.C > 0 && g.Co > 0 && g.H > 0 && g.W > 0 && g.kh > 0 && g.kw > 0 && g.stride > 0 && g.pad >= 0 && g.dil > 0 &&
           g.G > 0 && g.C % g.G == 0 && g.Ho > 0 && g.Wo > 0;
}
static DcnGeo make_geo(int B, int C, int H, int W, int Co, int kernel, int stride, int pad, int dil, int G)
{
    DcnGeo g{B, C, H, W, Co, kernel, kernel, stride, pad, dil, G, 0, 0};
    g.Ho = (H + 2 * pad - (dil * (kernel - 1) + 1)) / stride + 1;
    g.Wo = (W + 2 * pad - (dil * (kernel - 1) + 1)) / stride + 1;
    return g;
}
static unsigned grid1d(size_t total) { return (unsigned)(total / 256 + 1 > 65535u * 16u ? 65535u * 16u : total / 256 + 1); }

size_t dcn_generic_ws_bytes(int B, int C, int H, int W, int Co, int kernel, int stride, int pad, int dil, int G, int backward)
{
    const DcnGeo g = make_geo(B, C, H, W, Co, kernel, stride, pad, dil, G);
    if (!geo_ok(g)) return 0;
    const size_t cols = align_up((size_t)B * C * g.K() * g.Ho * g.Wo * sizeof(float), 256);
    return backward ? 2 * cols : cols;
}

int dcn_generic_forward(const float *input, const float *weight, const float *bias, const float *offset, const float *mask, int B,
                        int C, int H, int W, int Co, int kernel, int stride, int pad, int dil, int G, float *output,
                        void *workspace, size_t ws_bytes, cudaStream_t st)
{
    const DcnGeo g = make_geo(B, C, H, W, Co, kernel, stride, pad, dil, G);
    ESR_REQUIRE(geo_ok(g), "dcn_v2_forward: bad geometry (C=%d G=%d k=%d s=%d p=%d d=%d on %dx%d)", C, G, kernel, stride, pad, dil, H, W);
    const size_t need = dcn_generic_ws_bytes(B, C, H, W, Co, kernel, stride, pad, dil, G, 0);
    if (ws_bytes < need) { set_error("dcn_v2_forward: workspace %zu < %zu", ws_bytes, need); return ESR_EWORKSPACE; }
    float *cols = (float *)workspace;
    const int P = g.Ho * g.Wo, R = C * g.K();
    k_dcng_columns<<<grid1d((size_t)B * C * P), 256, 0, st>>>(g, input, offset, mask, cols);
    ESR_LAUNCH_CHECK();
    dim3 grid((P + 31) / 32, (Co + 31) / 32, B);
    k_dcng_gemm<0, 0><<<grid, 256, 0, st>>>(weight, cols, output, bias, Co, P, R, 0, (size_t)R * P, (size_t)Co * P, 0);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}

int dcn_generic_backward(const float *input, const float *weight, const float *offset, const float *mask, const float *grad_output,
                         int B, int C, int H, int W, int Co, int kernel, int stride, int pad, int dil, int G, float *grad_input,
                         float *grad_offset, float *grad_mask, float *grad_weight, float *grad_bias, void *workspace,
                         size_t ws_bytes, cudaStream_t st)
{
    const DcnGeo g = make_geo(B, C, H, W, Co, kernel, stride, pad, dil, G);
    ESR_REQUIRE(geo_ok(g), "dcn_v2_backward: bad geometry (C=%d G=%d k=%d s=%d p=%d d=%d on %dx%d)", C, G, kernel, stride, pad, dil, H, W);
    const size_t need = dcn_generic_ws_bytes(B, C, H, W, Co, kernel, stride, pad, dil, G, 1);
    if (ws_bytes < need) { set_error("dcn_v2_backward: workspace %zu < %zu", ws_bytes, need); return ESR_EWORKSPACE; }
    const int P = g.Ho * g.Wo, R = C * g.K();
    float *cols = (float *)workspace;
    float *gcols = (float *)((char *)workspace + need / 2);
    ESR_CUDA_CHECK(cudaMemsetAsync(grad_input, 0, (size_t)B * C * H * W * sizeof(float), st));
    ESR_CUDA_CHECK(cudaMemsetAsync(grad_weight, 0, (size_t)Co * R * sizeof(float), st));
    k_dcng_columns<<<grid1d((size_t)B * C * P), 256, 0, st>>>(g, input, offset, mask, cols);
    ESR_LAUNCH_CHECK();
    // grad_columns[b] = W^T [R x Co] . grad_out[b] [Co x P]
    k_dcng_gemm<1, 0><<<dim3((P + 31) / 32, (R + 31) / 32, B), 256, 0, st>>>(weight, grad_output, gcols, nullptr, R, P, Co, 0,
                                                                              (size_t)Co * P, (size_t)R * P, 0);
    ESR_LAUNCH_CHECK();
    // grad_weight [Co x R] = sum_b grad_out[b] [Co x P] . columns[b]^T [P x R]
    k_dcng_gemm<0, 1><<<dim3((R + 31) / 32, (Co + 31) / 32, B), 256, 0, st>>>(grad_output, cols, grad_weight, nullptr, Co, R, P,
                                                                               (size_t)Co * P, (size_t)R * P, 0, 1);
    ESR_LAUNCH_CHECK();
    k_dcng_bias_grad<<<Co, 256, 0, st>>>(grad_output, B, Co, P, grad_bias);
    ESR_LAUNCH_CHECK();
    k_dcng_bwd_sample<<<grid1d((size_t)B * G * g.K() * P), 256, 0, st>>>(g, input, offset, mask, gcols, grad_input, grad_offset, grad_mask);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}

} // namespace esr
