// train_ops.cu -- operators of the training step (SURVEY.md 8a row 17: train_ours_cnt_seq.py:206-235, 767-782).
//
// The reference's step is  sum over windows of MSELoss(forward(window), gt)  ->  one backward  ->  Adam(amsgrad).  Its
// backward is ATen's conv2d backward for every ConvLayer (models/submodules.py:159-200) plus `_ext.dcn_v2_backward`
// (dcn_bwd.cu here).  This file holds the convolution operator pair in the reference's own tensor layout (fp32 NCHW, the
// layout autograd hands over) and the loss / optimizer kernels:
//
//   esr_conv2d_forward   y = act(conv(x, w) + b)            3x3 pad 1 or 1x1 pad 0, stride 1 or 2
//   esr_conv2d_backward  g = dy * act'(y);  db = sum g;  dw = x (*) g;  dx = g (*) rot180(w)^T
//   esr_mse_loss         mean((p - t)^2) and its gradient
//   esr_adam_step        torch.optim.Adam semantics (L2 weight decay folded into the gradient, optional amsgrad)
//
// Stride-1 layers with 64-multiple input channels run on the wgmma implicit-GEMM kernel of tc_conv.cu (fp32 -> split
// bf16, 3-pass product, fp32 accumulate): the forward directly, dx as the same kernel over g with the weights transposed
// and rotated, and dw as a tensor-core reduction over pixels (k_wgrad_tc below, MN-major operands).  Every other shape
// (the <= 32-channel full-resolution layers, stride-2 encoder convs, 1- and 2-channel heads) uses the CUDA-core kernels
// in this file.  By default dw / db and the loss accumulate with fp32 atomics, so their summation order over pixels varies from
// run to run (as the reference's cuDNN / atomicAdd backward does when cudnn.deterministic is off).  With ESR_DETERMINISTIC in
// the flags of the _ex entry points every such sum goes through per-block partials and an ordered second pass instead, and
// the results are bitwise reproducible on a given GPU model.
#include "tc_common.cuh"
#include "net.cuh"

namespace esr {

// ------------------------------------------------------------------------------------------------------------------
// elementwise pieces
// ------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float act_fwd(float v, int act)
{
    if (act == ACT_RELU) return fmaxf(v, 0.0f);
    if (act == ACT_SIGMOID) return 1.0f / (1.0f + __expf(-v));
    if (act == ACT_TANH) return tanhf(v);
    return v;
}

__global__ void __launch_bounds__(256) k_act_bwd(const float *__restrict__ dy, const float *__restrict__ y, float *__restrict__ g,
                                                 size_t n, int act)
{
    for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (size_t)gridDim.x * 256) {
        const float o = y[i];
        float d = 1.0f;
        if (act == ACT_RELU) d = o > 0.0f ? 1.0f : 0.0f;
        else if (act == ACT_SIGMOID) d = o * (1.0f - o);
        else if (act == ACT_TANH) d = 1.0f - o * o;
        g[i] = dy[i] * d;
    }
}

// Deterministic mode (ESR_DETERMINISTIC): every reduction over pixels that ends in fp32 atomics by default has a variant that
// writes one partial per block (or per thread role) to slot s of a workspace buffer [slots][n] instead; k_sum_slices then adds
// the slots in slot order.  The slot a partial lands in depends only on the launch geometry, never on CTA scheduling.
// The variants share the kernel bodies below through a DET template parameter; the default kernels keep their names and code.
__global__ void __launch_bounds__(256) k_sum_slices(const float *__restrict__ part, int slices, size_t n, float *__restrict__ out)
{
    for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (size_t)gridDim.x * 256) {
        float s = 0.0f;
        for (int k = 0; k < slices; ++k) s += part[(size_t)k * n + i];
        out[i] = s;
    }
}

int sum_slices(const float *part, int slices, size_t n, float *out, cudaStream_t st)
{
    k_sum_slices<<<(unsigned)min((size_t)2048, (n + 255) / 256), 256, 0, st>>>(part, slices, n, out);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}

// db[co] += sum over (n, pixel) of g[n, co, pixel]; grid (Cout, chunks).  DET: partial of block (co, chunk) -> db[chunk][co]
template <bool DET>
__device__ __forceinline__ void bias_grad_body(const float *__restrict__ g, int B, int Cout, int HW, float *__restrict__ db)
{
    const int co = blockIdx.x;
    const size_t total = (size_t)B * HW;
    float s = 0.0f;
    for (size_t i = (size_t)blockIdx.y * 256 + threadIdx.x; i < total; i += (size_t)gridDim.y * 256) {
        const size_t n = i / HW, p = i - n * HW;
        s += g[(n * Cout + co) * HW + p];
    }
    __shared__ float red[8];
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x < 8) {
        s = red[threadIdx.x];
        for (int o = 4; o > 0; o >>= 1) s += __shfl_xor_sync(0xffu, s, o);
        if (threadIdx.x == 0) {
            if (DET) db[(size_t)blockIdx.y * Cout + co] = s;
            else atomicAdd(db + co, s);
        }
    }
}
__global__ void __launch_bounds__(256) k_bias_grad(const float *__restrict__ g, int B, int Cout, int HW, float *__restrict__ db)
{
    bias_grad_body<false>(g, B, Cout, HW, db);
}
__global__ void __launch_bounds__(256) k_bias_grad_det(const float *__restrict__ g, int B, int Cout, int HW, float *__restrict__ part)
{
    bias_grad_body<true>(g, B, Cout, HW, part);
}

// wT[ci][co][K-1-ky][K-1-kx] = w[co][ci][ky][kx]: the weights of the convolution that maps g to dx (co padded to CoutPad)
__global__ void k_weight_rot_t(const float *__restrict__ w, int Cout, int CoutPad, int Cin, int KK, float *__restrict__ wt)
{
    const int total = Cout * Cin * KK;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int t = i % KK, ci = (i / KK) % Cin, co = i / (KK * Cin);
        wt[((size_t)ci * CoutPad + co) * KK + (KK - 1 - t)] = w[i];
    }
}

// fp32 NCHW -> split bf16 NHWC with the channel count padded to Cpad (a multiple of 64; extra channels zero): 64-channel x
// 32-pixel tiles transposed through shared memory -- 128-byte coalesced reads per channel row, one 16-byte store per plane and
// thread (a pixel's 64 channels = one 128-byte line).  Padding lets Cout = 32 / 216 use the 64-channel tensor-core tiles.
// With dy/y/act/db it is the backward prologue of a tensor-core layer in ONE pass: g = dy * act'(y) -> split bf16, db[c] += sum g
// (warp reduction + one atomic per channel and block), optionally g in fp32 NCHW for the CUDA-core dw.
template <bool PROLOGUE>
__global__ void __launch_bounds__(256) k_to_split(const float *__restrict__ src, const float *__restrict__ y, int act, int C, int Cpad, int HW,
                                                  int tiles_per_block, __nv_bfloat16 *__restrict__ dst, size_t plane, float *__restrict__ db,
                                                  float *__restrict__ g_out)
{
    __shared__ float tile[64][33];
    const int n = blockIdx.z, c0 = blockIdx.y * 64;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int px = threadIdx.x >> 3, cg = threadIdx.x & 7;
    float bsum[8];                                                 // bias-gradient partial sums of this warp's 8 channel rows
#pragma unroll
    for (int j = 0; j < 8; ++j) bsum[j] = 0.0f;
    // several pixel tiles per block: the per-channel db atomics (all blocks hit the same <= 256 addresses) are issued once per
    // block, not once per tile -- same-address contention was the cost of the first version of this kernel
    for (int t = 0; t < tiles_per_block; ++t) {
        const int p0 = (blockIdx.x * tiles_per_block + t) * 32;
        if (p0 >= HW) break;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int r = ty + 8 * j;
            const int c = c0 + r, p = p0 + tx;
            float v = 0.0f;
            if (c < C && p < HW) {
                const size_t i = ((size_t)n * C + c) * HW + p;
                v = src[i];
                if (PROLOGUE) {
                    if (act != ACT_NONE) {
                        const float o = y[i];
                        v *= act == ACT_RELU ? (o > 0.0f ? 1.0f : 0.0f) : (act == ACT_SIGMOID ? o * (1.0f - o) : 1.0f - o * o);
                    }
                    if (g_out) g_out[i] = v;
                }
            }
            tile[r][tx] = v;
            if (PROLOGUE) bsum[j] += v;
        }
        __syncthreads();
        const int p = p0 + px;
        if (p < HW) {
            uint32_t hw[4], lw[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                split_pack2(tile[cg * 8 + 2 * e][px], tile[cg * 8 + 2 * e + 1][px], hw[e], lw[e]);
            }
            __nv_bfloat16 *o = dst + ((size_t)n * HW + p) * Cpad + c0 + cg * 8;
            *reinterpret_cast<uint4 *>(o) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
            *reinterpret_cast<uint4 *>(o + plane) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
        }
        __syncthreads();
    }
    if (PROLOGUE && db) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            float sum = bsum[j];
            for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
            const int c = c0 + ty + 8 * j;
            if (tx == 0 && c < C) atomicAdd(db + c, sum);
        }
    }
}

static inline int split_tiles_per_block(int HW, int cblocks, int B)
{
    const int tiles = (HW + 31) / 32;
    int t = 1;                                                     // grow while at least ~4 blocks per SM remain
    while (t < 16 && (int64_t)((tiles + 2 * t - 1) / (2 * t)) * cblocks * B >= 4 * dev_info().sm_count) t *= 2;
    return t;
}

static int split_from_nchw_pad(const float *src, int B, int C, int Cpad, int HW, __nv_bfloat16 *dst, cudaStream_t st)
{
    ESR_REQUIRE(Cpad % 64 == 0 && Cpad >= C, "split_from_nchw_pad: Cpad=%d", Cpad);
    const int tpb = split_tiles_per_block(HW, Cpad / 64, B), tiles = (HW + 31) / 32;
    k_to_split<false><<<dim3((tiles + tpb - 1) / tpb, Cpad / 64, B), 256, 0, st>>>(src, nullptr, ACT_NONE, C, Cpad, HW, tpb, dst,
                                                                                   (size_t)B * HW * Cpad, nullptr, nullptr);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}

// ------------------------------------------------------------------------------------------------------------------
// CUDA-core convolution, fp32 NCHW.  Block = 16 x 16 output pixels x 8 output channels; input channels in chunks of 8.
// ------------------------------------------------------------------------------------------------------------------
constexpr int G_T = 16, G_C = 8;

template <int KS>
__global__ void __launch_bounds__(256) k_conv_fwd_g(const float *__restrict__ x, const float *__restrict__ w,
                                                    const float *__restrict__ bias, float *__restrict__ y, int Cin, int H, int W,
                                                    int Cout, int Ho, int Wo, int stride, int act)
{
    extern __shared__ float sm[];
    const int PD = (G_T - 1) * stride + KS;                        // patch edge
    float *patch = sm;                                             // [G_C][PD][PD]
    float *wsm = sm + G_C * PD * PD;                               // [G_C co][G_C ci][KS*KS]
    constexpr int KK = KS * KS, pad = KS / 2;
    const int tiles_x = (Wo + G_T - 1) / G_T;
    const int ty0 = (blockIdx.x / tiles_x) * G_T, tx0 = (blockIdx.x % tiles_x) * G_T;
    const int co0 = blockIdx.y * G_C, n = blockIdx.z;
    const int tid = threadIdx.y * G_T + threadIdx.x;
    const int oy = ty0 + threadIdx.y, ox = tx0 + threadIdx.x;
    float acc[G_C];
#pragma unroll
    for (int c = 0; c < G_C; ++c) acc[c] = (co0 + c < Cout) ? bias[co0 + c] : 0.0f;
    for (int ci0 = 0; ci0 < Cin; ci0 += G_C) {
        for (int i = tid; i < G_C * PD * PD; i += 256) {
            const int ci = i / (PD * PD), r = i - ci * PD * PD;
            const int iy = ty0 * stride - pad + r / PD, ix = tx0 * stride - pad + r % PD;
            float v = 0.0f;
            if (ci0 + ci < Cin && iy >= 0 && iy < H && ix >= 0 && ix < W) v = x[(((size_t)n * Cin + ci0 + ci) * H + iy) * W + ix];
            patch[i] = v;
        }
        for (int i = tid; i < G_C * G_C * KK; i += 256) {
            const int t = i % KK, ci = (i / KK) % G_C, co = i / (KK * G_C);
            wsm[i] = (co0 + co < Cout && ci0 + ci < Cin) ? w[((size_t)(co0 + co) * Cin + ci0 + ci) * KK + t] : 0.0f;
        }
        __syncthreads();
#pragma unroll 2
        for (int ci = 0; ci < G_C; ++ci) {
#pragma unroll
            for (int t = 0; t < KK; ++t) {
                const float v = patch[(ci * PD + threadIdx.y * stride + t / KS) * PD + threadIdx.x * stride + t % KS];
#pragma unroll
                for (int c = 0; c < G_C; ++c) acc[c] = fmaf(v, wsm[(c * G_C + ci) * KK + t], acc[c]);
            }
        }
        __syncthreads();
    }
    if (oy < Ho && ox < Wo) {
#pragma unroll
        for (int c = 0; c < G_C; ++c)
            if (co0 + c < Cout) y[(((size_t)n * Cout + co0 + c) * Ho + oy) * Wo + ox] = act_fwd(acc[c], act);
    }
}

// Register-tiled variant for stride 1, 3x3: block = 64 x 16 output pixels, thread = 4 pixels along x  x  8 output channels.
// Per input channel a thread reads its 3 x 6 patch values with 16-/8-byte loads and the 9 x 8 weights as broadcast
// float4 pairs: 24 shared-memory instructions per 288 FMAs (the simple kernel above: 9 per 8).
constexpr int R_TW = 64, R_TH = 16, R_PW = 72, R_PH = 18;          // patch: image columns tx0-4 .. tx0+67, pitch 72 floats

__global__ void __launch_bounds__(256) k_conv_fwd_r(const float *__restrict__ x, const float *__restrict__ w,
                                                    const float *__restrict__ bias, float *__restrict__ y, int Cin, int H, int W,
                                                    int Cout, int act)
{
    extern __shared__ float sm[];
    float *patch = sm;                                             // [G_C ci][R_PH][R_PW], col j <-> image x0 - 1 + j ... shifted by 3
    float *wsm = sm + G_C * R_PH * R_PW;                           // [G_C ci][9][G_C co]
    const int tiles_x = (W + R_TW - 1) / R_TW;
    const int ty0 = (blockIdx.x / tiles_x) * R_TH, tx0 = (blockIdx.x % tiles_x) * R_TW;
    const int co0 = blockIdx.y * G_C, n = blockIdx.z;
    const int tid = threadIdx.x, lx = tid & 15, ly = tid >> 4;
    float acc[4][G_C];
#pragma unroll
    for (int c = 0; c < G_C; ++c) {
        const float b = (bias && co0 + c < Cout) ? bias[co0 + c] : 0.0f;
#pragma unroll
        for (int p = 0; p < 4; ++p) acc[p][c] = b;
    }
    // patch column jc holds image column tx0 - 4 + jc (so that a thread's first needed column 4*lx + 3 ... is 16-byte
    // aligned at 4*lx + 0 after loading [4*lx, 4*lx+8)): columns needed by thread lx: tx0 + 4*lx - 1 .. + 4 = jc 4*lx+3 .. 4*lx+8
    for (int ci0 = 0; ci0 < Cin; ci0 += G_C) {
        for (int i = tid; i < G_C * R_PH * R_PW; i += 256) {
            const int ci = i / (R_PH * R_PW), r = i - ci * R_PH * R_PW;
            const int iy = ty0 - 1 + r / R_PW, ix = tx0 - 4 + r % R_PW;
            float v = 0.0f;
            if (ci0 + ci < Cin && iy >= 0 && iy < H && ix >= 0 && ix < W) v = x[(((size_t)n * Cin + ci0 + ci) * H + iy) * W + ix];
            patch[i] = v;
        }
        for (int i = tid; i < G_C * 9 * G_C; i += 256) {
            const int co = i % G_C, t = (i / G_C) % 9, ci = i / (G_C * 9);
            wsm[i] = (co0 + co < Cout && ci0 + ci < Cin) ? w[((size_t)(co0 + co) * Cin + ci0 + ci) * 9 + t] : 0.0f;
        }
        __syncthreads();
#pragma unroll 1
        for (int ci = 0; ci < G_C; ++ci) {
            float v[3][6];
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                const float *row = patch + (ci * R_PH + ly + r) * R_PW + 4 * lx;
                const float4 a = *reinterpret_cast<const float4 *>(row), b = *reinterpret_cast<const float4 *>(row + 4);
                const float2 c = *reinterpret_cast<const float2 *>(row + 8);
                // needed: columns 3..8 of this 10-wide window
                v[r][0] = a.w; v[r][1] = b.x; v[r][2] = b.y; v[r][3] = b.z; v[r][4] = b.w; v[r][5] = c.x;
            }
#pragma unroll
            for (int t = 0; t < 9; ++t) {
                const float4 w0 = *reinterpret_cast<const float4 *>(wsm + (ci * 9 + t) * G_C);
                const float4 w1 = *reinterpret_cast<const float4 *>(wsm + (ci * 9 + t) * G_C + 4);
                const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
                for (int p = 0; p < 4; ++p) {
                    const float xv = v[t / 3][p + t % 3];
#pragma unroll
                    for (int c = 0; c < G_C; ++c) acc[p][c] = fmaf(xv, wv[c], acc[p][c]);
                }
            }
        }
        __syncthreads();
    }
    const int oy = ty0 + ly;
    if (oy < H) {
#pragma unroll
        for (int c = 0; c < G_C; ++c) {
            if (co0 + c >= Cout) continue;
            float *dst = y + (((size_t)n * Cout + co0 + c) * H + oy) * W + tx0 + 4 * lx;
#pragma unroll
            for (int p = 0; p < 4; ++p)
                if (tx0 + 4 * lx + p < W) dst[p] = act_fwd(acc[p][c], act);
        }
    }
}

// dx of a stride-2 3x3 pad-1 convolution by output parity: the four pixels of a 2x2 quad (y = 2m + a, x = 2n + b) receive
//   (0,0): g[m][n] w11        (0,1): g[m][n+1] w10 + g[m][n] w12        (1,0): g[m+1][n] w01 + g[m][n] w21
//   (1,1): g[m+1][n+1] w00 + g[m+1][n] w02 + g[m][n+1] w20 + g[m][n] w22
// i.e. exactly 9 useful FMAs per (co, ci) and quad -- no divisibility tests, no wasted taps.  Block = 16 x 16 quads
// (32 x 32 dx pixels) x 8 input channels; g patch 17 x 17 per output channel chunk of 8.
__global__ void __launch_bounds__(256) k_conv_dgrad_s2(const float *__restrict__ g, const float *__restrict__ w, float *__restrict__ dx,
                                                       int Cin, int H, int W, int Cout, int Ho, int Wo)
{
    __shared__ float patch[G_C][17][18];                           // [co][m][n]
    __shared__ __align__(16) float wsm[G_C][9][G_C];               // [co][tap][ci]
    const int tiles_x = (W + 31) / 32;
    const int m0 = (blockIdx.x / tiles_x) * 16, n0 = (blockIdx.x % tiles_x) * 16;     // quad coordinates of the tile
    const int ci0 = blockIdx.y * G_C, n = blockIdx.z;
    const int tid = threadIdx.x, qx = tid & 15, qy = tid >> 4;
    float acc[4][G_C];
#pragma unroll
    for (int p = 0; p < 4; ++p)
#pragma unroll
        for (int c = 0; c < G_C; ++c) acc[p][c] = 0.0f;
    for (int co0 = 0; co0 < Cout; co0 += G_C) {
        for (int i = tid; i < G_C * 17 * 17; i += 256) {
            const int co = i / 289, r = i % 289;
            const int gy = m0 + r / 17, gx = n0 + r % 17;
            float v = 0.0f;
            if (co0 + co < Cout && gy < Ho && gx < Wo) v = g[(((size_t)n * Cout + co0 + co) * Ho + gy) * Wo + gx];
            patch[co][r / 17][r % 17] = v;
        }
        for (int i = tid; i < G_C * 9 * G_C; i += 256) {
            const int ci = i % G_C, t = (i / G_C) % 9, co = i / (G_C * 9);
            wsm[co][t][ci] = (co0 + co < Cout && ci0 + ci < Cin) ? w[((size_t)(co0 + co) * Cin + ci0 + ci) * 9 + t] : 0.0f;
        }
        __syncthreads();
#pragma unroll 2
        for (int co = 0; co < G_C; ++co) {
            const float g00 = patch[co][qy][qx], g01 = patch[co][qy][qx + 1], g10 = patch[co][qy + 1][qx], g11 = patch[co][qy + 1][qx + 1];
            float wv[9][G_C];
#pragma unroll
            for (int t = 0; t < 9; ++t) {
                const float4 a = *reinterpret_cast<const float4 *>(&wsm[co][t][0]), b = *reinterpret_cast<const float4 *>(&wsm[co][t][4]);
                wv[t][0] = a.x; wv[t][1] = a.y; wv[t][2] = a.z; wv[t][3] = a.w; wv[t][4] = b.x; wv[t][5] = b.y; wv[t][6] = b.z; wv[t][7] = b.w;
            }
#pragma unroll
            for (int c = 0; c < G_C; ++c) {
                acc[0][c] = fmaf(g00, wv[4][c], acc[0][c]);
                acc[1][c] = fmaf(g01, wv[3][c], fmaf(g00, wv[5][c], acc[1][c]));
                acc[2][c] = fmaf(g10, wv[1][c], fmaf(g00, wv[7][c], acc[2][c]));
                acc[3][c] = fmaf(g11, wv[0][c], fmaf(g10, wv[2][c], fmaf(g01, wv[6][c], fmaf(g00, wv[8][c], acc[3][c]))));
            }
        }
        __syncthreads();
    }
#pragma unroll
    for (int p = 0; p < 4; ++p) {
        const int y = 2 * (m0 + qy) + (p >> 1), x = 2 * (n0 + qx) + (p & 1);
        if (y >= H || x >= W) continue;
#pragma unroll
        for (int c = 0; c < G_C; ++c)
            if (ci0 + c < Cin) dx[(((size_t)n * Cin + ci0 + c) * H + y) * W + x] = acc[p][c];
    }
}

// dw for 3x3: thread = (input channel, kernel row) x 3 kernel columns x 8 output channels (24 accumulators), pixels of the
// 16x16 tile split over 10 thread groups; 5 shared-memory instructions per 24 FMAs.
// DET: the partial of pixel group `split` in block (pair, y) goes to slot y * WR_NSPLIT + split of dw = [slots][Cout*Cin*9].
constexpr int WR_NSPLIT = 10;
template <bool DET>
__device__ __forceinline__ void wgrad_r_body(const float *__restrict__ x, const float *__restrict__ g, float *__restrict__ dw,
                                             int B, int Cin, int H, int W, int Cout, int Ho, int Wo, int stride)
{
    extern __shared__ float sm[];
    constexpr int NR = G_C * 3, NSPLIT = WR_NSPLIT;                // 24 roles x 10 pixel groups = 240 threads
    const int PD = (G_T - 1) * stride + 3;
    float *gs = sm;                                                // [256 px][G_C co]
    float *xs = sm + 256 * G_C;                                    // [G_C ci][PD][PD]
    const int ci_tiles = (Cin + G_C - 1) / G_C;
    const int co0 = (blockIdx.x / ci_tiles) * G_C, ci0 = (blockIdx.x % ci_tiles) * G_C;
    const int tiles_x = (Wo + G_T - 1) / G_T, tiles_y = (Ho + G_T - 1) / G_T;
    const int items = B * tiles_x * tiles_y;
    const int tid = threadIdx.x;
    const int role = tid % NR, split = tid / NR;
    const int pci = role / 3, ky = role % 3;
    const bool active = split < NSPLIT;
    float acc[3][G_C];
#pragma unroll
    for (int k = 0; k < 3; ++k)
#pragma unroll
        for (int c = 0; c < G_C; ++c) acc[k][c] = 0.0f;
    for (int it = blockIdx.y; it < items; it += gridDim.y) {
        const int n = it / (tiles_x * tiles_y), tr = it % (tiles_x * tiles_y);
        const int ty0 = (tr / tiles_x) * G_T, tx0 = (tr % tiles_x) * G_T;
        for (int i = tid; i < 256 * G_C; i += 256) {
            const int co = i / 256, p = i % 256;
            const int oy = ty0 + p / G_T, ox = tx0 + p % G_T;
            float v = 0.0f;
            if (co0 + co < Cout && oy < Ho && ox < Wo) v = g[(((size_t)n * Cout + co0 + co) * Ho + oy) * Wo + ox];
            gs[p * G_C + co] = v;
        }
        for (int i = tid; i < G_C * PD * PD; i += 256) {
            const int ci = i / (PD * PD), r = i - ci * PD * PD;
            const int iy = ty0 * stride - 1 + r / PD, ix = tx0 * stride - 1 + r % PD;
            float v = 0.0f;
            if (ci0 + ci < Cin && iy >= 0 && iy < H && ix >= 0 && ix < W) v = x[(((size_t)n * Cin + ci0 + ci) * H + iy) * W + ix];
            xs[i] = v;
        }
        __syncthreads();
        if (active) {
            for (int p = split; p < 256; p += NSPLIT) {
                const float *xr = xs + (pci * PD + (p / G_T) * stride + ky) * PD + (p % G_T) * stride;
                const float x0 = xr[0], x1 = xr[1], x2 = xr[2];
                const float4 g0 = *reinterpret_cast<const float4 *>(gs + p * G_C), g1 = *reinterpret_cast<const float4 *>(gs + p * G_C + 4);
                const float gv[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
#pragma unroll
                for (int c = 0; c < G_C; ++c) {
                    acc[0][c] = fmaf(x0, gv[c], acc[0][c]);
                    acc[1][c] = fmaf(x1, gv[c], acc[1][c]);
                    acc[2][c] = fmaf(x2, gv[c], acc[2][c]);
                }
            }
        }
        __syncthreads();
    }
    if (active && ci0 + pci < Cin) {
#pragma unroll
        for (int k = 0; k < 3; ++k)
#pragma unroll
            for (int c = 0; c < G_C; ++c)
                if (co0 + c < Cout) {
                    if (DET) dw[((size_t)blockIdx.y * NSPLIT + split) * ((size_t)Cout * Cin * 9) + ((size_t)(co0 + c) * Cin + ci0 + pci) * 9 + ky * 3 + k] = acc[k][c];
                    else atomicAdd(dw + ((size_t)(co0 + c) * Cin + ci0 + pci) * 9 + ky * 3 + k, acc[k][c]);
                }
    }
}
__global__ void __launch_bounds__(256) k_conv_wgrad_r(const float *__restrict__ x, const float *__restrict__ g, float *__restrict__ dw,
                                                      int B, int Cin, int H, int W, int Cout, int Ho, int Wo, int stride)
{
    wgrad_r_body<false>(x, g, dw, B, Cin, H, W, Cout, Ho, Wo, stride);
}
__global__ void __launch_bounds__(256) k_conv_wgrad_r_det(const float *__restrict__ x, const float *__restrict__ g, float *__restrict__ part,
                                                          int B, int Cin, int H, int W, int Cout, int Ho, int Wo, int stride)
{
    wgrad_r_body<true>(x, g, part, B, Cin, H, W, Cout, Ho, Wo, stride);
}

__device__ __forceinline__ int floor_div(int a, int b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }

// dx[n, ci, y, x] = sum over co, taps of g[n, co, (y + pad - ky) / s, (x + pad - kx) / s] * w[co, ci, ky, kx]  (when divisible)
template <int KS>
__global__ void __launch_bounds__(256) k_conv_dgrad_g(const float *__restrict__ g, const float *__restrict__ w, float *__restrict__ dx,
                                                      int Cin, int H, int W, int Cout, int Ho, int Wo, int stride)
{
    extern __shared__ float sm[];
    constexpr int KK = KS * KS, pad = KS / 2;
    const int GP = (G_T - 1 + KS - 1) / stride + 2;                // g patch edge
    float *patch = sm;                                             // [G_C co][GP][GP]
    float *wsm = sm + G_C * GP * GP;                               // [G_C co][G_C ci][KK]
    const int tiles_x = (W + G_T - 1) / G_T;
    const int ty0 = (blockIdx.x / tiles_x) * G_T, tx0 = (blockIdx.x % tiles_x) * G_T;
    const int ci0 = blockIdx.y * G_C, n = blockIdx.z;
    const int tid = threadIdx.y * G_T + threadIdx.x;
    const int yy = ty0 + threadIdx.y, xx = tx0 + threadIdx.x;
    const int gy0 = floor_div(ty0 + pad - (KS - 1), stride), gx0 = floor_div(tx0 + pad - (KS - 1), stride);
    float acc[G_C];
#pragma unroll
    for (int c = 0; c < G_C; ++c) acc[c] = 0.0f;
    for (int co0 = 0; co0 < Cout; co0 += G_C) {
        for (int i = tid; i < G_C * GP * GP; i += 256) {
            const int co = i / (GP * GP), r = i - co * GP * GP;
            const int gy = gy0 + r / GP, gx = gx0 + r % GP;
            float v = 0.0f;
            if (co0 + co < Cout && gy >= 0 && gy < Ho && gx >= 0 && gx < Wo) v = g[(((size_t)n * Cout + co0 + co) * Ho + gy) * Wo + gx];
            patch[i] = v;
        }
        for (int i = tid; i < G_C * G_C * KK; i += 256) {
            const int t = i % KK, ci = (i / KK) % G_C, co = i / (KK * G_C);
            wsm[i] = (co0 + co < Cout && ci0 + ci < Cin) ? w[((size_t)(co0 + co) * Cin + ci0 + ci) * KK + t] : 0.0f;
        }
        __syncthreads();
#pragma unroll
        for (int t = 0; t < KK; ++t) {
            const int ty = yy + pad - t / KS, tx = xx + pad - t % KS;
            if (ty < 0 || tx < 0 || ty % stride != 0 || tx % stride != 0) continue;
            const int py = ty / stride - gy0, px = tx / stride - gx0;
            if (py >= GP || px >= GP) continue;
            for (int co = 0; co < G_C; ++co) {
                const float v = patch[(co * GP + py) * GP + px];
#pragma unroll
                for (int c = 0; c < G_C; ++c) acc[c] = fmaf(v, wsm[(co * G_C + c) * KK + t], acc[c]);
            }
        }
        __syncthreads();
    }
    if (yy < H && xx < W) {
#pragma unroll
        for (int c = 0; c < G_C; ++c)
            if (ci0 + c < Cin) dx[(((size_t)n * Cin + ci0 + c) * H + yy) * W + xx] = acc[c];
    }
}

// dw[co, ci, ky, kx] += sum over (n, oy, ox) of g[n, co, oy, ox] * x[n, ci, oy*s + ky - pad, ox*s + kx - pad]
// grid (co-tiles * ci-tiles, work slices); each block walks (image, 16x16 output tile) items with stride gridDim.y
// DET: the partial of pixel split `split` in block (pair, y) goes to slot y * (256 / (8 KS^2)) + split of dw = [slots][Cout*Cin*KK]
template <int KS, bool DET>
__device__ __forceinline__ void wgrad_g_body(const float *__restrict__ x, const float *__restrict__ g, float *__restrict__ dw,
                                             int B, int Cin, int H, int W, int Cout, int Ho, int Wo, int stride)
{
    extern __shared__ float sm[];
    constexpr int KK = KS * KS, pad = KS / 2, NP = G_C * KK;       // (ci, tap) pairs per block
    constexpr int NSPLIT = 256 / NP;                               // pixel splits
    const int PD = (G_T - 1) * stride + KS;
    float *gs = sm;                                                // [256 px][G_C co]
    float *xs = sm + 256 * G_C;                                    // [G_C ci][PD][PD]
    const int ci_tiles = (Cin + G_C - 1) / G_C;
    const int co0 = (blockIdx.x / ci_tiles) * G_C, ci0 = (blockIdx.x % ci_tiles) * G_C;
    const int tiles_x = (Wo + G_T - 1) / G_T, tiles_y = (Ho + G_T - 1) / G_T;
    const int items = B * tiles_x * tiles_y;
    const int tid = threadIdx.x;
    const int pair = tid % NP, split = tid / NP;
    const int pci = pair / KK, pt = pair % KK;
    const bool active = split < NSPLIT;
    float acc[G_C];
#pragma unroll
    for (int c = 0; c < G_C; ++c) acc[c] = 0.0f;
    for (int it = blockIdx.y; it < items; it += gridDim.y) {
        const int n = it / (tiles_x * tiles_y), tr = it % (tiles_x * tiles_y);
        const int ty0 = (tr / tiles_x) * G_T, tx0 = (tr % tiles_x) * G_T;
        for (int i = tid; i < 256 * G_C; i += 256) {
            const int co = i / 256, p = i % 256;                   // coalesced along pixels
            const int oy = ty0 + p / G_T, ox = tx0 + p % G_T;
            float v = 0.0f;
            if (co0 + co < Cout && oy < Ho && ox < Wo) v = g[(((size_t)n * Cout + co0 + co) * Ho + oy) * Wo + ox];
            gs[p * G_C + co] = v;
        }
        for (int i = tid; i < G_C * PD * PD; i += 256) {
            const int ci = i / (PD * PD), r = i - ci * PD * PD;
            const int iy = ty0 * stride - pad + r / PD, ix = tx0 * stride - pad + r % PD;
            float v = 0.0f;
            if (ci0 + ci < Cin && iy >= 0 && iy < H && ix >= 0 && ix < W) v = x[(((size_t)n * Cin + ci0 + ci) * H + iy) * W + ix];
            xs[i] = v;
        }
        __syncthreads();
        if (active) {
            for (int p = split; p < 256; p += NSPLIT) {
                const float xv = xs[(pci * PD + (p / G_T) * stride + pt / KS) * PD + (p % G_T) * stride + pt % KS];
                const float4 g0 = *reinterpret_cast<const float4 *>(gs + p * G_C), g1 = *reinterpret_cast<const float4 *>(gs + p * G_C + 4);
                acc[0] = fmaf(xv, g0.x, acc[0]); acc[1] = fmaf(xv, g0.y, acc[1]); acc[2] = fmaf(xv, g0.z, acc[2]); acc[3] = fmaf(xv, g0.w, acc[3]);
                acc[4] = fmaf(xv, g1.x, acc[4]); acc[5] = fmaf(xv, g1.y, acc[5]); acc[6] = fmaf(xv, g1.z, acc[6]); acc[7] = fmaf(xv, g1.w, acc[7]);
            }
        }
        __syncthreads();
    }
    if (active && ci0 + pci < Cin) {
#pragma unroll
        for (int c = 0; c < G_C; ++c)
            if (co0 + c < Cout) {
                if (DET) dw[((size_t)blockIdx.y * NSPLIT + split) * ((size_t)Cout * Cin * KK) + ((size_t)(co0 + c) * Cin + ci0 + pci) * KK + pt] = acc[c];
                else atomicAdd(dw + ((size_t)(co0 + c) * Cin + ci0 + pci) * KK + pt, acc[c]);
            }
    }
}
template <int KS>
__global__ void __launch_bounds__(256) k_conv_wgrad_g(const float *__restrict__ x, const float *__restrict__ g, float *__restrict__ dw,
                                                      int B, int Cin, int H, int W, int Cout, int Ho, int Wo, int stride)
{
    wgrad_g_body<KS, false>(x, g, dw, B, Cin, H, W, Cout, Ho, Wo, stride);
}
template <int KS>
__global__ void __launch_bounds__(256) k_conv_wgrad_g_det(const float *__restrict__ x, const float *__restrict__ g, float *__restrict__ part,
                                                          int B, int Cin, int H, int W, int Cout, int Ho, int Wo, int stride)
{
    wgrad_g_body<KS, true>(x, g, part, B, Cin, H, W, Cout, Ho, Wo, stride);
}

// ------------------------------------------------------------------------------------------------------------------
// dw of the narrow 3x3 layers on the warp-level tensor cores.  Per tap the weight gradient is a GEMM over pixels:
//   D[co][n] += sum_px g[co][px] * x[ci(n)][py(px) * s + ky(n)][px(px) * s + kx(n)],   n = ci * 9 + tap  (= the dw memory order)
// mma.sync m16n8k16 with A = g (row-major, K = 16 consecutive output pixels of a tile row) and B = shifted x (col-major: two
// consecutive pixels per register).  fp32 inputs are split to bf16 (hi, lo) while staging a 16x16 output tile in shared
// memory -- g as [co][pixel], x as three column-shifted copies (one per kx) of PACKED pixel pairs so that every B fragment is
// one aligned 32-bit load for both strides -- and the usual three products (lo*hi + hi*lo + hi*hi) accumulate in fp32.
// Block = (16 output channels, 8 input channels) x a slice of the (image, tile) items; warp w owns tile rows w and w + 8;
// partial sums are combined through shared-memory atomics and added to dw once per block.
// ------------------------------------------------------------------------------------------------------------------
constexpr int WM_GP = 264;                                         // g row pitch (bf16 elements): conflict-free A fragment loads

__device__ __forceinline__ uint32_t pack_bf16x2(__nv_bfloat16 a, __nv_bfloat16 b)
{
    return (uint32_t)__bfloat16_as_ushort(a) | ((uint32_t)__bfloat16_as_ushort(b) << 16);
}
__device__ __forceinline__ void mma_bf16_k16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1)
{
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

template <int STRIDE>
__global__ void __launch_bounds__(256) k_conv_wgrad_mma(const float *__restrict__ x, const float *__restrict__ g, float *__restrict__ dw,
                                                        int B, int Cin, int H, int W, int Cout, int Ho, int Wo)
{
    constexpr int PD = 15 * STRIDE + 3;                            // input rows needed by a 16-row output tile
    constexpr int XW = 8 * PD * 8;                                 // words per (copy, plane): [ci 8][row PD][pair 8]
    extern __shared__ __align__(16) uint8_t wsm_raw[];
    __nv_bfloat16 *g_hi = reinterpret_cast<__nv_bfloat16 *>(wsm_raw), *g_lo = g_hi + 16 * WM_GP;
    uint32_t *x_hi = reinterpret_cast<uint32_t *>(g_lo + 16 * WM_GP), *x_lo = x_hi + 3 * XW;
    float *red = reinterpret_cast<float *>(x_lo + 3 * XW);          // [16][72] block-level partial sums

    const int ci_tiles = (Cin + 7) / 8;
    const int co0 = (blockIdx.x / ci_tiles) * 16, ci0 = (blockIdx.x % ci_tiles) * 8;
    const int tiles_x = (Wo + 15) / 16, tiles_y = (Ho + 15) / 16;
    const int items = B * tiles_x * tiles_y;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, gq = lane >> 2, t4 = lane & 3;
    float acc[9][4];
#pragma unroll
    for (int n = 0; n < 9; ++n) acc[n][0] = acc[n][1] = acc[n][2] = acc[n][3] = 0.0f;
    for (int i = tid; i < 16 * 72; i += 256) red[i] = 0.0f;

    for (int it = blockIdx.y; it < items; it += gridDim.y) {
        const int n_img = it / (tiles_x * tiles_y), tr = it % (tiles_x * tiles_y);
        const int ty0 = (tr / tiles_x) * 16, tx0 = (tr % tiles_x) * 16;
        __syncthreads();                                            // previous item's fragments are consumed
        // ---- stage g: 16 channels x 256 pixels, split
        for (int i = tid; i < 16 * 256; i += 256) {
            const int co = i >> 8, p = i & 255;
            const int oy = ty0 + (p >> 4), ox = tx0 + (p & 15);
            float v = 0.0f;
            if (co0 + co < Cout && oy < Ho && ox < Wo) v = g[(((size_t)n_img * Cout + co0 + co) * Ho + oy) * Wo + ox];
            __nv_bfloat16 h, l;
            split_bf16(v, h, l);
            g_hi[co * WM_GP + p] = h;
            g_lo[co * WM_GP + p] = l;
        }
        // ---- stage x: for each kx the pixel pairs (ox = 2j, 2j + 1) -> input columns (2j * s + kx, (2j + 1) * s + kx), packed
        for (int i = tid; i < 3 * XW; i += 256) {
            const int j = i & 7, row = (i >> 3) % PD, ci = (i / (8 * PD)) & 7, kx = i / XW;
            const int iy = ty0 * STRIDE - 1 + row;
            const int ix0 = (tx0 + 2 * j) * STRIDE - 1 + kx, ix1 = ix0 + STRIDE;
            float v0 = 0.0f, v1 = 0.0f;
            if (ci0 + ci < Cin && iy >= 0 && iy < H) {
                const float *xr = x + (((size_t)n_img * Cin + ci0 + ci) * H + iy) * W;
                if (ix0 >= 0 && ix0 < W) v0 = __ldg(xr + ix0);
                if (ix1 >= 0 && ix1 < W) v1 = __ldg(xr + ix1);
            }
            __nv_bfloat16 h0, l0, h1, l1;
            split_bf16(v0, h0, l0);
            split_bf16(v1, h1, l1);
            x_hi[i] = pack_bf16x2(h0, h1);
            x_lo[i] = pack_bf16x2(l0, l1);
        }
        __syncthreads();
        // ---- two K steps per warp: tile rows warp and warp + 8
#pragma unroll
        for (int kk = 0; kk < 2; ++kk) {
            const int oyl = warp + 8 * kk;                          // tile row = K step
            uint32_t ah[4], al[4];
            {
                const int o0 = gq * WM_GP + oyl * 16 + 2 * t4, o1 = (gq + 8) * WM_GP + oyl * 16 + 2 * t4;
                ah[0] = *reinterpret_cast<const uint32_t *>(g_hi + o0); ah[1] = *reinterpret_cast<const uint32_t *>(g_hi + o1);
                ah[2] = *reinterpret_cast<const uint32_t *>(g_hi + o0 + 8); ah[3] = *reinterpret_cast<const uint32_t *>(g_hi + o1 + 8);
                al[0] = *reinterpret_cast<const uint32_t *>(g_lo + o0); al[1] = *reinterpret_cast<const uint32_t *>(g_lo + o1);
                al[2] = *reinterpret_cast<const uint32_t *>(g_lo + o0 + 8); al[3] = *reinterpret_cast<const uint32_t *>(g_lo + o1 + 8);
            }
#pragma unroll
            for (int nt = 0; nt < 9; ++nt) {
                const int n = nt * 8 + gq;                          // this lane's B column: (ci, tap)
                const int ci = n / 9, tap = n - ci * 9, ky = tap / 3, kx = tap - ky * 3;
                const int wofs = kx * XW + (ci * PD + oyl * STRIDE + ky) * 8 + t4;
                const uint32_t bh0 = x_hi[wofs], bh1 = x_hi[wofs + 4], bl0 = x_lo[wofs], bl1 = x_lo[wofs + 4];
                mma_bf16_k16(acc[nt], al, bh0, bh1);
                mma_bf16_k16(acc[nt], ah, bl0, bl1);
                mma_bf16_k16(acc[nt], ah, bh0, bh1);
            }
        }
    }
    // ---- combine the 8 warps, then one global atomic per (co, n)
    __syncthreads();
#pragma unroll
    for (int nt = 0; nt < 9; ++nt) {
        atomicAdd(&red[gq * 72 + nt * 8 + 2 * t4], acc[nt][0]);
        atomicAdd(&red[gq * 72 + nt * 8 + 2 * t4 + 1], acc[nt][1]);
        atomicAdd(&red[(gq + 8) * 72 + nt * 8 + 2 * t4], acc[nt][2]);
        atomicAdd(&red[(gq + 8) * 72 + nt * 8 + 2 * t4 + 1], acc[nt][3]);
    }
    __syncthreads();
    for (int i = tid; i < 16 * 72; i += 256) {
        const int co = i / 72, n = i % 72, ci = n / 9, tap = n % 9;
        if (co0 + co < Cout && ci0 + ci < Cin) atomicAdd(dw + ((size_t)(co0 + co) * Cin + ci0 + ci) * 9 + tap, red[i]);
    }
}

// ------------------------------------------------------------------------------------------------------------------
// bilinear x2 (F.interpolate(scale_factor=2, mode='bilinear', align_corners=False), models/submodules.py:290) on fp32 NCHW
// planes, forward and backward.  For scale 2 the source coordinate is oy/2 - 0.25, so output row 2k reads rows (k-1, k)
// with weights (0.25, 0.75) and row 2k+1 reads (k, k+1) with (0.75, 0.25), clamped at the borders; the backward is the
// transposed 4-tap gather per input pixel (no atomics, deterministic).
// ------------------------------------------------------------------------------------------------------------------
// grid (ceil(2W / 256), 2H, planes): no integer divisions in the index math
__global__ void __launch_bounds__(256) k_upsample2x_fwd(const float *__restrict__ x, int H, int W, float *__restrict__ y)
{
    const int Wo = 2 * W, ox = blockIdx.x * 256 + threadIdx.x, oy = blockIdx.y;
    if (ox >= Wo) return;
    const size_t pl = blockIdx.z;
    const float fy = fmaxf(0.0f, ((float)oy + 0.5f) * 0.5f - 0.5f), fx = fmaxf(0.0f, ((float)ox + 0.5f) * 0.5f - 0.5f);
    const int y0 = (int)fy, x0 = (int)fx;
    const int y1 = min(y0 + 1, H - 1), x1 = min(x0 + 1, W - 1);
    const float ly = fy - (float)y0, lx = fx - (float)x0;
    const float *p = x + pl * H * W;
    const float v00 = p[(size_t)y0 * W + x0], v01 = p[(size_t)y0 * W + x1], v10 = p[(size_t)y1 * W + x0], v11 = p[(size_t)y1 * W + x1];
    y[(pl * 2 * H + oy) * Wo + ox] = (1.0f - ly) * ((1.0f - lx) * v00 + lx * v01) + ly * ((1.0f - lx) * v10 + lx * v11);
}

// weight of output index o (row or column) on input index k, per dimension: (o, weight) pairs, at most 4
__device__ __forceinline__ int up2_taps(int k, int n_in, int (&o)[4], float (&wt)[4])
{
    int c = 0;
    if (k >= 1) { o[c] = 2 * k - 1; wt[c++] = 0.25f; }
    o[c] = 2 * k; wt[c++] = k >= 1 ? 0.75f : 1.0f;
    o[c] = 2 * k + 1; wt[c++] = k < n_in - 1 ? 0.75f : 1.0f;
    if (k < n_in - 1) { o[c] = 2 * k + 2; wt[c++] = 0.25f; }
    return c;
}

__global__ void __launch_bounds__(256) k_upsample2x_bwd(const float *__restrict__ dy, int H, int W, float *__restrict__ dx)
{
    const int Wo = 2 * W, ix = blockIdx.x * 256 + threadIdx.x, iy = blockIdx.y;
    if (ix >= W) return;
    const size_t pl = blockIdx.z;
    int oy[4], ox[4];
    float wy[4], wx[4];
    const int ny = up2_taps(iy, H, oy, wy), nx = up2_taps(ix, W, ox, wx);
    const float *p = dy + pl * (size_t)(2 * H) * Wo;
    float s = 0.0f;
    for (int a = 0; a < ny; ++a) {
        float r = 0.0f;
        for (int b = 0; b < nx; ++b) r = fmaf(wx[b], p[(size_t)oy[a] * Wo + ox[b]], r);
        s = fmaf(wy[a], r, s);
    }
    dx[(pl * H + iy) * W + ix] = s;
}

// ------------------------------------------------------------------------------------------------------------------
// ConvGRU gate arithmetic (models/submodules.py:507-512) as two fused element-wise operators, forward and backward.
// zr = sigmoid(conv(cat(x, h))) holds the update gate z in channels [0, C) and the reset gate r in [C, 2C) of each image.
//   hr    = h * r                                   (input of the candidate convolution)
//   h_new = h * (1 - z) + o * z
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_gru_hr(const float *__restrict__ h, const float *__restrict__ zr, size_t n, int chw, float *__restrict__ out)
{
    const size_t b = blockIdx.y;                                   // grid (chunks, images): no 64-bit divisions
    for (int r = blockIdx.x * 256 + threadIdx.x; r < chw; r += gridDim.x * 256) {
        const size_t i = b * chw + r;
        out[i] = h[i] * zr[b * 2 * chw + chw + r];
    }
}
__global__ void __launch_bounds__(256) k_gru_hr_bwd(const float *__restrict__ h, const float *__restrict__ zr, const float *__restrict__ g, size_t n,
                                                    int chw, float *__restrict__ dh, float *__restrict__ dzr)
{
    const size_t b = blockIdx.y;
    for (int r = blockIdx.x * 256 + threadIdx.x; r < chw; r += gridDim.x * 256) {
        const size_t i = b * chw + r;
        const float gi = g[i];
        dh[i] = gi * zr[b * 2 * chw + chw + r];
        dzr[b * 2 * chw + r] = 0.0f;
        dzr[b * 2 * chw + chw + r] = gi * h[i];
    }
}
__global__ void __launch_bounds__(256) k_gru_blend(const float *__restrict__ h, const float *__restrict__ zr, const float *__restrict__ o, size_t n,
                                                   int chw, float *__restrict__ out)
{
    const size_t b = blockIdx.y;
    for (int r = blockIdx.x * 256 + threadIdx.x; r < chw; r += gridDim.x * 256) {
        const size_t i = b * chw + r;
        const float z = zr[b * 2 * chw + r];
        out[i] = h[i] * (1.0f - z) + o[i] * z;
    }
}
__global__ void __launch_bounds__(256) k_gru_blend_bwd(const float *__restrict__ h, const float *__restrict__ zr, const float *__restrict__ o,
                                                       const float *__restrict__ g, size_t n, int chw, float *__restrict__ dh,
                                                       float *__restrict__ dzr, float *__restrict__ d_o)
{
    const size_t b = blockIdx.y;
    for (int r = blockIdx.x * 256 + threadIdx.x; r < chw; r += gridDim.x * 256) {
        const size_t i = b * chw + r;
        const float z = zr[b * 2 * chw + r], gi = g[i];
        dh[i] = gi * (1.0f - z);
        d_o[i] = gi * z;
        dzr[b * 2 * chw + r] = gi * (o[i] - h[i]);
        dzr[b * 2 * chw + chw + r] = 0.0f;
    }
}

// ------------------------------------------------------------------------------------------------------------------
// loss and optimizer
// ------------------------------------------------------------------------------------------------------------------
// DET: block b writes its sum of squares to loss[b] (a workspace of gridDim.x floats); k_mse_finish adds them in block order
template <bool DET>
__device__ __forceinline__ void mse_body(const float *__restrict__ p, const float *__restrict__ t, size_t n, float inv_n,
                                         float *__restrict__ loss, float *__restrict__ grad, float grad_scale)
{
    float s = 0.0f;
    for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (size_t)gridDim.x * 256) {
        const float d = p[i] - t[i];
        s = fmaf(d, d, s);
        if (grad) grad[i] = 2.0f * d * inv_n * grad_scale;
    }
    __shared__ float red[8];
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x < 8) {
        s = red[threadIdx.x];
        for (int o = 4; o > 0; o >>= 1) s += __shfl_xor_sync(0xffu, s, o);
        if (threadIdx.x == 0) {
            if (DET) loss[blockIdx.x] = s;
            else atomicAdd(loss, s * inv_n);
        }
    }
}
__global__ void __launch_bounds__(256) k_mse(const float *__restrict__ p, const float *__restrict__ t, size_t n, float inv_n,
                                             float *__restrict__ loss, float *__restrict__ grad, float grad_scale)
{
    mse_body<false>(p, t, n, inv_n, loss, grad, grad_scale);
}
__global__ void __launch_bounds__(256) k_mse_det(const float *__restrict__ p, const float *__restrict__ t, size_t n, float inv_n,
                                                 float *__restrict__ part, float *__restrict__ grad, float grad_scale)
{
    mse_body<true>(p, t, n, inv_n, part, grad, grad_scale);
}
// one warp: lane l adds partials l, l + 32, ... in order, then a fixed butterfly
__global__ void k_mse_finish(const float *__restrict__ part, int blocks, float inv_n, float *__restrict__ loss)
{
    float s = 0.0f;
    for (int i = threadIdx.x; i < blocks; i += 32) s += part[i];
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (threadIdx.x == 0) *loss = s * inv_n;
}

__global__ void k_adam_tick(int *step) { *step += 1; }

__global__ void __launch_bounds__(256) k_adam(float *__restrict__ p, const float *__restrict__ g, float *__restrict__ m,
                                              float *__restrict__ v, float *__restrict__ vmax, size_t n, float lr, float b1, float b2,
                                              float eps, float wd, const int *__restrict__ step, const float *__restrict__ hyper)
{
    // hyper (optional, device): {lr, beta1, beta2, eps, weight_decay} read at run time, so that a replayed CUDA graph follows a
    // learning-rate schedule (train_ours_cnt_seq.py:784 esr_lr_scheduler) instead of freezing the values captured with it
    if (hyper) { lr = hyper[0]; b1 = hyper[1]; b2 = hyper[2]; eps = hyper[3]; wd = hyper[4]; }
    __shared__ float s_bc[2];
    if (threadIdx.x == 0) {                                        // bias corrections from the device-side step counter
        const int t = *step;
        s_bc[0] = (float)(1.0 - pow((double)b1, (double)t));
        s_bc[1] = (float)sqrt(1.0 - pow((double)b2, (double)t));
    }
    __syncthreads();
    const float bc1 = s_bc[0], bc2_sqrt = s_bc[1];
    for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (size_t)gridDim.x * 256) {
        const float pi = p[i];
        const float gi = fmaf(wd, pi, g[i]);                       // torch.optim.Adam: L2 term added to the gradient
        const float mi = b1 * m[i] + (1.0f - b1) * gi;
        const float vi = b2 * v[i] + (1.0f - b2) * gi * gi;
        m[i] = mi; v[i] = vi;
        float vh = vi;
        if (vmax) { vh = fmaxf(vmax[i], vi); vmax[i] = vh; }       // amsgrad
        const float denom = sqrtf(vh) / bc2_sqrt + eps;
        p[i] = pi - (lr / bc1) * (mi / denom);
    }
}

// ------------------------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------------------------
static inline bool tc_fwd_ok(int Cin, int Cout, int ksz, int stride) { return stride == 1 && Cin % 64 == 0 && Cout <= 256 && (ksz == 3 || ksz == 1); }
// dx / dw on the tensor cores: g is padded to a 64-multiple of channels; not worth it for the 1-, 2-, 8- and 16-channel layers
static inline bool tc_dgrad_ok(int Cin, int Cout, int ksz, int stride) { return stride == 1 && Cout >= 32 && Cout <= 256 && Cin <= 256 && (ksz == 3 || ksz == 1); }
static inline int pad64(int c) { return (c + 63) / 64 * 64; }

static size_t conv2d_ws(int B, int Cin, int H, int W, int Cout, int ksz, int stride)
{
    const int Ho = (H + 2 * (ksz / 2) - ksz) / stride + 1, Wo = (W + 2 * (ksz / 2) - ksz) / stride + 1;
    Bump f{nullptr, 0, 0}, b{nullptr, 0, 0};
    if (tc_fwd_ok(Cin, Cout, ksz, stride)) {
        f.take((size_t)B * Cin * H * W * 4); f.take(tc_packed_weight_bytes(Cout, Cin, ksz * ksz)); f.take(256 * 4);
        f.take((size_t)B * tc_npad(Cout) * H * W * 4);
    }
    b.take((size_t)B * Cout * Ho * Wo * 4);
    b.take((size_t)Cout * Cin * ksz * ksz * 4);                          // rotated weights of the CUDA-core dx path
    b.take(mma_weight_bytes(Cin, Cout)); f.take(mma_weight_bytes(Cout, Cin));   // weight images of the mma.sync kernels
    if (tc_dgrad_ok(Cin, Cout, ksz, stride)) {
        b.take((size_t)B * pad64(Cout) * Ho * Wo * 4); b.take((size_t)B * Cin * H * W * 4);      // g split, x split (dw on tensor cores)
        b.take((size_t)pad64(Cout) * Cin * ksz * ksz * 4);
        b.take(tc_packed_weight_bytes(Cin, pad64(Cout), ksz * ksz)); b.take(256 * 4); b.take((size_t)B * tc_npad(Cin) * H * W * 4);
    }
    return (f.off > b.off ? f.off : b.off) + 1024;
}

// y = act(conv(x)) on the tensor cores: fp32 NCHW -> split NHWC -> k_conv_tc -> fp32 NCHW
static int conv_tc_nchw(const float *x, const float *w, const float *bias, int B, int Cin, int H, int W, int Cout, int ksz, int act,
                        float *y, void *x_split_out, Bump &ws, cudaStream_t st)
{
    int rc;
    SplitTensor xs; xs.n_img = B; xs.H = H; xs.W = W; xs.C = Cin;
    xs.base = (__nv_bfloat16 *)(x_split_out ? x_split_out : ws.take((size_t)B * Cin * H * W * 4));   // kept by the caller for dw
    void *wp = ws.take(tc_packed_weight_bytes(Cout, Cin, ksz * ksz));
    float *bp = (float *)ws.take(256 * 4);
    ESR_REQUIRE(ws.off <= ws.cap, "conv2d: workspace too small (%zu > %zu)", ws.off, ws.cap);
    if ((rc = split_from_nchw_pad(x, B, Cin, Cin, H * W, xs.base, st))) return rc;
    if ((rc = pack_conv_weight(w, Cout, Cin, ksz, wp, st))) return rc;
    ESR_CUDA_CHECK(cudaMemsetAsync(bp, 0, 256 * 4, st));
    if (bias) ESR_CUDA_CHECK(cudaMemcpyAsync(bp, bias, (size_t)Cout * 4, cudaMemcpyDeviceToDevice, st));
    ConvTCDesc d;
    d.src[0] = xs; d.n_src = 1; d.ntaps = ksz * ksz; d.cout = Cout; d.wpacked = wp; d.bias = bp; d.n_img = B; d.act = act;
    d.out_f32 = y; d.out_f32_C = Cout; d.out_f32_nchw = 1;              // the epilogue writes fp32 NCHW directly
    ConvTCArgs a;
    if ((rc = conv_tc_prepare(d, &a))) return rc;
    return conv_tc_launch(a, st);
}

// work slices (gridDim.y) of the CUDA-core weight-gradient kernels: about 8 blocks per SM, at most one per (image, tile) item
static int wgrad_slices(int B, int Cin, int Cout, int Ho, int Wo)
{
    const int pairs = ((Cout + G_C - 1) / G_C) * ((Cin + G_C - 1) / G_C);
    const int items = B * ((Wo + G_T - 1) / G_T) * ((Ho + G_T - 1) / G_T);
    int slices = (dev_info().sm_count * 8 + pairs - 1) / pairs;
    if (slices > items) slices = items;
    if (slices < 1) slices = 1;
    return slices;
}
// partial slots of the deterministic variant: per block, one per pixel split of k_conv_wgrad_r (3x3) / k_conv_wgrad_g<1> (1x1)
static inline int wgrad_nsplit(int ksz) { return ksz == 3 ? WR_NSPLIT : 256 / G_C; }

// which: 0 forward, 1 dx, 2 dw.  part (dw only): deterministic mode -- partials go to part, then an ordered sum into out.
template <int KS>
static int launch_generic(int which, const float *x, const float *w, const float *bias, const float *g, float *out, int B, int Cin,
                          int H, int W, int Cout, int Ho, int Wo, int stride, int act, cudaStream_t st, float *part = nullptr)
{
    constexpr int KK = KS * KS;
    const dim3 blk(G_T, G_T);
    if (which == 2 && part) {
        if (KS == 3 && getenv("ESR_WGRAD_MMA") != nullptr) {
            set_error("conv2d_backward: the ESR_WGRAD_MMA weight gradient sums with atomics and has no deterministic variant; "
                      "unset ESR_WGRAD_MMA or leave deterministic mode");
            return ESR_EUNSUPPORTED;
        }
        const int PD = (G_T - 1) * stride + KS;
        const size_t smem = (size_t)(256 * G_C + G_C * PD * PD) * 4;
        const int pairs = ((Cout + G_C - 1) / G_C) * ((Cin + G_C - 1) / G_C);
        const int slices = wgrad_slices(B, Cin, Cout, Ho, Wo);
        static bool attr = false;
        if constexpr (KS == 3) {
            if (!attr) { ESR_CUDA_CHECK(cudaFuncSetAttribute(k_conv_wgrad_r_det, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024)); attr = true; }
            k_conv_wgrad_r_det<<<dim3(pairs, slices), 256, smem, st>>>(x, g, part, B, Cin, H, W, Cout, Ho, Wo, stride);
        } else {
            if (!attr) { ESR_CUDA_CHECK(cudaFuncSetAttribute(k_conv_wgrad_g_det<KS>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024)); attr = true; }
            k_conv_wgrad_g_det<KS><<<dim3(pairs, slices), 256, smem, st>>>(x, g, part, B, Cin, H, W, Cout, Ho, Wo, stride);
        }
        ESR_LAUNCH_CHECK();
        return sum_slices(part, slices * wgrad_nsplit(KS), (size_t)Cout * Cin * KK, out, st);
    }
    if (which == 0 && KS == 3 && stride == 1) {
        const size_t smem = (size_t)(G_C * R_PH * R_PW + G_C * 9 * G_C) * 4;
        const dim3 grid(((Wo + R_TW - 1) / R_TW) * ((Ho + R_TH - 1) / R_TH), (Cout + G_C - 1) / G_C, B);
        k_conv_fwd_r<<<grid, 256, smem, st>>>(x, w, bias, out, Cin, H, W, Cout, act);
    } else if (which == 2 && KS == 3 && getenv("ESR_WGRAD_MMA") != nullptr) {
        // opt-in experiment: parity-green but staging-bound (the three packed copies of the x patch cost more global loads than
        // the FFMA kernel's single patch): 3.29 ms vs 3.35 ms for the narrow layers of a cfg2 iteration, +0.7 ms on the whole step
        const int PD = 15 * stride + 3;
        const size_t smem = (size_t)2 * 16 * WM_GP * 2 + (size_t)2 * 3 * 8 * PD * 8 * 4 + 16 * 72 * 4;
        const int pairs = ((Cout + 15) / 16) * ((Cin + 7) / 8);
        const int items = B * ((Wo + 15) / 16) * ((Ho + 15) / 16);
        int slices = (dev_info().sm_count * 4 + pairs - 1) / pairs;
        if (slices > items) slices = items;
        if (slices < 1) slices = 1;
        static bool attr = false;
        if (!attr) {
            ESR_CUDA_CHECK(cudaFuncSetAttribute(k_conv_wgrad_mma<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
            ESR_CUDA_CHECK(cudaFuncSetAttribute(k_conv_wgrad_mma<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
            attr = true;
        }
        if (stride == 1) k_conv_wgrad_mma<1><<<dim3(pairs, slices), 256, smem, st>>>(x, g, out, B, Cin, H, W, Cout, Ho, Wo);
        else k_conv_wgrad_mma<2><<<dim3(pairs, slices), 256, smem, st>>>(x, g, out, B, Cin, H, W, Cout, Ho, Wo);
    } else if (which == 2 && KS == 3) {
        const int PD = (G_T - 1) * stride + 3;
        const size_t smem = (size_t)(256 * G_C + G_C * PD * PD) * 4;
        const int pairs = ((Cout + G_C - 1) / G_C) * ((Cin + G_C - 1) / G_C);
        const int items = B * ((Wo + G_T - 1) / G_T) * ((Ho + G_T - 1) / G_T);
        int slices = (dev_info().sm_count * 8 + pairs - 1) / pairs;
        if (slices > items) slices = items;
        if (slices < 1) slices = 1;
        static bool attr = false;
        if (!attr) { ESR_CUDA_CHECK(cudaFuncSetAttribute(k_conv_wgrad_r, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024)); attr = true; }
        k_conv_wgrad_r<<<dim3(pairs, slices), 256, smem, st>>>(x, g, out, B, Cin, H, W, Cout, Ho, Wo, stride);
    } else if (which == 0) {
        const int PD = (G_T - 1) * stride + KS;
        const size_t smem = (size_t)(G_C * PD * PD + G_C * G_C * KK) * 4;
        const dim3 grid(((Wo + G_T - 1) / G_T) * ((Ho + G_T - 1) / G_T), (Cout + G_C - 1) / G_C, B);
        static bool attr = false;
        if (!attr) { ESR_CUDA_CHECK(cudaFuncSetAttribute(k_conv_fwd_g<KS>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024)); attr = true; }
        k_conv_fwd_g<KS><<<grid, blk, smem, st>>>(x, w, bias, out, Cin, H, W, Cout, Ho, Wo, stride, act);
    } else if (which == 1 && KS == 3 && stride == 2) {
        const dim3 grid(((W + 31) / 32) * ((H + 31) / 32), (Cin + G_C - 1) / G_C, B);
        k_conv_dgrad_s2<<<grid, 256, 0, st>>>(g, w, out, Cin, H, W, Cout, Ho, Wo);
    } else if (which == 1) {
        const int GP = (G_T - 1 + KS - 1) / stride + 2;
        const size_t smem = (size_t)(G_C * GP * GP + G_C * G_C * KK) * 4;
        const dim3 grid(((W + G_T - 1) / G_T) * ((H + G_T - 1) / G_T), (Cin + G_C - 1) / G_C, B);
        k_conv_dgrad_g<KS><<<grid, blk, smem, st>>>(g, w, out, Cin, H, W, Cout, Ho, Wo, stride);
    } else {
        const int PD = (G_T - 1) * stride + KS;
        const size_t smem = (size_t)(256 * G_C + G_C * PD * PD) * 4;
        const int pairs = ((Cout + G_C - 1) / G_C) * ((Cin + G_C - 1) / G_C);
        const int items = B * ((Wo + G_T - 1) / G_T) * ((Ho + G_T - 1) / G_T);
        int slices = (dev_info().sm_count * 8 + pairs - 1) / pairs;
        if (slices > items) slices = items;
        if (slices < 1) slices = 1;
        static bool attr = false;
        if (!attr) { ESR_CUDA_CHECK(cudaFuncSetAttribute(k_conv_wgrad_g<KS>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024)); attr = true; }
        k_conv_wgrad_g<KS><<<dim3(pairs, slices), 256, smem, st>>>(x, g, out, B, Cin, H, W, Cout, Ho, Wo, stride);
    }
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}

static int generic(int which, int ksz, const float *x, const float *w, const float *bias, const float *g, float *out, int B, int Cin,
                   int H, int W, int Cout, int Ho, int Wo, int stride, int act, cudaStream_t st, float *part = nullptr)
{
    return ksz == 3 ? launch_generic<3>(which, x, w, bias, g, out, B, Cin, H, W, Cout, Ho, Wo, stride, act, st, part)
                    : launch_generic<1>(which, x, w, bias, g, out, B, Cin, H, W, Cout, Ho, Wo, stride, act, st, part);
}

// db = sum of g over (image, pixel); part != NULL: deterministic (per-block partials, then the ordered sum)
static int bias_grad(const float *g, int B, int Cout, int HW, float *db, float *part, cudaStream_t st)
{
    const size_t total = (size_t)B * HW;
    int chunks = (int)min((size_t)64, (total + 4095) / 4096);
    if (chunks < 1) chunks = 1;
    if (!part) {
        k_bias_grad<<<dim3(Cout, chunks), 256, 0, st>>>(g, B, Cout, HW, db);
        ESR_LAUNCH_CHECK();
        return ESR_OK;
    }
    k_bias_grad_det<<<dim3(Cout, chunks), 256, 0, st>>>(g, B, Cout, HW, part);
    ESR_LAUNCH_CHECK();
    return sum_slices(part, chunks, (size_t)Cout, db, st);
}

// wgrad_tc.cu (returns ESR_EINVAL when the shape is not supported).  part != NULL: deterministic (see wgrad_tc_part_bytes)
int wgrad_tc(const __nv_bfloat16 *x_split, const __nv_bfloat16 *g_split, int B, int Cin, int H, int W, int Cout, int CoutPad, int ksz,
             float *dw, float *part, cudaStream_t st);
size_t wgrad_tc_part_bytes(int B, int Cin, int H, int W, int Cout, int CoutPad, int ksz);

// the dw kernel esr_conv2d_backward picks: k_wgrad_tc for the 64-multiple layers, the CUDA-core kernels otherwise
static inline bool use_tc_dw(int Cin, int Cout, int ksz, int stride)
{
    return tc_dgrad_ok(Cin, Cout, ksz, stride) && Cin % 64 == 0 && getenv("ESR_WGRAD_GENERIC") == nullptr;
}

// deterministic mode's extra workspace, after the default layout: bias partials (<= 64 chunks), then the dw partials
static size_t conv2d_det_bias_bytes(int Cout) { return align_up((size_t)64 * Cout * 4, 256); }
static size_t conv2d_det_bytes(int B, int Cin, int H, int W, int Cout, int ksz, int stride)
{
    const int Ho = (H + 2 * (ksz / 2) - ksz) / stride + 1, Wo = (W + 2 * (ksz / 2) - ksz) / stride + 1;
    const size_t dw = use_tc_dw(Cin, Cout, ksz, stride)
                          ? wgrad_tc_part_bytes(B, Cin, H, W, Cout, pad64(Cout), ksz)
                          : (size_t)wgrad_slices(B, Cin, Cout, Ho, Wo) * wgrad_nsplit(ksz) * Cout * Cin * ksz * ksz * 4;
    return conv2d_det_bias_bytes(Cout) + dw;
}

} // namespace esr

using namespace esr;

extern "C" {

size_t esr_conv2d_workspace_bytes(int B, int Cin, int H, int W, int Cout, int ksz, int stride)
{
    return conv2d_ws(B, Cin, H, W, Cout, ksz, stride);
}

size_t esr_conv2d_workspace_bytes_ex(int B, int Cin, int H, int W, int Cout, int ksz, int stride, int flags)
{
    const size_t base = conv2d_ws(B, Cin, H, W, Cout, ksz, stride);
    return (flags & ESR_DETERMINISTIC) ? base + conv2d_det_bytes(B, Cin, H, W, Cout, ksz, stride) : base;
}

size_t esr_conv2d_split_bytes(int B, int Cin, int H, int W, int Cout, int ksz, int stride)
{
    const bool both = tc_fwd_ok(Cin, Cout, ksz, stride) && tc_dgrad_ok(Cin, Cout, ksz, stride) && Cin % 64 == 0;
    return both ? (size_t)B * Cin * H * W * 4 : 0;
}

int esr_conv2d_forward(const float *x, const float *w, const float *bias, int B, int Cin, int H, int W, int Cout, int ksz, int stride,
                       int act, float *y, void *x_split_out, void *workspace, size_t workspace_bytes, esr_stream_t stream)
{
    cudaStream_t st = (cudaStream_t)stream;
    ESR_REQUIRE(x && w && bias && y, "conv2d_forward: null pointer");
    ESR_REQUIRE((ksz == 3 || ksz == 1) && (stride == 1 || stride == 2) && act >= 0 && act <= 3, "conv2d_forward: ksz=%d stride=%d act=%d", ksz,
                stride, act);
    ESR_REQUIRE(B > 0 && Cin > 0 && Cout > 0 && H > 0 && W > 0, "conv2d_forward: bad shape");
    const int pad = ksz / 2, Ho = (H + 2 * pad - ksz) / stride + 1, Wo = (W + 2 * pad - ksz) / stride + 1;
    if (tc_fwd_ok(Cin, Cout, ksz, stride)) {
        ESR_REQUIRE(workspace, "conv2d_forward: workspace required");
        Bump ws{(uint8_t *)workspace, 0, workspace_bytes};
        return conv_tc_nchw(x, w, bias, B, Cin, H, W, Cout, ksz, act, y, x_split_out, ws, st);
    }
    static const bool no_mma = getenv("ESR_TRAIN_NO_MMA") != nullptr;
    if (ksz == 3 && !no_mma && workspace && workspace_bytes >= mma_weight_bytes(Cout, Cin)) {
        // narrow layers: warp-level tensor cores (mma_conv.cu) on fp32 NCHW; weights packed to the split-bf16 image first
        int rc = pack_mma_weight(w, Cout, Cin, workspace, st);
        if (rc) return rc;
        rc = conv_mma_nchw(x, workspace, bias, B, Cin, H, W, Cout, stride, act, y, st);
        if (rc != ESR_EINVAL) return rc;
    }
    return generic(0, ksz, x, w, bias, nullptr, y, B, Cin, H, W, Cout, Ho, Wo, stride, act, st);
}

int esr_conv2d_backward(const float *x, const void *x_split, const float *w, const float *y, const float *dy, int B, int Cin, int H,
                        int W, int Cout, int ksz, int stride, int act, float *dx, float *dw, float *db, void *workspace,
                        size_t workspace_bytes, esr_stream_t stream)
{
    return esr_conv2d_backward_ex(x, x_split, w, y, dy, B, Cin, H, W, Cout, ksz, stride, act, dx, dw, db, 0, workspace, workspace_bytes,
                                  stream);
}

int esr_conv2d_backward_ex(const float *x, const void *x_split, const float *w, const float *y, const float *dy, int B, int Cin, int H,
                           int W, int Cout, int ksz, int stride, int act, float *dx, float *dw, float *db, int flags, void *workspace,
                           size_t workspace_bytes, esr_stream_t stream)
{
    cudaStream_t st = (cudaStream_t)stream;
    ESR_REQUIRE((x || x_split) && w && dy && workspace && ((dw && db) || (!dw && !db && dx)), "conv2d_backward: null pointer");
    ESR_REQUIRE(!x_split || esr_conv2d_split_bytes(B, Cin, H, W, Cout, ksz, stride) > 0, "conv2d_backward: x_split given for a layer without a tensor-core dw");
    ESR_REQUIRE(x || getenv("ESR_WGRAD_GENERIC") == nullptr, "conv2d_backward: the CUDA-core dw needs x");
    const bool want_dw = dw != nullptr;                               // dw == db == NULL: input gradient only (deferred dw)
    ESR_REQUIRE(act == ACT_NONE || y, "conv2d_backward: the forward output is needed for the activation derivative");
    ESR_REQUIRE((ksz == 3 || ksz == 1) && (stride == 1 || stride == 2) && act >= 0 && act <= 3, "conv2d_backward: ksz=%d stride=%d act=%d", ksz,
                stride, act);
    const int pad = ksz / 2, Ho = (H + 2 * pad - ksz) / stride + 1, Wo = (W + 2 * pad - ksz) / stride + 1;
    // deterministic mode: the partial buffers sit after the default layout (esr_conv2d_workspace_bytes_ex)
    const bool det = (flags & ESR_DETERMINISTIC) != 0;
    const size_t base_bytes = conv2d_ws(B, Cin, H, W, Cout, ksz, stride);
    float *bias_part = nullptr, *dw_part = nullptr;
    if (det && want_dw) {
        ESR_REQUIRE(workspace_bytes >= base_bytes + conv2d_det_bytes(B, Cin, H, W, Cout, ksz, stride),
                    "conv2d_backward: deterministic mode needs esr_conv2d_workspace_bytes_ex(..., ESR_DETERMINISTIC) bytes");
        bias_part = (float *)((uint8_t *)workspace + base_bytes);
        dw_part = (float *)((uint8_t *)workspace + base_bytes + conv2d_det_bias_bytes(Cout));
    }
    Bump ws{(uint8_t *)workspace, 0, det ? base_bytes : workspace_bytes};
    int rc;
    const size_t ng = (size_t)B * Cout * Ho * Wo;
    const bool tcd = tc_dgrad_ok(Cin, Cout, ksz, stride);
    const int gC = pad64(Cout);
    const bool tc_dw = tcd && use_tc_dw(Cin, Cout, ksz, stride);
    float *g = (float *)ws.take(ng * 4);                           // fp32 g: only the CUDA-core kernels read it
    __nv_bfloat16 *gsplit = nullptr;
    if (want_dw) {
        ESR_CUDA_CHECK(cudaMemsetAsync(db, 0, (size_t)Cout * 4, st));
        ESR_CUDA_CHECK(cudaMemsetAsync(dw, 0, (size_t)Cout * Cin * ksz * ksz * 4, st));
    }
    if (tcd) {
        // one pass: activation derivative, bias gradient, fp32 -> split bf16 NHWC (padded to a 64-multiple of channels).
        // Deterministic mode: the pass writes fp32 g instead of adding db, and db is summed from g in a fixed order below.
        gsplit = (__nv_bfloat16 *)ws.take((size_t)B * gC * Ho * Wo * 4);
        ESR_REQUIRE(ws.off <= ws.cap, "conv2d_backward: workspace too small");
        const int tpb = split_tiles_per_block(Ho * Wo, gC / 64, B), tiles = (Ho * Wo + 31) / 32;
        k_to_split<true><<<dim3((tiles + tpb - 1) / tpb, gC / 64, B), 256, 0, st>>>(dy, y, act, Cout, gC, Ho * Wo, tpb, gsplit,
                                                                                   (size_t)B * Ho * Wo * gC, want_dw && !det ? db : nullptr,
                                                                                   tc_dw && !(det && want_dw) ? nullptr : g);
        ESR_LAUNCH_CHECK();
        if (det && want_dw && (rc = bias_grad(g, B, Cout, Ho * Wo, db, bias_part, st))) return rc;
    } else {
        ESR_REQUIRE(ws.off <= ws.cap, "conv2d_backward: workspace too small");
        if (act == ACT_NONE) {
            ESR_CUDA_CHECK(cudaMemcpyAsync(g, dy, ng * 4, cudaMemcpyDeviceToDevice, st));
        } else {
            k_act_bwd<<<(unsigned)min((size_t)4096, (ng + 255) / 256), 256, 0, st>>>(dy, y, g, ng, act);
            ESR_LAUNCH_CHECK();
        }
        if (want_dw && (rc = bias_grad(g, B, Cout, Ho * Wo, db, bias_part, st))) return rc;
    }
    // ---- dw
    bool dw_done = !want_dw;
    if (want_dw && tc_dw) {
        const __nv_bfloat16 *xsplit = (const __nv_bfloat16 *)x_split;       // saved by the forward, or converted here
        if (!xsplit) {
            Bump ws2 = ws;                                           // dead after the kernel: dx reuses the space
            __nv_bfloat16 *xs_ = (__nv_bfloat16 *)ws2.take((size_t)B * Cin * H * W * 4);
            ESR_REQUIRE(ws2.off <= ws2.cap, "conv2d_backward: workspace too small");
            if ((rc = split_from_nchw_pad(x, B, Cin, Cin, H * W, xs_, st))) return rc;
            xsplit = xs_;
        }
        if ((rc = wgrad_tc(xsplit, gsplit, B, Cin, H, W, Cout, gC, ksz, dw, dw_part, st))) return rc;
        dw_done = true;
    }
    if (!dw_done && (rc = generic(2, ksz, x, nullptr, nullptr, g, dw, B, Cin, H, W, Cout, Ho, Wo, stride, 0, st, dw_part))) return rc;
    // ---- dx
    if (dx) {
        if (tcd) {
            float *wt = (float *)ws.take((size_t)gC * Cin * ksz * ksz * 4);
            void *wp = ws.take(tc_packed_weight_bytes(Cin, gC, ksz * ksz));
            float *bp = (float *)ws.take(256 * 4);
            ESR_REQUIRE(ws.off <= ws.cap, "conv2d_backward: workspace too small (%zu > %zu)", ws.off, ws.cap);
            if (gC != Cout) ESR_CUDA_CHECK(cudaMemsetAsync(wt, 0, (size_t)gC * Cin * ksz * ksz * 4, st));
            k_weight_rot_t<<<(Cout * Cin * ksz * ksz + 255) / 256, 256, 0, st>>>(w, Cout, gC, Cin, ksz * ksz, wt);
            ESR_LAUNCH_CHECK();
            if ((rc = pack_conv_weight(wt, Cin, gC, ksz, wp, st))) return rc;
            ESR_CUDA_CHECK(cudaMemsetAsync(bp, 0, 256 * 4, st));
            SplitTensor gsrc; gsrc.base = gsplit; gsrc.n_img = B; gsrc.H = Ho; gsrc.W = Wo; gsrc.C = gC;
            ConvTCDesc d;
            d.src[0] = gsrc; d.n_src = 1; d.ntaps = ksz * ksz; d.cout = Cin; d.wpacked = wp; d.bias = bp; d.n_img = B; d.act = ACT_NONE;
            d.out_f32 = dx; d.out_f32_C = Cin; d.out_f32_nchw = 1;
            ConvTCArgs a;
            if ((rc = conv_tc_prepare(d, &a))) return rc;
            if ((rc = conv_tc_launch(a, st))) return rc;
        } else if (ksz == 3 && stride == 1 && getenv("ESR_TRAIN_NO_MMA") == nullptr &&
                   [&] {   // dx = conv(g, rot180(w)^T) on the warp-level tensor cores when the shape is instantiated
                       Bump w2 = ws;
                       void *img = w2.take(mma_weight_bytes(Cin, Cout));
                       if (w2.off > w2.cap) return false;
                       if (pack_mma_weight_dx(w, Cout, Cin, img, st)) return false;
                       return conv_mma_nchw(g, img, nullptr, B, Cout, H, W, Cin, 1, ACT_NONE, dx, st) == ESR_OK;
                   }()) {
        } else if (ksz == 3 && stride == 1) {
            // dx = conv(g, rot180(w)^T): the register-tiled forward kernel with the roles of Cin and Cout swapped
            float *wt = (float *)ws.take((size_t)Cout * Cin * 9 * 4);
            ESR_REQUIRE(ws.off <= ws.cap, "conv2d_backward: workspace too small (%zu > %zu)", ws.off, ws.cap);
            k_weight_rot_t<<<(Cout * Cin * 9 + 255) / 256, 256, 0, st>>>(w, Cout, Cout, Cin, 9, wt);
            ESR_LAUNCH_CHECK();
            if ((rc = generic(0, 3, g, wt, nullptr, nullptr, dx, B, Cout, H, W, Cin, H, W, 1, ACT_NONE, st))) return rc;
        } else {
            if ((rc = generic(1, ksz, nullptr, w, nullptr, g, dx, B, Cin, H, W, Cout, Ho, Wo, stride, 0, st))) return rc;
        }
    }
    return ESR_OK;
}

int esr_upsample2x_forward(const float *x, int planes, int H, int W, float *y, esr_stream_t stream)
{
    cudaStream_t st = (cudaStream_t)stream;
    ESR_REQUIRE(x && y && planes > 0 && H > 0 && W > 0, "upsample2x_forward: bad arguments");
    ESR_REQUIRE(2 * H <= 65535 && planes <= 65535, "upsample2x_forward: grid limits");
    k_upsample2x_fwd<<<dim3((2 * W + 255) / 256, 2 * H, planes), 256, 0, st>>>(x, H, W, y);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}

int esr_upsample2x_backward(const float *dy, int planes, int H, int W, float *dx, esr_stream_t stream)
{
    cudaStream_t st = (cudaStream_t)stream;
    ESR_REQUIRE(dy && dx && planes > 0 && H > 0 && W > 0, "upsample2x_backward: bad arguments");
    ESR_REQUIRE(H <= 65535 && planes <= 65535, "upsample2x_backward: grid limits");
    k_upsample2x_bwd<<<dim3((W + 255) / 256, H, planes), 256, 0, st>>>(dy, H, W, dx);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}

static inline dim3 ew_grid(int B, int chw) { return dim3((unsigned)min(256, (chw + 255) / 256), (unsigned)B); }

int esr_gru_hr(const float *h, const float *zr, int B, int chw, float *out, esr_stream_t stream)
{
    ESR_REQUIRE(h && zr && out && B > 0 && chw > 0, "gru_hr: bad arguments");
    const size_t n = (size_t)B * chw;
    k_gru_hr<<<ew_grid(B, chw), 256, 0, (cudaStream_t)stream>>>(h, zr, n, chw, out);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}
int esr_gru_hr_backward(const float *h, const float *zr, const float *grad, int B, int chw, float *dh, float *dzr, esr_stream_t stream)
{
    ESR_REQUIRE(h && zr && grad && dh && dzr && B > 0 && chw > 0, "gru_hr_backward: bad arguments");
    const size_t n = (size_t)B * chw;
    k_gru_hr_bwd<<<ew_grid(B, chw), 256, 0, (cudaStream_t)stream>>>(h, zr, grad, n, chw, dh, dzr);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}
int esr_gru_blend(const float *h, const float *zr, const float *o, int B, int chw, float *out, esr_stream_t stream)
{
    ESR_REQUIRE(h && zr && o && out && B > 0 && chw > 0, "gru_blend: bad arguments");
    const size_t n = (size_t)B * chw;
    k_gru_blend<<<ew_grid(B, chw), 256, 0, (cudaStream_t)stream>>>(h, zr, o, n, chw, out);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}
int esr_gru_blend_backward(const float *h, const float *zr, const float *o, const float *grad, int B, int chw, float *dh, float *dzr,
                           float *d_o, esr_stream_t stream)
{
    ESR_REQUIRE(h && zr && o && grad && dh && dzr && d_o && B > 0 && chw > 0, "gru_blend_backward: bad arguments");
    const size_t n = (size_t)B * chw;
    k_gru_blend_bwd<<<ew_grid(B, chw), 256, 0, (cudaStream_t)stream>>>(h, zr, o, grad, n, chw, dh, dzr, d_o);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}

int esr_mse_loss(const float *pred, const float *target, size_t n, float *loss, float *grad, float grad_scale, esr_stream_t stream)
{
    cudaStream_t st = (cudaStream_t)stream;
    ESR_REQUIRE(pred && target && loss && n > 0, "mse_loss: bad arguments");
    ESR_CUDA_CHECK(cudaMemsetAsync(loss, 0, 4, st));
    k_mse<<<(unsigned)min((size_t)1024, (n + 255) / 256), 256, 0, st>>>(pred, target, n, 1.0f / (float)n, loss, grad, grad_scale);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}

size_t esr_mse_loss_workspace_bytes_ex(size_t n, int flags)
{
    (void)n;
    return (flags & ESR_DETERMINISTIC) ? 1024 * sizeof(float) : 0;  // one partial per block (at most 1024 blocks)
}

int esr_mse_loss_ex(const float *pred, const float *target, size_t n, float *loss, float *grad, float grad_scale, int flags,
                    void *workspace, size_t workspace_bytes, esr_stream_t stream)
{
    if (!(flags & ESR_DETERMINISTIC)) return esr_mse_loss(pred, target, n, loss, grad, grad_scale, stream);
    cudaStream_t st = (cudaStream_t)stream;
    ESR_REQUIRE(pred && target && loss && n > 0, "mse_loss: bad arguments");
    ESR_REQUIRE(workspace && workspace_bytes >= esr_mse_loss_workspace_bytes_ex(n, flags), "mse_loss: workspace too small");
    const unsigned blocks = (unsigned)min((size_t)1024, (n + 255) / 256);
    float *part = (float *)workspace;
    k_mse_det<<<blocks, 256, 0, st>>>(pred, target, n, 1.0f / (float)n, part, grad, grad_scale);
    ESR_LAUNCH_CHECK();
    k_mse_finish<<<1, 32, 0, st>>>(part, (int)blocks, 1.0f / (float)n, loss);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}

int esr_adam_step(float *param, const float *grad, float *exp_avg, float *exp_avg_sq, float *max_exp_avg_sq, size_t n,
                  int32_t *step_counter, float lr, float beta1, float beta2, float eps, float weight_decay, esr_stream_t stream)
{
    cudaStream_t st = (cudaStream_t)stream;
    ESR_REQUIRE(param && grad && exp_avg && exp_avg_sq && step_counter && n > 0, "adam_step: bad arguments");
    k_adam_tick<<<1, 1, 0, st>>>(step_counter);
    ESR_LAUNCH_CHECK();
    k_adam<<<(unsigned)min((size_t)2048, (n + 255) / 256), 256, 0, st>>>(param, grad, exp_avg, exp_avg_sq, max_exp_avg_sq, n, lr, beta1, beta2, eps,
                                                                        weight_decay, step_counter, nullptr);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}

int esr_adam_step_dev(float *param, const float *grad, float *exp_avg, float *exp_avg_sq, float *max_exp_avg_sq, size_t n,
                      int32_t *step_counter, const float *hyper, esr_stream_t stream)
{
    cudaStream_t st = (cudaStream_t)stream;
    ESR_REQUIRE(param && grad && exp_avg && exp_avg_sq && step_counter && hyper && n > 0, "adam_step_dev: bad arguments");
    k_adam_tick<<<1, 1, 0, st>>>(step_counter);
    ESR_LAUNCH_CHECK();
    k_adam<<<(unsigned)min((size_t)2048, (n + 255) / 256), 256, 0, st>>>(param, grad, exp_avg, exp_avg_sq, max_exp_avg_sq, n, 0.f, 0.f, 0.f, 0.f,
                                                                        0.f, step_counter, hyper);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}

} // extern "C"
