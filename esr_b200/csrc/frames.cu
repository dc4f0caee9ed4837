// frames.cu -- the dataset's image frames: cv2.resize(..., interpolation=cv2.INTER_CUBIC) of uint8 frames, with
// augment_frame's flips and frame_formatting's / 255 (dataloader/h5dataset.py:300-315, 672-685, base_dataset.py:36-38),
// for a whole batch and both target sizes in one launch.
//
// The arithmetic is OpenCV's generic resize for 8-bit images (imgproc resize, ResizeCubic with HResizeCubic /
// VResizeCubic and the SIMD vertical pass VResizeCubicVec_32s8u); tests/frames_ref.py restates it in numpy and DESIGN §8b
// records what was measured against cv2 itself.  Every floating-point step is written with round-to-nearest intrinsics so
// that nvcc cannot contract or reorder it: the coefficients and the vertical pass must equal the host's bit for bit.
#include "common.cuh"

namespace esr {

// source tap k in [-1, 2] of output coordinate d and its 11-bit coefficient (interpolateCubic, saturate_cast<short>)
struct CubicTaps {
    int i[4];
    int c[4];
};

__device__ __forceinline__ CubicTaps cubic_taps(int d, int src, double scale)
{
    const float fx = __double2float_rn(__dsub_rn(__dmul_rn(__dadd_rn((double)d, 0.5), scale), 0.5));
    const float fl = floorf(fx);
    const int sx = (int)fl;
    const float x = __fsub_rn(fx, fl);
    const float A = -0.75f, x1 = __fadd_rn(x, 1.f), y = __fsub_rn(1.f, x);
    const float c0 = __fsub_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fsub_rn(__fmul_rn(A, x1), 5.f * A), x1), 8.f * A), x1), 4.f * A);
    const float c1 = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(A + 2.f, x), A + 3.f), x), x), 1.f);
    const float c2 = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(A + 2.f, y), A + 3.f), y), y), 1.f);
    const float c3 = __fsub_rn(__fsub_rn(__fsub_rn(1.f, c0), c1), c2);
    CubicTaps t;
    t.c[0] = __float2int_rn(c0 * 2048.f);
    t.c[1] = __float2int_rn(c1 * 2048.f);
    t.c[2] = __float2int_rn(c2 * 2048.f);
    t.c[3] = __float2int_rn(c3 * 2048.f);
#pragma unroll
    for (int k = 0; k < 4; ++k) t.i[k] = min(max(sx + k - 1, 0), src - 1);
    return t;
}

// one thread per output pixel of either target; blockIdx.y = frame
__global__ void __launch_bounds__(256)
k_resize_frames_cubic(const esr_frame_resize_desc *__restrict__ desc, int H, int W, int C, int oH0, int oW0, int oH1, int oW1,
                      double sx0, double sy0, double sx1, double sy1)
{
    const esr_frame_resize_desc d = desc[blockIdx.y];
    const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long n0 = (long long)oH0 * oW0;
    const bool second = p >= n0;
    if (second && (!d.out1 || p >= n0 + (long long)oH1 * oW1)) return;
    const int oW = second ? oW1 : oW0;
    const int q = (int)(second ? p - n0 : p);
    const int oy = q / oW, ox = q - oy * oW;
    const CubicTaps tx = cubic_taps(ox, W, second ? sx1 : sx0);
    const CubicTaps ty = cubic_taps(oy, H, second ? sy1 : sy0);
    float *out = (second ? d.out1 : d.out0) + (long long)q * C;
    const int simd_end = oW * C / 8 * 8;       // VResizeCubicVec_32s8u's 8-element steps; the rest of the row is scalar
    int col[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) col[k] = (d.flips & 1) ? W - 1 - tx.i[k] : tx.i[k];
    for (int c = 0; c < C; ++c) {
        int hs[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const int row = (d.flips & 2) ? H - 1 - ty.i[r] : ty.i[r];
            const uint8_t *s = d.src + ((long long)row * W) * C + c;
            int v = 0;
#pragma unroll
            for (int k = 0; k < 4; ++k) v += (int)s[(long long)col[k] * C] * tx.c[k];
            hs[r] = v;
        }
        int u;
        if (ox * C + c < simd_end) {
            const float sc = 1.f / (float)(1 << 22);
            float t = __fmul_rn((float)hs[3], (float)ty.c[3] * sc);
            t = __fmaf_rn((float)hs[2], (float)ty.c[2] * sc, t);
            t = __fmaf_rn((float)hs[1], (float)ty.c[1] * sc, t);
            t = __fmaf_rn((float)hs[0], (float)ty.c[0] * sc, t);
            u = __float2int_rn(t);
        } else {
            u = (hs[0] * ty.c[0] + hs[1] * ty.c[1] + hs[2] * ty.c[2] + hs[3] * ty.c[3] + (1 << 21)) >> 22;
        }
        out[c] = __fdiv_rn((float)min(max(u, 0), 255), 255.f);
    }
}

}  // namespace esr

extern "C" int esr_resize_frames_cubic(const esr_frame_resize_desc *desc, int n, int H, int W, int C, int oH0, int oW0, int oH1,
                                       int oW1, esr_stream_t stream)
{
    ESR_REQUIRE(desc && n >= 0 && (C == 1 || C == 3), "esr_resize_frames_cubic: bad arguments");
    ESR_REQUIRE(H > 0 && W > 0 && oH0 > 0 && oW0 > 0 && oH1 >= 0 && oW1 >= 0, "esr_resize_frames_cubic: bad sizes");
    ESR_REQUIRE((long long)H * W * C < (1LL << 40) && (long long)oH0 * oW0 + (long long)oH1 * oW1 < (1LL << 31),
                "esr_resize_frames_cubic: frames too large");
    ESR_REQUIRE(n <= 65535, "esr_resize_frames_cubic: at most 65535 frames per launch");
    if (n == 0) return ESR_OK;
    const long long total = (long long)oH0 * oW0 + (long long)oH1 * oW1;
    // OpenCV's scale_x = 1. / inv_scale_x with inv_scale_x = (double)dsize.width / ssize.width
    const double sx0 = 1.0 / ((double)oW0 / W), sy0 = 1.0 / ((double)oH0 / H);
    const double sx1 = oW1 ? 1.0 / ((double)oW1 / W) : 0.0, sy1 = oH1 ? 1.0 / ((double)oH1 / H) : 0.0;
    esr::k_resize_frames_cubic<<<dim3((unsigned)((total + 255) / 256), (unsigned)n), 256, 0, (cudaStream_t)stream>>>(
        desc, H, W, C, oH0, oW0, oH1, oW1, sx0, sy0, sx1, sy1);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}
