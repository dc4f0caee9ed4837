// dcn.cu -- modulated deformable sampling (DCNv2) producing the A operand of the 3x3xC contraction.
// Semantics restated from models/DCNv2/src/cuda/dcn_v2_im2col_cuda.cu:25-54 (bilinear with zero outside the image)
// and :125-195 (per deformable group g, tap k = i*3+j: offsets at channels g*18+2k (row) / +1 (col), mask at g*9+k;
// sample at (y-1+i+off_h, x-1+j+off_w) only if it lies in (-1, H) x (-1, W); columns = value * mask).
// Stride 1, pad 1, dilation 1, 3x3, 64 channels, 8 deformable groups of 8 channels (models/model.py:173).
//
// Layout choices: features are split-bf16 NHWC so the 8 channels of one group at one corner are one
// 16-byte load per plane; one thread = one (pixel, tap, group); its 8 outputs land at column tap*64 + g*8, i.e. eight
// consecutive threads (g = 0..7) write one contiguous 128-byte row segment.  The columns tensor is then consumed by the
// wgmma GEMM (tc_conv.cu, 1x1 mode over 9 K-chunks) with the DCN weight packed tap-major, which equals the
// reference's W[Co, Ci*9] . columns contraction (dcn_v2_cuda.cu:90-92).
#include "net.cuh"

namespace esr {

__device__ __forceinline__ void ld8(const __nv_bfloat16 *hi, size_t plane, float (&o)[8])
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

constexpr int DCN_PIX = 32;    // pixels per block

__global__ void __launch_bounds__(256)
k_dcn_columns(const __nv_bfloat16 *__restrict__ feat, size_t f_plane, const int *__restrict__ feat_img,
              const float *__restrict__ om, int n_img, int H, int W, __nv_bfloat16 *__restrict__ cols, size_t c_plane)
{
    // the 216 offset/mask values of DCN_PIX consecutive pixels, staged with coalesced 16-byte loads
    __shared__ float4 s_om4[DCN_PIX * 54];
    const float *s_om = reinterpret_cast<const float *>(s_om4);
    const size_t npix = (size_t)n_img * H * W;
    const size_t p0 = (size_t)blockIdx.x * DCN_PIX;
    const int cnt = (int)min((size_t)DCN_PIX, npix - p0);
    const float4 *src = reinterpret_cast<const float4 *>(om + p0 * 216);
    for (int i = threadIdx.x; i < cnt * 54; i += 256) s_om4[i] = src[i];
    __syncthreads();
    for (int it = threadIdx.x; it < cnt * 72; it += 256) {
        const int g = it % 8, k = (it / 8) % 9, lp = it / 72;
        const size_t p = p0 + lp;
        const int x = (int)(p % W), y = (int)((p / W) % H), img = (int)(p / ((size_t)W * H));
        const float *o = s_om + lp * 216;
        const float off_h = o[g * 18 + 2 * k], off_w = o[g * 18 + 2 * k + 1], m = o[144 + g * 9 + k];
        const float h_im = (float)(y - 1 + k / 3) + off_h;
        const float w_im = (float)(x - 1 + k % 3) + off_w;
        float v[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) v[e] = 0.0f;
        if (h_im > -1.0f && w_im > -1.0f && h_im < (float)H && w_im < (float)W) {
            const int h_low = (int)floorf(h_im), w_low = (int)floorf(w_im);
            const int h_high = h_low + 1, w_high = w_low + 1;
            const float lh = h_im - (float)h_low, lw = w_im - (float)w_low;
            const float hh = 1.0f - lh, hw = 1.0f - lw;
            const float w1 = hh * hw, w2 = hh * lw, w3 = lh * hw, w4 = lh * lw;
            const size_t base = (size_t)(feat_img ? feat_img[img] : img) * H * W;
            float c1[8], c2[8], c3[8], c4[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) c1[e] = c2[e] = c3[e] = c4[e] = 0.0f;
            if (h_low >= 0 && w_low >= 0) ld8(feat + ((base + (size_t)h_low * W + w_low) * 64 + g * 8), f_plane, c1);
            if (h_low >= 0 && w_high <= W - 1) ld8(feat + ((base + (size_t)h_low * W + w_high) * 64 + g * 8), f_plane, c2);
            if (h_high <= H - 1 && w_low >= 0) ld8(feat + ((base + (size_t)h_high * W + w_low) * 64 + g * 8), f_plane, c3);
            if (h_high <= H - 1 && w_high <= W - 1) ld8(feat + ((base + (size_t)h_high * W + w_high) * 64 + g * 8), f_plane, c4);
#pragma unroll
            for (int e = 0; e < 8; ++e) v[e] = (w1 * c1[e] + w2 * c2[e] + w3 * c3[e] + w4 * c4[e]) * m;
        }
        uint32_t hw_[4], lw_[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            split_pack2(v[2 * e], v[2 * e + 1], hw_[e], lw_[e]);
        }
        __nv_bfloat16 *dst = cols + p * 576 + k * 64 + g * 8;
        *reinterpret_cast<uint4 *>(dst) = make_uint4(hw_[0], hw_[1], hw_[2], hw_[3]);
        *reinterpret_cast<uint4 *>(dst + c_plane) = make_uint4(lw_[0], lw_[1], lw_[2], lw_[3]);
    }
}

int dcn_columns(const SplitTensor &feat, const int *feat_img, const float *om, int n_img, const SplitTensor &cols, cudaStream_t st)
{
    ESR_REQUIRE(feat.C == 64 && cols.C == 576 && cols.H == feat.H && cols.W == feat.W, "dcn_columns: bad shapes");
    const size_t npix = (size_t)n_img * feat.H * feat.W;
    k_dcn_columns<<<(unsigned)ceil_div64((int64_t)npix, DCN_PIX), 256, 0, st>>>(feat.base, feat.plane(), feat_img, om, n_img, feat.H,
                                                                             feat.W, cols.base, cols.plane());
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}

} // namespace esr

// ------------------------------------------------------------------------------------------------
// `_ext.dcn_v2_forward` operator boundary (models/DCNv2/src/dcn_v2.h:9-27, src/vision.cpp:4-8):
// fp32 NCHW tensors in the reference's own layout in, fp32 NCHW out.
// ------------------------------------------------------------------------------------------------
namespace esr {
__global__ void __launch_bounds__(256)
k_om_from_nchw(const float *__restrict__ offset, const float *__restrict__ mask, int B, int HW, float *__restrict__ om)
{
    const size_t total = (size_t)B * HW * 216;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % 216);
        const size_t p = i / 216;
        const int pix = (int)(p % HW), b = (int)(p / HW);
        om[i] = c < 144 ? offset[((size_t)b * 144 + c) * HW + pix] : mask[((size_t)b * 72 + (c - 144)) * HW + pix];
    }
}
int om_from_nchw(const float *offset, const float *mask, int B, int HW, float *om, cudaStream_t st)
{
    const size_t total = (size_t)B * HW * 216;
    k_om_from_nchw<<<(unsigned)ceil_div64((int64_t)total, 256), 256, 0, st>>>(offset, mask, B, HW, om);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}
} // namespace esr

using namespace esr;

static size_t dcn_ws_layout(int B, int H, int W, size_t *o_feat, size_t *o_om, size_t *o_cols, size_t *o_out, size_t *o_w, size_t *o_b)
{
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t r = off; off = align_up(off + bytes, 1024); return r; };
    const size_t px = (size_t)B * H * W;
    *o_feat = take(px * 64 * 4); *o_om = take(px * 216 * 4); *o_cols = take(px * 576 * 4); *o_out = take(px * 64 * 4);
    *o_w = take(tc_packed_weight_bytes(64, 64, 9)); *o_b = take(64 * 4);
    return off;
}

extern "C" size_t esr_dcn_v2_workspace_bytes(int B, int H, int W)
{
    size_t a, b, c, d, e, f;
    return dcn_ws_layout(B, H, W, &a, &b, &c, &d, &e, &f);
}

extern "C" size_t esr_dcn_v2_workspace_bytes_ex(int B, int C, int H, int W, int Co, int kernel, int stride, int pad, int dilation,
                                                int deformable_group, int backward)
{
    if (dcn_is_tuned(C, Co, kernel, stride, pad, dilation, deformable_group))
        return backward ? esr_dcn_v2_backward_workspace_bytes(B, H, W) : esr_dcn_v2_workspace_bytes(B, H, W);
    return dcn_generic_ws_bytes(B, C, H, W, Co, kernel, stride, pad, dilation, deformable_group, backward);
}

extern "C" int esr_dcn_v2_forward(const float *input, const float *weight, const float *bias, const float *offset,
                                  const float *mask, int B, int C, int H, int W, int Co, int kernel, int stride, int pad,
                                  int dilation, int deformable_group, float *output, void *workspace, size_t ws_bytes,
                                  esr_stream_t stream)
{
    ESR_REQUIRE(input && weight && bias && offset && mask && output && workspace, "esr_dcn_v2_forward: null pointer");
    if (!dcn_is_tuned(C, Co, kernel, stride, pad, dilation, deformable_group))      // any other configuration: dcn_generic.cu
        return dcn_generic_forward(input, weight, bias, offset, mask, B, C, H, W, Co, kernel, stride, pad, dilation, deformable_group,
                                   output, workspace, ws_bytes, (cudaStream_t)stream);
    size_t o_feat, o_om, o_cols, o_out, o_w, o_b;
    const size_t need = dcn_ws_layout(B, H, W, &o_feat, &o_om, &o_cols, &o_out, &o_w, &o_b);
    if (ws_bytes < need) { set_error("esr_dcn_v2_forward: workspace %zu < %zu", ws_bytes, need); return ESR_EWORKSPACE; }
    cudaStream_t st = (cudaStream_t)stream;
    char *ws = (char *)workspace;
    SplitTensor feat, cols, out;
    feat.base = (__nv_bfloat16 *)(ws + o_feat); feat.n_img = B; feat.H = H; feat.W = W; feat.C = 64;
    cols = feat; cols.base = (__nv_bfloat16 *)(ws + o_cols); cols.C = 576;
    out = feat; out.base = (__nv_bfloat16 *)(ws + o_out);
    float *om = (float *)(ws + o_om);
    int rc;
    if ((rc = split_from_nchw(input, B, 64, H, W, feat.base, st))) return rc;
    if ((rc = om_from_nchw(offset, mask, B, H * W, om, st))) return rc;
    if ((rc = dcn_columns(feat, nullptr, om, B, cols, st))) return rc;
    if ((rc = pack_conv_weight(weight, 64, 64, 3, ws + o_w, st))) return rc;
    ESR_CUDA_CHECK(cudaMemcpyAsync(ws + o_b, bias, 64 * sizeof(float), cudaMemcpyDeviceToDevice, st));
    ConvTCDesc d;
    d.src[0] = cols; d.n_src = 1; d.ntaps = 1; d.cout = 64; d.wpacked = ws + o_w; d.bias = (const float *)(ws + o_b);
    d.n_img = B; d.act = ACT_NONE; d.out = out;
    ConvTCArgs args;
    if ((rc = conv_tc_prepare(d, &args))) return rc;
    if ((rc = conv_tc_launch(args, st))) return rc;
    return split_to_nchw(out.base, B, 64, H, W, output, st);
}
