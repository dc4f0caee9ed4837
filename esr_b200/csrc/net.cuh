// net.cuh -- shared declarations of the DeepRecurrNet forward pipeline (direct convs, element-wise kernels, DCN).
#pragma once
#include "tc_conv.cuh"

namespace esr {

enum Fmt : int { FMT_NCHW_F32 = 0, FMT_SPLIT = 1, FMT_NHWC_F32 = 2, FMT_HEAD_FUSED = 3 };

enum DirectKind : int { DK_HEAD, DK_HEAD_ENC0, DK_ENC0, DK_ENC1, DK_ENC2, DK_ATT32, DK_ATT16, DK_RECON0, DK_RECON1, DK_RECON2, DK_TAIL };

struct DirectArgs {
    // input
    const float *in_f32 = nullptr;              // NCHW fp32 [*, CIN, Hin, Win]   (head)
    const __nv_bfloat16 *in_split = nullptr;    // split NHWC [*, Hin, Win, CIN]
    size_t in_plane = 0;
    const int *in_img = nullptr;                // output image -> input image (nullptr = identity)
    int Hin = 0, Win = 0;
    int pad_top = 0, pad_bottom = 0, pad_left = 0, pad_right = 0;   // CropSize zero padding of the network input
    // weights
    const float *w = nullptr;                   // [9][CIN][COUT]
    const void *w_mma = nullptr;                // mma_conv.cu: split bf16 image [2 planes][9][max(COUT,8)][CIN+8] (pack_mma_weight)
    const float *bias = nullptr;                // [COUT]
    const float *w0 = nullptr, *b0 = nullptr;   // fused head (2->8): [9][2][8], [8]
    int act = ACT_NONE;
    // output
    int n_img = 0, Hout = 0, Wout = 0;
    __nv_bfloat16 *out_split = nullptr;
    size_t out_plane = 0;
    float *out_f32 = nullptr;
    int crop_top = 0, crop_left = 0, out_H = 0, out_W = 0;          // NCHW output window (tail)
};

int conv_direct(DirectKind kind, const DirectArgs &a, cudaStream_t st);
// conv_direct with the kernel family chosen by the caller (ffma: the fp32 FFMA kernels even where an mma variant exists)
int conv_direct_choice(DirectKind kind, const DirectArgs &a, bool ffma, cudaStream_t st);
// mma_conv.cu: the same layers on mma.sync tensor cores; ESR_EINVAL = this kind has no mma variant (use the FFMA kernel)
int conv_mma(DirectKind kind, const DirectArgs &a, cudaStream_t st);
int pack_direct_weight(const float *w, int cout, int cin, float *dst, cudaStream_t st);
// fp32 [Cout,Cin,3,3] -> the shared-memory image the mma kernels copy: split bf16 [plane][tap][co (padded to >= 8)][ci + 8 pad]
size_t mma_weight_bytes(int cout, int cin);
int pack_mma_weight(const float *w, int cout, int cin, void *dst, cudaStream_t st);
int pack_mma_weight_dx(const float *w, int layer_cout, int layer_cin, void *dst, cudaStream_t st);
int conv_mma_nchw(const float *x, const void *w_img, const float *bias, int B, int Cin, int H, int W, int Cout, int stride, int act,
                  float *y, cudaStream_t st);

// ---- element-wise / reduction kernels (elementwise.cu)
// local_fusion input: out[img=(b,i)] = cat(f[i0]*map[p0], f[i1], f[i2]*map[p1])  (models/model.py:82-86)
int ltc_cat(const SplitTensor &f, const float *maps, const int *idx /*[n_img][5]: f0,f1,f2,map0,map1*/, int n_img,
            const SplitTensor &out /*C=192*/, cudaStream_t st);
// per-image channel max of a 64-channel split tensor -> [n_img, 64] fp32   (models/model.py:221)
int chan_max(const SplitTensor &t, int n_img, float *out, cudaStream_t st);
// channel attention MLP 64 -> 32 relu -> 128 sigmoid (models/submodules.py:67-77, model.py:186-189)
int attn_mlp(const float *mx, int n_img, const float *w0, const float *b0, const float *w1, const float *b1, float *ck,
             cudaStream_t st);
// y = cat(aligned * sk[...,0] * ck[:64], mid * sk[...,1] * ck[64:])   (models/model.py:224-227)
int attn_apply(const SplitTensor &aligned, const SplitTensor &mid_src, const int *mid_img, const float *sk, const float *ck,
               int n_img, const SplitTensor &out /*C=128*/, cudaStream_t st);
// out[b] = x[b] + mean_n(feats[f] * att[f]), f = fidx[b*N+n] (or b*N+n)     (models/model.py:259-267)
int scale_aggregate(const SplitTensor &x, const SplitTensor &feats, const float *att, const int *fidx, int B, int N,
                    const SplitTensor &out, cudaStream_t st);
// bilinear x2 (align_corners=False) of a split tensor (models/submodules.py:290)
int upsample2x(const SplitTensor &src, int n_img, const SplitTensor &dst, cudaStream_t st);
int copy_split(const SplitTensor &src, const int *src_img, int n_img, const SplitTensor &dst, cudaStream_t st);
// Cout = 1 / 2 convolutions (3x3 or 1x1, sigmoid) of a 64-channel split tensor on CUDA cores: fp32 NHWC out [n_img, H, W, cout]
int conv_narrow(const SplitTensor &x, const int *src_img, const float *w, const float *bias, int cout, int ntaps, int n_img, float *out,
                cudaStream_t st);
int pack_narrow_weight(const float *w, int cout, int ntaps, float *dst, cudaStream_t st);

// ---- deformable sampling (dcn.cu): columns[img][y][x][tap*64 + c] = bilinear(feat[c], y-1+i+off_h, x-1+j+off_w) * mask
// om: fp32 NHWC [n_img, H, W, 216] = {144 offsets (group-major, (h,w) pairs per tap), 72 masks (already sigmoid)}
int dcn_columns(const SplitTensor &feat, const int *feat_img, const float *om, int n_img, const SplitTensor &cols /*C=576*/,
                cudaStream_t st);

// ---- DCNv2 with the sampling fused into the wgmma contraction (dcn_fused.cu): no columns tensor in HBM
int dcn_fused_prepare(const SplitTensor &feat, const int *feat_img, const float *om, const void *wpacked, const float *bias,
                      int n_img, int act, const SplitTensor &out, void **plan_out);
int dcn_fused_launch(void *plan, cudaStream_t st);
void dcn_fused_destroy(void *plan);

// ---- the operators for any other configuration (dcn_generic.cu): fp32 CUDA-core kernels, reference NCHW layouts
size_t dcn_generic_ws_bytes(int B, int C, int H, int W, int Co, int kernel, int stride, int pad, int dil, int G, int backward);
int dcn_generic_forward(const float *input, const float *weight, const float *bias, const float *offset, const float *mask, int B,
                        int C, int H, int W, int Co, int kernel, int stride, int pad, int dil, int G, float *output,
                        void *workspace, size_t ws_bytes, cudaStream_t st);
int dcn_generic_backward(const float *input, const float *weight, const float *offset, const float *mask, const float *grad_output,
                         int B, int C, int H, int W, int Co, int kernel, int stride, int pad, int dil, int G, float *grad_input,
                         float *grad_offset, float *grad_mask, float *grad_weight, float *grad_bias, void *workspace,
                         size_t ws_bytes, cudaStream_t st);
static inline bool dcn_is_tuned(int C, int Co, int kernel, int stride, int pad, int dil, int G)
{
    return C == 64 && Co == 64 && kernel == 3 && stride == 1 && pad == 1 && dil == 1 && G == 8;   // models/model.py:173
}

// out[i] = part[0][i] + part[1][i] + ... + part[slices-1][i] (part = [slices][n]), added in slot order: the second pass of
// the deterministic reductions (train_ops.cu)
int sum_slices(const float *part, int slices, size_t n, float *out, cudaStream_t st);

// offset [B,144,HW] + mask [B,72,HW] (reference NCHW) -> om [B*HW, 216]
int om_from_nchw(const float *offset, const float *mask, int B, int HW, float *om, cudaStream_t st);

} // namespace esr
