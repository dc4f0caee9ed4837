// tc_conv.cuh -- interface of the wgmma implicit-GEMM convolution (see tc_conv.cu).
#pragma once
#include "common.cuh"
#include <cuda.h>   // CUtensorMap (types only; the driver entry point is resolved at run time)
#include <vector>

namespace esr {
enum Act : int { ACT_NONE = 0, ACT_RELU = 1, ACT_SIGMOID = 2, ACT_TANH = 3 };
enum EpiMode : int { EPI_STD = 0, EPI_GRU_ZR = 1, EPI_GRU_OUT = 2 };
enum ResMode : int { RES_NONE = 0, RES_PRE_ACT = 1, RES_POST_ACT = 2 };

// A "split" activation tensor: [2 planes][n_img][H][W][C] bf16, value = hi + lo.
struct SplitTensor {
    __nv_bfloat16 *base = nullptr;
    int n_img = 0, H = 0, W = 0, C = 0;
    size_t plane_override = 0;      // set on views into a larger tensor (distance between the hi and lo planes)
    size_t plane() const { return plane_override ? plane_override : (size_t)n_img * H * W * C; }
    size_t bytes() const { return plane() * 2 * sizeof(__nv_bfloat16); }
};

constexpr int TC_MAX_SRC = 3;

// Everything one launch needs.  Passed to the kernel by value (__grid_constant__).
struct ConvTCArgs {
    CUtensorMap amap[TC_MAX_SRC];   // 5-D maps over the source split tensors (C, W, H, img, plane), box (64, TW, tc_box_h, 1, 1)
    CUtensorMap bmap;               // 3-D map over packed weights (64, npad, 2*nkb), box (64, npad, 1)
    const int *src_img[TC_MAX_SRC]; // output image -> source image (nullptr = identity)
    int chunk_end[TC_MAX_SRC];      // cumulative number of 64-channel chunks after source s
    int n_src, ntaps, nkb, npad, cout;
    int H, W, TW, TH, tiles_x, tiles_y, n_img;
    int a_stages, b_stages;         // ring depths: A boxes (one per chunk and dx), B slots (one per tap)
    // epilogue
    const float *bias;              // [npad]
    int act, act_from, res_mode, epi_mode;
    const __nv_bfloat16 *res; size_t res_plane; int res_C; const int *res_img;
    __nv_bfloat16 *out; size_t out_plane; int out_C, out_coff;   // split output (may be null)
    float *out_f32; int out_f32_C;                                // fp32 NHWC output (may be null)
    int out_f32_nchw;                                             // 1: out_f32 is NCHW [n_img][out_f32_C][H][W] instead
    // GRU extras
    const __nv_bfloat16 *h_prev; size_t h_plane;                  // [*,H,W,64] split
    float *z_buf;                                                 // [n_img,H,W,64] fp32 (ZR writes, OUT reads)
    // 0: chunk c of source s is channels 64 (c - chunk base); k != 0: channels 0-63 of image src_img + (c - chunk base) * k.
    // Last, so that the offsets of the fields above (and the register allocation of every k_conv_tc instantiation) do not move.
    int chunk_img_step[TC_MAX_SRC];
};

static_assert(sizeof(ConvTCArgs) <= 1024, "ConvTCArgs: keep the kernel argument block within 1 KB");

// Host-side description used to build ConvTCArgs.
struct ConvTCDesc {
    SplitTensor src[TC_MAX_SRC];
    const int *src_img[TC_MAX_SRC] = {nullptr, nullptr, nullptr};
    // A source with chunk_img_step[s] = k != 0 is a 64-channel tensor that contributes src_chunks[s] chunks: chunk j reads image
    // src_img[s][img] + j * k.  This concatenates images of one tensor along channels without materialising the concatenation
    // (dense_fusion's N-1 aligned neighbours, stored k-major).  The caller keeps the last image inside the tensor.
    int src_chunks[TC_MAX_SRC] = {0, 0, 0};
    int chunk_img_step[TC_MAX_SRC] = {0, 0, 0};
    int n_src = 1;
    int ntaps = 9;                  // 9 (3x3, pad 1), 1 (1x1) or 25 (5x5, pad 2; npad 192 only)
    int cout = 64;
    const void *wpacked = nullptr;  // packed by pack_conv_weight: [2][nkb][npad][64] bf16
    const float *bias = nullptr;    // [npad] fp32, zero padded
    int n_img = 0;                  // number of output images
    int act = ACT_NONE, act_from = 0, res_mode = RES_NONE, epi_mode = EPI_STD;
    SplitTensor res; const int *res_img = nullptr;
    SplitTensor out; int out_coff = 0;
    float *out_f32 = nullptr; int out_f32_C = 0; int out_f32_nchw = 0;
    SplitTensor h_prev; float *z_buf = nullptr;
};

static inline int tc_npad(int cout) { return (cout + 15) / 16 * 16; }
// Rows of one A box: a 3x3 layer's box has the tile's TH rows plus a halo row above and below, so that its three dy taps
// read it at row offsets 0, TW and 2 TW; a 1x1 layer's box is the tile.
__host__ __device__ inline int tc_box_h(int TH, int ntaps) { return ntaps == 9 ? TH + 2 : TH; }
// bytes of one A box, both planes (64 channels = 128 bytes per pixel and plane)
__host__ __device__ inline uint32_t tc_a_box_bytes(int TW, int TH, int ntaps) { return 2u * 128u * (uint32_t)(TW * tc_box_h(TH, ntaps)); }
// A 5x5 layer (ntaps 25, LPIPS's conv2) has two halo rows above and below; the kernel knows it at compile time, so the
// 3x3 / 1x1 helpers above stay as they are and the host sizes every kind through these two.
__host__ __device__ inline uint32_t tc_a_box_bytes5(int TW, int TH) { return 2u * 128u * (uint32_t)(TW * (TH + 4)); }
static inline int tc_conv_box_h(int TH, int ntaps) { return ntaps == 25 ? TH + 4 : tc_box_h(TH, ntaps); }
static inline uint32_t tc_conv_a_box(int TW, int TH, int ntaps) { return ntaps == 25 ? tc_a_box_bytes5(TW, TH) : tc_a_box_bytes(TW, TH, ntaps); }
static inline int tc_nkb(int cin_total, int ntaps) { return cin_total / 64 * ntaps; }
static inline size_t tc_packed_weight_bytes(int cout, int cin_total, int ntaps)
{
    return (size_t)2 * tc_nkb(cin_total, ntaps) * tc_npad(cout) * 64 * sizeof(__nv_bfloat16);
}

// Builds tensor maps + launch geometry.  H, W taken from src[0].
int conv_tc_prepare(const ConvTCDesc &d, ConvTCArgs *args);
int conv_tc_launch(const ConvTCArgs &args, cudaStream_t st);
// the ConvGRU recurrence as one cooperative launch over the prepared gate layers of every step (EPI_GRU_ZR / EPI_GRU_OUT)
int gru_chain_prepare(const std::vector<ConvTCArgs> &zr, const std::vector<ConvTCArgs> &go, void **plan_out);
int gru_chain_launch(void *plan, cudaStream_t st);
void gru_chain_destroy(void *plan);
// tensor-map builders (shared with dcn_fused.cu, wgrad_tc.cu)
int tc_make_amap(const SplitTensor &t, int box_w, int box_h, CUtensorMap *out);
int tc_make_bmap(const void *w, int npad, int nkb, int box_rows, CUtensorMap *out);

// w: fp32 [cout, cin, k, k] (device) -> packed split bf16 [2][nkb][npad][64]; kb = chunk*ntaps + tap
int pack_conv_weight(const float *w, int cout, int cin, int ksz, void *dst, cudaStream_t st);
// concatenates two [cout_i, cin, k, k] weights along cout before packing (GRU update|reset gates)
int pack_conv_weight2(const float *w0, const float *w1, int cout_each, int cin, int ksz, void *dst, cudaStream_t st);

// NCHW fp32 <-> split NHWC
int split_from_nchw(const float *src, int n_img, int C, int H, int W, __nv_bfloat16 *dst, cudaStream_t st);
int split_to_nchw(const __nv_bfloat16 *src, int n_img, int C, int H, int W, float *dst, cudaStream_t st);
// same, with an explicit hi->lo plane distance (views into a larger split tensor)
int split_from_nchw_planes(const float *src, int n_img, int C, int H, int W, __nv_bfloat16 *dst, size_t plane, cudaStream_t st);
int split_to_nchw_planes(const __nv_bfloat16 *src, size_t plane, int n_img, int C, int H, int W, float *dst, cudaStream_t st);

} // namespace esr
