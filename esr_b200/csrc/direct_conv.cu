// direct_conv.cu -- CUDA-core 3x3 convolutions for the small-channel, full-resolution layers (Cin <= 64 and
// Cout <= 64 with too few channels to fill a tensor-core tile; HBM / FFMA bound):
//   head 2->8 (models/model.py:301,330), encoder 8->16->32->64 stride 2 (models/model.py:20-45),
//   attention maps C->1 sigmoid (models/model.py:195-199,262), decoder bilinear x2 + conv (models/submodules.py:254-299),
//   tail 8->2 (models/model.py:309,337).
// One block = a 16x16 / 32x16 / 32x32 output tile (wider for narrower layers), all output channels.
//   stage 1: the input patch (+halo) is staged in shared memory as [ci][py][px] fp32 -- 16-byte loads of 8 channels of
//            the split-bf16 NHWC source per thread (the bilinear x2 upsampling of the decoder is applied on the fly);
//   stage 2: register tiling -- a thread owns a 2x2 pixel patch x COUT/4 channels (its 4x4 / 5x5 input window is read
//            once per input channel and reused over the 9 taps; weights are warp-uniform LDS.128 broadcasts);
//            layers with COUT < 8 use one pixel x all channels per thread;
//   stage 3: 16-byte split-bf16 stores.
// fp32 math throughout.
#include "net.cuh"
#include "direct_common.cuh"

namespace esr {

// Output tile geometry.  Tiled layers: a thread owns TPW x 2 pixels x C channels, C = 16 (COUT=64) or 8; the COUT/C
// channel groups are spread over warps, so narrower layers get wider tiles (more pixels per block, 16-byte stores
// everywhere).  TPW = 4 (more weight reuse per thread) is implemented; every layer currently uses TPW = 2 (more resident
// blocks per SM).
template <int COUT, int TPW> struct DcGeom {
    static constexpr bool TILED = COUT >= 8;
    static constexpr int C = COUT >= 64 ? 16 : (COUT >= 8 ? 8 : COUT);
    static constexpr int CG = TILED ? COUT / C : 1;
    static constexpr int PG = 256 / CG;                         // pixel groups (threads per channel group)
    static constexpr int GW = PG == 64 ? 8 : 16;                // pixel groups along x
    static constexpr int GH = PG / GW;
    static constexpr int TW = TILED ? GW * TPW : 16;            // output tile width
    static constexpr int TH = TILED ? GH * 2 : 16;              // output tile height
};

template <int CIN, int COUT, int STRIDE, bool UPS, int INF, int OUTF, int TPW>
__global__ void __launch_bounds__(256) k_conv_direct(const DirectArgs a)
{
    using G = DcGeom<COUT, TPW>;
    constexpr int PW = (G::TW - 1) * STRIDE + 3;          // patch width actually needed
    constexpr int PH = (G::TH - 1) * STRIDE + 3;          // patch height
    constexpr int PP = (PW + 3) / 4 * 4;                  // row pitch (floats)
    constexpr bool TILED = G::TILED;
    extern __shared__ float dsm[];
    float *patch = dsm;                                   // [CIN][PH][PP]
    float *wsm = dsm + CIN * PH * PP;                     // [9][CIN][COUT]
    float *bsm = wsm + 9 * CIN * COUT;                    // [COUT]
    constexpr int IPP = (PW + 2 + 3) / 4 * 4;             // fused head: input patch pitch
    float *inp = bsm + ((COUT + 3) / 4 * 4);              // fused head: [2][PH+2][IPP] input patch, then [9][2][8] + [8]
    float *w0s = inp + 2 * (PH + 2) * IPP;

    const int img = blockIdx.z;
    const int oy0 = blockIdx.y * G::TH, ox0 = blockIdx.x * G::TW;
    const int tid = threadIdx.x;

    for (int i = tid; i < 9 * CIN * COUT / 4; i += 256)
        reinterpret_cast<float4 *>(wsm)[i] = reinterpret_cast<const float4 *>(a.w)[i];
    if (tid < COUT) bsm[tid] = a.bias[tid];

    // ---- stage 1: input patch.  Conv input coordinates (after padding / upsampling): [0,Hc) x [0,Wc)
    const int Hc = UPS ? 2 * a.Hin : a.Hin + a.pad_top + a.pad_bottom;
    const int Wc = UPS ? 2 * a.Win : a.Win + a.pad_left + a.pad_right;
    const int iy0 = oy0 * STRIDE - 1, ix0 = ox0 * STRIDE - 1;
    const int simg = a.in_img ? a.in_img[img] : img;
    if constexpr (INF == FMT_HEAD_FUSED) {
        // head (2 -> 8, relu; models/model.py:301,330) evaluated on the fly for the (PH x PW) patch this tile needs:
        // the full-resolution 8-channel tensor (the largest activation of the network) never goes to HBM.
        static_assert(INF != FMT_HEAD_FUSED || CIN == 8, "fused head feeds the 8-channel encoder layer");
        for (int i = tid; i < 9 * 2 * 8 + 8; i += 256) w0s[i] = i < 144 ? a.w0[i] : a.b0[i - 144];
        for (int i = tid; i < 2 * (PH + 2) * (PW + 2); i += 256) {
            const int px = i % (PW + 2), py = (i / (PW + 2)) % (PH + 2), ci = i / ((PW + 2) * (PH + 2));
            const int y = iy0 - 1 + py, x = ix0 - 1 + px;                 // head-input coordinates (padded frame)
            float v = 0.0f;
            const int sy = y - a.pad_top, sx = x - a.pad_left;           // CropSize zero padding (model_util.py:148-152)
            if (sy >= 0 && sy < a.Hin && sx >= 0 && sx < a.Win)
                v = a.in_f32[(((size_t)simg * 2 + ci) * a.Hin + sy) * a.Win + sx];
            inp[(ci * (PH + 2) + py) * IPP + px] = v;
        }
        __syncthreads();
        for (int i = tid; i < PH * PW; i += 256) {
            const int px = i % PW, py = i / PW;
            const int y = iy0 + py, x = ix0 + px;
            float o[8];
            const bool inside = (y >= 0 && y < Hc && x >= 0 && x < Wc);   // outside = the encoder conv's zero padding
#pragma unroll
            for (int c = 0; c < 8; ++c) o[c] = w0s[144 + c];
#pragma unroll
            for (int ci = 0; ci < 2; ++ci)
#pragma unroll
                for (int ky = 0; ky < 3; ++ky)
#pragma unroll
                    for (int kx = 0; kx < 3; ++kx) {
                        const float xv = inp[(ci * (PH + 2) + py + ky) * IPP + px + kx];
                        const float *wp = w0s + ((ky * 3 + kx) * 2 + ci) * 8;
#pragma unroll
                        for (int c = 0; c < 8; ++c) o[c] = fmaf(xv, wp[c], o[c]);
                    }
#pragma unroll
            for (int c = 0; c < 8; ++c) patch[(c * PH + py) * PP + px] = inside ? fmaxf(o[c], 0.0f) : 0.0f;
        }
    } else if constexpr (INF == FMT_NCHW_F32) {
        for (int i = tid; i < CIN * PW * PH; i += 256) {
            const int px = i % PW, py = (i / PW) % PH, ci = i / (PW * PH);
            const int y = iy0 + py, x = ix0 + px;
            float v = 0.0f;
            if (y >= 0 && y < Hc && x >= 0 && x < Wc) {
                const int sy = y - a.pad_top, sx = x - a.pad_left;      // CropSize zero padding (model_util.py:148-152)
                if (sy >= 0 && sy < a.Hin && sx >= 0 && sx < a.Win)
                    v = a.in_f32[(((size_t)simg * CIN + ci) * a.Hin + sy) * a.Win + sx];
            }
            patch[(ci * PH + py) * PP + px] = v;
        }
    } else {
        static_assert(INF != FMT_SPLIT || CIN % 8 == 0, "split input needs CIN % 8 == 0");
        const __nv_bfloat16 *hi = a.in_split;
        const size_t plane = a.in_plane;
        constexpr int Q = CIN / 8;
        for (int i = tid; i < Q * PW * PH; i += 256) {
            const int pp = i % (PW * PH), q = i / (PW * PH);            // lanes <-> pixels: conflict-free smem writes
            const int px = pp % PW, py = pp / PW;
            const int y = iy0 + py, x = ix0 + px;
            float v[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) v[e] = 0.0f;
            if (y >= 0 && y < Hc && x >= 0 && x < Wc) {
                if constexpr (!UPS) {
                    dc_ld8(hi + (((size_t)simg * a.Hin + y) * a.Win + x) * CIN + q * 8, plane, v);
                } else {
                    // F.interpolate(scale_factor=2, mode='bilinear', align_corners=False) (submodules.py:290):
                    // src = max(0, (dst + 0.5) * 0.5 - 0.5); neighbours clamped to the image
                    const float fy = fmaxf(0.0f, ((float)y + 0.5f) * 0.5f - 0.5f);
                    const float fx = fmaxf(0.0f, ((float)x + 0.5f) * 0.5f - 0.5f);
                    const int y_0 = (int)fy, x_0 = (int)fx;
                    const int y_1 = min(y_0 + 1, a.Hin - 1), x_1 = min(x_0 + 1, a.Win - 1);
                    const float ly = fy - (float)y_0, lx = fx - (float)x_0;
                    const size_t b0 = ((size_t)simg * a.Hin + y_0) * a.Win, b1 = ((size_t)simg * a.Hin + y_1) * a.Win;
                    float v00[8], v01[8], v10[8], v11[8];
                    dc_ld8(hi + (b0 + x_0) * CIN + q * 8, plane, v00);
                    dc_ld8(hi + (b0 + x_1) * CIN + q * 8, plane, v01);
                    dc_ld8(hi + (b1 + x_0) * CIN + q * 8, plane, v10);
                    dc_ld8(hi + (b1 + x_1) * CIN + q * 8, plane, v11);
#pragma unroll
                    for (int e = 0; e < 8; ++e)   // ATen: h0*(w0*v00 + w1*v01) + h1*(w0*v10 + w1*v11)
                        v[e] = (1.0f - ly) * ((1.0f - lx) * v00[e] + lx * v01[e]) + ly * ((1.0f - lx) * v10[e] + lx * v11[e]);
                }
            }
#pragma unroll
            for (int e = 0; e < 8; ++e) patch[((q * 8 + e) * PH + py) * PP + px] = v[e];
        }
    }
    __syncthreads();

    if constexpr (TILED) {
        // ---- stage 2 (tiled): thread = (cout group cg, pixel group pg): TPW x 2 pixels x C channels
        constexpr int C = G::C;
        constexpr int NP = TPW * 2;                       // pixels per thread
        constexpr int WINW = (TPW - 1) * STRIDE + 3;      // input window of the thread's pixel patch
        constexpr int WINH = STRIDE + 3;
        const int cg = tid / G::PG, pg = tid % G::PG;     // cg is warp-uniform -> weight reads are broadcasts
        const int gy = pg / G::GW, gx = pg % G::GW;
        float acc[NP][C];
#pragma unroll
        for (int p = 0; p < NP; ++p)
#pragma unroll
            for (int c = 0; c < C; ++c) acc[p][c] = bsm[cg * C + c];
#pragma unroll 1
        for (int ci = 0; ci < CIN; ++ci) {
            float win[WINH][WINW];
            const float *pb = patch + (ci * PH + gy * 2 * STRIDE) * PP + gx * TPW * STRIDE;
            // the window starts at an even float offset (PP % 4 == 0, gx * TPW * STRIDE even): 8-byte shared loads
#pragma unroll
            for (int r = 0; r < WINH; ++r) {
#pragma unroll
                for (int s2 = 0; s2 + 1 < WINW; s2 += 2) {
                    const float2 t = *reinterpret_cast<const float2 *>(pb + r * PP + s2);
                    win[r][s2] = t.x; win[r][s2 + 1] = t.y;
                }
                if (WINW & 1) win[r][WINW - 1] = pb[r * PP + WINW - 1];
            }
#pragma unroll
            for (int ky = 0; ky < 3; ++ky)
#pragma unroll
                for (int kx = 0; kx < 3; ++kx) {
                    const float *wp = wsm + ((ky * 3 + kx) * CIN + ci) * COUT + cg * C;
                    float wv[C];
#pragma unroll
                    for (int c4 = 0; c4 < C / 4; ++c4) {                 // warp-uniform 16-byte broadcast loads
                        const float4 t = reinterpret_cast<const float4 *>(wp)[c4];
                        wv[4 * c4] = t.x; wv[4 * c4 + 1] = t.y; wv[4 * c4 + 2] = t.z; wv[4 * c4 + 3] = t.w;
                    }
#pragma unroll
                    for (int p = 0; p < NP; ++p) {
                        const float xv = win[(p / TPW) * STRIDE + ky][(p % TPW) * STRIDE + kx];
#pragma unroll
                        for (int c = 0; c < C; ++c) acc[p][c] = fmaf(xv, wv[c], acc[p][c]);
                    }
                }
        }
        // ---- stage 3
#pragma unroll
        for (int p = 0; p < NP; ++p) {
            const int oy = oy0 + gy * 2 + p / TPW, ox = ox0 + gx * TPW + p % TPW;
            if (oy >= a.Hout || ox >= a.Wout) continue;
            float v[C];
#pragma unroll
            for (int c = 0; c < C; ++c) v[c] = dc_act(acc[p][c], a.act);
            static_assert(OUTF == FMT_SPLIT, "tiled path writes split tensors");
            __nv_bfloat16 *dst = a.out_split + (((size_t)img * a.Hout + oy) * a.Wout + ox) * COUT + cg * C;
#pragma unroll
            for (int c8 = 0; c8 < C / 8; ++c8) dc_store<8>(dst + c8 * 8, a.out_plane, v + c8 * 8);
        }
    } else {
        // ---- stage 2 (narrow): one pixel x all COUT (1 or 2) per thread
        const int ty = tid / G::TW, tx = tid % G::TW;
        const int oy = oy0 + ty, ox = ox0 + tx;
        float acc[COUT];
#pragma unroll
        for (int co = 0; co < COUT; ++co) acc[co] = bsm[co];
#pragma unroll 4
        for (int ci = 0; ci < CIN; ++ci) {
#pragma unroll
            for (int ky = 0; ky < 3; ++ky)
#pragma unroll
                for (int kx = 0; kx < 3; ++kx) {
                    const float xv = patch[(ci * PH + ty * STRIDE + ky) * PP + tx * STRIDE + kx];
                    const float *wp = wsm + ((ky * 3 + kx) * CIN + ci) * COUT;
#pragma unroll
                    for (int co = 0; co < COUT; ++co) acc[co] = fmaf(xv, wp[co], acc[co]);
                }
        }
        if (oy >= a.Hout || ox >= a.Wout) return;
#pragma unroll
        for (int co = 0; co < COUT; ++co) acc[co] = dc_act(acc[co], a.act);
        if constexpr (OUTF == FMT_NHWC_F32) {
            const size_t o = (((size_t)img * a.Hout + oy) * a.Wout + ox) * COUT;
#pragma unroll
            for (int co = 0; co < COUT; ++co) a.out_f32[o + co] = acc[co];
        } else {
            // NCHW fp32 with the CropSize crop (model_util.py:154-164): only pixels inside the crop window are stored
            const int cy = oy - a.crop_top, cx = ox - a.crop_left;
            if (cy >= 0 && cy < a.out_H && cx >= 0 && cx < a.out_W) {
#pragma unroll
                for (int co = 0; co < COUT; ++co) a.out_f32[(((size_t)img * COUT + co) * a.out_H + cy) * a.out_W + cx] = acc[co];
            }
        }
    }
}

template <int CIN, int COUT, int STRIDE, bool UPS, int INF, int OUTF, int TPW = 2>
static int launch_direct(const DirectArgs &a, cudaStream_t st)
{
    using G = DcGeom<COUT, TPW>;
    constexpr int PW = (G::TW - 1) * STRIDE + 3;
    constexpr int PH = (G::TH - 1) * STRIDE + 3;
    constexpr int PP = (PW + 3) / 4 * 4;
    constexpr int IPP = (PW + 2 + 3) / 4 * 4;
    constexpr size_t extra = INF == FMT_HEAD_FUSED ? (size_t)(2 * (PH + 2) * IPP + 9 * 2 * 8 + 8) : 0;
    constexpr size_t smem = sizeof(float) * ((size_t)(CIN * PH * PP + 9 * CIN * COUT + (COUT + 3) / 4 * 4) + extra);
    static_assert(smem <= 227 * 1024, "direct conv tile does not fit in shared memory");
    static bool attr_set = false;
    if (!attr_set) {
        ESR_CUDA_CHECK(cudaFuncSetAttribute(k_conv_direct<CIN, COUT, STRIDE, UPS, INF, OUTF, TPW>,
                                            cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr_set = true;
    }
    dim3 grid((a.Wout + G::TW - 1) / G::TW, (a.Hout + G::TH - 1) / G::TH, a.n_img);
    k_conv_direct<CIN, COUT, STRIDE, UPS, INF, OUTF, TPW><<<grid, 256, smem, st>>>(a);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}

int conv_direct(DirectKind kind, const DirectArgs &a, cudaStream_t st)
{
    // default: warp-level tensor-core variant (mma_conv.cu) where one exists; ESR_DIRECT_FFMA=1 keeps the fp32 FFMA kernels
    static const bool ffma = getenv("ESR_DIRECT_FFMA") != nullptr;
    return conv_direct_choice(kind, a, ffma, st);
}

int conv_direct_choice(DirectKind kind, const DirectArgs &a, bool ffma, cudaStream_t st)
{
    if (!ffma) {
        const int rc = conv_mma(kind, a, st);
        if (rc != ESR_EINVAL) return rc;
    }
    switch (kind) {
    case DK_HEAD:    return launch_direct<2, 8, 1, false, FMT_NCHW_F32, FMT_SPLIT>(a, st);
    case DK_HEAD_ENC0: return launch_direct<8, 16, 2, false, FMT_HEAD_FUSED, FMT_SPLIT>(a, st);
    case DK_ENC0:    return launch_direct<8, 16, 2, false, FMT_SPLIT, FMT_SPLIT>(a, st);
    case DK_ENC1:    return launch_direct<16, 32, 2, false, FMT_SPLIT, FMT_SPLIT>(a, st);
    case DK_ENC2:    return launch_direct<32, 64, 2, false, FMT_SPLIT, FMT_SPLIT>(a, st);
    case DK_ATT32:   return launch_direct<32, 1, 1, false, FMT_SPLIT, FMT_NHWC_F32>(a, st);
    case DK_ATT16:   return launch_direct<16, 1, 1, false, FMT_SPLIT, FMT_NHWC_F32>(a, st);
    case DK_RECON0:  return launch_direct<64, 32, 1, true, FMT_SPLIT, FMT_SPLIT>(a, st);
    case DK_RECON1:  return launch_direct<32, 16, 1, true, FMT_SPLIT, FMT_SPLIT>(a, st);
    case DK_RECON2:  return launch_direct<16, 8, 1, true, FMT_SPLIT, FMT_SPLIT>(a, st);
    case DK_TAIL:    return launch_direct<8, 2, 1, false, FMT_SPLIT, FMT_NCHW_F32>(a, st);
    }
    set_error("conv_direct: unknown kind %d", (int)kind);
    return ESR_EINVAL;
}

// fp32 [Cout, Cin, 3, 3] -> [tap][ci][co]
__global__ void k_pack_direct_weight(const float *__restrict__ w, int cout, int cin, float *__restrict__ dst)
{
    const int total = 9 * cin * cout;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int co = i % cout, ci = (i / cout) % cin, tap = i / (cout * cin);
        dst[i] = w[((size_t)co * cin + ci) * 9 + tap];
    }
}
int pack_direct_weight(const float *w, int cout, int cin, float *dst, cudaStream_t st)
{
    k_pack_direct_weight<<<(9 * cin * cout + 255) / 256, 256, 0, st>>>(w, cout, cin, dst);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}

// ---- esr_conv_small: one launch of the plan's small-channel / narrow-output layers, kernel family chosen per call
namespace {
struct SmallKind {
    int cin, cout, ntaps, stride;
    bool ups;
    int dk;        // DirectKind of paths 0 and 1 (-1: narrow only)
    int paths;     // bit p: path p runs this kind in the plan
};
// indexed by ESR_CONV_SMALL_*; 8 and 9 are unassigned (no path runs them)
const SmallKind SMALL_KINDS[] = {
    {8, 16, 9, 2, false, DK_HEAD_ENC0, 3}, {16, 32, 9, 2, false, DK_ENC1, 3}, {32, 64, 9, 2, false, DK_ENC2, 3},
    {32, 1, 9, 1, false, DK_ATT32, 3},     {16, 1, 9, 1, false, DK_ATT16, 3}, {32, 16, 9, 1, true, DK_RECON1, 3},
    {16, 8, 9, 1, true, DK_RECON2, 3},     {8, 2, 9, 1, false, DK_TAIL, 3},   {},
    {},                                    {64, 2, 1, 1, false, -1, 4},
};
constexpr int N_SMALL_KINDS = (int)(sizeof(SMALL_KINDS) / sizeof(SMALL_KINDS[0]));
bool small_ok(int kind, int path) { return kind >= 0 && kind < N_SMALL_KINDS && path >= 0 && path <= 2 && (SMALL_KINDS[kind].paths >> path & 1); }
size_t align256(size_t b) { return (b + 255) / 256 * 256; }
// the packed weights of the kind's layer (path 0: pack_mma_weight; otherwise fp32 [tap][ci][co], as pack_direct_weight and
// pack_narrow_weight write it), then for HEAD_ENC0 the head's [9][2][8]
size_t small_w_bytes(const SmallKind &k, int path)
{
    return path == 0 ? mma_weight_bytes(k.cout, k.cin) : sizeof(float) * k.ntaps * k.cin * k.cout;
}
} // namespace

} // namespace esr

using namespace esr;

extern "C" size_t esr_conv_small_workspace_bytes(int kind, int path)
{
    if (!small_ok(kind, path)) return 0;
    return align256(small_w_bytes(SMALL_KINDS[kind], path)) + (kind == ESR_CONV_SMALL_HEAD_ENC0 ? align256(sizeof(float) * 9 * 2 * 8) : 0);
}

extern "C" int esr_conv_small(const esr_conv_small_desc *d, esr_stream_t stream)
{
    ESR_REQUIRE(d, "esr_conv_small: null descriptor");
    if (!small_ok(d->kind, d->path)) {
        set_error("esr_conv_small: kind %d has no path %d in the network", d->kind, d->path);
        return ESR_EUNSUPPORTED;
    }
    const SmallKind &k = SMALL_KINDS[d->kind];
    const bool head = d->kind == ESR_CONV_SMALL_HEAD_ENC0, tail = d->kind == ESR_CONV_SMALL_TAIL;
    const bool split_out = k.cout >= 8;
    ESR_REQUIRE(d->n_img > 0 && d->H_in > 0 && d->W_in > 0, "esr_conv_small: n_img=%d H_in=%d W_in=%d", d->n_img, d->H_in, d->W_in);
    ESR_REQUIRE(d->workspace && d->workspace_bytes >= esr_conv_small_workspace_bytes(d->kind, d->path), "esr_conv_small: workspace");
    ESR_REQUIRE(d->w && d->bias && (head ? d->in_f32 && d->w_head && d->b_head : d->in && d->in_n_img > 0),
                "esr_conv_small: missing input or weights");
    ESR_REQUIRE(split_out ? d->out && d->out_n_img >= d->n_img : d->out_f32 != nullptr, "esr_conv_small: missing output");
    ESR_REQUIRE(head || (d->pad_top | d->pad_bottom | d->pad_left | d->pad_right) == 0, "esr_conv_small: pads are HEAD_ENC0's");
    ESR_REQUIRE(d->pad_top >= 0 && d->pad_bottom >= 0 && d->pad_left >= 0 && d->pad_right >= 0, "esr_conv_small: negative pad");
    const int Hc = d->H_in + d->pad_top + d->pad_bottom, Wc = d->W_in + d->pad_left + d->pad_right;
    const int Hout = k.ups ? 2 * Hc : (k.stride == 2 ? (Hc - 1) / 2 + 1 : Hc);
    const int Wout = k.ups ? 2 * Wc : (k.stride == 2 ? (Wc - 1) / 2 + 1 : Wc);
    ESR_REQUIRE(!tail || (d->crop_top >= 0 && d->crop_left >= 0 && d->out_H > 0 && d->out_W > 0 && d->crop_top + d->out_H <= Hout &&
                          d->crop_left + d->out_W <= Wout),
                "esr_conv_small: crop window (%d, %d) %d x %d outside %d x %d", d->crop_top, d->crop_left, d->out_H, d->out_W, Hout, Wout);

    cudaStream_t st = (cudaStream_t)stream;
    uint8_t *ws = (uint8_t *)d->workspace;
    int rc;
    if (d->path == 0) rc = pack_mma_weight(d->w, k.cout, k.cin, ws, st);
    else if (k.cin == 64) rc = pack_narrow_weight(d->w, k.cout, k.ntaps, (float *)ws, st);
    else rc = pack_direct_weight(d->w, k.cout, k.cin, (float *)ws, st);
    if (rc) return rc;
    float *w_head = (float *)(ws + align256(small_w_bytes(k, d->path)));
    if (head && (rc = pack_direct_weight(d->w_head, 8, 2, w_head, st))) return rc;

    const size_t in_plane = (size_t)d->in_n_img * d->H_in * d->W_in * k.cin;
    if (d->path == 2) {
        SplitTensor x;
        x.base = (__nv_bfloat16 *)d->in; x.n_img = d->in_n_img; x.H = d->H_in; x.W = d->W_in; x.C = k.cin;
        return conv_narrow(x, d->in_img, (const float *)ws, d->bias, k.cout, k.ntaps, d->n_img, d->out_f32, st);
    }
    DirectArgs a;
    a.in_img = d->in_img; a.Hin = d->H_in; a.Win = d->W_in;
    a.w = (const float *)ws; a.w_mma = ws; a.bias = d->bias;
    a.act = k.cout == 1 ? ACT_SIGMOID : ACT_RELU;
    a.n_img = d->n_img; a.Hout = Hout; a.Wout = Wout;
    if (head) {
        a.in_f32 = d->in_f32; a.w0 = w_head; a.b0 = d->b_head;
        a.pad_top = d->pad_top; a.pad_bottom = d->pad_bottom; a.pad_left = d->pad_left; a.pad_right = d->pad_right;
    } else {
        a.in_split = (const __nv_bfloat16 *)d->in; a.in_plane = in_plane;
    }
    if (split_out) {
        a.out_split = (__nv_bfloat16 *)d->out; a.out_plane = (size_t)d->out_n_img * Hout * Wout * k.cout;
    } else {
        a.out_f32 = d->out_f32;
        if (tail) { a.crop_top = d->crop_top; a.crop_left = d->crop_left; a.out_H = d->out_H; a.out_W = d->out_W; }
    }
    if (d->path == 1) return conv_direct_choice((DirectKind)k.dk, a, true, st);
    rc = conv_mma((DirectKind)k.dk, a, st);
    if (rc == ESR_EINVAL) set_error("esr_conv_small: kind %d has no mma instantiation", d->kind);
    return rc;
}
