// mma_conv.cu -- the small-channel 3x3 convolutions (Cin 8..32, full / half resolution) on the warp-level tensor-core
// path (mma.sync m16n8k16 / m16n8k8, bf16 operands, fp32 accumulate) instead of FFMA loops.
//
// These layers (head+encoder 8->16->32->64 stride 2, decoder bilinear x2 + conv 32->16->8, tail 8->2;
// models/model.py:20-45, 264-291, 309) have too few channels for a 128 x N wgmma tile and their inputs are produced on
// the fly (fused head, fused bilinear upsampling), which TMA cannot do -- so the operand tile is built by the CTA itself:
//   stage 1  the input patch of the output tile (+1 halo) is written to shared memory as split bf16 (hi and lo planes),
//            pixel-major [py][px][CIN] with a 16-byte pad per pixel (conflict-free ldmatrix rows); the split source is
//            copied as is, the decoder's bilinear x2 and the fused head conv are evaluated in fp32 and split here;
//   stage 2  implicit GEMM per warp: A fragments (16 consecutive output pixels x 16 channels of one tap) by ldmatrix
//            straight from the patch (lane addresses carry the stride and the tap shift), B fragments (weights, split,
//            [tap][co][ci]) by 32-bit shared loads, three MMAs per K step (lo*hi + hi*lo + hi*hi) like the wgmma path;
//   stage 3  accumulators -> shared memory (fp32) -> bias/activation already applied -> 16-byte split-bf16 stores (or the
//            cropped fp32 NCHW output of the tail).
// Same DirectArgs interface and results within the split-bf16 operand error (2^-17) of the fp32 kernels in direct_conv.cu,
// which remain available with ESR_DIRECT_FFMA=1.
#include "direct_common.cuh"

namespace esr {

// weight row pitch in elements ([tap][co][ci + pad]): rows of 8 lanes (g) x 4 lanes (t4) 32-bit loads must cover 32 distinct banks
__host__ __device__ constexpr int mma_wp(int cinp) { return cinp == 8 ? 8 : cinp + 8; }

template <int CIN, int COUT, int STRIDE, int TW, int TH> struct MmGeom {
    static constexpr int NP = COUT < 8 ? 8 : COUT;             // N padded to the MMA's 8
    static constexpr int NT = NP / 8;
    static constexpr int MTILES = TW * TH / 16;                // 16-pixel row segments per block
    static constexpr int MT = MTILES / 8;                      // per warp
    static constexpr int PW = (TW - 1) * STRIDE + 3, PH = (TH - 1) * STRIDE + 3;
    static constexpr int CINP = CIN < 8 ? 8 : CIN;             // K per tap padded to the MMA's 8 (1- and 2-channel inputs)
    // bytes per pixel per plane: + 16 makes the 8 rows of an ldmatrix fall into distinct 16-byte bank groups for 32- and 64-byte
    // pixels; 16-byte pixels (CINP = 8) are conflict-free unpadded at stride 1 (8 consecutive pixels = 128 contiguous bytes)
    // 32-byte pixels at stride 1 are stored unpadded with the 16-byte halves of pixels 4..7 (mod 8) swapped (SWZ): any 8
    // consecutive pixels then cover the 8 distinct 16-byte bank groups, and the patch is a third smaller (one more resident block)
    static constexpr bool SWZ = CINP == 16 && STRIDE == 1;
    // 16-byte pixels read at stride 2: pixels 8..15 (mod 16) swap places pairwise (slot = px ^ 1), so that 8 rows two pixels
    // apart cover the 8 distinct 16-byte bank groups (padding cannot: any pitch puts them 32 * k bytes apart)
    static constexpr bool SWZ8 = CINP == 8 && STRIDE == 2;
    static constexpr int PITCH = (CINP == 8 || SWZ) ? CINP * 2 : CINP * 2 + 16;
    static constexpr int WP = mma_wp(CINP);                    // weight row pitch (elements): conflict-free B loads
    // decoder layers: the source (half-resolution) patch of the tile, unpacked once to fp32
    static constexpr int SW = TW / 2 + 2, SH = TH / 2 + 2, SPITCH = CINP * 4 + 16;
    static constexpr int KS = CINP >= 16 ? CINP / 16 : 1;
    static constexpr size_t PATCH_BYTES = (size_t)((PH * PW + 15) / 16 * 16) * PITCH;   // (SWZ8 swaps within pixel pairs)
    static constexpr size_t W_BYTES = (size_t)9 * NP * WP * 2;
    static_assert(TW % 16 == 0 && MTILES % 8 == 0, "tile must hold a multiple of 8 16-pixel segments");
};

__device__ __forceinline__ uint32_t smem_u32_generic(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t (&r)[4])
{
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x2(uint32_t addr, uint32_t (&r)[4])
{
    asm volatile("ldmatrix.sync.aligned.m8n8.x2.shared.b16 {%0, %1}, [%2];" : "=r"(r[0]), "=r"(r[1]) : "r"(addr));
}
__device__ __forceinline__ void mma_k16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1)
{
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void mma_k8(float (&d)[4], const uint32_t (&a)[4], uint32_t b0)
{
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5}, {%6}, {%0, %1, %2, %3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]) : "r"(a[0]), "r"(a[1]), "r"(b0));
}
// byte offset of 16-byte chunk q of patch pixel pp
template <typename G> __device__ __forceinline__ uint32_t patch_off(int pp, int q)
{
    if constexpr (G::SWZ) return (uint32_t)(pp * 32 + ((q ^ ((pp >> 2) & 1)) << 4));
    else if constexpr (G::SWZ8) return (uint32_t)((pp ^ ((pp >> 3) & 1)) << 4);
    else return (uint32_t)(pp * G::PITCH + q * 16);
}
// 8 fp32 -> split bf16, one 16-byte store per plane (shared memory)
__device__ __forceinline__ void st_split8(uint8_t *hi, uint8_t *lo, const float (&v)[8])
{
    uint32_t hw[4], lw[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        split_pack2(v[2 * e], v[2 * e + 1], hw[e], lw[e]);
    }
    *reinterpret_cast<uint4 *>(hi) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
    *reinterpret_cast<uint4 *>(lo) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
}

template <int CIN, int COUT, int STRIDE, bool UPS, int INF, int OUTF, int TW, int TH>
__global__ void __launch_bounds__(256) k_conv_mma(const DirectArgs a)
{
    PDL_LAUNCH_DEPENDENTS();
    PDL_WAIT();
    using G = MmGeom<CIN, COUT, STRIDE, TW, TH>;
    constexpr int NP = G::NP, NT = G::NT, MT = G::MT, PW = G::PW, PH = G::PH, PITCH = G::PITCH, WP = G::WP, KS = G::KS;
    constexpr int CINP = G::CINP;
    extern __shared__ __align__(16) uint8_t msm[];
    uint8_t *p_hi = msm, *p_lo = msm + G::PATCH_BYTES;
    __nv_bfloat16 *w_hi = reinterpret_cast<__nv_bfloat16 *>(msm + 2 * G::PATCH_BYTES);
    __nv_bfloat16 *w_lo = w_hi + 9 * NP * WP;
    float *bsm = reinterpret_cast<float *>(w_lo + 9 * NP * WP);            // [NP]
    constexpr int IPP = (PW + 2 + 3) / 4 * 4;
    float *inp = bsm + NP;                                                 // fused head: [2][PH+2][IPP], then [9][2][8] + [8]

    const int img = blockIdx.z;
    const int oy0 = blockIdx.y * TH, ox0 = blockIdx.x * TW;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

    // ---- weights: the pre-packed split-bf16 image ([plane][tap][co][ci + pad], pack_mma_weight) by asynchronous 16-byte copies
    {
        const uint8_t *src = reinterpret_cast<const uint8_t *>(a.w_mma);
        const uint32_t dst = smem_u32_generic(w_hi);
        for (int i = tid; i < (int)(2 * G::W_BYTES / 16); i += 256)
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + 16u * i), "l"(src + 16 * (size_t)i) : "memory");
        asm volatile("cp.async.commit_group;" ::: "memory");
    }
    if (tid < NP) bsm[tid] = (a.bias && tid < COUT) ? a.bias[tid] : 0.0f;

    // ---- stage 1: the input patch as split bf16, pixel-major
    const int Hc = UPS ? 2 * a.Hin : a.Hin + a.pad_top + a.pad_bottom;
    const int Wc = UPS ? 2 * a.Win : a.Win + a.pad_left + a.pad_right;
    const int iy0 = oy0 * STRIDE - 1, ix0 = ox0 * STRIDE - 1;
    const int simg = a.in_img ? a.in_img[img] : img;
    if constexpr (INF == FMT_HEAD_FUSED) {
        // head (2 -> 8, relu; models/model.py:301,330) evaluated for the PH x PW patch this tile needs, on the tensor cores too:
        // K = 18 = 3 rows of (3 pixels x 2 channels), padded to 3 x 8 with a fourth pixel whose weights are zero, so that the
        // A fragment of row ky is just the split input words (one 32-bit word = both channels of a pixel) at pixels x .. x + 3.
        static_assert(INF != FMT_HEAD_FUSED || CIN == 8, "fused head feeds the 8-channel encoder layer");
        constexpr int IW = PW + 2, IH = PH + 2, IN_N = IW * IH, NPX = PH * PW;
        static_assert(INF != FMT_HEAD_FUSED || 2 * (IN_N + 4) <= 2 * IH * IPP, "input patch does not fit its region");
        uint32_t *in_hi = reinterpret_cast<uint32_t *>(inp), *in_lo = in_hi + IN_N + 4;
        for (int i = tid; i < IN_N + 4; i += 256) {                        // (+4: the zero-weight fourth pixel of the last rows)
            float v0 = 0.0f, v1 = 0.0f;
            if (i < IN_N) {
                const int y = iy0 - 1 + i / IW, x = ix0 - 1 + i % IW;      // head-input coordinates (padded frame)
                const int sy = y - a.pad_top, sx = x - a.pad_left;       // CropSize zero padding (model_util.py:148-152)
                if (sy >= 0 && sy < a.Hin && sx >= 0 && sx < a.Win) {
                    const float *src = a.in_f32 + ((size_t)simg * 2 * a.Hin + sy) * a.Win + sx;
                    v0 = __ldg(src); v1 = __ldg(src + (size_t)a.Hin * a.Win);
                }
            }
            split_pack2(v0, v1, in_hi[i], in_lo[i]);
        }
        const int hg = lane >> 2, ht = lane & 3;
        uint32_t hbh[3], hbl[3];                                           // B fragments: k = (kx = ht, ci), n = hg
#pragma unroll
        for (int ky = 0; ky < 3; ++ky) {
            float w_a = 0.0f, w_b = 0.0f;
            if (ht < 3) { w_a = a.w0[((ky * 3 + ht) * 2 + 0) * 8 + hg]; w_b = a.w0[((ky * 3 + ht) * 2 + 1) * 8 + hg]; }
            split_pack2(w_a, w_b, hbh[ky], hbl[ky]);
        }
        const float hb0 = a.b0[2 * ht], hb1 = a.b0[2 * ht + 1];
        __syncthreads();
        for (int mt = warp; mt < (NPX + 15) / 16; mt += 8) {
            const int pa = mt * 16 + hg, pb = pa + 8;
            const int qa = min(pa, NPX - 1), qb = min(pb, NPX - 1);
            const int oa = (qa / PW) * IW + qa % PW + ht, ob = (qb / PW) * IW + qb % PW + ht;
            float acc[4] = {hb0, hb1, hb0, hb1};
#pragma unroll
            for (int ky = 0; ky < 3; ++ky) {
                const uint32_t ah[4] = {in_hi[oa + ky * IW], in_hi[ob + ky * IW], 0, 0}, al[4] = {in_lo[oa + ky * IW], in_lo[ob + ky * IW], 0, 0};
                mma_k8(acc, al, hbh[ky]);
                mma_k8(acc, ah, hbl[ky]);
                mma_k8(acc, ah, hbh[ky]);
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int pp = h ? pb : pa;
                if (pp >= NPX) continue;
                const int y = iy0 + pp / PW, x = ix0 + pp % PW;
                const bool inside = (y >= 0 && y < Hc && x >= 0 && x < Wc);   // outside = the encoder conv's zero padding
                uint32_t vh, vl;
                split_pack2(inside ? fmaxf(acc[2 * h], 0.0f) : 0.0f, inside ? fmaxf(acc[2 * h + 1], 0.0f) : 0.0f, vh, vl);
                *reinterpret_cast<uint32_t *>(p_hi + patch_off<G>(pp, 0) + 4 * ht) = vh;
                *reinterpret_cast<uint32_t *>(p_lo + patch_off<G>(pp, 0) + 4 * ht) = vl;
            }
        }
    } else if constexpr (INF == FMT_NCHW_F32) {
        // training operators: fp32 NCHW planes.  A thread gathers the 8 channels of one pixel (each of the 8 loads is
        // coalesced across the warp: consecutive lanes = consecutive pixels of a row), splits and stores 16 bytes per plane.
        constexpr int Q = CINP / 8;
        const size_t cs = (size_t)a.Hin * a.Win;
        for (int i = tid; i < Q * PW * PH; i += 256) {
            const int pp = i % (PW * PH), q = i / (PW * PH);
            const int y = iy0 + pp / PW, x = ix0 + pp % PW;
            float v[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) v[e] = 0.0f;
            if (y >= 0 && y < Hc && x >= 0 && x < Wc) {
                const float *src = a.in_f32 + ((size_t)simg * CIN + q * 8) * cs + (size_t)y * a.Win + x;
#pragma unroll
                for (int e = 0; e < 8; ++e)
                    if (q * 8 + e < CIN) v[e] = __ldg(src + e * cs);
            }
            st_split8(p_hi + patch_off<G>(pp, q), p_lo + patch_off<G>(pp, q), v);
        }
    } else {
        static_assert(INF == FMT_HEAD_FUSED || INF == FMT_SPLIT || INF == FMT_NCHW_F32, "unsupported input format");
        const __nv_bfloat16 *hi = a.in_split;
        const size_t plane = a.in_plane;
        constexpr int Q = CIN / 8;
        constexpr int NI = Q * PW * PH;
        if constexpr (!UPS) {
            // already split: asynchronous 16-byte copies global -> shared (all in flight at once), zeros outside the image
            for (int i = tid; i < NI; i += 256) {
                const int q = i % Q, pp = i / Q;                          // consecutive lanes: the 16-byte groups of a pixel
                const int px = pp % PW, py = pp / PW;
                const int y = iy0 + py, x = ix0 + px;
                uint8_t *dh = p_hi + patch_off<G>(pp, q), *dl = p_lo + patch_off<G>(pp, q);
                if (y >= 0 && y < Hc && x >= 0 && x < Wc) {
                    const __nv_bfloat16 *s = hi + (((size_t)simg * a.Hin + y) * a.Win + x) * CIN + q * 8;
                    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32_generic(dh)), "l"(s) : "memory");
                    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32_generic(dl)), "l"(s + plane) : "memory");
                } else {
                    *reinterpret_cast<uint4 *>(dh) = make_uint4(0, 0, 0, 0);
                    *reinterpret_cast<uint4 *>(dl) = make_uint4(0, 0, 0, 0);
                }
            }
            asm volatile("cp.async.commit_group;" ::: "memory");
            asm volatile("cp.async.wait_group 0;" ::: "memory");
        } else {
            // F.interpolate(scale_factor=2, bilinear, align_corners=False) (submodules.py:290), as in direct_conv.cu, in two
            // phases so that every source pixel is loaded and unpacked ONCE (the direct form unpacked 4 corners per patch
            // pixel and was bound by those integer instructions):
            //  A  the (TH/2+2) x (TW/2+2) source patch, indices clamped to the image, split bf16 -> fp32 in shared memory;
            //  B  per patch pixel: 4 corner reads, ATen's h0*(w0*v00 + w1*v01) + h1*(w0*v10 + w1*v11), split, store.
            // Output row y of the x2 image reads source rows y_0 = floor(max(0, y/2 - 0.25)) and min(y_0 + 1, Hin - 1); for the
            // tile rows iy0 .. iy0 + PH - 1 (iy0 = oy0 - 1, oy0 even) that is oy0/2 - 1 .. oy0/2 + TH/2, and because the stored
            // patch is clamped the same way, "y_0 + 1" is simply the next stored row.
            constexpr int SW = G::SW, SH = G::SH, SPITCH = G::SPITCH;
            uint8_t *srcp = reinterpret_cast<uint8_t *>(inp);
            const int sy0 = oy0 / 2 - 1, sx0 = ox0 / 2 - 1;
            for (int i = tid; i < Q * SW * SH; i += 256) {
                const int q = i % Q, sp = i / Q;
                const int sy = min(max(sy0 + sp / SW, 0), a.Hin - 1), sx = min(max(sx0 + sp % SW, 0), a.Win - 1);
                const __nv_bfloat16 *s = hi + (((size_t)simg * a.Hin + sy) * a.Win + sx) * CIN + q * 8;
                float v[8];
                dc_unpack8(__ldg(reinterpret_cast<const uint4 *>(s)), __ldg(reinterpret_cast<const uint4 *>(s + plane)), v);
                float4 *d = reinterpret_cast<float4 *>(srcp + (size_t)sp * SPITCH + q * 32);
                d[0] = make_float4(v[0], v[1], v[2], v[3]);
                d[1] = make_float4(v[4], v[5], v[6], v[7]);
            }
            __syncthreads();
            for (int i = tid; i < NI; i += 256) {
                const int q = i % Q, pp = i / Q;
                const int y = iy0 + pp / PW, x = ix0 + pp % PW;
                uint8_t *dh = p_hi + patch_off<G>(pp, q), *dl = p_lo + patch_off<G>(pp, q);
                if (!(y >= 0 && y < Hc && x >= 0 && x < Wc)) {
                    *reinterpret_cast<uint4 *>(dh) = make_uint4(0, 0, 0, 0);
                    *reinterpret_cast<uint4 *>(dl) = make_uint4(0, 0, 0, 0);
                    continue;
                }
                const float fy = fmaxf(0.0f, ((float)y + 0.5f) * 0.5f - 0.5f);
                const float fx = fmaxf(0.0f, ((float)x + 0.5f) * 0.5f - 0.5f);
                const int y_0 = (int)fy, x_0 = (int)fx;
                const float ly = fy - (float)y_0, lx = fx - (float)x_0;
                const int r0 = y_0 - sy0, c0 = x_0 - sx0;                    // in [0, SH - 2] x [0, SW - 2]
                const uint8_t *b00 = srcp + (size_t)(r0 * SW + c0) * SPITCH + q * 32;
                const float4 *p00 = reinterpret_cast<const float4 *>(b00), *p01 = reinterpret_cast<const float4 *>(b00 + SPITCH);
                const float4 *p10 = reinterpret_cast<const float4 *>(b00 + SW * SPITCH), *p11 = reinterpret_cast<const float4 *>(b00 + (SW + 1) * SPITCH);
                const float w0 = 1.0f - lx, h0 = 1.0f - ly;
                float v[8];
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const float4 a00 = p00[h], a01 = p01[h], a10 = p10[h], a11 = p11[h];
                    v[4 * h + 0] = h0 * (w0 * a00.x + lx * a01.x) + ly * (w0 * a10.x + lx * a11.x);
                    v[4 * h + 1] = h0 * (w0 * a00.y + lx * a01.y) + ly * (w0 * a10.y + lx * a11.y);
                    v[4 * h + 2] = h0 * (w0 * a00.z + lx * a01.z) + ly * (w0 * a10.z + lx * a11.z);
                    v[4 * h + 3] = h0 * (w0 * a00.w + lx * a01.w) + ly * (w0 * a10.w + lx * a11.w);
                }
                st_split8(dh, dl, v);
            }
        }
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");                   // weights (and the copied patch) have landed
    __syncthreads();

    // ---- stage 2: implicit GEMM on the warp-level tensor cores
    const int g = lane >> 2, t4 = lane & 3;
    float acc[MT][NT][4];
#pragma unroll
    for (int m = 0; m < MT; ++m)
#pragma unroll
        for (int n = 0; n < NT; ++n) {
            acc[m][n][0] = acc[m][n][2] = bsm[n * 8 + 2 * t4];
            acc[m][n][1] = acc[m][n][3] = bsm[n * 8 + 2 * t4 + 1];
        }
    // ldmatrix lane roles: matrix = lane / 8 -> pixel half (mat & 1) and channel half (mat >> 1); row = lane % 8
    const int lm_px = (lane & 7) + ((lane >> 3) & 1) * 8;
    const int lm_koff = CINP >= 16 ? (lane >> 4) * 16 : 0;                   // bytes
    const uint32_t hi_base = smem_u32_generic(p_hi), lo_base = smem_u32_generic(p_lo);
    uint32_t a_off[MT];                                                      // byte offset of this lane's row for tap (0,0)
    int a_px[MT];                                                            // (SWZ) its patch pixel
#pragma unroll
    for (int m = 0; m < MT; ++m) {
        const int mt = warp * MT + m;
        const int ty = mt / (TW / 16), cx = mt % (TW / 16);
        a_px[m] = (ty * STRIDE) * PW + (cx * 16 + lm_px) * STRIDE;
        a_off[m] = (uint32_t)(a_px[m] * PITCH + lm_koff);
    }
#pragma unroll 1
    for (int tap = 0; tap < 9; ++tap) {
        const int tap_px = (tap / 3) * PW + tap % 3;
        const uint32_t tap_off = (uint32_t)(tap_px * PITCH);
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
            uint32_t ah[MT][4], al[MT][4];
#pragma unroll
            for (int m = 0; m < MT; ++m) {
                const uint32_t o = (G::SWZ || G::SWZ8) ? patch_off<G>(a_px[m] + tap_px, lane >> 4) : a_off[m] + tap_off + ks * 32;
                if constexpr (CINP >= 16) { ldsm_x4(hi_base + o, ah[m]); ldsm_x4(lo_base + o, al[m]); }
                else { ldsm_x2(hi_base + o, ah[m]); ldsm_x2(lo_base + o, al[m]); }
            }
#pragma unroll
            for (int n = 0; n < NT; ++n) {
                const int wrow = ((tap * NP + n * 8 + g) * WP + ks * 16 + 2 * t4);
                const uint32_t bh0 = *reinterpret_cast<const uint32_t *>(w_hi + wrow), bl0 = *reinterpret_cast<const uint32_t *>(w_lo + wrow);
                if constexpr (CINP >= 16) {
                    const uint32_t bh1 = *reinterpret_cast<const uint32_t *>(w_hi + wrow + 8), bl1 = *reinterpret_cast<const uint32_t *>(w_lo + wrow + 8);
#pragma unroll
                    for (int m = 0; m < MT; ++m) {
                        mma_k16(acc[m][n], al[m], bh0, bh1);
                        mma_k16(acc[m][n], ah[m], bl0, bl1);
                        mma_k16(acc[m][n], ah[m], bh0, bh1);
                    }
                } else {
#pragma unroll
                    for (int m = 0; m < MT; ++m) {
                        mma_k8(acc[m][n], al[m], bh0);
                        mma_k8(acc[m][n], ah[m], bl0);
                        mma_k8(acc[m][n], ah[m], bh0);
                    }
                }
            }
        }
    }
    __syncthreads();                                                         // the patch is dead: reuse it as the output stage

    // ---- stage 3: accumulators (+activation) -> shared fp32 [pixel][NP] -> global
    float *stage = reinterpret_cast<float *>(msm);
    // (the launcher sizes the dynamic shared memory as max(patch + weights + ..., this stage); patch and weights are dead here)
#pragma unroll
    for (int m = 0; m < MT; ++m) {
        const int mt = warp * MT + m;
        const int ty = mt / (TW / 16), cx = mt % (TW / 16);
        const int p0 = ty * TW + cx * 16 + g;
#pragma unroll
        for (int n = 0; n < NT; ++n) {
            *reinterpret_cast<float2 *>(stage + (size_t)p0 * NP + n * 8 + 2 * t4) = make_float2(dc_act(acc[m][n][0], a.act), dc_act(acc[m][n][1], a.act));
            *reinterpret_cast<float2 *>(stage + (size_t)(p0 + 8) * NP + n * 8 + 2 * t4) = make_float2(dc_act(acc[m][n][2], a.act), dc_act(acc[m][n][3], a.act));
        }
    }
    __syncthreads();
    if constexpr (OUTF == FMT_SPLIT) {
        constexpr int QO = COUT / 8;
        for (int i = tid; i < TW * TH * QO; i += 256) {
            const int q = i % QO, p = i / QO;
            const int oy = oy0 + p / TW, ox = ox0 + p % TW;
            if (oy >= a.Hout || ox >= a.Wout) continue;
            const float4 v0 = *reinterpret_cast<const float4 *>(stage + (size_t)p * NP + q * 8), v1 = *reinterpret_cast<const float4 *>(stage + (size_t)p * NP + q * 8 + 4);
            const float v[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
            dc_store<8>(a.out_split + (((size_t)img * a.Hout + oy) * a.Wout + ox) * COUT + q * 8, a.out_plane, v);
        }
    } else if constexpr (OUTF == FMT_NHWC_F32) {
        for (int i = tid; i < TW * TH * COUT; i += 256) {                  // attention maps: [img][y][x][COUT] fp32
            const int co = i % COUT, p = i / COUT;
            const int oy = oy0 + p / TW, ox = ox0 + p % TW;
            if (oy < a.Hout && ox < a.Wout) a.out_f32[(((size_t)img * a.Hout + oy) * a.Wout + ox) * COUT + co] = stage[(size_t)p * NP + co];
        }
    } else {
        // fp32 NCHW with the CropSize crop (model_util.py:154-164): only pixels inside the crop window are stored
        static_assert(OUTF == FMT_SPLIT || OUTF == FMT_NCHW_F32 || OUTF == FMT_NHWC_F32, "unsupported output format");
        for (int i = tid; i < TW * TH * COUT; i += 256) {
            const int p = i % (TW * TH), co = i / (TW * TH);
            const int oy = oy0 + p / TW, ox = ox0 + p % TW;
            const int cy = oy - a.crop_top, cx = ox - a.crop_left;
            if (oy < a.Hout && ox < a.Wout && cy >= 0 && cy < a.out_H && cx >= 0 && cx < a.out_W)
                a.out_f32[(((size_t)img * COUT + co) * a.out_H + cy) * a.out_W + cx] = stage[(size_t)p * NP + co];
        }
    }
}

template <int CIN, int COUT, int STRIDE, bool UPS, int INF, int OUTF, int TW, int TH>
static int launch_mma(const DirectArgs &a, cudaStream_t st)
{
    using G = MmGeom<CIN, COUT, STRIDE, TW, TH>;
    constexpr int IPP = (G::PW + 2 + 3) / 4 * 4;
    constexpr size_t extra = INF == FMT_HEAD_FUSED ? sizeof(float) * (size_t)(2 * (G::PH + 2) * IPP + 9 * 2 * 8 + 8)
                             : (UPS ? (size_t)G::SW * G::SH * G::SPITCH : 0);
    constexpr size_t smem_in = 2 * G::PATCH_BYTES + 2 * G::W_BYTES + sizeof(float) * G::NP + extra + 16;
    constexpr size_t smem_stage = (size_t)TW * TH * G::NP * sizeof(float);
    constexpr size_t smem = smem_in > smem_stage ? smem_in : smem_stage;
    static_assert(smem <= 227 * 1024, "mma conv tile does not fit in shared memory");
    static_assert((2 * G::PATCH_BYTES) % 16 == 0 && G::W_BYTES % 16 == 0, "alignment");
    static bool attr_set = false;
    if (!attr_set) {
        ESR_CUDA_CHECK(cudaFuncSetAttribute(k_conv_mma<CIN, COUT, STRIDE, UPS, INF, OUTF, TW, TH>,
                                            cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr_set = true;
    }
    dim3 grid((a.Wout + TW - 1) / TW, (a.Hout + TH - 1) / TH, a.n_img);
    ESR_CUDA_CHECK(launch_pdl(k_conv_mma<CIN, COUT, STRIDE, UPS, INF, OUTF, TW, TH>, dim3(grid), dim3(256), smem, st, a));
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}

// rot = 0: v(co, ci, tap) = w[co][ci][tap], w = [cout][cin][3][3].  rot = 1 (the convolution that maps g to dx; cout / cin are
// those of THAT convolution, w is the forward layer's [cin][cout][3][3]): v(co, ci, tap) = w[ci][co][8 - tap].
__global__ void k_pack_mma_weight(const float *__restrict__ w, int cout, int cin, int rot, __nv_bfloat16 *__restrict__ dst)
{
    const int np = cout < 8 ? 8 : cout, wp = mma_wp(cin < 8 ? 8 : cin);
    const int total = 9 * np * wp;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int ci = i % wp, co = (i / wp) % np, tap = i / (wp * np);
        float v = 0.0f;
        if (ci < cin && co < cout) v = rot ? w[((size_t)ci * cout + co) * 9 + (8 - tap)] : w[((size_t)co * cin + ci) * 9 + tap];
        __nv_bfloat16 h, l;
        split_bf16(v, h, l);
        dst[i] = h;
        dst[total + i] = l;
    }
}
size_t mma_weight_bytes(int cout, int cin) { return (size_t)2 * 9 * (cout < 8 ? 8 : cout) * mma_wp(cin < 8 ? 8 : cin) * sizeof(__nv_bfloat16); }
int pack_mma_weight(const float *w, int cout, int cin, void *dst, cudaStream_t st)
{
    k_pack_mma_weight<<<(int)(mma_weight_bytes(cout, cin) / 4 + 255) / 256, 256, 0, st>>>(w, cout, cin, 0, (__nv_bfloat16 *)dst);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}
// image of the dx convolution (cin_dx = the layer's Cout -> cout_dx = the layer's Cin) from the layer's w [Cout][Cin][3][3]:
// rotated by 180 degrees and transposed
int pack_mma_weight_dx(const float *w, int layer_cout, int layer_cin, void *dst, cudaStream_t st)
{
    k_pack_mma_weight<<<(int)(mma_weight_bytes(layer_cin, layer_cout) / 4 + 255) / 256, 256, 0, st>>>(w, layer_cin, layer_cout, 1, (__nv_bfloat16 *)dst);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}

// returns ESR_EINVAL for kinds that stay on the FFMA kernels
int conv_mma(DirectKind kind, const DirectArgs &a, cudaStream_t st)
{
    if (!a.w_mma) return ESR_EINVAL;
    switch (kind) {
    case DK_HEAD_ENC0: return launch_mma<8, 16, 2, false, FMT_HEAD_FUSED, FMT_SPLIT, 16, 16>(a, st);
    case DK_ENC0:      return launch_mma<8, 16, 2, false, FMT_SPLIT, FMT_SPLIT, 16, 16>(a, st);
    case DK_ENC1:      return launch_mma<16, 32, 2, false, FMT_SPLIT, FMT_SPLIT, 16, 8>(a, st);
    case DK_ENC2:      return launch_mma<32, 64, 2, false, FMT_SPLIT, FMT_SPLIT, 16, 8>(a, st);
    case DK_RECON1:    return launch_mma<32, 16, 1, true, FMT_SPLIT, FMT_SPLIT, 32, 8>(a, st);
    case DK_RECON2:    return launch_mma<16, 8, 1, true, FMT_SPLIT, FMT_SPLIT, 32, 16>(a, st);
    case DK_TAIL:      return launch_mma<8, 2, 1, false, FMT_SPLIT, FMT_NCHW_F32, 32, 16>(a, st);
    case DK_ATT32:     return launch_mma<32, 1, 1, false, FMT_SPLIT, FMT_NHWC_F32, 32, 8>(a, st);
    case DK_ATT16:     return launch_mma<16, 1, 1, false, FMT_SPLIT, FMT_NHWC_F32, 32, 16>(a, st);
    default: break;
    }
    return ESR_EINVAL;
}

// The fp32 NCHW instantiations of the training operators: MMA_CASE(Cin, Cout, stride, tile width, tile height)
#define MMA_NCHW_CASES(MMA_CASE)                                                                                                   \
    MMA_CASE(2, 8, 1, 32, 16) MMA_CASE(32, 16, 1, 32, 8) MMA_CASE(16, 8, 1, 32, 16) MMA_CASE(8, 2, 1, 32, 16)                      \
    MMA_CASE(32, 1, 1, 32, 8) MMA_CASE(16, 1, 1, 32, 16)                                                                           \
    MMA_CASE(16, 32, 1, 32, 16) MMA_CASE(8, 16, 1, 32, 16) MMA_CASE(1, 32, 1, 32, 16) MMA_CASE(1, 16, 1, 32, 16) MMA_CASE(1, 64, 1, 32, 8) \
    MMA_CASE(8, 16, 2, 16, 16) MMA_CASE(16, 32, 2, 16, 8) MMA_CASE(32, 64, 2, 16, 8)

bool conv_mma_nchw_ok(int Cin, int Cout, int stride, int act)
{
    if (act != ACT_NONE && act != ACT_RELU && act != ACT_SIGMOID) return false;
#define MMA_CASE(ci, co, s, tw, th) if (Cin == ci && Cout == co && stride == s) return true;
    MMA_NCHW_CASES(MMA_CASE)
#undef MMA_CASE
    return false;
}

// fp32 NCHW in / out (the training operators): y = act(conv3x3(x) + bias), stride 1 or 2, weights as a pack_mma_weight image.
int conv_mma_nchw(const float *x, const void *w_img, const float *bias, int B, int Cin, int H, int W, int Cout, int stride, int act,
                  float *y, cudaStream_t st)
{
    ESR_REQUIRE(conv_mma_nchw_ok(Cin, Cout, stride, act), "conv_mma_nchw: no instantiation for %d -> %d, stride %d, act %d", Cin,
                Cout, stride, act);
    DirectArgs a;
    a.in_f32 = x; a.Hin = H; a.Win = W; a.w_mma = w_img; a.bias = bias; a.act = act;
    a.n_img = B; a.Hout = (H + 2 - 3) / stride + 1; a.Wout = (W + 2 - 3) / stride + 1;
    a.out_f32 = y; a.out_H = a.Hout; a.out_W = a.Wout;
#define MMA_CASE(ci, co, s, tw, th) \
    if (Cin == ci && Cout == co && stride == s) return launch_mma<ci, co, s, false, FMT_NCHW_F32, FMT_NCHW_F32, tw, th>(a, st);
    MMA_NCHW_CASES(MMA_CASE)
#undef MMA_CASE
    return ESR_EINVAL;                                                   // not reached: conv_mma_nchw_ok reads the same list
}

} // namespace esr
