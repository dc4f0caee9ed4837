// tc_conv.cu -- 3x3 / 1x1 (and LPIPS's 5x5) convolution as an implicit GEMM on the Hopper tensor cores (sm_90a, wgmma).
//
//   D[128 pixels, Cout] += A[128 pixels, 64 ch of one tap] * B[Cout, 64]^T      per K-block (tap x 64-channel chunk)
//
// * Activations live in HBM as "split bf16" NHWC tensors (value = hi + lo).  A 3x3 layer's A operand is ONE TMA box
//   (64 ch, TW, TH + 2, 1 image, 1 plane) per 64-channel chunk and dx shift, read by the three dy taps at row offsets
//   0, TW, 2 TW; out-of-image coordinates are zero-filled by TMA, which is exactly the conv's zero padding.  The box lands
//   in shared memory in the 128B-swizzled K-major layout that wgmma reads, so no thread touches the operands.
// * Channel concatenation (torch.cat in the reference) is a K-split over up to 3 source tensors.  A 64-channel source can also
//   stand for several chunks, chunk j at image + j * step (the num_frame-way concatenation of dense_fusion): one multiply-add
//   in the producer per K-block.
// * fp32 parity: three bf16 MMAs per K-step (lo*hi + hi*lo + hi*hi) accumulate in fp32 registers => ~2^-17 relative
//   operand error instead of bf16's 2^-9 (the reference network is fp32-only).
// * Warp roles: warps 0-7 = two consumer warpgroups (pixel rows 0-63 / 64-127 of the tile, accumulators in registers,
//   then the epilogue: staging through shared memory -> bias / residual / activation / GRU gating -> split-bf16 or fp32
//   stores); warp 8 = TMA producer.
// * Two mbarrier rings, A boxes and per-tap weights: full[s] (TMA -> consumers), empty[s] (one arrival per consumer warp
//   once its MMAs on s retired -> TMA).
//
// Reference layers served: every Conv2d of models/model.py at feature resolution (Cin multiple of 64), the ConvGRU
// gates (models/submodules.py:496-514) and the DCNv2 contraction (models/DCNv2/src/cuda/dcn_v2_cuda.cu:90-92).
#include "tc_common.cuh"
#include <algorithm>
#include <cstdlib>

namespace esr {

constexpr int TC_THREADS = 288;

// ------------------------------------------------------------------------------------------------
// Persistent conv body: the CTA walks tiles tile0, tile0 + step, ... of one layer (128 output pixels (TH x TW) of one image x
// all NP (= npad) output channels each).  K-blocks run in the order (chunk, dx, dy).  A 3x3 layer loads ONE A box of
// TW x (TH + 2) pixels per (chunk, dx), taken at (x0 + dx, y0 - 1); its three dy taps are the 128 rows starting (dy + 1) TW
// rows into it (a multiple of 1024 bytes, so every tap starts on a SWIZZLE_128B atom).  A 1x1 layer loads the tile itself, one
// tap per box.  A boxes and per-tap weights (B) have separate rings: a consumer frees an A box once the MMAs of its last tap
// retired, and each B slot once its own MMAs did.  The TMA producer streams both across tile boundaries, so the loads of
// tile i+1 overlap the epilogue of tile i; the ring positions of each role persist across tiles.
// The epilogue stages accumulators in a dedicated area beside the rings (the rings are already refilling).
// ------------------------------------------------------------------------------------------------
struct TcSmem {
    uint32_t a_ring, a_box, b_ring, b_slot;              // shared-memory addresses and slot strides
    uint32_t bar;                                        // mbarriers: A full [na], A empty [na], B full [nb], B empty [nb]
    float *stg;                                          // epilogue staging: [2 warpgroups][64][TC_STG_LD] fp32
    int na, nb;
    __device__ uint32_t a_full(uint32_t s) const { return bar + 8u * s; }
    __device__ uint32_t a_empty(uint32_t s) const { return bar + 8u * (na + s); }
    __device__ uint32_t b_full(uint32_t s) const { return bar + 8u * (2 * na + s); }
    __device__ uint32_t b_empty(uint32_t s) const { return bar + 8u * (2 * na + nb + s); }
};
// Ring position: the count of slots used modulo twice the depth n, i.e. slot c % n with phase c / n (one register per ring).
__device__ __forceinline__ uint32_t ring_slot(uint32_t c, int n) { return c < (uint32_t)n ? c : c - n; }
__device__ __forceinline__ uint32_t ring_phase(uint32_t c, int n) { return c < (uint32_t)n ? 0u : 1u; }
__device__ __forceinline__ uint32_t ring_next(uint32_t c, int n) { return c + 1 == 2u * n ? 0u : c + 1; }
__device__ __forceinline__ uint32_t ring_prev_slot(uint32_t c, int n) { return ring_slot(c == 0 ? 2u * n - 1 : c - 1, n); }

// 1024: worst-case alignment of the rings; then the A ring, the B ring, the two staging tiles and the full / empty mbarriers of
// both rings.  conv_tc_prepare sizes the rings so that this fits the 227 KB (232448 B) an H100 block
// may opt in to.
static size_t tc_smem_bytes(int npad, uint32_t a_box, int na, int nb)
{
    return 1024 + (size_t)na * (a_box + 16) + (size_t)nb * (2 * (size_t)npad * 128 + 16) + 2 * TC_STG_BYTES;
}
// Ring depths for one CTA per SM: two A boxes and two B slots (one A box where that does not fit: npad = 256), then one more slot
// for whichever ring is fewer K-blocks ahead (B on a tie) while it fits, up to 4 A boxes and 9 B slots.  false: nothing fits.
// Rings that end at two A boxes and two B slots keep the weights only one K-block ahead of the MMAs.  Where a third B slot fits in
// place of the second A box (npad 160-192), take it: one box still feeds `taps` K-blocks, and npad 192 at 3x3 ran 13 % faster
// per launch on H100 (1 + 3 against 2 + 2).  Not for 1x1 layers: a single box there would stall every K-block.
static bool tc_rings(int npad, uint32_t a_box, int taps, size_t cap, int *na_out, int *nb_out)
{
    int na = 2, nb = 2;
    if (tc_smem_bytes(npad, a_box, na, nb) > cap) na = 1;
    if (tc_smem_bytes(npad, a_box, na, nb) > cap) return false;
    for (;;) {
        const bool a_can = na < 4 && tc_smem_bytes(npad, a_box, na + 1, nb) <= cap;
        const bool b_can = nb < 9 && tc_smem_bytes(npad, a_box, na, nb + 1) <= cap;
        if (a_can && (!b_can || (na - 1) * taps < nb - 1)) ++na;
        else if (b_can) ++nb;
        else break;
    }
    if (na == 2 && nb == 2 && taps > 1 && tc_smem_bytes(npad, a_box, 1, 3) <= cap) { na = 1; nb = 3; }
    *na_out = na; *nb_out = nb;
    return true;
}
__device__ __forceinline__ TcSmem tc_smem_layout(int np_max, uint32_t a_box, int na, int nb)
{
    extern __shared__ uint8_t smem_raw[];
    TcSmem m;
    m.a_ring = (smem_u32(smem_raw) + 1023u) & ~1023u;                  // SWIZZLE_128B needs 1024-B alignment
    m.a_box = a_box;                                                    // a multiple of 1024 (TW is)
    m.b_ring = m.a_ring + (uint32_t)na * a_box;
    m.b_slot = 2u * (uint32_t)np_max * 128u;
    const uint32_t stg = m.b_ring + (uint32_t)nb * m.b_slot;
    m.stg = reinterpret_cast<float *>(smem_raw + (stg - smem_u32(smem_raw)));
    m.bar = stg + 2u * TC_STG_BYTES;
    m.na = na; m.nb = nb;
    return m;
}
__device__ __forceinline__ void tc_init_barriers(const TcSmem &m)
{
    if (threadIdx.x == 0) {
        for (int s = 0; s < m.na; ++s) { mbar_init(m.a_full(s), 1); mbar_init(m.a_empty(s), 8); }
        for (int s = 0; s < m.nb; ++s) { mbar_init(m.b_full(s), 1); mbar_init(m.b_empty(s), 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
}

// KS = 0: 3x3 or 1x1 (a.ntaps 9 or 1); KS = 5: 5x5, pad 2 (a.ntaps 25) -- one box of TW x (TH + 4) pixels per (chunk, dx),
// read by the five dy taps, and the packing's order chunk * 25 + 5 (dy + 2) + dx + 2.
template <int NP, int KS = 0>
__device__ __forceinline__ void conv_tiles(const ConvTCArgs &a, int tile0, int step, const TcSmem &m)
{
    static_assert(KS == 0 || KS == 5, "conv_tiles: KS is 0 (3x3 / 1x1) or 5");
    constexpr bool k5 = KS == 5;
    constexpr uint32_t b_bytes = (uint32_t)NP * 128u;                  // one plane of one tap's weights
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tiles_per_img = a.tiles_x * a.tiles_y, n_tiles = a.n_img * tiles_per_img;
    const bool k3 = a.ntaps == 9;
    const int taps = k5 ? 5 : k3 ? 3 : 1, nbox = a.nkb / taps;         // dy taps per A box, A boxes per tile
    const uint32_t a_plane = m.a_box / 2;

    if (warp == 8) {
        // ===================== TMA producer (one elected lane; the others idle until the caller's next barrier) =====================
        if (elect_one_sync()) {
            uint32_t ca = 0, cb = 0;
            for (int tile = tile0; tile < n_tiles; tile += step) {
                const int img = tile / tiles_per_img, trem = tile - img * tiles_per_img;
                const int y0 = (trem / a.tiles_x) * a.TH, x0 = (trem % a.tiles_x) * a.TW;
                int src = 0, chunk_base = 0;
                for (int bx = 0; bx < nbox; ++bx) {
                    const int gchunk = k5 ? bx / 5 : k3 ? bx / 3 : bx, dx = k5 ? bx - 5 * gchunk - 2 : k3 ? bx - 3 * gchunk - 1 : 0;
                    const int ytop = y0 - (k5 ? 2 : k3 ? 1 : 0);
                    while (gchunk >= a.chunk_end[src]) { chunk_base = a.chunk_end[src]; ++src; }
                    const int cc = gchunk - chunk_base, istep = a.chunk_img_step[src];
                    const int simg = (a.src_img[src] ? a.src_img[src][img] : img) + cc * istep;
                    const int c0 = istep ? 0 : cc * 64;
                    const uint32_t sa = ring_slot(ca, m.na);
                    mbar_wait(m.a_empty(sa), ring_phase(ca, m.na) ^ 1u);
                    mbar_expect_tx(m.a_full(sa), m.a_box);
                    const uint32_t as = m.a_ring + sa * m.a_box;
                    tma_load_5d(&a.amap[src], m.a_full(sa), as, c0, x0 + dx, ytop, simg, 0);
                    tma_load_5d(&a.amap[src], m.a_full(sa), as + a_plane, c0, x0 + dx, ytop, simg, 1);
                    ca = ring_next(ca, m.na);
                    for (int t = 0; t < taps; ++t) {
                        // the packing's order: chunk * 9 + 3 (dy + 1) + dx + 1 (5x5: chunk * 25 + 5 (dy + 2) + dx + 2)
                        const int kb = k5 ? gchunk * 25 + 5 * t + dx + 2 : k3 ? gchunk * 9 + 3 * t + dx + 1 : gchunk;
                        const uint32_t sb = ring_slot(cb, m.nb);
                        mbar_wait(m.b_empty(sb), ring_phase(cb, m.nb) ^ 1u);
                        mbar_expect_tx(m.b_full(sb), 2u * b_bytes);
                        const uint32_t bs = m.b_ring + sb * m.b_slot;
                        tma_load_3d(&a.bmap, m.b_full(sb), bs, 0, 0, kb);
                        tma_load_3d(&a.bmap, m.b_full(sb), bs + b_bytes, 0, 0, a.nkb + kb);
                        cb = ring_next(cb, m.nb);
                    }
                }
            }
        }
        return;
    }

    // ===================== consumers: warpgroup wg owns tile rows [64 wg, 64 wg + 64) =====================
    const int wg = warp >> 2;
    float *stg = m.stg + wg * (TC_STG_BYTES / 4);
    const int r = threadIdx.x & 63, h = (threadIdx.x >> 6) & 1;
    const uint32_t tap_rows = (uint32_t)a.TW * 128u;                   // bytes between the dy taps of a box
    uint32_t ca = 0, cb = 0;
    for (int tile = tile0; tile < n_tiles; tile += step) {
        const int img = tile / tiles_per_img, trem = tile - img * tiles_per_img;
        const int y0 = (trem / a.tiles_x) * a.TH, x0 = (trem % a.tiles_x) * a.TW;
        float acc[NP / 2];
#pragma unroll
        for (int i = 0; i < NP / 2; ++i) acc[i] = 0.0f;
        for (int kb = 0, t = 0; kb < a.nkb; ++kb) {                    // t: the K-block's tap within its A box
            const uint32_t sa = ring_slot(ca, m.na), sb = ring_slot(cb, m.nb);
            if (t == 0) mbar_wait(m.a_full(sa), ring_phase(ca, m.na));
            mbar_wait(m.b_full(sb), ring_phase(cb, m.nb));
            const uint32_t ah = m.a_ring + sa * m.a_box + (uint32_t)wg * 8192u + (uint32_t)t * tap_rows;
            const uint32_t bs = m.b_ring + sb * m.b_slot;
            const uint64_t dah = wgmma_desc(ah), dal = wgmma_desc(ah + a_plane);
            const uint64_t dbh = wgmma_desc(bs), dbl = wgmma_desc(bs + b_bytes);
            acc_fence<NP / 2>(acc);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k) {                           // 4 x (K = 16 bf16 = 32 bytes) per 128-byte row
                wgmma_rows<NP, 0>(acc, dal + 2 * k, dbh + 2 * k);   // small terms first
                wgmma_rows<NP, 0>(acc, dah + 2 * k, dbl + 2 * k);
                wgmma_rows<NP, 0>(acc, dah + 2 * k, dbh + 2 * k);
            }
            wgmma_commit();
            // the previous K-block's MMAs have retired: free its B slot, and at a box's first tap the previous box.  With a
            // single A box (npad >= 224) the box's last tap waits for its own MMAs and frees it at once: the next box needs it.
            const bool drain = m.na == 1 && t == taps - 1;
            if (drain) wgmma_wait<0>();
            else wgmma_wait<1>();
            acc_fence<NP / 2>(acc);
            if (lane == 0) {
                if (kb != 0) mbar_arrive(m.b_empty(ring_prev_slot(cb, m.nb)));
                if (kb != 0 && t == 0 && m.na > 1) mbar_arrive(m.a_empty(ring_prev_slot(ca, m.na)));
                if (drain) mbar_arrive(m.a_empty(0));                 // the only slot
            }
            cb = ring_next(cb, m.nb);
            if (++t == taps) { t = 0; ca = ring_next(ca, m.na); }
        }
        wgmma_wait<0>();
        acc_fence<NP / 2>(acc);
        if (lane == 0) {                                            // the tile's last K-block and box
            mbar_arrive(m.b_empty(ring_prev_slot(cb, m.nb)));
            if (m.na > 1) mbar_arrive(m.a_empty(ring_prev_slot(ca, m.na)));
        }

        // ===================== epilogue: thread = (tile row r, 32-column half h) per 64-column pass =====================
        const int mrow = wg * 64 + r;                               // accumulator row = pixel within the tile
        const int y = y0 + mrow / a.TW, x = x0 + mrow % a.TW;
        const bool valid = (y < a.H) && (x < a.W);
        const size_t pix = ((size_t)img * a.H + (valid ? y : 0)) * a.W + (valid ? x : 0);
#pragma unroll
        for (int p = 0; p < (NP + 63) / 64; ++p) {
            stage_acc<NP>(acc, p, stg);
            named_sync(2 + wg, 128);
            const int n0 = 64 * p + 32 * h;
            if (n0 < NP) {
                uint32_t raw[32];
                staged_row32(stg, r, h, NP - n0, raw);
                if (valid) epilogue_chunk(a, raw, n0, pix, img, y, x);
            }
            named_sync(2 + wg, 128);
        }
    }
}

// one layer: grid = min(tiles, resident CTAs); CTA b takes tiles b, b + gridDim.x, ...
template <int NP, int KS = 0>
__global__ void __launch_bounds__(TC_THREADS, 1) k_conv_tc(const __grid_constant__ ConvTCArgs a)
{
    PDL_LAUNCH_DEPENDENTS();
    const uint32_t a_box = KS == 5 ? tc_a_box_bytes5(a.TW, a.TH) : tc_a_box_bytes(a.TW, a.TH, a.ntaps);
    const TcSmem m = tc_smem_layout(NP, a_box, a.a_stages, a.b_stages);
    tc_init_barriers(m);
    PDL_WAIT();                      // everything above is CTA-local set-up; global memory only from here on
    conv_tiles<NP, KS>(a, blockIdx.x, gridDim.x, m);
}

// ------------------------------------------------------------------------------------------------
// host side: tensor maps and launch
// ------------------------------------------------------------------------------------------------
typedef CUresult (*PFN_tmapEncodeTiled)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                        const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                        CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_tmapEncodeTiled get_encode()
{
    static PFN_tmapEncodeTiled fn = [] {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
            q != cudaDriverEntryPointSuccess)
            p = nullptr;
        return (PFN_tmapEncodeTiled)p;
    }();
    return fn;
}

static int make_amap(const SplitTensor &t, int BW, int BH, CUtensorMap *out)
{
    PFN_tmapEncodeTiled enc = get_encode();
    if (!enc) { set_error("cuTensorMapEncodeTiled unavailable"); return ESR_ECUDA; }
    const cuuint64_t C = t.C, W = t.W, H = t.H, N = t.n_img;
    cuuint64_t gdim[5] = {C, W, H, N, 2};
    cuuint64_t gstr[4] = {C * 2, W * C * 2, H * W * C * 2, N * H * W * C * 2};
    cuuint32_t box[5] = {64, (cuuint32_t)BW, (cuuint32_t)BH, 1, 1};
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, t.base, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(A) failed: %d (C=%d W=%d H=%d N=%d)", (int)r, t.C, t.W, t.H, t.n_img); return ESR_ECUDA; }
    return ESR_OK;
}

static int make_bmap(const void *w, int npad, int nkb, int box_rows, CUtensorMap *out)
{
    PFN_tmapEncodeTiled enc = get_encode();
    if (!enc) { set_error("cuTensorMapEncodeTiled unavailable"); return ESR_ECUDA; }
    cuuint64_t gdim[3] = {64, (cuuint64_t)npad, (cuuint64_t)2 * nkb};
    cuuint64_t gstr[2] = {128, (cuuint64_t)npad * 128};
    cuuint32_t box[3] = {64, (cuuint32_t)box_rows, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void *>(w), gdim, gstr, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(B) failed: %d (npad=%d nkb=%d)", (int)r, npad, nkb); return ESR_ECUDA; }
    return ESR_OK;
}

int tc_make_amap(const SplitTensor &t, int BW, int BH, CUtensorMap *out) { return make_amap(t, BW, BH, out); }
int tc_make_bmap(const void *w, int npad, int nkb, int box_rows, CUtensorMap *out) { return make_bmap(w, npad, nkb, box_rows, out); }

int conv_tc_prepare(const ConvTCDesc &d, ConvTCArgs *args)
{
    ConvTCArgs &a = *args;
    memset(&a, 0, sizeof(a));
    ESR_REQUIRE(d.n_src >= 1 && d.n_src <= TC_MAX_SRC, "conv_tc: n_src=%d", d.n_src);
    ESR_REQUIRE(d.ntaps == 9 || d.ntaps == 1 || d.ntaps == 25, "conv_tc: ntaps=%d", d.ntaps);
    const int H = d.src[0].H, W = d.src[0].W;
    int chunks = 0;
    // tile shape: 128 pixels, 16 x 8 (8 x 16 on images narrower than 12, so that at most half a tile is wasted).  A 3x3 box of
    // 16 x 10 pixels serves three taps: 2.4x fewer A bytes per tap than one box per tap (32 x 4 tiles: 2.0x).
    const int TW = W >= 12 ? 16 : 8;
    const int TH = TC_BLOCK_M / TW;
    for (int s = 0; s < d.n_src; ++s) {
        const SplitTensor &t = d.src[s];
        ESR_REQUIRE(t.base && t.C % 64 == 0 && t.H == H && t.W == W, "conv_tc: source %d has C=%d H=%d W=%d", s, t.C, t.H, t.W);
        if (d.chunk_img_step[s] != 0) {
            ESR_REQUIRE(t.C == 64 && d.src_chunks[s] >= 1, "conv_tc: source %d with an image step needs C=64 and src_chunks >= 1", s);
            chunks += d.src_chunks[s];
        } else {
            ESR_REQUIRE(d.src_chunks[s] == 0 || d.src_chunks[s] == t.C / 64, "conv_tc: source %d has %d chunks, not %d", s, t.C / 64,
                        d.src_chunks[s]);
            chunks += t.C / 64;
        }
        a.chunk_end[s] = chunks;
        a.chunk_img_step[s] = d.chunk_img_step[s];
        a.src_img[s] = d.src_img[s];
        int rc = make_amap(t, TW, tc_conv_box_h(TH, d.ntaps), &a.amap[s]);
        if (rc) return rc;
    }
    for (int s = d.n_src; s < TC_MAX_SRC; ++s) a.chunk_end[s] = 1 << 30;
    a.n_src = d.n_src; a.ntaps = d.ntaps; a.nkb = chunks * d.ntaps;
    a.npad = tc_npad(d.cout); a.cout = d.cout;
    ESR_REQUIRE(a.npad <= 256, "conv_tc: cout=%d too large", d.cout);
    int rc = make_bmap(d.wpacked, a.npad, a.nkb, a.npad, &a.bmap);
    if (rc) return rc;
    a.H = H; a.W = W; a.TW = TW; a.TH = TH;
    a.tiles_x = (W + TW - 1) / TW; a.tiles_y = (H + TH - 1) / TH; a.n_img = d.n_img;
    // Ring depths: as many slots as fit beside one CTA per SM (two 40 KB A boxes already rule out a second CTA).
    const size_t smem_cap = (size_t)dev_info().max_smem_optin;
    const uint32_t a_box = tc_conv_a_box(TW, TH, d.ntaps);
    ESR_REQUIRE(tc_rings(a.npad, a_box, d.ntaps == 25 ? 5 : d.ntaps == 9 ? 3 : 1, smem_cap, &a.a_stages, &a.b_stages),
                "conv_tc: npad=%d needs %zu B of shared memory, the device allows %zu", a.npad, tc_smem_bytes(a.npad, a_box, 1, 2),
                smem_cap);
    a.bias = d.bias;
    a.act = d.act; a.act_from = d.act_from; a.res_mode = d.res_mode; a.epi_mode = d.epi_mode;
    if (d.res_mode != RES_NONE) {
        ESR_REQUIRE(d.res.base && d.res.H == H && d.res.W == W && d.cout % 32 == 0 && d.res.C >= d.cout, "conv_tc: bad residual");
        a.res = d.res.base; a.res_plane = d.res.plane(); a.res_C = d.res.C; a.res_img = d.res_img;
    }
    if (d.out.base) {
        ESR_REQUIRE(d.out.H == H && d.out.W == W && d.out.n_img >= d.n_img && d.out.C % 8 == 0 && d.out_coff % 8 == 0,
                    "conv_tc: bad split output");
        a.out = d.out.base; a.out_plane = d.out.plane(); a.out_C = d.out.C; a.out_coff = d.out_coff;
    }
    a.out_f32 = d.out_f32; a.out_f32_C = d.out_f32_C; a.out_f32_nchw = d.out_f32_nchw;
    if (d.epi_mode != EPI_STD) {
        ESR_REQUIRE(d.h_prev.base && d.h_prev.C == 64 && d.z_buf && d.out.base, "conv_tc: GRU epilogue needs h_prev, z_buf, out");
        ESR_REQUIRE((d.epi_mode == EPI_GRU_ZR && a.npad == 128) || (d.epi_mode == EPI_GRU_OUT && a.npad == 64), "conv_tc: GRU epilogue width");
        a.h_prev = d.h_prev.base; a.h_plane = d.h_prev.plane(); a.z_buf = d.z_buf;
    } else {
        ESR_REQUIRE(!d.out.base || d.cout % 32 == 0, "conv_tc: split output needs cout %% 32 == 0");
    }
    return ESR_OK;
}

// one instantiation per padded width (multiples of 16 up to 256): the accumulator is a register array of npad / 2 floats
template <int NP, int KS = 0>
static int launch_np(const ConvTCArgs &a, cudaStream_t st)
{
    static int max_set = 0;
    const size_t smem = tc_smem_bytes(NP, tc_conv_a_box(a.TW, a.TH, a.ntaps), a.a_stages, a.b_stages);
    if ((int)smem > max_set) {
        ESR_CUDA_CHECK(cudaFuncSetAttribute(k_conv_tc<NP, KS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        max_set = (int)smem;
    }
    int per_sm = 0;
    ESR_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_conv_tc<NP, KS>, TC_THREADS, smem));
    const int n_tiles = a.n_img * a.tiles_x * a.tiles_y;
    const unsigned grid = (unsigned)std::max(1, std::min(n_tiles, std::max(per_sm, 1) * dev_info().sm_count));
    ESR_CUDA_CHECK(launch_pdl(k_conv_tc<NP, KS>, dim3(grid), dim3(TC_THREADS), smem, st, a));
    esr::count_launch();
    return ESR_OK;
}

int conv_tc_launch(const ConvTCArgs &a, cudaStream_t st)
{
    if (a.ntaps == 25) {                 // 5x5: the width LPIPS's conv2 uses (AlexNet features.3, 64 -> 192)
        if (a.npad == 192) return launch_np<192, 5>(a, st);
        set_error("conv_tc: 5x5 taps are instantiated for npad 192 only, not %d", a.npad);
        return ESR_EUNSUPPORTED;
    }
    switch (a.npad) {
    case 16: return launch_np<16>(a, st);
    case 32: return launch_np<32>(a, st);
    case 48: return launch_np<48>(a, st);
    case 64: return launch_np<64>(a, st);
    case 80: return launch_np<80>(a, st);
    case 96: return launch_np<96>(a, st);
    case 112: return launch_np<112>(a, st);
    case 128: return launch_np<128>(a, st);
    case 144: return launch_np<144>(a, st);
    case 160: return launch_np<160>(a, st);
    case 176: return launch_np<176>(a, st);
    case 192: return launch_np<192>(a, st);
    case 208: return launch_np<208>(a, st);
    case 224: return launch_np<224>(a, st);
    case 240: return launch_np<240>(a, st);
    case 256: return launch_np<256>(a, st);
    }
    set_error("conv_tc: npad=%d", a.npad);
    return ESR_EINVAL;
}

// ------------------------------------------------------------------------------------------------
// weight packing and layout conversion kernels
// ------------------------------------------------------------------------------------------------
__global__ void k_pack_weight(const float *__restrict__ w0, const float *__restrict__ w1, int cout_each, int cin, int ksz,
                              int npad, int nkb, __nv_bfloat16 *__restrict__ dst)
{
    const int ntaps = ksz * ksz;
    const size_t total = (size_t)nkb * npad * 64;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % 64);
        const int n = (int)((i / 64) % npad);
        const int kb = (int)(i / ((size_t)64 * npad));
        const int chunk = kb / ntaps, tap = kb % ntaps;
        const int ci = chunk * 64 + c;
        float v = 0.0f;
        const int cout_tot = w1 ? 2 * cout_each : cout_each;
        if (n < cout_tot) {
            const float *w = (n < cout_each) ? w0 : w1;
            const int nn = n < cout_each ? n : n - cout_each;
            v = w[((size_t)nn * cin + ci) * ntaps + tap];
        }
        __nv_bfloat16 hi, lo;
        split_bf16(v, hi, lo);
        dst[i] = hi;
        dst[total + i] = lo;
    }
}

int pack_conv_weight2(const float *w0, const float *w1, int cout_each, int cin, int ksz, void *dst, cudaStream_t st)
{
    ESR_REQUIRE(cin % 64 == 0 && (ksz == 1 || ksz == 3 || ksz == 5), "pack_conv_weight: cin=%d ksz=%d", cin, ksz);
    const int cout = w1 ? 2 * cout_each : cout_each;
    const int npad = tc_npad(cout), nkb = tc_nkb(cin, ksz * ksz);
    const size_t total = (size_t)nkb * npad * 64;
    k_pack_weight<<<(unsigned)ceil_div64((int64_t)total, 256), 256, 0, st>>>(w0, w1, cout_each, cin, ksz, npad, nkb,
                                                                             (__nv_bfloat16 *)dst);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}
int pack_conv_weight(const float *w, int cout, int cin, int ksz, void *dst, cudaStream_t st)
{
    return pack_conv_weight2(w, nullptr, cout, cin, ksz, dst, st);
}

__global__ void k_split_from_nchw(const float *__restrict__ src, int n_img, int C, int H, int W, __nv_bfloat16 *__restrict__ dst,
                                  size_t plane)
{
    const size_t count = (size_t)n_img * H * W * C;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (size_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const size_t p = i / C;
        const int x = (int)(p % W), y = (int)((p / W) % H), n = (int)(p / ((size_t)W * H));
        __nv_bfloat16 hi, lo;
        split_bf16(src[(((size_t)n * C + c) * H + y) * W + x], hi, lo);
        dst[i] = hi;
        dst[plane + i] = lo;
    }
}
__global__ void k_split_to_nchw(const __nv_bfloat16 *__restrict__ src, size_t plane, int n_img, int C, int H, int W,
                                float *__restrict__ dst)
{
    const size_t count = (size_t)n_img * H * W * C;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (size_t)gridDim.x * blockDim.x) {
        const int x = (int)(i % W), y = (int)((i / W) % H);
        const int c = (int)((i / ((size_t)W * H)) % C), n = (int)(i / ((size_t)W * H * C));
        const size_t s = (((size_t)n * H + y) * W + x) * C + c;
        dst[i] = join_bf16(src[s], src[plane + s]);
    }
}
int split_from_nchw_planes(const float *src, int n_img, int C, int H, int W, __nv_bfloat16 *dst, size_t plane, cudaStream_t st)
{
    const size_t count = (size_t)n_img * H * W * C;
    k_split_from_nchw<<<(unsigned)ceil_div64((int64_t)count, 256), 256, 0, st>>>(src, n_img, C, H, W, dst, plane);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}
int split_to_nchw_planes(const __nv_bfloat16 *src, size_t plane, int n_img, int C, int H, int W, float *dst, cudaStream_t st)
{
    const size_t count = (size_t)n_img * H * W * C;
    k_split_to_nchw<<<(unsigned)ceil_div64((int64_t)count, 256), 256, 0, st>>>(src, plane, n_img, C, H, W, dst);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}
int split_from_nchw(const float *src, int n_img, int C, int H, int W, __nv_bfloat16 *dst, cudaStream_t st)
{
    return split_from_nchw_planes(src, n_img, C, H, W, dst, (size_t)n_img * H * W * C, st);
}
int split_to_nchw(const __nv_bfloat16 *src, int n_img, int C, int H, int W, float *dst, cudaStream_t st)
{
    return split_to_nchw_planes(src, (size_t)n_img * H * W * C, n_img, C, H, W, dst, st);
}

} // namespace esr

// ------------------------------------------------------------------------------------------------
// C ABI (layer level)
// ------------------------------------------------------------------------------------------------
using namespace esr;

static SplitTensor mk_split(const void *p, int n_img, int H, int W, int C)
{
    SplitTensor t;
    t.base = (__nv_bfloat16 *)const_cast<void *>(p);
    t.n_img = n_img; t.H = H; t.W = W; t.C = C;
    return t;
}

static int conv_tc_abi(const esr_conv_desc *c, const int *src_chunks, const int *chunk_img_step, esr_stream_t stream)
{
    ESR_REQUIRE(c, "esr_conv_tc: null descriptor");
    ConvTCDesc d;
    d.n_src = c->n_src;
    for (int s = 0; s < c->n_src && s < TC_MAX_SRC; ++s) {
        d.src[s] = mk_split(c->src[s], c->src_n_img[s], c->H, c->W, c->src_C[s]);
        d.src_img[s] = c->src_img[s];
        if (src_chunks) d.src_chunks[s] = src_chunks[s];
        if (chunk_img_step) d.chunk_img_step[s] = chunk_img_step[s];
    }
    d.ntaps = c->ntaps; d.cout = c->cout; d.wpacked = c->wpacked; d.bias = c->bias; d.n_img = c->n_img;
    d.act = c->act; d.act_from = c->act_from; d.res_mode = c->res_mode; d.epi_mode = c->epi_mode;
    if (c->res) { d.res = mk_split(c->res, c->res_n_img, c->H, c->W, c->res_C); d.res_img = c->res_img; }
    if (c->out) { d.out = mk_split(c->out, c->out_n_img, c->H, c->W, c->out_C); d.out_coff = c->out_coff; }
    d.out_f32 = c->out_f32; d.out_f32_C = c->out_f32_C;
    if (c->h_prev) d.h_prev = mk_split(c->h_prev, c->h_n_img, c->H, c->W, 64);
    d.z_buf = c->z_buf;
    ConvTCArgs args;
    int rc = conv_tc_prepare(d, &args);
    if (rc) return rc;
    return conv_tc_launch(args, (cudaStream_t)stream);
}
extern "C" int esr_conv_tc(const esr_conv_desc *c, esr_stream_t stream) { return conv_tc_abi(c, nullptr, nullptr, stream); }
extern "C" int esr_conv_tc_chunked(const esr_conv_desc *c, const int *src_chunks, const int *chunk_img_step, esr_stream_t stream)
{
    return conv_tc_abi(c, src_chunks, chunk_img_step, stream);
}
extern "C" size_t esr_conv_weight_bytes(int cout, int cin, int ksz) { return tc_packed_weight_bytes(cout, cin, ksz * ksz); }
extern "C" int esr_pack_conv_weight(const float *w0, const float *w1, int cout_each, int cin, int ksz, void *dst, esr_stream_t st)
{
    return pack_conv_weight2(w0, w1, cout_each, cin, ksz, dst, (cudaStream_t)st);
}
extern "C" int esr_split_from_nchw(const float *src, int n_img, int C, int H, int W, void *dst, esr_stream_t st)
{
    return split_from_nchw(src, n_img, C, H, W, (__nv_bfloat16 *)dst, (cudaStream_t)st);
}
extern "C" int esr_split_to_nchw(const void *src, int n_img, int C, int H, int W, float *dst, esr_stream_t st)
{
    return split_to_nchw((const __nv_bfloat16 *)src, n_img, C, H, W, dst, (cudaStream_t)st);
}
