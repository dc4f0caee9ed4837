// wgrad_tc.cu -- weight gradient of a stride-1 3x3 (pad 1) / 1x1 convolution on the tensor cores (sm_90a, wgmma).
//
//   dw[co, ci, ky, kx] = sum over (image, y, x) of g[image, y, x, co] * x[image, y + ky - 1, x + kx - 1, ci]
//
// is, per tap, a GEMM whose reduction dimension is the PIXEL index: D[a-channel, b-channel] += A^T B with A and B both
// stored pixel-major (NHWC rows of 64 channels = one 128-byte shared-memory row per pixel).  That is exactly the
// MN-major SWIZZLE_128B operand layout of wgmma (canonical ((8,n),(8,k)) : ((1,LBO),(8,SBO)) in 16-byte units: 64
// channels contiguous in a row, 8 pixel rows per 1024-byte swizzle atom, SBO = 1024 between K atoms), so the same TMA
// boxes the forward kernel loads (64 ch x TW x TH pixels, tap shift + zero fill = padding) feed the MMA directly -- no
// transposition anywhere.  fp32 parity: operands are split bf16 (hi, lo), three MMAs per K step (lo*hi + hi*lo + hi*hi)
// into fp32 accumulators, like the forward.
//
// One CTA owns (128 M-side channels, 64 N-side channels, a group of <= 3 taps, a slice of the pixel tiles): each of its two
// consumer warpgroups keeps one 64 x 64 fp32 accumulator per tap in registers (M-side channels [64 w, 64 w + 64)), streams
// the pixel tiles through a TMA/mbarrier pipeline (the unshifted tensor once per tile, the shifted one once per tap) and adds
// its partial sums to dw with fp32 atomics at the end.  Which tensor sits on the 128-row M side is chosen per layer:
// g (Cout >= 128) or x (Cout == 64 and Cin >= 128); a 64-channel tensor on the M side is loaded twice (rows 64..127
// ignored).  Warps: 0-7 = MMA + epilogue (two warpgroups), 8 = TMA producer.
#include "tc_common.cuh"
#include "net.cuh"

namespace esr {

constexpr int WG_THREADS = 288;
constexpr int WG_TAPS = 3;                            // taps per CTA (accumulators: 3 x 32 registers per thread)
constexpr uint32_t WG_TILE = TC_BLOCK_M * 128u;       // one 64-channel x 128-pixel plane: 16 KB

struct WgradArgs {
    CUtensorMap gmap, xmap;           // 5-D (C, W, H, img, plane), box (64, TW, TH, 1, 1)
    float *dw;                        // [Cout][Cin][KK]
    int Cout, CoutPad, Cin, KK;       // g has CoutPad (64-multiple) channels, the first Cout are real
    int a_is_x;                       // 1: M side = x channels (shifted per tap), N side = g; 0: M side = g, N side = x
    int m_blocks, n_chunks, groups;   // grid decomposition
    int n_img, H, W, TW, TH, tiles_x, tiles_y, slices;
};

// DET: instead of the atomics, the CTA of slice s stores its tile to slot s of a.dw = [slices][Cout*Cin*KK] (every CTA of a
// slice owns distinct elements, and every slice walks at least one tile, so each slot is written in full); sum_slices adds them.
template <bool DET>
__device__ __forceinline__ void wgrad_tc_body(const WgradArgs &a)
{
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    // shared memory: [once buffers x2][per-tap ring x2][barriers]; sizes depend on which tensor is on the M side
    const uint32_t m_bytes = 4u * WG_TILE, n_bytes = 2u * WG_TILE;      // M side: 2 tiles x 2 planes; N side: 1 tile x 2 planes
    const uint32_t once_bytes = a.a_is_x ? n_bytes : m_bytes;           // the unshifted tensor (g)
    const uint32_t tap_bytes = a.a_is_x ? m_bytes : n_bytes;            // the shifted tensor (x)
    const uint32_t once_base = smem_base, ring_base = smem_base + 2u * once_bytes;
    const uint32_t bar_base = ring_base + 2u * tap_bytes;
    const uint32_t bar_gfull = bar_base, bar_gempty = bar_base + 16u, bar_xfull = bar_base + 32u, bar_xempty = bar_base + 48u;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    // block -> (M block, N chunk, tap group, slice)
    int bid = blockIdx.x;
    const int slice = bid % a.slices; bid /= a.slices;
    const int grp = bid % a.groups; bid /= a.groups;
    const int nch = bid % a.n_chunks; const int mblk = bid / a.n_chunks;
    const int tap0 = grp * WG_TAPS;
    const int ntap = a.KK == 1 ? 1 : WG_TAPS;
    const int m_ch = a.a_is_x ? a.Cin : a.CoutPad;               // channels of the M-side tensor as stored
    const int m_real = a.a_is_x ? a.Cin : a.Cout;
    const int m0 = mblk * 128;
    const bool m_dup = m0 + 64 >= m_ch;                                  // only 64 channels left on the M side
    const int n0 = nch * 64;
    const int tiles_per_img = a.tiles_x * a.tiles_y, n_tiles = a.n_img * tiles_per_img;

    if (threadIdx.x == 0) {
        for (int s = 0; s < 2; ++s) {
            mbar_init(bar_gfull + 8u * s, 1); mbar_init(bar_gempty + 8u * s, 8);
            mbar_init(bar_xfull + 8u * s, 1); mbar_init(bar_xempty + 8u * s, 8);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == 8) {
        if (elect_one_sync()) {
            uint32_t gs = 0, gph = 0, xs = 0, xph = 0;
            for (int t = slice; t < n_tiles; t += a.slices) {
                const int img = t / tiles_per_img, tr = t - img * tiles_per_img;
                const int y0 = (tr / a.tiles_x) * a.TH, x0 = (tr % a.tiles_x) * a.TW;
                // ---- g tile(s), unshifted
                mbar_wait(bar_gempty + 8u * gs, gph ^ 1u);
                mbar_expect_tx(bar_gfull + 8u * gs, once_bytes);
                const uint32_t gb = once_base + gs * once_bytes;
                if (!a.a_is_x) {                                         // M side: [hi: tile0, tile1][lo: tile0, tile1]
                    const int c1 = m_dup ? m0 : m0 + 64;
                    tma_load_5d(&a.gmap, bar_gfull + 8u * gs, gb, m0, x0, y0, img, 0);
                    tma_load_5d(&a.gmap, bar_gfull + 8u * gs, gb + WG_TILE, c1, x0, y0, img, 0);
                    tma_load_5d(&a.gmap, bar_gfull + 8u * gs, gb + 2u * WG_TILE, m0, x0, y0, img, 1);
                    tma_load_5d(&a.gmap, bar_gfull + 8u * gs, gb + 3u * WG_TILE, c1, x0, y0, img, 1);
                } else {
                    tma_load_5d(&a.gmap, bar_gfull + 8u * gs, gb, n0, x0, y0, img, 0);
                    tma_load_5d(&a.gmap, bar_gfull + 8u * gs, gb + WG_TILE, n0, x0, y0, img, 1);
                }
                if (++gs == 2) { gs = 0; gph ^= 1u; }
                // ---- x tile(s), one per tap, shifted; out-of-image pixels are zero-filled = the conv padding
                for (int j = 0; j < ntap; ++j) {
                    const int tap = tap0 + j;
                    const int dy = a.KK == 9 ? tap / 3 - 1 : 0, dx = a.KK == 9 ? tap % 3 - 1 : 0;
                    mbar_wait(bar_xempty + 8u * xs, xph ^ 1u);
                    mbar_expect_tx(bar_xfull + 8u * xs, tap_bytes);
                    const uint32_t xb = ring_base + xs * tap_bytes;
                    if (a.a_is_x) {
                        const int c1 = m_dup ? m0 : m0 + 64;
                        tma_load_5d(&a.xmap, bar_xfull + 8u * xs, xb, m0, x0 + dx, y0 + dy, img, 0);
                        tma_load_5d(&a.xmap, bar_xfull + 8u * xs, xb + WG_TILE, c1, x0 + dx, y0 + dy, img, 0);
                        tma_load_5d(&a.xmap, bar_xfull + 8u * xs, xb + 2u * WG_TILE, m0, x0 + dx, y0 + dy, img, 1);
                        tma_load_5d(&a.xmap, bar_xfull + 8u * xs, xb + 3u * WG_TILE, c1, x0 + dx, y0 + dy, img, 1);
                    } else {
                        tma_load_5d(&a.xmap, bar_xfull + 8u * xs, xb, n0, x0 + dx, y0 + dy, img, 0);
                        tma_load_5d(&a.xmap, bar_xfull + 8u * xs, xb + WG_TILE, n0, x0 + dx, y0 + dy, img, 1);
                    }
                    if (++xs == 2) { xs = 0; xph ^= 1u; }
                }
            }
        }
        return;
    }

    // ===================== consumers: warpgroup wg = M-side channels [m0 + 64 wg, +64) =====================
    const int wg = warp >> 2;
    float acc[WG_TAPS][32];
#pragma unroll
    for (int j = 0; j < WG_TAPS; ++j)
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[j][i] = 0.0f;
    uint32_t gs = 0, gph = 0, xs = 0, xph = 0;
    for (int t = slice; t < n_tiles; t += a.slices) {
        mbar_wait(bar_gfull + 8u * gs, gph);
        const uint32_t gb = once_base + gs * once_bytes;
#pragma unroll
        for (int j = 0; j < WG_TAPS; ++j) {
            if (j >= ntap) break;
            mbar_wait(bar_xfull + 8u * xs, xph);
            const uint32_t xb = ring_base + xs * tap_bytes;
            const uint32_t m_hi = (a.a_is_x ? xb : gb) + (uint32_t)wg * WG_TILE, m_lo = m_hi + 2u * WG_TILE;   // this warpgroup's M tile
            const uint32_t n_hi = a.a_is_x ? gb : xb, n_lo = n_hi + WG_TILE;                                   // N side planes
            const uint64_t dah = wgmma_desc(m_hi, WG_TILE), dal = wgmma_desc(m_lo, WG_TILE);
            const uint64_t dbh = wgmma_desc(n_hi, WG_TILE), dbl = wgmma_desc(n_lo, WG_TILE);
            acc_fence<32>(acc[j]);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 8; ++k) {                        // 8 x (K = 16 pixels = 16 rows = 2048 bytes)
                wgmma_rows<64, 1>(acc[j], dal + 128 * k, dbh + 128 * k);
                wgmma_rows<64, 1>(acc[j], dah + 128 * k, dbl + 128 * k);
                wgmma_rows<64, 1>(acc[j], dah + 128 * k, dbh + 128 * k);
            }
            wgmma_commit();
            wgmma_wait<0>();
            acc_fence<32>(acc[j]);
            if (lane == 0) mbar_arrive(bar_xempty + 8u * xs);
            if (++xs == 2) { xs = 0; xph ^= 1u; }
        }
        if (lane == 0) mbar_arrive(bar_gempty + 8u * gs);
        if (++gs == 2) { gs = 0; gph ^= 1u; }
    }
    if (slice >= n_tiles) return;

    // ===================== epilogue: accumulator fragments -> fp32 atomics into dw =====================
    const int w = warp & 3;
#pragma unroll
    for (int j = 0; j < WG_TAPS; ++j) {
        if (j >= ntap) break;
        const int tap = tap0 + j;
#pragma unroll
        for (int i = 0; i < 32; ++i) {
            const int m = wg * 64 + 16 * w + (lane >> 2) + 8 * ((i >> 1) & 1);   // accumulator row = M-side channel
            const int nc = n0 + 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);        // column = N-side channel
            const bool row_ok = (m < 64 || !m_dup) && (m0 + m < m_real);
            const int co = a.a_is_x ? nc : m0 + m, ci = a.a_is_x ? m0 + m : nc;
            if (row_ok && co < a.Cout) {
                if (DET) a.dw[(size_t)slice * a.Cout * a.Cin * a.KK + ((size_t)co * a.Cin + ci) * a.KK + tap] = acc[j][i];
                else atomicAdd(a.dw + ((size_t)co * a.Cin + ci) * a.KK + tap, acc[j][i]);
            }
        }
    }
}
__global__ void __launch_bounds__(WG_THREADS, 1) k_wgrad_tc(const __grid_constant__ WgradArgs a) { wgrad_tc_body<false>(a); }
__global__ void __launch_bounds__(WG_THREADS, 1) k_wgrad_tc_det(const __grid_constant__ WgradArgs a) { wgrad_tc_body<true>(a); }

// CTAs per (M block, N chunk, tap group): one CTA per SM in all.  (Every CTA ends with 128 x 64 x taps fp32 atomics; giving small
// problems fewer, longer CTAs was measured slower: min 6 tiles per CTA +0.3 ms, min 16 +2 ms per cfg2 training iteration --
// ESR_WGRAD_MIN_TILES to retest.)
static int wgrad_tc_slices(int n_tiles, int base)
{
    int slices = (dev_info().sm_count + base - 1) / base;
    static const int min_tiles = getenv("ESR_WGRAD_MIN_TILES") ? atoi(getenv("ESR_WGRAD_MIN_TILES")) : 1;
    if (slices > n_tiles / min_tiles) slices = n_tiles / min_tiles;
    if (slices < 1) slices = 1;
    return slices;
}

static void wgrad_tc_geometry(int B, int Cin, int H, int W, int Cout, int CoutPad, int ksz, WgradArgs &a)
{
    a.Cout = Cout; a.Cin = Cin; a.KK = ksz * ksz; a.CoutPad = CoutPad;
    a.a_is_x = (Cout == 64 && Cin >= 128) ? 1 : 0;
    a.TW = W >= 24 ? 32 : (W >= 12 ? 16 : 8); a.TH = TC_BLOCK_M / a.TW;
    const int m_ch = a.a_is_x ? Cin : CoutPad, n_ch = a.a_is_x ? CoutPad : Cin;
    a.m_blocks = (m_ch + 127) / 128; a.n_chunks = n_ch / 64; a.groups = ksz == 3 ? 9 / WG_TAPS : 1;
    a.n_img = B; a.H = H; a.W = W;
    a.tiles_x = (W + a.TW - 1) / a.TW; a.tiles_y = (H + a.TH - 1) / a.TH;
    a.slices = wgrad_tc_slices(B * a.tiles_x * a.tiles_y, a.m_blocks * a.n_chunks * a.groups);
}

// partial buffer of the deterministic variant: [slices][Cout][Cin][KK] fp32
size_t wgrad_tc_part_bytes(int B, int Cin, int H, int W, int Cout, int CoutPad, int ksz)
{
    WgradArgs a;
    memset(&a, 0, sizeof(a));
    wgrad_tc_geometry(B, Cin, H, W, Cout, CoutPad, ksz, a);
    return (size_t)a.slices * Cout * Cin * ksz * ksz * 4;
}

// x_split: split NHWC [2][B][H][W][Cin]; g_split: split NHWC [2][B][H][W][CoutPad] (channels >= Cout zero); dw pre-zeroed.
// part != NULL: deterministic mode -- per-slice partial tiles into part (wgrad_tc_part_bytes), then the ordered sum into dw.
int wgrad_tc(const __nv_bfloat16 *x_split, const __nv_bfloat16 *g_split, int B, int Cin, int H, int W, int Cout, int CoutPad, int ksz,
             float *dw, float *part, cudaStream_t st)
{
    if (Cin % 64 != 0 || CoutPad % 64 != 0 || CoutPad < Cout || (ksz != 3 && ksz != 1)) return ESR_EINVAL;
    int rc;
    SplitTensor xs; xs.base = const_cast<__nv_bfloat16 *>(x_split); xs.n_img = B; xs.H = H; xs.W = W; xs.C = Cin;
    SplitTensor gs; gs.base = const_cast<__nv_bfloat16 *>(g_split); gs.n_img = B; gs.H = H; gs.W = W; gs.C = CoutPad;
    WgradArgs a;
    memset(&a, 0, sizeof(a));
    wgrad_tc_geometry(B, Cin, H, W, Cout, CoutPad, ksz, a);
    a.dw = part ? part : dw;
    if ((rc = tc_make_amap(gs, a.TW, a.TH, &a.gmap))) return rc;
    if ((rc = tc_make_amap(xs, a.TW, a.TH, &a.xmap))) return rc;
    const int base = a.m_blocks * a.n_chunks * a.groups;
    const size_t smem = 1024 + 2 * (size_t)(4 * WG_TILE) + 2 * (size_t)(2 * WG_TILE) + 64;
    static size_t attr_done = 0, attr_det = 0;
    if (!part) {
        if (smem > attr_done) {
            ESR_CUDA_CHECK(cudaFuncSetAttribute(k_wgrad_tc, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            attr_done = smem;
        }
        k_wgrad_tc<<<(unsigned)(base * a.slices), WG_THREADS, smem, st>>>(a);
        ESR_LAUNCH_CHECK();
        return ESR_OK;
    }
    if (smem > attr_det) {
        ESR_CUDA_CHECK(cudaFuncSetAttribute(k_wgrad_tc_det, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr_det = smem;
    }
    k_wgrad_tc_det<<<(unsigned)(base * a.slices), WG_THREADS, smem, st>>>(a);
    ESR_LAUNCH_CHECK();
    return sum_slices(part, a.slices, (size_t)Cout * Cin * ksz * ksz, dw, st);
}

} // namespace esr
