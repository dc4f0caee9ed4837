// events.cu -- the integer/byte side of the hot path on sm_90a:
//   events -> polarity count images (atomic scatter), dense counts / stacks -> time-sorted event lists
//   (round-half-even -> exclusive scan -> expand -> stable LSD radix sort on (sample, t) -> padded rows).
// Reference behaviour restated from dataloader/encodings.py:243-304, dataloader/h5dataset.py:508-528,
// dataloader/cython_cnt2event/cnt2event.pyx:18-116, dataloader/cython_event_redistribute/event_redistribute.pyx:17-153.
// All of this is HBM/L2-bound integer work: coalesced streaming reads, L2-resident atomics, no tensor cores.
#include "common.cuh"
#include <cstdlib>

namespace esr {

// =============================================================================================
// 1. events -> count images
// =============================================================================================
// One thread per event (grid-stride inside a frame).  Each event contributes ps*ps to its polarity
// channel (encodings.py:296-302: ps * mask where mask is ps with the other sign zeroed).
// Quirk bookkeeping (encodings.py:251-256 mutates xs/ys in place during the FIRST, positive, call):
//   out-of-range event:  positive -> dropped (its weight was zeroed);  negative -> lands on neg[0,0]
//   because by the second call its coordinates are already (0,0) and nothing masks it any more.
__global__ void __launch_bounds__(256)
k_scatter_cnt(float *__restrict__ xs, float *__restrict__ ys, const float *__restrict__ ps,
              const int64_t *__restrict__ frame_off, int64_t n_single, int H, int W, float w_lr, float w_hr, float h_lr,
              float h_hr, int do_lift, int writeback, float *__restrict__ out)
{
    const int f = blockIdx.y;
    const int64_t beg = frame_off ? frame_off[f] : 0, end = frame_off ? frame_off[f + 1] : n_single;
    float *img = out + (size_t)f * 2 * H * W;
    const float fW = (float)W, fH = (float)H;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = beg + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < end; i += stride) {
        float x = xs[i], y = ys[i];
        const float p = ps[i];
        if (do_lift) {
            // h5dataset.py:515 then :526 -- two separately rounded fp32 ops; intrinsics forbid FMA contraction
            x = __fmul_rn(__fdiv_rn(x, w_lr), w_hr);
            y = __fmul_rn(__fdiv_rn(y, h_lr), h_hr);
        }
        const bool oor = (x >= fW) | (x < 0.0f) | (y >= fH) | (y < 0.0f);
        float vpos = __fmul_rn(p, p < 0.0f ? 0.0f : p);
        const float vneg = __fmul_rn(p, p > 0.0f ? 0.0f : p);
        float vn = vneg;
        if (oor) {
            x = 0.0f; y = 0.0f; vpos = 0.0f;
            // writeback == 2, the order of H5Dataset.__getitem__ (h5dataset.py:337-354): create_stack_encoding has already zeroed x, y AND p
            // of out-of-range events in place when the frame holds more than 3 events (encodings.py:219-220, 251-256), so they add nothing
            if (writeback == 2 && end - beg > 3) vn = 0.0f;
        }
        const long long xi = (long long)x, yi = (long long)y;   // .long(): truncation toward zero
        const size_t pix = (size_t)yi * W + (size_t)xi;
        if (vpos != 0.0f) atomicAdd(img + pix, vpos);
        if (vn != 0.0f) atomicAdd(img + (size_t)H * W + pix, vn);
        if (writeback == 1 && oor) { xs[i] = 0.0f; ys[i] = 0.0f; }
    }
}

// Measured dead end (profiles/r1_notes.md): tiling the image over the shared memory of an 8/16-CTA cluster and routing
// the contributions with distributed-shared-memory reductions (red.shared::cluster.add.u32) is exact but 3x SLOWER than
// the L2 atomics above (48 vs 142 G events/s at 1e8 events onto 256x256); shared-memory fp32 adds compile to CAS loops.

// events_to_image (encodings.py:243-268): one image, raw weights ps, out-of-range events dropped and
// xs/ys/ps zeroed in place when writeback is set.
__global__ void __launch_bounds__(256)
k_scatter_image(float *__restrict__ xs, float *__restrict__ ys, float *__restrict__ ps, int64_t n, int H, int W,
                int writeback, float *__restrict__ img)
{
    const float fW = (float)W, fH = (float)H;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const float x = xs[i], y = ys[i], p = ps[i];
        const bool oor = (x >= fW) | (x < 0.0f) | (y >= fH) | (y < 0.0f);
        if (oor) {
            if (writeback) { xs[i] = 0.0f; ys[i] = 0.0f; ps[i] = 0.0f; }
            continue;
        }
        if (p != 0.0f) atomicAdd(img + (size_t)(long long)y * W + (size_t)(long long)x, p);
    }
}

// time-bin slice bounds of events_to_stack_no_polarity (encodings.py:204-240) with the reference's own
// binary_search_torch_tensor (encodings.py:77-99) -- including its early exits on exact matches, which decide which of
// several equal timestamps ends a bin.  One thread per bin; fp32 arithmetic rounded step by step like torch's.
__global__ void k_time_bin_bounds(const float *__restrict__ ts, long long n, int B, long long *__restrict__ out)
{
    const int bi = blockIdx.x * blockDim.x + threadIdx.x;
    if (bi >= B) return;
    const float t0 = ts[0];
    const float dt = __fadd_rn(__fsub_rn(ts[n - 1], t0), 1e-6f);            // ts[-1]-ts[0] + 1e-6
    const float delta = __fdiv_rn(dt, (float)B);
    const float tstart = __fadd_rn(t0, __fmul_rn(delta, (float)bi));
    const float tend = __fadd_rn(tstart, delta);
    for (int side = 0; side < 2; ++side) {
        const float x = side == 0 ? tstart : tend;
        long long l = 0, r = n - 1, res = 0;
        bool found = false;
        while (l <= r) {
            if (ts[l] == x) { res = l; found = true; break; }
            if (ts[r] == x) { res = r; found = true; break; }
            const long long mid = l + (r - l) / 2;
            const float mv = ts[mid];
            if (mv == x) { res = mid; found = true; break; }
            else if (mv < x) l = mid + 1;
            else r = mid - 1;
        }
        if (!found) res = side == 0 ? l : r;
        out[2 * bi + side] = side == 0 ? res : res + 1;                      // end = search(..., side='right') + 1
    }
}

// events_to_voxel (encodings.py:271-286): bin b accumulates ps * max(0, 1 - |ts*(nb-1) - b|) through events_to_image.
// Quirk kept: the first bin's call zeroes out-of-range xs/ys in place, so in bins >= 1 those events are no longer
// out of range and their weight lands on pixel (0,0).
__global__ void __launch_bounds__(256)
k_scatter_voxel(float *__restrict__ xs, float *__restrict__ ys, const float *__restrict__ ts, const float *__restrict__ ps,
                long long n, int nb, int H, int W, int writeback, float *__restrict__ out)
{
    const float fW = (float)W, fH = (float)H;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        float x = xs[i], y = ys[i];
        const float p = ps[i];
        const float tt = __fmul_rn(ts[i], (float)(nb - 1));
        const bool oor = (x >= fW) | (x < 0.0f) | (y >= fH) | (y < 0.0f);
        if (oor) { x = 0.0f; y = 0.0f; }
        const size_t pix = (size_t)(long long)y * W + (size_t)(long long)x;
        for (int b = 0; b < nb; ++b) {
            const float w = fmaxf(0.0f, __fsub_rn(1.0f, fabsf(__fsub_rn(tt, (float)b))));
            const float v = __fmul_rn(p, w);
            if (oor && b == 0) continue;                                     // dropped only in the first bin
            if (v != 0.0f) atomicAdd(out + (size_t)b * H * W + pix, v);
        }
        if (writeback && oor) { xs[i] = 0.0f; ys[i] = 0.0f; }
    }
}

// events_to_mask (encodings.py:307-331): mask[(long)y,(long)x] = |ps| with accumulate=False, i.e. the LAST event that
// hits a pixel decides (torch's CPU index_put_ walks the indices in order).  Out-of-range events are zeroed in place
// first, so they write 0 to pixel (0,0) when they come last.  Two passes: atomicMax of the event index per pixel, then
// the winning event writes its |ps|.
__global__ void __launch_bounds__(256)
k_mask_last_index(float *__restrict__ xs, float *__restrict__ ys, float *__restrict__ ps, long long n, int H, int W,
                  int writeback, int *__restrict__ last)
{
    const float fW = (float)W, fH = (float)H;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        float x = xs[i], y = ys[i];
        const bool oor = (x >= fW) | (x < 0.0f) | (y >= fH) | (y < 0.0f);
        if (oor) { x = 0.0f; y = 0.0f; if (writeback) { xs[i] = 0.0f; ys[i] = 0.0f; ps[i] = 0.0f; } }
        atomicMax(last + (size_t)(long long)y * W + (size_t)(long long)x, (int)i);
    }
}
__global__ void __launch_bounds__(256)
k_mask_write(const float *__restrict__ xs, const float *__restrict__ ys, const float *__restrict__ ps, long long n, int H, int W,
             const int *__restrict__ last, float *__restrict__ out)
{
    const float fW = (float)W, fH = (float)H;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        float x = xs[i], y = ys[i], p = ps[i];
        const bool oor = (x >= fW) | (x < 0.0f) | (y >= fH) | (y < 0.0f);
        if (oor) { x = 0.0f; y = 0.0f; p = 0.0f; }
        const size_t pix = (size_t)(long long)y * W + (size_t)(long long)x;
        if (last[pix] == (int)i) out[pix] = fabsf(p);
    }
}

// =============================================================================================
// 2. exclusive scan of uint32 (multi-level, tile = 1024 threads x 4)
// =============================================================================================
constexpr int SCAN_THREADS = 1024;
constexpr int SCAN_TILE = SCAN_THREADS * 4;

__global__ void __launch_bounds__(SCAN_THREADS)
k_scan_tiles(const uint32_t *__restrict__ in, uint32_t *__restrict__ out, uint32_t *__restrict__ tile_sums, int64_t n)
{
    __shared__ uint32_t warp_sums[32];
    const int64_t base = (int64_t)blockIdx.x * SCAN_TILE + (int64_t)threadIdx.x * 4;
    uint32_t v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) v[k] = (base + k < n) ? in[base + k] : 0u;
    const uint32_t tsum = v[0] + v[1] + v[2] + v[3];
    uint32_t incl = tsum;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        uint32_t t = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += t;
    }
    if (lane == 31) warp_sums[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        uint32_t w = warp_sums[lane];
        uint32_t wi = w;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            uint32_t t = __shfl_up_sync(0xffffffffu, wi, d);
            if (lane >= d) wi += t;
        }
        warp_sums[lane] = wi - w;                 // exclusive prefix of warp totals
        if (lane == 31 && tile_sums) tile_sums[blockIdx.x] = wi;
    }
    __syncthreads();
    uint32_t run = warp_sums[warp] + incl - tsum;  // exclusive prefix of this thread within the tile
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        if (base + k < n) out[base + k] = run;
        run += v[k];
    }
}

__global__ void __launch_bounds__(SCAN_THREADS)
k_scan_add(uint32_t *__restrict__ out, const uint32_t *__restrict__ tile_prefix, int64_t n)
{
    const uint32_t add = tile_prefix[blockIdx.x];
    const int64_t base = (int64_t)blockIdx.x * SCAN_TILE + (int64_t)threadIdx.x * 4;
#pragma unroll
    for (int k = 0; k < 4; ++k)
        if (base + k < n) out[base + k] += add;
}

static size_t scan_ws_elems(int64_t n)
{
    size_t tot = 0;
    while (n > SCAN_TILE) { n = ceil_div64(n, SCAN_TILE); tot += align_up((size_t)n, 64); }
    return tot + 64;
}

// in-place allowed (in == out).  ws needs scan_ws_elems(n) uint32.
// defer_add: skip the final pass over `out`; out[i] is then exclusive WITHIN its SCAN_TILE and the consumer adds
// (*tile_prefix)[i / SCAN_TILE] itself (nullptr when there is a single tile).
static int exclusive_scan_u32(const uint32_t *in, uint32_t *out, int64_t n, uint32_t *ws, cudaStream_t st,
                              const uint32_t **tile_prefix = nullptr)
{
    if (tile_prefix) *tile_prefix = nullptr;
    if (n <= 0) return ESR_OK;
    const int64_t nt = ceil_div64(n, SCAN_TILE);
    if (nt == 1) {
        k_scan_tiles<<<1, SCAN_THREADS, 0, st>>>(in, out, nullptr, n);
        ESR_LAUNCH_CHECK();
        return ESR_OK;
    }
    k_scan_tiles<<<(unsigned)nt, SCAN_THREADS, 0, st>>>(in, out, ws, n);
    ESR_LAUNCH_CHECK();
    int rc = exclusive_scan_u32(ws, ws, nt, ws + align_up((size_t)nt, 64), st);
    if (rc) return rc;
    if (tile_prefix) { *tile_prefix = ws; return ESR_OK; }
    k_scan_add<<<(unsigned)nt, SCAN_THREADS, 0, st>>>(out, ws, n);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}

// =============================================================================================
// 3. round + count (phase 1 of cnt2event / event_redistribute)
// =============================================================================================
// grid = (tiles per sample, B).  counts[slot] = number of events the slot emits; per-sample stats are
// reduced in the block and added with one atomic per block.
template <bool VEC>
__global__ void __launch_bounds__(256)
k_expand_count(const float *__restrict__ vals, int64_t S, int kind, uint32_t *__restrict__ counts,
               unsigned long long *__restrict__ stats /*[B,4]: sum(as i64), nev, neg, maxn*/)
{
    const int b = blockIdx.y;
    const float *v = vals + (size_t)b * S;
    uint32_t *c = counts + (size_t)b * S;
    long long sum = 0, nev = 0;
    int neg = 0;
    unsigned int mx = 0;
    auto one = [&](float x) -> unsigned int {
        const float r = rintf(x);                  // numpy round(): half to even (cnt2event.pyx:31)
        const long long ri = (long long)r;
        sum += ri;
        unsigned int n;
        if (kind == 0) { if (ri < 0) { neg = 1; n = 0; } else n = (unsigned int)ri; }
        else n = (unsigned int)(ri < 0 ? -ri : ri);
        nev += n;
        mx = max(mx, n);
        return n;
    };
    if constexpr (VEC) {                           // S % 4 == 0 and 16-byte aligned bases: 16-byte loads / stores
        const int64_t S4 = S >> 2;
        for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < S4; q += (int64_t)gridDim.x * blockDim.x) {
            const float4 x = __ldg(reinterpret_cast<const float4 *>(v) + q);
            reinterpret_cast<uint4 *>(c)[q] = make_uint4(one(x.x), one(x.y), one(x.z), one(x.w));
        }
    } else {
        for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < S; s += (int64_t)gridDim.x * blockDim.x) c[s] = one(v[s]);
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        sum += __shfl_xor_sync(0xffffffffu, sum, d);
        nev += __shfl_xor_sync(0xffffffffu, nev, d);
        neg |= __shfl_xor_sync(0xffffffffu, neg, d);
        mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, d));
    }
    __shared__ long long s_sum[8], s_nev[8];
    __shared__ int s_neg[8];
    __shared__ unsigned int s_mx[8];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) { s_sum[warp] = sum; s_nev[warp] = nev; s_neg[warp] = neg; s_mx[warp] = mx; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < 8; ++w) { sum += s_sum[w]; nev += s_nev[w]; neg |= s_neg[w]; mx = max(mx, s_mx[w]); }
        unsigned long long *st = stats + (size_t)b * 4;
        if (sum != 0) atomicAdd(st + 0, (unsigned long long)sum);   // two's complement add == signed add
        if (nev != 0) atomicAdd(st + 1, (unsigned long long)nev);
        if (neg) atomicOr(st + 2, 1ull);
        if (mx) atomicMax(st + 3, (unsigned long long)mx);
    }
}

// =============================================================================================
// 4. expand: one sort item per event, in emission order
// =============================================================================================
// item = { t_bits | (negative polarity << 31), global slot }.  t >= 0 always, so bit 31 is free.
struct __align__(8) Item { uint32_t tkey; uint32_t slot; };

// numpy.linspace(t0, t1, n)[j] in float64, rounded once to fp32 (cnt2event.pyx:74; event_redistribute.pyx:63).
// __d*_rn intrinsics keep the three float64 roundings separate (no FMA), like numpy's array ops.
__device__ __forceinline__ float linspace_f32(double t0, double t1, unsigned int n, unsigned int j)
{
    if (n == 1) return (float)t0;
    if (j == n - 1) return (float)t1;
    const double step = __ddiv_rn(__dsub_rn(t1, t0), (double)(n - 1));
    return (float)__dadd_rn(__dmul_rn((double)j, step), t0);
}

// Compact keys (cnt2event, linear timestamps, max count <= 255): the timestamp of event (n, j) is one of the few values
// float32(linspace(0,1,n)[j]); `rank[n*rank_m + j]` is its index among the sorted distinct values, so the sort key is
// ceil(log2(#distinct)) bits instead of 30 and one or two radix passes replace four.  The item then carries
// rank | j << 16 | negative << 31 and the timestamp is re-derived from (n, j) when the row is written.
// one slot with n > 0 events starting at output offset `off`
__device__ __forceinline__ void emit_slot(int64_t s, uint32_t n, uint32_t off, const float *__restrict__ vals, int C, int HW, int kind,
                                          int mode, const double *__restrict__ rnd, const uint16_t *__restrict__ rank, int rank_m,
                                          Item *__restrict__ items)
{
    uint32_t negbit;
    double t0 = 0.0, t1 = 1.0;
    float t0f = 0.0f, t1f = 1.0f;
    if (kind == 0) {
        negbit = ((uint32_t)s / (uint32_t)HW) & 1u;           // channel 1 = negative (cnt2event.pyx:80-90); slots < 2^32
    } else {
        negbit = vals[s] < 0.0f ? 1u : 0u;                    // p = sign(value); P index ignored
        const int c = (int)(((uint32_t)s / (uint32_t)HW) % (uint32_t)C);
        // cdef float t0, t1 <- float64 expressions (event_redistribute.pyx:61-62)
        t0f = (float)__dadd_rn(__ddiv_rn((double)c, (double)C), __ddiv_rn(1.0, (double)(100 * C)));
        t1f = (float)__ddiv_rn((double)(c + 1), (double)C);
        t0 = (double)t0f; t1 = (double)t1f;
    }
    if (rank) {                                                   // compact-key path (kind 0, mode 0, n <= rank_m)
        const uint16_t *rk = rank + (size_t)n * rank_m;
        for (uint32_t j = 0; j < n; ++j) {
            Item it;
            it.tkey = (uint32_t)rk[j] | (j << 16) | (negbit << 31);
            it.slot = (uint32_t)s;
            items[(size_t)off + j] = it;
        }
        return;
    }
    for (uint32_t j = 0; j < n; ++j) {
        float t;
        if (mode == 0) t = linspace_f32(t0, t1, n, j);
        else if (kind == 0) t = (float)rnd[(size_t)off + j];
        else t = (float)__dadd_rn(__dmul_rn(rnd[(size_t)off + j], (double)__fsub_rn(t1f, t0f)), t0);
        Item it;
        it.tkey = __float_as_uint(t) | (negbit << 31);
        it.slot = (uint32_t)s;
        items[(size_t)off + j] = it;
    }
}

// VEC (total_slots % 4 == 0, 16-byte aligned counts / offs): a thread takes 4 consecutive slots, so the count and offset
// loads of a group are two independent 16-byte loads in flight instead of a dependent chain per slot (the kernel is
// latency-bound: ncu long_scoreboard 15 per issue).
template <bool VEC>
__global__ void __launch_bounds__(256)
k_expand_emit(const float *__restrict__ vals, const uint32_t *__restrict__ counts, const uint32_t *__restrict__ offs,
              const uint32_t *__restrict__ offs_tile_prefix /*nullable: offs is exclusive per SCAN_TILE, add this*/, int64_t total_slots,
              int C, int HW, int kind, int mode, const double *__restrict__ rnd,
              const uint16_t *__restrict__ rank, int rank_m, Item *__restrict__ items)
{
    if constexpr (VEC) {
        const int64_t groups = total_slots >> 2;
        for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < groups; q += (int64_t)gridDim.x * blockDim.x) {
            const uint4 c4 = __ldg(reinterpret_cast<const uint4 *>(counts) + q);
            const uint4 o4 = __ldg(reinterpret_cast<const uint4 *>(offs) + q);
            if ((c4.x | c4.y | c4.z | c4.w) == 0) continue;
            const uint32_t tp = offs_tile_prefix ? offs_tile_prefix[(q * 4) / SCAN_TILE] : 0u;   // SCAN_TILE % 4 == 0: one tile per group
            const uint32_t cn[4] = {c4.x, c4.y, c4.z, c4.w}, co[4] = {o4.x, o4.y, o4.z, o4.w};
#pragma unroll
            for (int e = 0; e < 4; ++e)
                if (cn[e]) emit_slot(q * 4 + e, cn[e], co[e] + tp, vals, C, HW, kind, mode, rnd, rank, rank_m, items);
        }
    } else {
        for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < total_slots; s += (int64_t)gridDim.x * blockDim.x) {
            const uint32_t n = counts[s];
            if (n == 0) continue;
            emit_slot(s, n, offs[s] + (offs_tile_prefix ? offs_tile_prefix[s / SCAN_TILE] : 0u), vals, C, HW, kind, mode, rnd, rank, rank_m, items);
        }
    }
}

// =============================================================================================
// 5. stable LSD radix sort, 8 bits per pass, key = (sample, t)
// =============================================================================================
// pass p < 4 : digit = byte p of the fp32 timestamp bits (non-negative floats order like integers);
// pass 4     : digit = sample index (emission order is sample-major, so this pass only matters when
//              B > 1; B <= 256 per call, larger batches are split by the host wrapper).
// Each warp owns a contiguous sub-tile so that (warp, round, lane) order == input order => stable.
constexpr int RS_WARPS = 8;
constexpr int RS_IPT = 8;                                  // rounds of 32 consecutive items per warp
constexpr int RS_TILE = RS_WARPS * 32 * RS_IPT;            // 2048 items per block

// key digits: 4 passes over the raw fp32 timestamp bits, or 1-2 over the compact ranks (low 16 bits of tkey)
__device__ __forceinline__ uint32_t rs_digit(const Item &it, int pass) { return ((it.tkey & 0x7fffffffu) >> (8 * pass)) & 255u; }

// The sort is SEGMENTED by sample: events are emitted sample-major, so every pass only permutes items inside their own
// sample's range [start[b], start[b] + n[b]) and no pass over the sample index is needed.  Tiles are aligned to the sample
// starts: block -> (sample b, local tile lt) through the prefix of per-sample tile counts; the histogram of sample b's tiles
// lives at hist[256 * tile_prefix[b] + digit * T_b + lt], so ONE exclusive scan over the whole array yields, for each
// (sample, digit, tile), exactly the output offset of the sample-major, then key, then input-order (stable) arrangement.
struct SegTile { int b, lt, nt; int64_t base, end; uint32_t hoff; };

__device__ __forceinline__ SegTile rs_tile(const int64_t *__restrict__ seg /*[3][B]: start, n, tile_prefix*/, int B)
{
    const int64_t *start = seg, *nev = seg + B, *tpre = seg + 2 * B;
    int lo = 0, hi = B - 1;                                     // last b with tile_prefix[b] <= blockIdx.x
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (tpre[mid] <= (int64_t)blockIdx.x) lo = mid; else hi = mid - 1;
    }
    SegTile t;
    t.b = lo; t.lt = (int)((int64_t)blockIdx.x - tpre[lo]);
    t.nt = (int)((nev[lo] + RS_TILE - 1) / RS_TILE);
    t.base = start[lo] + (int64_t)t.lt * RS_TILE;
    t.end = start[lo] + nev[lo];
    t.hoff = (uint32_t)(256 * tpre[lo]) + (uint32_t)t.lt;
    return t;
}

__global__ void __launch_bounds__(RS_WARPS * 32)
k_radix_hist(const Item *__restrict__ items, const int64_t *__restrict__ seg, int B, int pass, uint32_t *__restrict__ hist)
{
    __shared__ uint32_t h[256];
    h[threadIdx.x] = 0;
    __syncthreads();
    const SegTile t = rs_tile(seg, B);
    for (int k = threadIdx.x; k < RS_TILE; k += RS_WARPS * 32) {
        const int64_t i = t.base + k;
        if (i < t.end) atomicAdd(&h[rs_digit(items[i], pass)], 1u);
    }
    __syncthreads();
    hist[t.hoff + (uint32_t)threadIdx.x * (uint32_t)t.nt] = h[threadIdx.x];
}

// Final pass writes the padded [B, maxlen, 4] rows directly instead of items.
__global__ void __launch_bounds__(RS_WARPS * 32)
k_radix_scatter(const Item *__restrict__ in, Item *__restrict__ out, const int64_t *__restrict__ seg, int B, int pass,
                uint32_t slots_per_sample, const uint32_t *__restrict__ hist_scanned /*segmented layout, exclusive*/,
                const uint32_t *__restrict__ hist_tile_prefix /*nullable: hist_scanned is exclusive per SCAN_TILE*/,
                int final_pass, float *__restrict__ rows, int64_t maxlen,
                int W, int H, const uint32_t *__restrict__ counts /*non-null: compact keys*/)
{
    __shared__ uint32_t cnt[RS_WARPS][256];     // per-warp digit counters -> then per-warp bases
    __shared__ uint32_t gbase[256];
    const SegTile t = rs_tile(seg, B);
    const int64_t n = t.end;
    for (int k = threadIdx.x; k < RS_WARPS * 256; k += RS_WARPS * 32) (&cnt[0][0])[k] = 0;
    {
        const uint32_t hi = t.hoff + (uint32_t)threadIdx.x * (uint32_t)t.nt;
        gbase[threadIdx.x] = hist_scanned[hi] + (hist_tile_prefix ? hist_tile_prefix[hi / SCAN_TILE] : 0u);
    }
    __syncthreads();

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t wbase = t.base + (int64_t)warp * (32 * RS_IPT);
    Item it[RS_IPT];
    uint32_t dig[RS_IPT], rank[RS_IPT];
#pragma unroll
    for (int r = 0; r < RS_IPT; ++r) {                     // all loads first: the ranking rounds below are serial (shared counters)
        const int64_t i = wbase + r * 32 + lane;
        if (i < n) it[r] = in[i];
    }
#pragma unroll
    for (int r = 0; r < RS_IPT; ++r) {
        const int64_t i = wbase + r * 32 + lane;
        const bool valid = i < n;
        dig[r] = valid ? rs_digit(it[r], pass) : 0xffffffffu;
        // rank among the lanes of this round holding the same digit
        const uint32_t peers = __match_any_sync(0xffffffffu, dig[r]);
        const uint32_t before = __popc(peers & ((1u << lane) - 1u));
        uint32_t old = 0;
        if (valid) {
            const int leader = __ffs(peers) - 1;
            if (lane == leader) { old = cnt[warp][dig[r]]; cnt[warp][dig[r]] = old + __popc(peers); }
            old = __shfl_sync(peers, old, leader);
        }
        rank[r] = old + before;
        __syncwarp();
    }
    __syncthreads();
    // exclusive prefix over warps for every digit (thread d handles digit d)
    {
        uint32_t run = 0;
        const int d = threadIdx.x;
#pragma unroll
        for (int w = 0; w < RS_WARPS; ++w) { const uint32_t c = cnt[w][d]; cnt[w][d] = run; run += c; }
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < RS_IPT; ++r) {
        const int64_t i = wbase + r * 32 + lane;
        if (i >= n) continue;
        const size_t pos = (size_t)gbase[dig[r]] + cnt[warp][dig[r]] + rank[r];
        if (!final_pass) { out[pos] = it[r]; continue; }
        const uint32_t slot = it[r].slot;
        const uint32_t b = slot / slots_per_sample;
        const uint32_t in_s = slot - b * slots_per_sample;
        const uint32_t x = in_s % (uint32_t)W, y = (in_s / (uint32_t)W) % (uint32_t)H;
        float4 row;
        row.x = (float)x; row.y = (float)y;
        row.z = counts ? linspace_f32(0.0, 1.0, counts[slot], (it[r].tkey >> 16) & 255u)
                       : __uint_as_float(it[r].tkey & 0x7fffffffu);
        row.w = (it[r].tkey >> 31) ? -1.0f : 1.0f;
        const int64_t local = (int64_t)pos - seg[b];              // seg[0..B) = sample starts
        reinterpret_cast<float4 *>(rows)[(size_t)b * maxlen + local] = row;
    }
}

} // namespace esr

// =============================================================================================
// C ABI
// =============================================================================================
using namespace esr;

extern "C" int esr_scatter_cnt(float *xs, float *ys, const float *ps, const int64_t *frame_off, int F,
                               int64_t n_max_frame, int H, int W, int lift_w_lr, int lift_w_hr, int lift_h_lr,
                               int lift_h_hr, int writeback, float *out, esr_stream_t stream)
{
    ESR_REQUIRE(F >= 0 && H > 0 && W > 0 && out, "esr_scatter_cnt: bad dims F=%d H=%d W=%d", F, H, W);
    cudaStream_t st = (cudaStream_t)stream;
    if (F == 0) return ESR_OK;
    ESR_CUDA_CHECK(cudaMemsetAsync(out, 0, sizeof(float) * (size_t)F * 2 * H * W, st));
    if (n_max_frame <= 0) return ESR_OK;
    ESR_REQUIRE(xs && ys && ps, "esr_scatter_cnt: null event arrays");
    ESR_REQUIRE(frame_off || F == 1, "esr_scatter_cnt: frame_off may be null only for a single frame");
    const int do_lift = (lift_w_lr > 0 && lift_w_hr > 0 && lift_h_lr > 0 && lift_h_hr > 0) ? 1 : 0;
    // enough blocks per frame to cover the longest frame at ~8 events per thread, capped for huge frames
    int64_t bx = ceil_div64(n_max_frame, 256 * 8);
    const int64_t cap = (int64_t)dev_info().sm_count * 16;
    if (bx > cap) bx = cap;
    if (bx < 1) bx = 1;
    ESR_REQUIRE(F <= 65535, "esr_scatter_cnt: at most 65535 frames per call");
    dim3 grid((unsigned)bx, (unsigned)F);
    k_scatter_cnt<<<grid, 256, 0, st>>>(xs, ys, ps, frame_off, n_max_frame, H, W, (float)lift_w_lr, (float)lift_w_hr,
                                         (float)lift_h_lr, (float)lift_h_hr, do_lift, writeback == 2 ? 2 : (writeback && !do_lift), out);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}

extern "C" int esr_scatter_image(float *xs, float *ys, float *ps, int64_t n, int H, int W, int writeback, float *out,
                                 esr_stream_t stream)
{
    ESR_REQUIRE(H > 0 && W > 0 && out && n >= 0, "esr_scatter_image: bad dims");
    cudaStream_t st = (cudaStream_t)stream;
    ESR_CUDA_CHECK(cudaMemsetAsync(out, 0, sizeof(float) * (size_t)H * W, st));
    if (n == 0) return ESR_OK;
    ESR_REQUIRE(xs && ys && ps, "esr_scatter_image: null event arrays");
    int64_t bx = ceil_div64(n, 256 * 8);
    const int64_t cap = (int64_t)dev_info().sm_count * 16;
    if (bx > cap) bx = cap;
    k_scatter_image<<<(unsigned)bx, 256, 0, st>>>(xs, ys, ps, n, H, W, writeback, out);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}

extern "C" int esr_scatter_mask(float *xs, float *ys, float *ps, int64_t n, int H, int W, int writeback, int32_t *last_tmp,
                                float *out, esr_stream_t stream)
{
    ESR_REQUIRE(H > 0 && W > 0 && out && last_tmp && n >= 0 && n < (1ll << 31), "esr_scatter_mask: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    ESR_CUDA_CHECK(cudaMemsetAsync(out, 0, sizeof(float) * (size_t)H * W, st));
    if (n == 0) return ESR_OK;
    ESR_REQUIRE(xs && ys && ps, "esr_scatter_mask: null event arrays");
    ESR_CUDA_CHECK(cudaMemsetAsync(last_tmp, 0xff, sizeof(int32_t) * (size_t)H * W, st));     // -1
    int64_t bx = ceil_div64(n, 256 * 4);
    const int64_t cap = (int64_t)dev_info().sm_count * 16;
    if (bx > cap) bx = cap;
    // pass 2 must see the ORIGINAL coordinates: with writeback the first pass zeroes them, which maps to the same pixel
    // (0,0) and weight 0 as the recomputed out-of-range case, so reading the mutated arrays is equivalent
    k_mask_last_index<<<(unsigned)bx, 256, 0, st>>>(xs, ys, ps, (long long)n, H, W, writeback, last_tmp);
    ESR_LAUNCH_CHECK();
    k_mask_write<<<(unsigned)bx, 256, 0, st>>>(xs, ys, ps, (long long)n, H, W, last_tmp, out);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}

extern "C" int esr_time_bin_bounds(const float *ts, int64_t n, int B, int64_t *bounds, esr_stream_t stream)
{
    ESR_REQUIRE(ts && bounds && n > 0 && B > 0, "esr_time_bin_bounds: bad arguments");
    k_time_bin_bounds<<<(B + 63) / 64, 64, 0, (cudaStream_t)stream>>>(ts, (long long)n, B, (long long *)bounds);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}

extern "C" int esr_scatter_voxel(float *xs, float *ys, const float *ts, const float *ps, int64_t n, int num_bins, int H, int W,
                                 int writeback, float *out, esr_stream_t stream)
{
    ESR_REQUIRE(H > 0 && W > 0 && num_bins > 0 && out && n >= 0, "esr_scatter_voxel: bad dims");
    cudaStream_t st = (cudaStream_t)stream;
    ESR_CUDA_CHECK(cudaMemsetAsync(out, 0, sizeof(float) * (size_t)num_bins * H * W, st));
    if (n == 0) return ESR_OK;
    ESR_REQUIRE(xs && ys && ts && ps, "esr_scatter_voxel: null event arrays");
    int64_t bx = ceil_div64(n, 256 * 4);
    const int64_t cap = (int64_t)dev_info().sm_count * 16;
    if (bx > cap) bx = cap;
    k_scatter_voxel<<<(unsigned)bx, 256, 0, st>>>(xs, ys, ts, ps, (long long)n, num_bins, H, W, writeback, out);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}

extern "C" int esr_expand_count(const float *vals, int B, int P, int C, int H, int W, int kind, int64_t *stats,
                                uint32_t *counts, esr_stream_t stream)
{
    ESR_REQUIRE(vals && stats && counts, "esr_expand_count: null pointer");
    ESR_REQUIRE(B > 0 && P > 0 && C > 0 && H > 0 && W > 0 && (kind == 0 || kind == 1), "esr_expand_count: bad dims");
    ESR_REQUIRE(kind != 0 || (P == 2 && C == 1), "esr_expand_count: cnt2event needs [B,2,H,W]");
    ESR_REQUIRE(B <= 256, "esr_expand_count: at most 256 samples per call");
    const int64_t S = (int64_t)P * C * H * W;
    ESR_REQUIRE((int64_t)B * S < (1ll << 32), "esr_expand_count: more than 2^32 slots");
    cudaStream_t st = (cudaStream_t)stream;
    ESR_CUDA_CHECK(cudaMemsetAsync(stats, 0, sizeof(int64_t) * 4 * (size_t)B, st));
    int64_t bx = ceil_div64(S, 256 * 4);
    const int64_t cap = (int64_t)dev_info().sm_count * 8;
    if (bx > cap) bx = cap;
    dim3 grid((unsigned)bx, (unsigned)B);
    const bool vec = S % 4 == 0 && ((uintptr_t)vals & 15) == 0 && ((uintptr_t)counts & 15) == 0;
    if (vec) k_expand_count<true><<<grid, 256, 0, st>>>(vals, S, kind, counts, reinterpret_cast<unsigned long long *>(stats));
    else k_expand_count<false><<<grid, 256, 0, st>>>(vals, S, kind, counts, reinterpret_cast<unsigned long long *>(stats));
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}

static size_t expand_ws_layout(int64_t slots, int64_t E, size_t *o_offs, size_t *o_scanws, size_t *o_items0,
                               size_t *o_items1, size_t *o_hist, size_t *o_histws, size_t *o_start)
{
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t r = off; off = align_up(off + bytes, 256); return r; };
    const int64_t nblk = ceil_div64(E > 0 ? E : 1, RS_TILE) + 256;   // sample-aligned tiles: at most one partial tile per sample more
    *o_offs = take(sizeof(uint32_t) * (size_t)slots);
    *o_scanws = take(sizeof(uint32_t) * scan_ws_elems(slots));
    *o_items0 = take(sizeof(Item) * (size_t)(E > 0 ? E : 1));
    *o_items1 = take(sizeof(Item) * (size_t)(E > 0 ? E : 1));
    *o_hist = take(sizeof(uint32_t) * 256 * (size_t)nblk);
    *o_histws = take(sizeof(uint32_t) * scan_ws_elems(256 * nblk));
    *o_start = take(sizeof(int64_t) * 3 * 256);                      // [start | n | tile_prefix] per sample
    return off;
}

extern "C" size_t esr_expand_workspace_bytes(int B, int P, int C, int H, int W, int64_t total_events)
{
    size_t a, b, c, d, e, f, g;
    return expand_ws_layout((int64_t)B * P * C * H * W, total_events, &a, &b, &c, &d, &e, &f, &g);
}

extern "C" int esr_expand_emit(const float *vals, uint32_t *counts, int B, int P, int C, int H, int W, int kind,
                               int mode, const double *rnd, const uint16_t *rank_table, int rank_m, int rank_bits,
                               const int32_t *active_host, const int64_t *start_host,
                               int64_t total_events, int64_t maxlen, float *out, void *workspace,
                               size_t workspace_bytes, esr_stream_t stream)
{
    ESR_REQUIRE(!rank_table || (kind == 0 && mode == 0 && rank_m >= 1 && rank_m <= 255 && rank_bits >= 1 && rank_bits <= 16),
                "esr_expand_emit: compact keys need cnt2event, linear timestamps and max count <= 255");
    ESR_REQUIRE(vals && counts && active_host && start_host && out && workspace, "esr_expand_emit: null pointer");
    ESR_REQUIRE(B > 0 && B <= 256 && (mode == 0 || mode == 1), "esr_expand_emit: bad B/mode");
    ESR_REQUIRE(mode == 0 || rnd, "esr_expand_emit: mode 1 needs the random stream");
    ESR_REQUIRE(total_events >= 0 && total_events < (1ll << 31), "esr_expand_emit: more than 2^31 events");
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t S = (int64_t)P * C * H * W, slots = (int64_t)B * S;
    if (total_events == 0) return ESR_OK;
    size_t o_offs, o_scanws, o_i0, o_i1, o_hist, o_histws, o_start;
    const size_t need = expand_ws_layout(slots, total_events, &o_offs, &o_scanws, &o_i0, &o_i1, &o_hist, &o_histws, &o_start);
    if (workspace_bytes < need) { set_error("esr_expand_emit: workspace %zu < %zu", workspace_bytes, need); return ESR_EWORKSPACE; }
    char *ws = (char *)workspace;
    uint32_t *offs = (uint32_t *)(ws + o_offs), *scanws = (uint32_t *)(ws + o_scanws);
    Item *items[2] = {(Item *)(ws + o_i0), (Item *)(ws + o_i1)};
    uint32_t *hist = (uint32_t *)(ws + o_hist), *histws = (uint32_t *)(ws + o_histws);
    int64_t *d_start = (int64_t *)(ws + o_start);

    // samples the reference treats as empty (rounded values sum to zero) emit nothing
    for (int b = 0; b < B; ++b)
        if (!active_host[b]) ESR_CUDA_CHECK(cudaMemsetAsync(counts + (size_t)b * S, 0, sizeof(uint32_t) * (size_t)S, st));
    // per-sample segments of the sort: start, event count, prefix of the per-sample tile counts
    int64_t seg_host[3 * 256];
    int64_t n_tiles_total = 0;
    for (int b = 0; b < B; ++b) {
        const int64_t nb = (b + 1 < B ? start_host[b + 1] : total_events) - start_host[b];
        seg_host[b] = start_host[b]; seg_host[B + b] = nb; seg_host[2 * B + b] = n_tiles_total;
        n_tiles_total += ceil_div64(nb, RS_TILE);
    }
    ESR_CUDA_CHECK(cudaMemcpyAsync(d_start, seg_host, sizeof(int64_t) * 3 * (size_t)B, cudaMemcpyHostToDevice, st));
    // (pageable source: the driver stages the bytes before the call returns, so the stack buffer is safe)

    const uint32_t *offs_tp = nullptr;
    int rc = exclusive_scan_u32(counts, offs, slots, scanws, st, &offs_tp);       // the emit kernel adds the tile prefixes itself
    if (rc) return rc;
    {
        const bool vec = slots % 4 == 0 && ((uintptr_t)counts & 15) == 0 && ((uintptr_t)offs & 15) == 0;
        int64_t bx = ceil_div64(slots, 256 * 4);
        const int64_t cap = (int64_t)dev_info().sm_count * 32;
        if (bx > cap) bx = cap;
        if (vec) k_expand_emit<true><<<(unsigned)bx, 256, 0, st>>>(vals, counts, offs, offs_tp, slots, C, H * W, kind, mode, rnd, rank_table, rank_m, items[0]);
        else k_expand_emit<false><<<(unsigned)bx, 256, 0, st>>>(vals, counts, offs, offs_tp, slots, C, H * W, kind, mode, rnd, rank_table, rank_m, items[0]);
        ESR_LAUNCH_CHECK();
    }
    const int64_t nblk = n_tiles_total;
    const int npass = rank_table ? (rank_bits + 7) / 8 : 4;          // key passes only: the sort is segmented by sample
    int cur = 0;
    for (int p = 0; p < npass; ++p) {
        k_radix_hist<<<(unsigned)nblk, RS_WARPS * 32, 0, st>>>(items[cur], d_start, B, p, hist);
        ESR_LAUNCH_CHECK();
        const uint32_t *hist_tp = nullptr;
        rc = exclusive_scan_u32(hist, hist, 256 * nblk, histws, st, &hist_tp);
        if (rc) return rc;
        const int fin = p == npass - 1;
        k_radix_scatter<<<(unsigned)nblk, RS_WARPS * 32, 0, st>>>(items[cur], items[cur ^ 1], d_start, B, p, (uint32_t)S,
                                                                  hist, hist_tp, fin, out, maxlen, W, H, rank_table ? counts : nullptr);
        ESR_LAUNCH_CHECK();
        cur ^= 1;
    }
    return ESR_OK;
}
