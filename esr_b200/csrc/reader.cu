// reader.cu -- device side of the columnar event reader (SURVEY 8f rank 2): window indexing by timestamp search and the
// gather of per-frame event slices from the (pinned, host-mapped or device-resident) columns straight into the fp32 SoA the
// count-scatter kernels consume.
//
// Replaces, for whole batches at once:
//   BaseDataset.binary_search_h5_dset   dataloader/base_dataset.py:78-91 (= dataloader/binary_search/binary_search.pyx:17-38):
//       bisection over the sorted float64 timestamps that returns `mid` as soon as dset[mid] == x, else the left insertion
//       point -- with duplicate timestamps this is NOT numpy.searchsorted; the same probe sequence is reproduced so the indices
//       are bit-identical;
//   H5Dataset.get_events / get_gt_events + BaseDataset.event_formatting   dataloader/h5dataset.py:492-506,
//       dataloader/base_dataset.py:26-33: int16 x / y and float64 t / p slices -> float32, t normalised per frame
//       (ts - ts[0]) / (ts[-1] - ts[0] + 1e-6) in float32 arithmetic, as torch evaluates it;
//   H5Dataset.augment_event + SequenceDataset's paused frames   dataloader/h5dataset.py:652-670, 769-789: per-frame flips
//       and the zero event of a paused frame, applied in registers during the same gather.
#include "common.cuh"

namespace esr {

__global__ void __launch_bounds__(256)
k_ts_search(const double *__restrict__ ts, long long n, const double *__restrict__ q, long long nq, long long *__restrict__ out)
{
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nq; i += (long long)gridDim.x * blockDim.x) {
        const double x = q[i];
        long long l = 0, r = n - 1, res = -1;
        while (l <= r) {
            const long long mid = l + (r - l) / 2;
            const double v = ts[mid];
            if (v == x) { res = mid; break; }
            if (v < x) l = mid + 1; else r = mid - 1;
        }
        out[i] = res >= 0 ? res : l;
    }
}

// one block per frame: events [start[f], start[f] + len[f]) of the columns -> out[off[f] ...] as fp32.
// xform (optional) = one word per frame, H5Dataset.augment_event (h5dataset.py:652-670) and SequenceDataset's pause
// (h5dataset.py:780-784, 317-319):
//   bit 0: x -> W - 1 - x, bit 1: y -> H - 1 - y, bit 2: p -> -p  (the reference flips the float64 values before the fp32 cast;
//          for int16 coordinates and W, H < 2^23 both sides are exact integers, so one fp32 subtraction gives the same bits);
//   bit 3: paused, every output event is (x, y, t, p) = 0 (torch.zeros([4, 1]) for the one slot the host reserves); start ignored.
__global__ void __launch_bounds__(256)
k_gather_events(const short *__restrict__ xs, const short *__restrict__ ys, const double *__restrict__ ts,
                const double *__restrict__ ps, const long long *__restrict__ start, const long long *__restrict__ off,
                const int *__restrict__ xform, float wm1, float hm1,
                float *__restrict__ oxs, float *__restrict__ oys, float *__restrict__ ots, float *__restrict__ ops)
{
    const int f = blockIdx.x;
    const int xf = xform ? xform[f] : 0;
    const bool paused = xf & 8;
    const long long s = paused ? 0 : start[f], o = off[f], n = off[f + 1] - o;
    float t0 = 0.f, den = 1.f;
    if (ots && n > 0 && !paused) {
        t0 = (float)ts[s];
        den = __fadd_rn(__fsub_rn((float)ts[s + n - 1], t0), 1e-6f);          // fp32, like the torch expression
    }
    for (long long i = (long long)blockIdx.y * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.y * blockDim.x) {
        float x = 0.f, y = 0.f, p = 0.f, t = 0.f;
        if (!paused) {
            x = (float)xs[s + i];
            y = (float)ys[s + i];
            p = (float)ps[s + i];
            if (xf & 1) x = __fsub_rn(wm1, x);
            if (xf & 2) y = __fsub_rn(hm1, y);
            if (xf & 4) p = -p;
            if (ots) t = __fdiv_rn(__fsub_rn((float)ts[s + i], t0), den);
        }
        oxs[o + i] = x;
        oys[o + i] = y;
        ops[o + i] = p;
        if (ots) ots[o + i] = t;
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// Columns of many recordings -> count banks in one pass (the batch of HDF5DataLoaderSequence, dataloader/h5dataloader.py:
// 180-233, whose samples come from different SequenceDatasets of one ConcatDataset).  The same arithmetic as
// k_gather_events followed by k_scatter_cnt with writeback == 2 (events.cu), without the fp32 SoA in between:
//   x, y (int16) and p (float64) are read once per event (12 B; ts is not read), cast to fp32 and flipped in registers;
//   LR bank: the event as it is; lifted bank: x / W * kW, y / H * kH with two fp32 roundings (h5dataset.py:515, 526);
//   out of range: positive weight dropped; the negative weight lands on neg[0, 0] unless the frame holds more than 3 events
//   (create_stack_encoding zeroed x, y and p first, h5dataset.py:337-354, encodings.py:219-220, 251-256);
//   a paused frame is the reference's one zero event (p = 0): it adds nothing, so its block returns at once.
// Counts are fp32 sums of p * p, exact and order-independent for p = +-1, so the banks equal the two-step path bit for bit.
struct FrameDesc {
    long long start, len;     // rows [start, start + len) of recording rec's columns
    int rec, xform;           // xform: the transform word of k_gather_events (bit 3 = paused)
};

__device__ __forceinline__ void scatter_pn(float *__restrict__ img, int H, int W, float x, float y, float vpos, float vneg, bool many)
{
    if ((x >= (float)W) | (x < 0.0f) | (y >= (float)H) | (y < 0.0f)) {
        x = 0.0f; y = 0.0f; vpos = 0.0f;
        if (many) vneg = 0.0f;
    }
    const size_t pix = (size_t)(long long)y * W + (size_t)(long long)x;     // .long(): truncation toward zero
    if (vpos != 0.0f) atomicAdd(img + pix, vpos);
    if (vneg != 0.0f) atomicAdd(img + (size_t)H * W + pix, vneg);
}

// grid (frames, blocks per frame); cols = [R][3] addresses of the xs, ys, ps columns of recording r (pinned host or HBM)
template <bool LIFT>
__global__ void __launch_bounds__(256)
k_encode_frames_multi(const unsigned long long *__restrict__ cols, const FrameDesc *__restrict__ desc, int H, int W, int kH, int kW,
                      float *__restrict__ out, float *__restrict__ out_hr)
{
    const unsigned f = blockIdx.x;
    const FrameDesc d = desc[f];
    if (d.xform & 8) return;
    const short *__restrict__ xs = reinterpret_cast<const short *>(cols[3 * d.rec]) + d.start;
    const short *__restrict__ ys = reinterpret_cast<const short *>(cols[3 * d.rec + 1]) + d.start;
    const double *__restrict__ ps = reinterpret_cast<const double *>(cols[3 * d.rec + 2]) + d.start;
    const bool many = d.len > 3;
    const float wm1 = (float)(W - 1), hm1 = (float)(H - 1);
    float *img = out + (size_t)f * 2 * H * W;
    float *img_hr = LIFT ? out_hr + (size_t)f * 2 * kH * kW : nullptr;
    for (long long i = (long long)blockIdx.y * blockDim.x + threadIdx.x; i < d.len; i += (long long)gridDim.y * blockDim.x) {
        float x = (float)xs[i], y = (float)ys[i], p = (float)ps[i];
        if (d.xform & 1) x = __fsub_rn(wm1, x);
        if (d.xform & 2) y = __fsub_rn(hm1, y);
        if (d.xform & 4) p = -p;
        const float vpos = __fmul_rn(p, p < 0.0f ? 0.0f : p);
        const float vneg = __fmul_rn(p, p > 0.0f ? 0.0f : p);
        scatter_pn(img, H, W, x, y, vpos, vneg, many);
        if (LIFT)
            scatter_pn(img_hr, kH, kW, __fmul_rn(__fdiv_rn(x, (float)W), (float)kW), __fmul_rn(__fdiv_rn(y, (float)H), (float)kH),
                       vpos, vneg, many);
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// Many live streams' new events -> their HBM rings in one launch (esr_b200.stream.EventStreamPool).  Segment d = rows
// [src, src + count) of the packed source columns goes to ring positions position, position + 1, ... mod capacity.
struct RingDesc {
    unsigned long long xs, ys, ps;     // the ring's columns: int16, int16, float64
    long long capacity, position, count, src;
};

// grid (blocks per segment, segments), both with stride loops; consecutive threads write consecutive ring elements
__global__ void __launch_bounds__(256)
k_append_rings(const RingDesc *__restrict__ desc, int n_desc, const short *__restrict__ src_xs, const short *__restrict__ src_ys,
               const double *__restrict__ src_ps)
{
    for (int s = blockIdx.y; s < n_desc; s += gridDim.y) {
        const RingDesc d = desc[s];
        if (d.capacity <= 0) continue;
        const long long n = min(max(d.count, 0LL), d.capacity), p0 = d.position % d.capacity;
        short *xs = reinterpret_cast<short *>(d.xs), *ys = reinterpret_cast<short *>(d.ys);
        double *ps = reinterpret_cast<double *>(d.ps);
        for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
            long long j = p0 + i;
            if (j >= d.capacity) j -= d.capacity;                  // the wrap: n <= capacity
            xs[j] = src_xs[d.src + i];
            ys[j] = src_ys[d.src + i];
            ps[j] = src_ps[d.src + i];
        }
    }
}

} // namespace esr

using namespace esr;

static_assert(sizeof(FrameDesc) == sizeof(esr_frame_desc), "esr_frame_desc layout");
static_assert(sizeof(RingDesc) == sizeof(esr_ring_desc), "esr_ring_desc layout");

extern "C" int esr_events_append_rings(const esr_ring_desc *desc, int n_desc, int64_t max_count, const int16_t *src_xs,
                                       const int16_t *src_ys, const double *src_ps, esr_stream_t stream)
{
    ESR_REQUIRE(n_desc >= 0 && max_count >= 0, "esr_events_append_rings: negative count");
    if (n_desc == 0 || max_count == 0) return ESR_OK;
    ESR_REQUIRE(desc && src_xs && src_ys && src_ps, "esr_events_append_rings: null pointer");
    // ~4 events per thread for the longest segment, capped; segments on grid y
    const int64_t bx = max((int64_t)1, min(ceil_div64(max_count, 256 * 4), (int64_t)dev_info().sm_count * 16));
    const dim3 grid((unsigned)bx, (unsigned)min(n_desc, 65535));
    k_append_rings<<<grid, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const RingDesc *>(desc), n_desc, src_xs, src_ys, src_ps);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}

extern "C" int esr_encode_frames_multi(const uint64_t *cols, const esr_frame_desc *desc, int n_frames, int64_t max_len, int H, int W,
                                       int kH, int kW, float *out_cnt, float *out_scaled_cnt, esr_stream_t stream)
{
    ESR_REQUIRE(n_frames >= 0 && H > 0 && W > 0 && H < (1 << 23) && W < (1 << 23) && out_cnt && max_len >= 0,
                "esr_encode_frames_multi: bad arguments");
    ESR_REQUIRE(!out_scaled_cnt || (kH > 0 && kW > 0), "esr_encode_frames_multi: bad lifted resolution");
    cudaStream_t st = (cudaStream_t)stream;
    if (n_frames == 0) return ESR_OK;
    ESR_CUDA_CHECK(cudaMemsetAsync(out_cnt, 0, sizeof(float) * (size_t)n_frames * 2 * H * W, st));
    if (out_scaled_cnt) ESR_CUDA_CHECK(cudaMemsetAsync(out_scaled_cnt, 0, sizeof(float) * (size_t)n_frames * 2 * kH * kW, st));
    if (max_len == 0) return ESR_OK;
    ESR_REQUIRE(cols && desc, "esr_encode_frames_multi: null tables");
    // as esr_scatter_cnt: ~8 events per thread for the longest frame, capped for huge frames; frames on grid x (up to 2^31 - 1)
    const int64_t by = max((int64_t)1, min(ceil_div64(max_len, 256 * 8), min((int64_t)dev_info().sm_count * 16, (int64_t)65535)));
    const dim3 grid((unsigned)n_frames, (unsigned)by);
    const FrameDesc *dd = reinterpret_cast<const FrameDesc *>(desc);
    const unsigned long long *cc = reinterpret_cast<const unsigned long long *>(cols);
    if (out_scaled_cnt)
        k_encode_frames_multi<true><<<grid, 256, 0, st>>>(cc, dd, H, W, kH, kW, out_cnt, out_scaled_cnt);
    else
        k_encode_frames_multi<false><<<grid, 256, 0, st>>>(cc, dd, H, W, 0, 0, out_cnt, nullptr);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}

extern "C" int esr_ts_search(const double *ts, int64_t n, const double *queries, int64_t nq, int64_t *out, esr_stream_t stream)
{
    ESR_REQUIRE(ts && queries && out && n >= 0 && nq >= 0, "esr_ts_search: bad arguments");
    if (nq == 0) return ESR_OK;
    k_ts_search<<<(unsigned)min((int64_t)4096, (nq + 255) / 256), 256, 0, (cudaStream_t)stream>>>(ts, (long long)n, queries, (long long)nq,
                                                                                              (long long *)out);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}

extern "C" int esr_gather_events_aug(const int16_t *xs, const int16_t *ys, const double *ts, const double *ps, const int64_t *start,
                                     const int64_t *off, const int32_t *xform, int W, int H, int n_frames, int64_t max_len,
                                     float *out_xs, float *out_ys, float *out_ts, float *out_ps, esr_stream_t stream)
{
    ESR_REQUIRE(xs && ys && ps && start && off && out_xs && out_ys && out_ps && n_frames >= 0, "esr_gather_events: bad arguments");
    ESR_REQUIRE(!out_ts || ts, "esr_gather_events: out_ts needs the ts column");
    ESR_REQUIRE(!xform || (W > 0 && H > 0 && W < (1 << 23) && H < (1 << 23)), "esr_gather_events_aug: bad flip resolution");
    if (n_frames == 0) return ESR_OK;
    ESR_REQUIRE(n_frames <= 0x7fffffff, "esr_gather_events: too many frames");
    const unsigned gy = (unsigned)max((int64_t)1, min((int64_t)64, (max_len + 2047) / 2048));
    k_gather_events<<<dim3((unsigned)n_frames, gy), 256, 0, (cudaStream_t)stream>>>(xs, ys, ts, ps, (const long long *)start, (const long long *)off,
                                                                                (const int *)xform, (float)(W - 1), (float)(H - 1),
                                                                                out_xs, out_ys, out_ts, out_ps);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}

extern "C" int esr_gather_events(const int16_t *xs, const int16_t *ys, const double *ts, const double *ps, const int64_t *start,
                                 const int64_t *off, int n_frames, int64_t max_len, float *out_xs, float *out_ys, float *out_ts,
                                 float *out_ps, esr_stream_t stream)
{
    return esr_gather_events_aug(xs, ys, ts, ps, start, off, nullptr, 0, 0, n_frames, max_len, out_xs, out_ys, out_ts, out_ps, stream);
}
