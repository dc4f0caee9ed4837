// columns.cu -- padded cnt2event rows -> the four columns of an event file, with sensor timestamps.
//
// Completes dataloader/cython_cnt2event/cnt2event_api.py:25-35 (cnt2eventAPI, whose [B, maxlen, 4] rows have no caller in the
// reference's scripts) towards the file layout of generate_dataset/tools/event_packagers.py:121-224 (xs, ys int16; ts, ps
// float64): sample s contributes its first `valid` rows -- the padding and the zero row of an empty sample are left out -- to rows
// [dst, dst + valid) of the columns, and its per-window fp32 timestamp t32 in [0, 1] becomes the sensor time
//     t = t0 + double(t32) * (t1 - t0)
// with one IEEE subtraction per sample, then one multiplication and one addition per event, never contracted into an FMA, so that
// numpy's float64 arithmetic gives the same bits.  This inverts BaseDataset.event_formatting (dataloader/base_dataset.py:26-33)
// without its 1e-6, which would push the last event past t1.
#include "common.cuh"

namespace esr {

struct ColumnDesc {
    long long valid, dst;     // rows [0, valid) of the sample -> rows [dst, dst + valid) of the columns
    double t0, t1;            // sensor time of the first / last input event of the window's middle frame
};

// grid (blocks per sample, samples), both with stride loops.  A thread reads one 16-byte row; consecutive threads write
// consecutive elements of each column (device memory or pinned host memory).
__global__ void __launch_bounds__(256)
k_events_to_columns(const float4 *__restrict__ rows, int n_samples, long long maxlen, const ColumnDesc *__restrict__ desc,
                    short *__restrict__ xs, short *__restrict__ ys, double *__restrict__ ts, double *__restrict__ ps)
{
    for (int s = blockIdx.y; s < n_samples; s += gridDim.y) {
        const ColumnDesc d = desc[s];
        const long long n = min(max(d.valid, 0LL), maxlen);
        const double dt = __dsub_rn(d.t1, d.t0);
        const float4 *__restrict__ src = rows + (size_t)s * maxlen;
        for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
            const float4 e = __ldg(src + i);                       // (x, y, t, p)
            xs[d.dst + i] = (short)(int)e.x;                       // exact: small non-negative integers in fp32
            ys[d.dst + i] = (short)(int)e.y;
            ts[d.dst + i] = __dadd_rn(d.t0, __dmul_rn((double)e.z, dt));
            ps[d.dst + i] = (double)e.w;
        }
    }
}

} // namespace esr

using namespace esr;

static_assert(sizeof(ColumnDesc) == sizeof(esr_column_desc), "esr_column_desc layout");

extern "C" int esr_events_to_columns(const float *rows, int n_samples, int64_t maxlen, const esr_column_desc *desc, int64_t max_valid,
                                     int16_t *xs, int16_t *ys, double *ts, double *ps, esr_stream_t stream)
{
    ESR_REQUIRE(n_samples >= 0 && maxlen >= 0 && max_valid >= 0, "esr_events_to_columns: negative length");
    ESR_REQUIRE(max_valid <= maxlen, "esr_events_to_columns: %lld valid rows in samples of %lld rows", (long long)max_valid,
                (long long)maxlen);
    if (n_samples == 0 || max_valid == 0) return ESR_OK;
    ESR_REQUIRE(rows && desc && xs && ys && ts && ps, "esr_events_to_columns: null pointer");
    ESR_REQUIRE(((uintptr_t)rows & 15) == 0, "esr_events_to_columns: rows must be 16-byte aligned");
    // ~4 events per thread for the longest sample, capped for huge samples; samples on grid y
    const int64_t bx = max((int64_t)1, min(ceil_div64(max_valid, 256 * 4), (int64_t)dev_info().sm_count * 16));
    const dim3 grid((unsigned)bx, (unsigned)min(n_samples, 65535));
    k_events_to_columns<<<grid, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float4 *>(rows), n_samples, (long long)maxlen,
                                                                reinterpret_cast<const ColumnDesc *>(desc), xs, ys, ts, ps);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}
