/*
 * esr_b200.h -- C ABI of libesr_b200.so, the H100 (sm_90a) implementation of WarranWeng/ESR's
 * per-timestep hot path.  Plain pointers and sizes only; every pointer is a DEVICE pointer unless
 * its name ends in _host.  The caller owns every buffer and the stream; the library allocates no
 * user-visible memory (workspaces are sized by *_workspace_bytes and passed in).  All functions return
 * ESR_OK (0) or a negative error code; esr_last_error() gives the message for the calling thread.
 * Calls are asynchronous on `stream` unless stated otherwise.
 *
 * Each entry point names the reference interface it replaces (paths relative to the reference root).
 */
#ifndef ESR_B200_H
#define ESR_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ESR_OK 0
#define ESR_EINVAL (-1)       /* bad argument */
#define ESR_ENEGCOUNT (-2)    /* negative rounded count: the reference raises ValueError (cnt2event.pyx:71) */
#define ESR_ECUDA (-3)        /* CUDA runtime / driver error */
#define ESR_EUNSUPPORTED (-4) /* configuration outside what the sm_90a kernels implement */
#define ESR_EWORKSPACE (-5)   /* workspace too small */

/* `flags` bits of the *_ex training entry points.  ESR_DETERMINISTIC: every reduction that sums with fp32 atomics by default
 * (bias and weight gradients, the loss, the deformable convolution's grad_input) runs as per-block partials added in a fixed
 * order, or in int64 fixed point, so repeated calls on the same GPU model give bitwise identical results -- what
 * torch.backends.cudnn.deterministic / torch.use_deterministic_algorithms ask of cuDNN.  Paths without such a variant return
 * ESR_EUNSUPPORTED in this mode.  The workspace queries with the same flags include the partial buffers. */
#define ESR_DETERMINISTIC 1

typedef void *esr_stream_t; /* cudaStream_t */

int esr_version(void);
const char *esr_last_error(void);
/* number of kernels this library has launched since load (bench.py's gpu_launches claim) */
int64_t esr_launch_count(void);

/* ---------------------------------------------------------------------------------------------
 * events -> 2-channel polarity count images
 * Replaces: dataloader/encodings.py:289-304 events_to_channels (+ :243-268 events_to_image), and, with
 * lift_* set, the LR->HR coordinate lift of dataloader/h5dataset.py:508-528 (x / W_lr * W_hr in fp32,
 * two roundings).  F frames in one launch: frame f owns events [frame_off[f], frame_off[f+1]).
 *   xs, ys, ps : fp32 [n_total]        frame_off : int64 [F+1] (device)
 *   out        : fp32 [F, 2, H, W], overwritten (zeroed by the call)
 *   lift_w_lr/lift_w_hr/lift_h_lr/lift_h_hr : 0 = coordinates used as given
 *   writeback  : 1 = reproduce the reference's in-place side effect (out-of-range xs, ys set to 0)
 * Reference quirks kept: out-of-range positive events are dropped, out-of-range NEGATIVE events are
 * counted at neg[0,0]; fractional coordinates truncate toward zero; each event adds ps*ps.
 * writeback: 0 = leave xs / ys alone, 1 = zero them in place for out-of-range events (standalone events_to_channels), 2 = the
 * order of H5Dataset.__getitem__ (h5dataset.py:337-354): in frames of more than 3 events out-of-range events of EITHER polarity add
 * nothing, because create_stack_encoding has sanitised the event tensor before the count encodings see it.
 * --------------------------------------------------------------------------------------------- */
int esr_scatter_cnt(float *xs, float *ys, const float *ps, const int64_t *frame_off, int F, int64_t n_max_frame,
                    int H, int W, int lift_w_lr, int lift_w_hr, int lift_h_lr, int lift_h_hr, int writeback,
                    float *out, esr_stream_t stream);

/* Replaces: dataloader/encodings.py:243-268 events_to_image.  One image, raw weights: out[(long)y,(long)x] += ps;
 * out-of-range events are dropped and, with writeback = 1, xs/ys/ps are zeroed in place like the reference. */
int esr_scatter_image(float *xs, float *ys, float *ps, int64_t n, int H, int W, int writeback, float *out,
                      esr_stream_t stream);

/* Replaces: dataloader/encodings.py:307-331 events_to_mask (index_put_ with accumulate=False: the last event hitting a
 * pixel writes |ps|; out-of-range events are zeroed in place and then write 0 to pixel (0,0)).  last_tmp: int32 [H*W]. */
int esr_scatter_mask(float *xs, float *ys, float *ps, int64_t n, int H, int W, int writeback, int32_t *last_tmp, float *out,
                     esr_stream_t stream);

/* Replaces: the slicing of dataloader/encodings.py:204-240 events_to_stack_no_polarity, i.e. its calls to
 * binary_search_torch_tensor (encodings.py:77-99).  ts: sorted fp32 [n]; bounds: int64 [B,2] = (beg, end) of every time
 * bin, identical to the reference's search (incl. which of several equal timestamps it stops on). */
int esr_time_bin_bounds(const float *ts, int64_t n, int B, int64_t *bounds, esr_stream_t stream);

/* Replaces: dataloader/encodings.py:271-286 events_to_voxel (temporal bilinear voxel grid through events_to_image).
 * out: fp32 [num_bins,H,W], overwritten.  Keeps the reference's side effect (xs, ys zeroed in place for out-of-range
 * events) and its consequence (those events land on pixel (0,0) in bins >= 1). */
int esr_scatter_voxel(float *xs, float *ys, const float *ts, const float *ps, int64_t n, int num_bins, int H, int W,
                      int writeback, float *out, esr_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * dense counts / time-bin stacks -> time-sorted event lists
 * Replaces: dataloader/cython_cnt2event/cnt2event.pyx:18-116 (kind 0: vals = [B,2,H,W], P=2, C=1) and
 * dataloader/cython_event_redistribute/event_redistribute.pyx:17-83 / :88-153 (kind 1: vals =
 * [B,P,C,H,W], P=1 for the NoPolarity form).
 *
 * Two phases, because the output length depends on the data:
 *  1. esr_expand_count: rounds (half-to-even) and counts.  stats : int64 [B,4] (device) =
 *     {sum of rounded values, number of events, any-negative flag, max per-slot count}; counts : uint32
 *     [B*P*C*H*W] (device, kept for phase 2).
 *  2. the host reads stats, applies the reference's emptiness rules (a sample whose rounded values sum to
 *     zero yields one zero row; an all-zero call yields [B,1,4]), sizes out = [B, maxlen, 4] (zero-filled)
 *     and calls esr_expand_emit with active_host[b] / start_host[b] (first sorted row of sample b in the
 *     global event order).  mode 0 = linear timestamps (float64 linspace -> fp32), mode 1 = the caller's
 *     random stream rnd[total_events] (float64, numpy MT19937 seed 123, one value per event in emission order).
 * --------------------------------------------------------------------------------------------- */
int esr_expand_count(const float *vals, int B, int P, int C, int H, int W, int kind, int64_t *stats, uint32_t *counts,
                     esr_stream_t stream);
size_t esr_expand_workspace_bytes(int B, int P, int C, int H, int W, int64_t total_events);
/* rank_table (optional, device uint16 [(rank_m+1) * rank_m]): compact sort keys for cnt2event with linear timestamps and
 * max per-pixel count rank_m <= 255 -- rank_table[n*rank_m + j] = index of float32(linspace(0,1,n)[j]) among the sorted
 * distinct timestamps, rank_bits = bits needed; NULL = sort on the raw fp32 timestamp bits (always valid). */
int esr_expand_emit(const float *vals, uint32_t *counts, int B, int P, int C, int H, int W, int kind, int mode,
                    const double *rnd, const uint16_t *rank_table, int rank_m, int rank_bits, const int32_t *active_host,
                    const int64_t *start_host, int64_t total_events, int64_t maxlen, float *out, void *workspace,
                    size_t workspace_bytes, esr_stream_t stream);

/* cnt2event with linear timestamps, whole operator in three launches without a host round trip
 * (dataloader/cython_cnt2event/cnt2event.pyx:18-116, mode 'linear'; csrc/expand_fused.cu).  vals: device fp32 [B,2,H,W].
 * The caller supplies `out` with room for cap_rows rows of 4 floats; the kernels compute maxlen = max over samples of the
 * event count (1 for a sample whose rounded values sum to zero) on the device and write the padded [B, maxlen, 4] result,
 * zero padding included, at the start of `out`.  stats (device int64 [B,4], same meaning as esr_expand_count) is how the caller
 * learns maxlen afterwards and whether the result is valid: it is NOT when an active sample holds a negative count (the
 * reference raises), when the largest count of an active sample exceeds max_count rounded up to a power of two (max_count <= 64:
 * the caller's guess, it sizes the per-key counters in shared memory), when B * maxlen > cap_rows, or when no sample is
 * active -- then nothing was written and the caller applies the reference's rules / uses esr_expand_count + esr_expand_emit.
 * tables: device blob of the 7 key tables for m = 1, 2, 4 .. 64 -- rank uint16 [(m+1)*m] (index of float32(linspace(0,1,n)[j])
 * among the K distinct values for counts <= m) and uniq float [K]; tables_desc_host: int32 [7][3] = {rank byte offset, uniq
 * byte offset, K}.  The host builds them with numpy.linspace, the reference's own arithmetic. */
size_t esr_cnt2event_fused_workspace_bytes(int B, int H, int W);
int esr_cnt2event_fused(const float *vals, int B, int H, int W, const void *tables, const int32_t *tables_desc_host,
                        int max_count, int64_t *stats, float *out, int64_t cap_rows, void *workspace, size_t workspace_bytes,
                        esr_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Tensor-core convolution (wgmma, TMA-tiled implicit GEMM), layer-level entry point.
 * Replaces: every stride-1 nn.Conv2d at feature resolution in models/model.py / models/submodules.py
 * (3x3 pad 1 or 1x1; Cin a multiple of 64, Cout <= 256), including torch.cat inputs (K-split over up to 3
 * sources), the fused bias / residual / activation tail of ConvLayer / ResidualBlock
 * (models/submodules.py:159-200, 347-409) and the ConvGRU gating (models/submodules.py:496-514).
 *
 * Activation tensors are "split bf16" NHWC: [2 planes][n_img][H][W][C] bf16, value = hi + lo
 * (esr_split_from_nchw / esr_split_to_nchw convert from / to the reference's fp32 NCHW layout).
 * Weights are packed once by esr_pack_conv_weight (fp32 [Cout,Cin,k,k] -> split bf16 K-blocks).
 * --------------------------------------------------------------------------------------------- */
typedef struct esr_conv_desc {
    const void *src[3];        /* split tensors */
    int src_C[3];              /* channels of each source (multiple of 64) */
    int src_n_img[3];          /* images in each source tensor */
    const int32_t *src_img[3]; /* optional: output image -> source image index (device), NULL = identity */
    int n_src;
    int H, W;                  /* spatial size (input == output) */
    int n_img;                 /* output images */
    int ntaps;                 /* 9 = 3x3 pad 1, 1 = 1x1 */
    int cout;
    const void *wpacked;       /* from esr_pack_conv_weight */
    const float *bias;         /* fp32 [ceil16(cout)], zero padded */
    int act;                   /* 0 none, 1 relu, 2 sigmoid, 3 tanh; applied to channels >= act_from */
    int act_from;
    int res_mode;              /* 0 none, 1 add before activation, 2 add after activation */
    int epi_mode;              /* 0 standard, 1 ConvGRU update|reset gates, 2 ConvGRU candidate + blend */
    const void *res; int res_C; int res_n_img; const int32_t *res_img;
    void *out; int out_C; int out_n_img; int out_coff;   /* split output (NULL = none), channel offset */
    float *out_f32; int out_f32_C;                        /* fp32 NHWC output (NULL = none) */
    const void *h_prev; int h_n_img; float *z_buf;        /* ConvGRU: previous state (split, 64 ch), z gate fp32 */
} esr_conv_desc;

int esr_conv_tc(const esr_conv_desc *desc, esr_stream_t stream);
/* Same, with sources that repeat over images: for each s < n_src, chunk_img_step[s] = k != 0 makes source s (64 channels)
 * contribute src_chunks[s] 64-channel chunks, chunk j read from image src_img[s][img] + j*k (identity map: img + j*k).
 * This is the channel concatenation of images of one tensor (dense_fusion.0 over the num_frame-1 aligned neighbours).
 * Host arrays of 3 ints; NULL = all zero (then the call is esr_conv_tc). */
int esr_conv_tc_chunked(const esr_conv_desc *desc, const int *src_chunks, const int *chunk_img_step, esr_stream_t stream);
size_t esr_conv_weight_bytes(int cout, int cin, int ksz);
/* w1 != NULL: two [cout_each,cin,k,k] tensors concatenated along Cout (GRU update|reset) */
int esr_pack_conv_weight(const float *w0, const float *w1, int cout_each, int cin, int ksz, void *dst,
                         esr_stream_t stream);
int esr_split_from_nchw(const float *src, int n_img, int C, int H, int W, void *dst, esr_stream_t stream);
int esr_split_to_nchw(const void *src, int n_img, int C, int H, int W, float *dst, esr_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Small-channel and narrow-output convolutions, layer by layer (for tests and tools; the network launches the same kernels
 * from esr_net_forward).  One call runs one launch of the network's plan on a chosen kernel family:
 *   path 0 = warp-level tensor cores (mma.sync, split bf16), 1 = fp32 FFMA twins, 2 = the narrow-output CUDA-core kernel.
 * A (kind, path) pair the network never runs, or an unknown kind, returns ESR_EUNSUPPORTED.
 *   kind             Cin -> Cout, stride, act; input; output                                       paths
 *   HEAD_ENC0        2 -> 8 relu (head, w_head / b_head) fused into 8 -> 16 stride 2 relu; fp32 NCHW [*, 2, H_in, W_in]
 *                    zero-padded by pad_* (CropSize); split out                                    0, 1
 *   ENC1 / ENC2      16 -> 32 / 32 -> 64, stride 2, relu; split in and out                         0, 1
 *   ATT32 / ATT16    32 -> 1 / 16 -> 1, sigmoid; split in; fp32 NHWC out [n_img, H_in, W_in, 1]    0, 1
 *   RECON1 / RECON2  bilinear x2, then 32 -> 16 / 16 -> 8 relu; split in and out (2 H_in x 2 W_in) 0, 1
 *   TAIL             8 -> 2 relu; split in; fp32 NCHW out [n_img, 2, out_H, out_W] = the window at (crop_top, crop_left)
 *                    of the H_in x W_in result                                                     0, 1
 *   SPATIAL_KERNEL   64 -> 2, 1x1, sigmoid; split in; fp32 NHWC out [n_img, H_in, W_in, 2]         2
 * Weights are fp32 [Cout, Cin, k, k], packed into `workspace` (esr_conv_small_workspace_bytes(kind, path) bytes) on `stream` by
 * the network's own packers.  Split tensors are [2 planes][n_img][H][W][C] bf16; in_n_img / out_n_img give the images per
 * plane.  in_img (optional): output image -> input image.  Stride-2 outputs are (H - 1) / 2 + 1 high for a conv input of H rows
 * (H_in + pad_top + pad_bottom for HEAD_ENC0).
 * --------------------------------------------------------------------------------------------- */
enum {
    ESR_CONV_SMALL_HEAD_ENC0 = 0, ESR_CONV_SMALL_ENC1, ESR_CONV_SMALL_ENC2, ESR_CONV_SMALL_ATT32, ESR_CONV_SMALL_ATT16,
    ESR_CONV_SMALL_RECON1, ESR_CONV_SMALL_RECON2, ESR_CONV_SMALL_TAIL, ESR_CONV_SMALL_SPATIAL_KERNEL = 10
};
typedef struct esr_conv_small_desc {
    int kind, path;
    const float *in_f32;                    /* HEAD_ENC0 */
    const void *in; int in_n_img;           /* the other kinds */
    const int32_t *in_img;
    int H_in, W_in;
    int pad_top, pad_bottom, pad_left, pad_right;   /* HEAD_ENC0 */
    const float *w, *bias;
    const float *w_head, *b_head;           /* HEAD_ENC0: [8, 2, 3, 3], [8] */
    int n_img;
    void *out; int out_n_img;               /* split output */
    float *out_f32;                         /* fp32 output */
    int crop_top, crop_left, out_H, out_W;  /* TAIL */
    void *workspace; size_t workspace_bytes;
} esr_conv_small_desc;
size_t esr_conv_small_workspace_bytes(int kind, int path);
int esr_conv_small(const esr_conv_small_desc *desc, esr_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * The element-wise glue of the network, launcher by launcher (for tests and tools; esr_net_forward calls the same launchers).
 * One call runs one of them, chosen by `op`, on n_img images of H x W.  Split tensors are [2 planes][*_n_img][H][W][C] bf16,
 * and each one's image count sets its plane stride.  `idx` is the op's int32 index table; NULL = identity where allowed.
 *   op            reads                                                       writes                                   C
 *   LTC_CAT       in [*, H, W, 64]; maps fp32 [*, H, W]; idx [n_img][5] =    out [out_n_img, H, W, 192]               64
 *                 (f0, f1, f2, map0, map1) (required): cat(f0 m0, f1, f2 m1)
 *   CHAN_MAX      in [>= n_img, H, W, 64]: the per-image channel max          mx int32 [out_n_img, 64], the fp32 max   64
 *                                                                             as ordered ints (i >= 0 ? i : i ^ 0x7fffffff)
 *   ATTN_MLP      mx (as CHAN_MAX writes it); w0 [32, 64], b0 [32],           ck fp32 [out_n_img, 128]                 64
 *                 w1 [128, 32], b1 [128]: sigmoid(w1 relu(w0 max + b0) + b1)
 *   ATTN_APPLY    in [>= n_img, H, W, 64]; in2 [*, H, W, 64] at image         out [out_n_img, H, W, 128]               64
 *                 idx[img] (or img); sk fp32 [n_img, H, W, 2]; ck [n_img, 128]:
 *                 cat(in sk0 ck[:64], in2 sk1 ck[64:])
 *   SCALE_AGGREGATE  in [>= n_img, H, W, C]; in2 [*, H, W, C] and att fp32   out [out_n_img, H, W, C]                 8k
 *                 [*, H, W] at frame f = idx[img * N + n] (or img * N + n):
 *                 in + mean over n < N of in2[f] att[f]
 *   UPSAMPLE2X    in [>= n_img, H, W, C]: bilinear x2, align_corners=False    out [out_n_img, 2H, 2W, C]               8k
 *   COPY_SPLIT    in [*, H, W, C] at image idx[img] (or img)                  out [out_n_img, H, W, C]                 8k
 * ESR_EINVAL before any launch: a missing pointer, a C the op is not written for, n_img, H, W (or N) < 1, too few images in
 * an output or in an input read without a table, n_img > 65535 for CHAN_MAX and UPSAMPLE2X, 2H > 65535 for UPSAMPLE2X.
 * --------------------------------------------------------------------------------------------- */
enum {
    ESR_GLUE_LTC_CAT = 0, ESR_GLUE_CHAN_MAX, ESR_GLUE_ATTN_MLP, ESR_GLUE_ATTN_APPLY, ESR_GLUE_SCALE_AGGREGATE,
    ESR_GLUE_UPSAMPLE2X, ESR_GLUE_COPY_SPLIT
};
typedef struct esr_glue_desc {
    int op;
    int n_img, N, H, W, C;
    const void *in; int in_n_img;           /* split inputs */
    const void *in2; int in2_n_img;
    const int32_t *idx;
    const float *maps, *sk, *ck_in, *att;   /* fp32 side inputs (ck_in: ATTN_APPLY) */
    const float *w0, *b0, *w1, *b1;         /* ATTN_MLP */
    int32_t *mx;                            /* CHAN_MAX output, ATTN_MLP input */
    float *ck;                              /* ATTN_MLP output */
    void *out; int out_n_img;               /* split output; out_n_img also counts mx / ck images */
} esr_glue_desc;
int esr_glue(const esr_glue_desc *desc, esr_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * The network: DeepRecurrNet.forward with carried ConvGRU states.
 * Replaces: models/model.py:294-344 (DeepRecurrNet.forward / reset_states), and underneath it
 * models/model.py:20-291, models/submodules.py (ConvLayer, UpsampleConvLayer, ResidualBlock, RecurrentConvLayer,
 * ConvGRU, MLP), models/model_util.py:133-164 (CropSize) and the `_ext.dcn_v2_forward` operator
 * (models/DCNv2/src/dcn_v2.h:9-27, src/cuda/dcn_v2_cuda.cu:20-95) for the shipped configuration
 * (inch=2, basech=8, norm=None, relu, all sub-blocks enabled; config/train_ours_enfssyn.yml:21-26) and any odd
 * num_frame N >= 3 (the config's SEQN; the shipped value is 3).
 *
 *  params    : 68 device pointers to fp32 tensors in the reference's state_dict order
 *              (head.conv2d.weight, head.conv2d.bias, feat_extract.convblock.0.conv2d.weight, ... tail.conv2d.bias)
 *  blob      : esr_net_param_bytes_n(N) bytes, packed by esr_net_pack_params_n(N, ...) for the N the net is created with;
 *              repack whenever the parameters change.  Only dense_fusion.0's weight (N*64 input channels) depends on N,
 *              so a blob packed for another N has a different layout: esr_net_create refuses one that is too short for N
 *              when the device allocation holding it says so, and cannot detect the other mismatches.
 *              esr_net_param_bytes() / esr_net_pack_params() are the N = 3 forms.
 *  workspace : esr_net_workspace_bytes(B,N,L,H,W) bytes, owned by the caller, must outlive the net; holds all
 *              intermediates AND the recurrent states (which persist across esr_net_forward calls)
 *  N         : num_frame, odd and >= 3 (anything else: ESR_EUNSUPPORTED).  The middle frame (N-1)/2 of each window is
 *              the one super-resolved.
 *  L         : frames per sequence handled by one call.  L == N is the reference's forward: one window,
 *              input fp32 [B,N,2,H,W], output fp32 [B,2,H,W].  L > N is the sequence form used by the pipeline:
 *              input fp32 [B,L,2,H,W], output fp32 [(L-N+1)*B,2,H,W] (window-major: w*B+b) = the L-N+1 sliding-window
 *              forwards the reference would run one after another with the state carried (train_ours_cnt_seq.py:217-231,
 *              dataloader/h5dataloader.py:229-231).  Per-frame work (encoder, attention maps) is done once per frame
 *              and all state-independent layers once for all windows; only the ConvGRU chain is serial.  Results are
 *              identical to L-N+1 single-window calls.
 *  in_img    : optional device int32 [B*L]: frame (b,l) is read from input image in_img[b*L+l] (frame banks)
 * H, W need not be multiples of 8: the CropSize pad / crop is folded into the first and last kernels.
 * --------------------------------------------------------------------------------------------- */
typedef void *esr_net_t;
size_t esr_net_param_bytes(void);                 /* num_frame = 3 */
int esr_net_pack_params(const float *const *params_host_array_of_device_ptrs, void *blob, esr_stream_t stream);
size_t esr_net_param_bytes_n(int num_frame);      /* 0 for an unsupported num_frame */
int esr_net_pack_params_n(int num_frame, const float *const *params_host_array_of_device_ptrs, void *blob, esr_stream_t stream);
size_t esr_net_workspace_bytes(int B, int N, int L, int H, int W);
int esr_net_create(esr_net_t *net, int B, int N, int L, int H, int W, void *blob, void *workspace, size_t workspace_bytes,
                   esr_stream_t stream);
int esr_net_destroy(esr_net_t net);
int esr_net_reset_states(esr_net_t net, esr_stream_t stream);
/* Zero the carried states of sample b alone (both directions: images b and B + b of the state slot, both split planes) with
 * memsets on `stream`; graph-capturable.  The other samples' states are untouched, so a batch can start a new recording
 * in one slot while the others continue theirs. */
int esr_net_reset_sample_states(esr_net_t net, int b, esr_stream_t stream);
int esr_net_forward(esr_net_t net, const float *input, const int32_t *in_img, float *output, esr_stream_t stream);
/* Same as esr_net_forward, but brackets every kernel launch with CUDA events on `stream`, synchronises, and reports
 * per-launch {class (0 tensor-core conv, 1 CUDA-core conv, 2 element-wise/sampling),
 * milliseconds, algorithmic FLOPs, algorithmic bytes (every input / output element once at 4 bytes), layer name (32 chars each)}
 * into host arrays (measurement aid for bench.py's roofline objects; not on the production path).  bytes_host / names_host
 * may be null. */
int esr_net_forward_profiled(esr_net_t net, const float *input, const int32_t *in_img, float *output, int max_entries,
                             int *n_entries_host, int *cls_host, float *ms_host, double *flops_host, double *bytes_host,
                             char *names_host, esr_stream_t stream);
/* states: fp32 [2,B,64,H/8,W/8] (forward-direction state, reverse-direction state), the reference's self.states */
int esr_net_get_states(esr_net_t net, float *states, esr_stream_t stream);
int esr_net_set_states(esr_net_t net, const float *states, esr_stream_t stream);
/* State rows: the carried ConvGRU state of one sample kept outside any plan, so that many independent streams can share the
 * plans' batch slots (esr_b200.stream.EventStreamPool).  A row holds both directions and both split-bf16 planes in a layout
 * private to the library, esr_net_state_bytes(H, W) bytes for a net of input size H x W (0 for a non-positive size); a pool
 * is an array of rows, 16-byte aligned.  row_of_slot: device int32 [B] (B of the net).
 *   gather : sample b's state (slot 0, images b and B + b, both planes) := pool row row_of_slot[b]; row -1 gives zeros, a new
 *            stream's state.  Rows may repeat.
 *   scatter: pool row row_of_slot[b] := sample b's state; row -1 is skipped.  Rows other than -1 must not repeat.
 * Bit-exact copies (no fp32 round trip); one launch each on `stream`, no allocation, no host synchronisation:
 * graph-capturable.  The plans' own states need no reset when every call is framed by a gather and a scatter. */
size_t esr_net_state_bytes(int H, int W);
int esr_net_gather_states(esr_net_t net, const void *pool, const int32_t *row_of_slot, esr_stream_t stream);
int esr_net_scatter_states(esr_net_t net, void *pool, const int32_t *row_of_slot, esr_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * The `_ext.dcn_v2_forward` operator (modulated deformable convolution), reference layouts in and out.
 * Replaces: models/DCNv2/src/dcn_v2.h:9-27 dcn_v2_forward -> src/cuda/dcn_v2_cuda.cu:20-95 (+ the im2col kernel
 * src/cuda/dcn_v2_im2col_cuda.cu:125-195), as bound by src/vision.cpp:4-8 and called from models/DCNv2/dcn_v2.py:27.
 * input [B,C,H,W], weight [Co,C,k,k], bias [Co], offset [B,dg*2*k*k,Ho,Wo], mask [B,dg*k*k,Ho,Wo], output [B,Co,Ho,Wo];
 * fp32; Ho = (H + 2*pad - dilation*(k-1) - 1) / stride + 1, likewise Wo.  The kernel, stride, padding and dilation are
 * square (one value each).  The configuration ESR instantiates (C=Co=64, 3x3, stride 1, pad 1, dilation 1, dg=8) runs on
 * the wgmma path; any other with C % dg == 0 and Ho, Wo >= 1 on fp32 CUDA-core kernels (csrc/dcn_generic.cu); a bad
 * geometry returns ESR_EINVAL.  The tensor shapes are not checked here: the caller passes tensors of the sizes above.
 * --------------------------------------------------------------------------------------------- */
size_t esr_dcn_v2_workspace_bytes(int B, int H, int W);   /* the configuration ESR uses (64 -> 64, 3x3, s1 p1 d1, 8 groups) */
/* workspace for ANY configuration the reference operator accepts (backward = 1: for esr_dcn_v2_backward).  The configuration
 * of models/model.py:173 runs on the wgmma path; every other one (the reference's own tests use 2 -> 2 channels and
 * deformable_groups 1 / 2, models/DCNv2/testcuda.py:14-17,169-180) on fp32 CUDA-core kernels (csrc/dcn_generic.cu). */
size_t esr_dcn_v2_workspace_bytes_ex(int B, int C, int H, int W, int Co, int kernel, int stride, int pad, int dilation,
                                     int deformable_group, int backward);
/* Replaces: models/DCNv2/src/dcn_v2.h:29-50 dcn_v2_backward -> src/cuda/dcn_v2_cuda.cu:97-216 (+ the col2im / coord kernels
 * src/cuda/dcn_v2_im2col_cuda.cu:197-327), called from models/DCNv2/dcn_v2.py:50.  Same five gradients, reference layouts:
 * grad_input [B,C,H,W], grad_offset [B,dg*18,H,W], grad_mask [B,dg*9,H,W], grad_weight [Co,C,3,3], grad_bias [Co].
 * By default grad_input, grad_weight and grad_bias sum with fp32 atomics like the reference, so their summation order varies
 * from call to call; esr_dcn_v2_backward_ex with ESR_DETERMINISTIC makes them bitwise reproducible. */
size_t esr_dcn_v2_backward_workspace_bytes(int B, int H, int W);
int esr_dcn_v2_backward(const float *input, const float *weight, const float *bias, const float *offset, const float *mask,
                        const float *grad_output, int B, int C, int H, int W, int Co, int kernel, int stride, int pad,
                        int dilation, int deformable_group, float *grad_input, float *grad_offset, float *grad_mask,
                        float *grad_weight, float *grad_bias, void *workspace, size_t workspace_bytes, esr_stream_t stream);
/* Replaces the same dcn_v2_backward (models/DCNv2/src/dcn_v2.h:29-50, called from models/DCNv2/dcn_v2.py:50) with `flags`
 * (ESR_DETERMINISTIC or 0; 0 is esr_dcn_v2_backward).  Deterministic mode: grad_input accumulates in int64 fixed point (scale
 * chosen from the largest |grad_columns * mask| of the call so that no element can overflow), grad_weight / grad_bias from
 * per-slice partials.  Only the configuration of models/model.py:173 has this mode; any other returns ESR_EUNSUPPORTED.
 * Workspace: esr_dcn_v2_backward_workspace_bytes_ex with the same configuration and flags. */
size_t esr_dcn_v2_backward_workspace_bytes_ex(int B, int C, int H, int W, int Co, int kernel, int stride, int pad, int dilation,
                                              int deformable_group, int flags);
int esr_dcn_v2_backward_ex(const float *input, const float *weight, const float *bias, const float *offset, const float *mask,
                           const float *grad_output, int B, int C, int H, int W, int Co, int kernel, int stride, int pad,
                           int dilation, int deformable_group, float *grad_input, float *grad_offset, float *grad_mask,
                           float *grad_weight, float *grad_bias, int flags, void *workspace, size_t workspace_bytes,
                           esr_stream_t stream);
int esr_dcn_v2_forward(const float *input, const float *weight, const float *bias, const float *offset, const float *mask,
                       int B, int C, int H, int W, int Co, int kernel, int stride, int pad, int dilation,
                       int deformable_group, float *output, void *workspace, size_t workspace_bytes, esr_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Training step operators (SURVEY.md 8a row 17).
 * Replaces, for one ConvLayer (models/submodules.py:159-200: Conv2d(bias) -> activation), ATen's conv2d forward and
 * backward as autograd calls them inside train_ours_cnt_seq.py:217-231 (forward) and :232 (loss.backward()); and
 * nn.MSELoss (:774) and torch.optim.Adam(lr, weight_decay, amsgrad) (:781, config/train_ours_enfssyn.yml optimizer).
 * Tensors are fp32 NCHW (x [B,Cin,H,W], w [Cout,Cin,k,k], y/dy [B,Cout,Ho,Wo]); k = 3 (pad 1) or 1 (pad 0); stride 1|2;
 * act: 0 none, 1 relu, 2 sigmoid, 3 tanh (fused into the forward; backward multiplies dy by act'(y)).
 * backward: dx may be NULL (first layer); dw [Cout,Cin,k,k] and db [Cout] are overwritten (not accumulated); dw == db ==
 * NULL computes dx only (a caller that batches the weight gradient of a weight-shared layer, e.g. the ConvGRU steps).
 * workspace: esr_conv2d_workspace_bytes() bytes of device memory owned by the caller; a NULL or shorter one is refused (ESR_EINVAL).
 * --------------------------------------------------------------------------------------------- */
size_t esr_conv2d_workspace_bytes(int B, int Cin, int H, int W, int Cout, int ksz, int stride);
/* x_split (optional): layers whose forward, dx and dw all run on the tensor cores convert x to the split-bf16 NHWC operand
 * format once; esr_conv2d_split_bytes() > 0 says so and gives the size of the buffer the forward fills (x_split_out) and the
 * backward reads (x_split) instead of converting x again -- the backward then does not need x itself (x may be NULL). */
size_t esr_conv2d_split_bytes(int B, int Cin, int H, int W, int Cout, int ksz, int stride);
int esr_conv2d_forward(const float *x, const float *w, const float *bias, int B, int Cin, int H, int W, int Cout, int ksz,
                       int stride, int act, float *y, void *x_split_out, void *workspace, size_t workspace_bytes,
                       esr_stream_t stream);
int esr_conv2d_backward(const float *x, const void *x_split, const float *w, const float *y, const float *dy, int B, int Cin,
                        int H, int W, int Cout, int ksz, int stride, int act, float *dx, float *dw, float *db, void *workspace,
                        size_t workspace_bytes, esr_stream_t stream);
/* Replaces the same ATen conv2d backward (train_ops.cu, for a ConvLayer of models/submodules.py:159-200) with `flags`: 0 is
 * esr_conv2d_backward; ESR_DETERMINISTIC sums db and dw from per-block partials in a fixed order (what
 * torch.backends.cudnn.deterministic asks of cuDNN), with esr_conv2d_workspace_bytes_ex(..., flags) bytes of workspace. */
size_t esr_conv2d_workspace_bytes_ex(int B, int Cin, int H, int W, int Cout, int ksz, int stride, int flags);
int esr_conv2d_backward_ex(const float *x, const void *x_split, const float *w, const float *y, const float *dy, int B, int Cin,
                           int H, int W, int Cout, int ksz, int stride, int act, float *dx, float *dw, float *db, int flags,
                           void *workspace, size_t workspace_bytes, esr_stream_t stream);
/* Bilinear x2 upsampling of `planes` = B*C fp32 planes [H,W] -> [2H,2W] and its backward (dy [2H,2W] -> dx [H,W]):
 * F.interpolate(scale_factor=2, mode='bilinear', align_corners=False) of UpsampleConvLayer (models/submodules.py:290). */
int esr_upsample2x_forward(const float *x, int planes, int H, int W, float *y, esr_stream_t stream);
int esr_upsample2x_backward(const float *dy, int planes, int H, int W, float *dx, esr_stream_t stream);
/* Resize of `planes` fp32 planes [Hin,Win] -> [Hout,Wout] as torch.nn.functional.interpolate(size=..., align_corners=False)
 * does on the CPU: mode 1 = 'bicubic' (Keys, A = -0.75, clamped taps), mode 0 = legacy 'nearest'.  Replaces the per-frame
 * calls of the dataset's tensor factory (dataloader/h5dataset.py:341-344: inp_bicubic_cnt / _stack, inp_near_cnt / _stack)
 * and the bicubic baseline of infer_ours_cnt.py:76-78. */
int esr_resize_planes(const float *x, int planes, int Hin, int Win, int Hout, int Wout, int mode, float *out,
                      esr_stream_t stream);
/* ConvGRU gate arithmetic (models/submodules.py:507-512), fp32, B images of chw = C*H*W elements; zr [B, 2C, H, W] holds
 * the update gate z in channels [0,C) and the reset gate r in [C,2C).  hr = h*r;  blend = h*(1-z) + o*z.  The backward
 * entry points write full-size dzr (the half they do not touch is zero-filled). */
int esr_gru_hr(const float *h, const float *zr, int B, int chw, float *out, esr_stream_t stream);
int esr_gru_hr_backward(const float *h, const float *zr, const float *grad, int B, int chw, float *dh, float *dzr,
                        esr_stream_t stream);
int esr_gru_blend(const float *h, const float *zr, const float *o, int B, int chw, float *out, esr_stream_t stream);
int esr_gru_blend_backward(const float *h, const float *zr, const float *o, const float *grad, int B, int chw, float *dh,
                           float *dzr, float *d_o, esr_stream_t stream);
/* loss[0] = mean((pred - target)^2); grad (optional) = grad_scale * 2 (pred - target) / n */
int esr_mse_loss(const float *pred, const float *target, size_t n, float *loss, float *grad, float grad_scale,
                 esr_stream_t stream);
/* Replaces the same nn.MSELoss (train_ours_cnt_seq.py:774) with `flags`: 0 is esr_mse_loss; ESR_DETERMINISTIC writes one
 * partial per block and adds them in block order (workspace: esr_mse_loss_workspace_bytes_ex bytes, 0 without the flag). */
size_t esr_mse_loss_workspace_bytes_ex(size_t n, int flags);
int esr_mse_loss_ex(const float *pred, const float *target, size_t n, float *loss, float *grad, float grad_scale, int flags,
                    void *workspace, size_t workspace_bytes, esr_stream_t stream);
/* One torch.optim.Adam step over a flat fp32 parameter buffer; max_exp_avg_sq != NULL = amsgrad.  step_counter is a
 * DEVICE int32 holding the number of steps taken so far (0 before the first); the call increments it on the stream and
 * uses the new value for the bias corrections, so the call can sit inside a replayed CUDA graph. */
int esr_adam_step(float *param, const float *grad, float *exp_avg, float *exp_avg_sq, float *max_exp_avg_sq, size_t n,
                  int32_t *step_counter, float lr, float beta1, float beta2, float eps, float weight_decay,
                  esr_stream_t stream);
/* Same step with the hyper-parameters {lr, beta1, beta2, eps, weight_decay} read from DEVICE memory when the kernel runs: a
 * CUDA graph that contains the call follows a learning-rate schedule (train_ours_cnt_seq.py:784) by rewriting 20 bytes. */
int esr_adam_step_dev(float *param, const float *grad, float *exp_avg, float *exp_avg_sq, float *max_exp_avg_sq, size_t n,
                      int32_t *step_counter, const float *hyper, esr_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Evaluation metrics on the GPU (SURVEY 8f rank 3).  Replaces the per-channel CPU calls of infer_ours_cnt.py:81-100:
 * nn.L1Loss / nn.MSELoss, loss/restore.py:42-61 ssim_loss (skimage structural_similarity, 7x7 uniform window, sample
 * covariance, K1 0.01, K2 0.03) and :64-90 psnr_loss (skimage peak_signal_noise_ratio).
 * pred, tgt: fp32 [n_planes, H, W] (plane = sample x channel).  stats: fp64 [n_planes][6] =
 *   {sum |pred - tgt|, sum (pred - tgt)^2, max tgt, min tgt, sum of the SSIM map over the valid region, its pixel count};
 * the host side (esr_b200/metrics.py) turns them into the reference's scalars. */
size_t esr_metrics_workspace_bytes(int n_planes, int H, int W, int win);
int esr_metrics_planes(const float *pred, const float *tgt, int n_planes, int H, int W, int win, double data_range, double *stats,
                       void *workspace, size_t workspace_bytes, esr_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * LPIPS distance (version 0.1, AlexNet backbone, linear heads, spatial=False) of infer_ours_cnt.py:85,90.
 * Replaces: loss/restore.py:10-39 perceptual_loss.__call__'s per-image work, i.e.
 * loss/PerceptualSimilarity/models/__init__.py:32-46 PerceptualLoss.forward (normalize: 2x - 1) ->
 * networks_basic.py:73-101 PNetLin.forward with ScalingLayer (:103-110), pretrained_networks.py:57-95 alexnet (torchvision
 * alexnet().features up to relu5), normalize_tensor (__init__.py:48-50), NetLinLayer (:113-120) and spatial_average.
 *  params    : 15 device pointers to fp32 tensors: torchvision's features.{0,3,6,8,10}.{weight,bias} in that order, then the
 *              v0.1 heads lin{0..4}.model.1.weight ([1,C,1,1]); blob: esr_lpips_param_bytes() bytes.
 *  workspace : esr_lpips_workspace_bytes(n_img, H, W) bytes (0: the size is too small -- the second max-pool needs H, W >= 31,
 *              where the reference raises too), owned by the caller, must outlive the plan; the plan is bound to it.
 *  forward   : planes fp32 [*][H][W]; channel_src int32 [n_img][3] = the plane of each of image i's three input channels (a
 *              count plane repeated to 3 channels, or three planes of an RGB image); normalize != 0 applies 2x - 1 first.
 *              out[p] (fp64) = LPIPS(image pair_a[p], image pair_b[p]) for p < n_pairs; n_img, n_pairs <= the plan's n_img;
 *              indices must be < n_img.  Deterministic, and a pair's value does not depend on the other pairs or images.
 *              No allocation and no host synchronisation: graph-capturable.
 * --------------------------------------------------------------------------------------------- */
typedef void *esr_lpips_t;
size_t esr_lpips_param_bytes(void);
int esr_lpips_pack_params(const float *const *params_host_array_of_device_ptrs, void *blob, esr_stream_t stream);
size_t esr_lpips_workspace_bytes(int n_img, int H, int W);
int esr_lpips_create(esr_lpips_t *plan, int n_img, int H, int W, const void *blob, void *workspace, size_t workspace_bytes);
int esr_lpips_destroy(esr_lpips_t plan);
int esr_lpips_forward(esr_lpips_t plan, const float *planes, const int32_t *channel_src, int n_img, int normalize, int n_pairs,
                      const int32_t *pair_a, const int32_t *pair_b, double *out, esr_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Event-count images of the evaluation script (myutils/vis_events/matplotlib_plot_events.py:125-248, plot_event_cnt with
 * is_save=False) for B images at once.  cnt: fp32 [B, 2, H, W] (0 positive, 1 negative), H * W < 2^24.
 * color_scheme: 0 gray, 1 green_red, 2 blue_red.  out: uint8 [B, H, W, 3] (gray: [B, H, W]); channels in BGR order when
 * bgr != 0 (use_opencv=True), else RGB (the script's cv2.cvtColor(BGR2RGB)).  The 1st / 99th percentiles of every plane
 * are numpy 2.x np.percentile's float32 values, from a radix select; percentiles (optional, device) receives them as
 * fp32 [B, 2 planes, 2] = {p1, p99}.  workspace: esr_render_workspace_bytes(B, H, W) bytes of device memory. */
size_t esr_render_workspace_bytes(int B, int H, int W);
int esr_render_event_cnt(const float *cnt, int B, int H, int W, int color_scheme, int black_background, int is_norm, int bgr,
                         unsigned char *out, float *percentiles, void *workspace, size_t workspace_bytes, esr_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Columnar event reader, device side (SURVEY 8f rank 2).  Replaces, for whole batches of frames:
 *   BaseDataset.binary_search_h5_dset (dataloader/base_dataset.py:78-91; same algorithm as
 *   dataloader/binary_search/binary_search.pyx:17-38) used by H5Dataset.find_ts_index / get_gt_event_indices_num
 *   (dataloader/h5dataset.py:264-270, 451-475): out[i] = the index that bisection returns for queries[i] (exact hit -> the probed
 *   index, else the left insertion point); ts sorted float64 [n], device or host-mapped memory;
 *   H5Dataset.get_events / get_gt_events + BaseDataset.event_formatting (h5dataset.py:492-506, base_dataset.py:26-33):
 *   frame f = rows [start[f], start[f] + off[f+1] - off[f]) of the int16 x / y and float64 t / p columns -> fp32 SoA at
 *   out_*[off[f] ...]; out_ts (optional) = per-frame normalised time (ts - ts[0]) / (ts[-1] - ts[0] + 1e-6) in fp32.
 * esr_gather_events_aug adds H5Dataset.augment_event and SequenceDataset's pause (h5dataset.py:652-670, 769-789, 317-319) as one
 * word per frame, xform[f] (device memory; NULL = esr_gather_events): bit 0 x -> W - 1 - x, bit 1 y -> H - 1 - y, bit 2 p -> -p,
 * bit 3 paused: the frame's events are all (0, 0, 0, 0) (the host gives it length 1, the reference's torch.zeros([4, 1]))
 * and start[f] is not read.  W, H: the stream's sensor resolution, 0 < W, H < 2^23 when xform is given. */
int esr_ts_search(const double *ts, int64_t n, const double *queries, int64_t nq, int64_t *out, esr_stream_t stream);
int esr_gather_events(const int16_t *xs, const int16_t *ys, const double *ts, const double *ps, const int64_t *start,
                      const int64_t *off, int n_frames, int64_t max_len, float *out_xs, float *out_ys, float *out_ts,
                      float *out_ps, esr_stream_t stream);
int esr_gather_events_aug(const int16_t *xs, const int16_t *ys, const double *ts, const double *ps, const int64_t *start,
                          const int64_t *off, const int32_t *xform, int W, int H, int n_frames, int64_t max_len,
                          float *out_xs, float *out_ys, float *out_ts, float *out_ps, esr_stream_t stream);

/* Columns of many recordings -> count banks, one launch per event stream: the batch of HDF5DataLoaderSequence
 * (dataloader/h5dataloader.py:180-233: SequenceDatasets joined by ConcatDataset, stacked by custom_collate), each sample
 * encoded as H5Dataset.__getitem__ does (h5dataset.py:337-354, 508-528) with SequenceDataset's flips and pauses (:652-670,
 * 769-789).  Equal, bit for bit, to esr_gather_events_aug followed by esr_scatter_cnt(writeback = 2) per frame: without and
 * (out_scaled_cnt) with the x / W * kW, y / H * kH lift.
 *   cols: device table [R][3] of the addresses of recording r's int16 xs, int16 ys and float64 ps columns (pinned host
 *         memory or HBM); desc: device table [n_frames]; frame f = rows [start, start + len) of recording rec, transformed
 *         by xform (the word of esr_gather_events_aug; bit 3 paused: the frame adds nothing, len should be 1);
 *   H, W: the stream's resolution (flips and out_cnt [n_frames, 2, H, W]); kH, kW: out_scaled_cnt [n_frames, 2, kH, kW];
 *   max_len: the longest len (grid sizing).  Both banks are zeroed by the call.  Up to 2^31 - 1 frames. */
typedef struct {
    int64_t start, len;
    int32_t rec, xform;
} esr_frame_desc;
int esr_encode_frames_multi(const uint64_t *cols, const esr_frame_desc *desc, int n_frames, int64_t max_len, int H, int W, int kH,
                            int kW, float *out_cnt, float *out_scaled_cnt, esr_stream_t stream);

/* New events of many live streams -> each stream's ring, in one launch (esr_b200.stream.EventStreamPool uploads a round
 * this way).  desc: device table [n_desc], one segment per stream: rows [src, src + count) of the source columns src_xs,
 * src_ys (int16) and src_ps (float64) go to ring elements (position + i) mod capacity of the ring columns xs, ys, ps (device
 * addresses; position is the stream's event count before the segment).  0 <= count <= capacity and capacity > 0; rings must
 * not overlap.  The source may be pinned host memory or device memory.  max_count: the largest count (grid sizing).
 * No allocation, no synchronisation: graph-capturable. */
typedef struct {
    uint64_t xs, ys, ps;
    int64_t capacity, position, count, src;
} esr_ring_desc;
int esr_events_append_rings(const esr_ring_desc *desc, int n_desc, int64_t max_count, const int16_t *src_xs,
                            const int16_t *src_ys, const double *src_ps, esr_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Padded cnt2event rows -> the columns of an event file (esr_b200/superresolve.py).  Completes
 * dataloader/cython_cnt2event/cnt2event_api.py:25-35 (cnt2eventAPI: its [B, maxlen, 4] rows have no caller in the reference's
 * scripts) towards the column types of generate_dataset/tools/event_packagers.py:121-224 (xs, ys int16; ts, ps float64).
 *   rows : fp32 [n_samples, maxlen, 4] = (x, y, t, p) as esr_cnt2event_fused / esr_expand_emit write them (device, 16-byte
 *          aligned); desc: device table [n_samples]: the first `valid` rows of sample s go to rows [dst, dst + valid) of the
 *          columns -- the padding and the zero row of an empty sample (valid = 0) are not written -- and its timestamp t32 becomes
 *          t = t0 + (double)t32 * (t1 - t0): one IEEE subtraction, multiplication and addition, no fused multiply-add, so
 *          numpy's float64 arithmetic reproduces every bit (BaseDataset.event_formatting, dataloader/base_dataset.py:26-33,
 *          inverted without its 1e-6);
 *   max_valid : the largest `valid` (grid sizing; must not exceed maxlen);
 *   xs, ys, ts, ps : device memory or pinned host memory.  x and y must fit int16: the caller refuses resolutions above 32767.
 * One launch, no allocation and no synchronisation: graph-capturable.  Negative lengths, max_valid > maxlen, a null or
 * misaligned pointer return ESR_EINVAL before anything is launched. */
typedef struct {
    int64_t valid, dst;
    double t0, t1;
} esr_column_desc;
int esr_events_to_columns(const float *rows, int n_samples, int64_t maxlen, const esr_column_desc *desc, int64_t max_valid,
                          int16_t *xs, int16_t *ys, double *ts, double *ps, esr_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * uint8 frames -> the dataset's fp32 frames (esr_b200/frames.py): BaseDataset.frame_formatting(cv2.resize(augment_frame(img),
 * dsize, interpolation=cv2.INTER_CUBIC)) of dataloader/h5dataset.py:300-315, 672-685 and base_dataset.py:36-38, many frames
 * and two target sizes in one launch.  The resize is OpenCV's generic fixed-point bicubic for 8-bit images (A = -0.75,
 * source position (float)((d + 0.5) * (1 / (dst / src)) - 0.5) in double, coefficients of fp32 polynomials rounded to
 * nearest-even at 2^11, replicated borders, an exact int32 horizontal pass, then a vertical pass that is an fp32
 * fused-multiply-add chain rounded to nearest-even for the first floor(oW * C / 8) * 8 elements of a row and
 * (sum + 2^21) >> 22 for the rest), saturated to uint8; the result is float(u8) / 255 with an IEEE division.
 *   desc : device table [n]: frame i reads image `src` [H, W(, C)] (pinned host memory or HBM) mirrored by `flips`
 *          (bit 0: x -> W - 1 - x, bit 1: y -> H - 1 - y, applied to the source before the resize) and writes out0
 *          [oH0, oW0(, C)] and, unless NULL, out1 [oH1, oW1(, C)], fp32 device memory;
 *   C    : 1 (grey) or 3 (interleaved colour).  No allocation, no synchronisation. */
typedef struct {
    const uint8_t *src;
    float *out0, *out1;
    int32_t flips, pad_;
} esr_frame_resize_desc;
int esr_resize_frames_cubic(const esr_frame_resize_desc *desc, int n, int H, int W, int C, int oH0, int oW0, int oH1, int oW1,
                            esr_stream_t stream);

/* The same resize with cv2.resize's own uint8 output: the saturated level esr_resize_frames_cubic divides by 255, stored as
 * it is (infer_ours_cnt.py:109 writes (gt_img * 255).astype('uint8'), which is that level: float32(k) / 255 * 255 truncates
 * back to k for every k in 0..255).  One target size; frame i of desc [n] reads `src` [H, W(, C)] mirrored by `flips` (as
 * above) and writes out [oH, oW(, C)] uint8 device memory.  No allocation, no synchronisation. */
typedef struct {
    const uint8_t *src;
    uint8_t *out;
    int32_t flips, pad_;
} esr_frame_resize_u8_desc;
int esr_resize_frames_cubic_u8(const esr_frame_resize_u8_desc *desc, int n, int H, int W, int C, int oH, int oW,
                               esr_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* ESR_B200_H */
