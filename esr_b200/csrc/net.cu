// net.cu -- DeepRecurrNet.forward (models/model.py:294-344) as a fixed launch sequence over the sm_90a kernels.
//
// A "net" is a plan for one (B, N, L, H, W), N = num_frame any odd number >= 3: every intermediate tensor has a fixed place in a
// caller-provided
// workspace, every TMA tensor map / launch descriptor is built once at creation, and forward() only enqueues
// kernels on the caller's stream (no allocation, no host synchronisation, CUDA-graph capturable).
// Recurrent ConvGRU states (models/model.py:72,102-114) live in the workspace and persist across forward() calls
// until esr_net_reset_states, exactly like the reference's `self.states`.
//
// Frame/image ordering everywhere: image = b * N + n.  Fuse images: j = k * B + b (k-th non-middle frame).
// GRU step images: j < B forward direction (sample j), j >= B time-reversed direction (sample j - B).
#include "net.cuh"
#include <cstdlib>
#include <vector>
#include <string>

namespace esr {

// ---- parameter inventory: the reference's state_dict order (68 tensors, SURVEY 8b) ----------------------------
enum P : int {
    P_HEAD_W, P_HEAD_B, P_FE0_W, P_FE0_B, P_FE1_W, P_FE1_B, P_FE2_W, P_FE2_B,
    P_PM0_W, P_PM0_B, P_PM1_W, P_PM1_B, P_LF1_W, P_LF1_B, P_LF2_W, P_LF2_B, P_LF3_W, P_LF3_B,
    P_GX_W, P_GX_B, P_GR_W, P_GR_B, P_GU_W, P_GU_B, P_GO_W, P_GO_B, P_GF_W, P_GF_B,
    P_OF0_W, P_OF0_B, P_OF1_W, P_OF1_B, P_DCN_W, P_DCN_B, P_COM_W, P_COM_B,
    P_CB0_W, P_CB0_B, P_CB1_W, P_CB1_B, P_KER_W, P_KER_B, P_FC0_W, P_FC0_B, P_FC1_W, P_FC1_B,
    P_DF0_W, P_DF0_B, P_DF1_W, P_DF1_B, P_DN0_W, P_DN0_B, P_DN1_W, P_DN1_B,
    P_AT0_W, P_AT0_B, P_AT1_W, P_AT1_B, P_AT2_W, P_AT2_B,
    P_RC0_W, P_RC0_B, P_RC1_W, P_RC1_B, P_RC2_W, P_RC2_B, P_TAIL_W, P_TAIL_B, P_COUNT
};
static_assert(P_COUNT == 68, "reference state_dict has 68 tensors");

// tensor-core layers
enum TL : int { T_PM0, T_PM1, T_LF1, T_LF2, T_LF3, T_GX, T_GZR, T_GO, T_GF, T_OF0, T_OF1, T_COM, T_DCN, T_CB0, T_CB1,
                T_KER, T_DF0, T_DF1, T_DN0, T_DN1, T_AT0, T_RC0, T_COUNT };
struct TLInfo { int w, b, w2, b2, cout, cin, k; };
static const TLInfo TLS[T_COUNT] = {
    {P_PM0_W, P_PM0_B, -1, -1, 64, 128, 3}, {P_PM1_W, P_PM1_B, -1, -1, 1, 64, 3},
    {P_LF1_W, P_LF1_B, -1, -1, 192, 192, 3}, {P_LF2_W, P_LF2_B, -1, -1, 192, 192, 3}, {P_LF3_W, P_LF3_B, -1, -1, 64, 192, 3},
    {P_GX_W, P_GX_B, -1, -1, 64, 64, 3}, {P_GU_W, P_GU_B, P_GR_W, P_GR_B, 128, 128, 3}, {P_GO_W, P_GO_B, -1, -1, 64, 128, 3},
    {P_GF_W, P_GF_B, -1, -1, 64, 128, 1}, {P_OF0_W, P_OF0_B, -1, -1, 64, 128, 3}, {P_OF1_W, P_OF1_B, -1, -1, 64, 64, 3},
    {P_COM_W, P_COM_B, -1, -1, 216, 64, 3}, {P_DCN_W, P_DCN_B, -1, -1, 64, 64, 3}, {P_CB0_W, P_CB0_B, -1, -1, 64, 128, 3},
    {P_CB1_W, P_CB1_B, -1, -1, 64, 64, 3}, {P_KER_W, P_KER_B, -1, -1, 2, 64, 1}, {P_DF0_W, P_DF0_B, -1, -1, 64, 128, 3},
    {P_DF1_W, P_DF1_B, -1, -1, 64, 64, 3}, {P_DN0_W, P_DN0_B, -1, -1, 64, 0, 3}, {P_DN1_W, P_DN1_B, -1, -1, 64, 64, 3},
    {P_AT0_W, P_AT0_B, -1, -1, 1, 64, 3}, {P_RC0_W, P_RC0_B, -1, -1, 32, 64, 3},
};
// input channels of a tensor-core layer: dense_fusion.0 reads cat(N-1 aligned neighbours, middle frame) = N x 64
static int tl_cin(int t, int N) { return t == T_DN0 ? 64 * N : TLS[t].cin; }
static bool num_frame_ok(int N) { return N >= 3 && N % 2 == 1 && N <= 255; }
// direct (CUDA-core) layers
enum DL : int { D_HEAD, D_ENC0, D_ENC1, D_ENC2, D_AT1, D_AT2, D_RC0, D_RC1, D_RC2, D_TAIL, D_COUNT };
struct DLInfo { int w, b, cout, cin; DirectKind kind; };
static const DLInfo DLS[D_COUNT] = {
    {P_HEAD_W, P_HEAD_B, 8, 2, DK_HEAD}, {P_FE0_W, P_FE0_B, 16, 8, DK_ENC0}, {P_FE1_W, P_FE1_B, 32, 16, DK_ENC1},
    {P_FE2_W, P_FE2_B, 64, 32, DK_ENC2}, {P_AT1_W, P_AT1_B, 1, 32, DK_ATT32}, {P_AT2_W, P_AT2_B, 1, 16, DK_ATT16},
    {P_RC0_W, P_RC0_B, 32, 64, DK_RECON0}, {P_RC1_W, P_RC1_B, 16, 32, DK_RECON1}, {P_RC2_W, P_RC2_B, 8, 16, DK_RECON2},
    {P_TAIL_W, P_TAIL_B, 2, 8, DK_TAIL},
};

struct ParamLayout {
    size_t tw[T_COUNT], tb[T_COUNT];     // packed weights / padded bias of TC layers
    size_t dw[D_COUNT], db[D_COUNT];     // direct layers
    size_t dm[D_COUNT];                  // the same weights as the split-bf16 image of the mma.sync kernels
    size_t fc0w, fc0b, fc1w, fc1b;
    size_t nw_ker;                       // fp32 [ci][co] weights of the spatial-attention kernel (conv_narrow)
    size_t total;
};
// Only dense_fusion.0's packed weight depends on N; the entries after it move with its size.  N = 3 is the layout of
// esr_net_param_bytes() / esr_net_pack_params().
static ParamLayout param_layout(int N)
{
    ParamLayout l{};
    {
        size_t off = 0;
        auto take = [&](size_t bytes) { size_t r = off; off = align_up(off + bytes, 256); return r; };
        for (int i = 0; i < T_COUNT; ++i) {
            l.tw[i] = take(tc_packed_weight_bytes(TLS[i].cout, tl_cin(i, N), TLS[i].k * TLS[i].k));
            l.tb[i] = take(sizeof(float) * tc_npad(TLS[i].cout));
        }
        for (int i = 0; i < D_COUNT; ++i) {
            l.dw[i] = take(sizeof(float) * 9 * DLS[i].cin * DLS[i].cout);
            l.db[i] = take(sizeof(float) * DLS[i].cout);
            l.dm[i] = take(mma_weight_bytes(DLS[i].cout, DLS[i].cin));
        }
        l.fc0w = take(sizeof(float) * 32 * 64); l.fc0b = take(sizeof(float) * 32);
        l.fc1w = take(sizeof(float) * 128 * 32); l.fc1b = take(sizeof(float) * 128);
        l.nw_ker = take(sizeof(float) * 64 * 2);
        l.total = off;
    }
    return l;
}

// ---- the plan ---------------------------------------------------------------------------------------------------
// Sequence plan: B sequences x L frames, Wn = L-N+1 sliding windows.  Everything that does not depend on the
// recurrent state is evaluated ONCE for all windows (virtual batch VB = Wn*B, window-major vb = w*B + b), per-frame
// work (encoder, attention maps) once per bank frame (FR = B*L frames, frame = b*L + l); only the ConvGRU chain runs
// window after window.  L = N gives the reference's single-window forward.
struct Net {
    int B, N, L, Wn, VB, FR, H, W, Hc, Wc, h, w;
    int pad_top, pad_bottom, pad_left, pad_right;
    ParamLayout P;  // layout of the packed blob for this N
    char *params;   // packed blob
    char *ws;       // workspace
    size_t ws_bytes;
    // tensors
    SplitTensor t_e0, t_e1, F, t_pm0, t_cat, t_lf1, t_lf2, ltc, xc, hs, rh, tp;
    SplitTensor t_of0, t_off, cols, aligned, t_cb0, feat, ycat, t_df0, fused, t_dn0, x0, pre0, up0, x1, pre1, x2, pre2, x3;
    float *maps, *zbuf, *om, *sk, *mx, *ck, *att0, *att1, *att2;
    // index maps (device)
    int *m_fr, *m_pairA, *m_pairB, *m_ltc5, *m_lf3res, *m_f0, *m_fm, *m_gf_f, *m_gf_r, *m_gfres;
    std::vector<int *> m_gx, m_gh;     // per GRU step (Wn * N of them)
    // prepared tensor-core launches
    ConvTCArgs c_pm0, c_pm1, c_lf1, c_lf2, c_lf3, c_gx, c_gf, c_of0, c_of1, c_com, c_dcn, c_cb0, c_cb1, c_ker, c_df0, c_df1,
        c_dn0, c_dn1, c_at0, c_rc0;
    std::vector<ConvTCArgs> c_gzr, c_go;
    void *dcn_plan = nullptr;          // fused sampling + contraction (dcn_fused.cu); nullptr = columns + 1x1 GEMM
    DirectArgs d[D_COUNT];
};

static size_t split_bytes(int n_img, int H, int W, int C) { return (size_t)2 * n_img * H * W * C * sizeof(__nv_bfloat16); }

struct Arena {
    char *base; size_t off = 0; size_t cap;
    Arena(char *b, size_t c) : base(b), cap(c) {}
    void *take(size_t bytes) { size_t r = off; off = align_up(off + bytes, 1024); return base ? base + r : nullptr; }
    SplitTensor split(int n_img, int H, int W, int C)
    {
        SplitTensor t; t.n_img = n_img; t.H = H; t.W = W; t.C = C;
        t.base = (__nv_bfloat16 *)take(split_bytes(n_img, H, W, C));
        return t;
    }
};

// lays out every tensor; with net.ws == nullptr it only measures
static size_t layout(Net &n)
{
    Arena A(n.ws, n.ws_bytes);
    const int B = n.B, N = n.N, VB = n.VB, FR = n.FR, VN = VB * N, h = n.h, w = n.w, Hc = n.Hc, Wc = n.Wc;
    const int nf = (N - 1) * VB, np = VB * (N + 1), nsteps = n.Wn * N;
    // recurrent state first so that its address does not depend on later changes
    n.hs = A.split((nsteps + 1) * 2 * B, h, w, 64);
    n.t_e0 = A.split(FR, Hc / 2, Wc / 2, 16);
    n.t_e1 = A.split(FR, Hc / 4, Wc / 4, 32);
    n.F = A.split(FR, h, w, 64);
    n.att0 = (float *)A.take(sizeof(float) * FR * h * w);
    n.att1 = (float *)A.take(sizeof(float) * FR * 4 * h * w);
    n.att2 = (float *)A.take(sizeof(float) * FR * 16 * h * w);
    n.t_pm0 = A.split(np, h, w, 64);
    n.maps = (float *)A.take(sizeof(float) * np * h * w);
    n.t_cat = A.split(VN, h, w, 192);
    n.t_lf1 = A.split(VN, h, w, 192);
    n.t_lf2 = A.split(VN, h, w, 192);
    n.ltc = A.split(VN, h, w, 64);
    n.xc = A.split(VN, h, w, 64);
    n.rh = A.split(2 * B, h, w, 64);
    n.zbuf = (float *)A.take(sizeof(float) * 2 * B * h * w * 64);
    n.tp = A.split(VN, h, w, 64);
    n.t_of0 = A.split(nf, h, w, 64);
    n.t_off = A.split(nf, h, w, 64);
    n.om = (float *)A.take(sizeof(float) * nf * h * w * 216);
    n.cols = A.split(nf, h, w, 576);
    n.aligned = A.split(nf, h, w, 64);
    n.t_cb0 = A.split(nf, h, w, 64);
    n.feat = A.split(nf, h, w, 64);
    n.sk = (float *)A.take(sizeof(float) * nf * h * w * 2);
    n.mx = (float *)A.take(sizeof(float) * nf * 64);
    n.ck = (float *)A.take(sizeof(float) * nf * 128);
    n.ycat = A.split(nf, h, w, 128);
    n.t_df0 = A.split(nf, h, w, 64);
    n.fused = A.split(nf, h, w, 64);
    n.t_dn0 = A.split(VB, h, w, 64);
    n.x0 = A.split(VB, h, w, 64);
    n.pre0 = A.split(VB, h, w, 64);
    n.up0 = A.split(VB, 2 * h, 2 * w, 64);
    n.x1 = A.split(VB, 2 * h, 2 * w, 32);
    n.pre1 = A.split(VB, 2 * h, 2 * w, 32);
    n.x2 = A.split(VB, 4 * h, 4 * w, 16);
    n.pre2 = A.split(VB, 4 * h, 4 * w, 16);
    n.x3 = A.split(VB, Hc, Wc, 8);
    // index maps
    auto ints = [&](size_t cnt) { return (int *)A.take(sizeof(int) * cnt); };
    n.m_fr = ints(VN);
    n.m_pairA = ints(np); n.m_pairB = ints(np); n.m_ltc5 = ints((size_t)VN * 5); n.m_lf3res = ints(VN);
    n.m_f0 = ints(nf); n.m_fm = ints(nf);
    n.m_gf_f = ints(VN); n.m_gf_r = ints(VN); n.m_gfres = ints(VN);
    n.m_gx.resize(nsteps); n.m_gh.resize(nsteps);
    for (int s = 0; s < nsteps; ++s) { n.m_gx[s] = ints(2 * B); n.m_gh[s] = ints(2 * B); }
    return A.off;
}

static int upload(int *dst, const std::vector<int> &v, cudaStream_t st)
{
    ESR_CUDA_CHECK(cudaMemcpyAsync(dst, v.data(), sizeof(int) * v.size(), cudaMemcpyHostToDevice, st));
    ESR_CUDA_CHECK(cudaStreamSynchronize(st));   // v is a temporary
    return ESR_OK;
}

static const void *pw(const Net &n, int t) { return n.params + n.P.tw[t]; }
static const float *pb(const Net &n, int t) { return (const float *)(n.params + n.P.tb[t]); }

static ConvTCDesc mk(const Net &n, int t, int n_img, int act)
{
    ConvTCDesc d;
    d.wpacked = pw(n, t); d.bias = pb(n, t); d.cout = TLS[t].cout; d.ntaps = TLS[t].k * TLS[t].k; d.n_img = n_img; d.act = act;
    return d;
}

static SplitTensor view_imgs(const SplitTensor &t, int first_img)
{
    // a window starting at image `first_img`; planes keep the parent's distance
    SplitTensor v = t;
    v.base = t.base + (size_t)first_img * t.H * t.W * t.C;
    v.plane_override = t.plane();
    return v;
}

static int build(Net &n, cudaStream_t st)
{
    const int B = n.B, N = n.N, L = n.L, Wn = n.Wn, VB = n.VB, FR = n.FR, VN = VB * N;
    const int nf = (N - 1) * VB, np = VB * (N + 1), mid = (N - 1) / 2;
    int rc;
    // bank frame of window slot (vb = w*B + b, n): b*L + w + n
    auto fr = [&](int vb, int i) { const int w = vb / B, b = vb % B; return b * L + w + i; };
    // ---------------- index maps
    {
        std::vector<int> mfr(VN), a(np), b(np), l5((size_t)VN * 5), r(VN);
        for (int vb = 0; vb < VB; ++vb) {
            for (int p = 0; p <= N; ++p) {           // pair p: (0,0), (0,1), ..., (N-2,N-1), (N-1,N-1)
                const int fa = p == 0 ? 0 : p - 1, fb = p == N ? N - 1 : p;
                a[vb * (N + 1) + p] = fr(vb, fa);
                b[vb * (N + 1) + p] = fr(vb, fb);
            }
            for (int i = 0; i < N; ++i) {            // window slot i: frames (i-1, i, i+1) edge-replicated (model.py:133-143)
                const int i0 = i == 0 ? 0 : i - 1, i2 = i == N - 1 ? N - 1 : i + 1;
                int *q = &l5[(size_t)(vb * N + i) * 5];
                q[0] = fr(vb, i0); q[1] = fr(vb, i); q[2] = fr(vb, i2);
                q[3] = vb * (N + 1) + i;             // map of pair (i0, i)
                q[4] = vb * (N + 1) + i + 1;         // map of pair (i, i2)
                r[vb * N + i] = fr(vb, i);
                mfr[vb * N + i] = fr(vb, i);
            }
        }
        if ((rc = upload(n.m_fr, mfr, st)) || (rc = upload(n.m_pairA, a, st)) || (rc = upload(n.m_pairB, b, st)) ||
            (rc = upload(n.m_ltc5, l5, st)) || (rc = upload(n.m_lf3res, r, st)) || (rc = upload(n.m_gfres, r, st)))
            return rc;
        std::vector<int> f0(nf), fm(nf);
        int k = 0;
        for (int i = 0; i < N; ++i) {
            if (i == mid) continue;
            for (int vb = 0; vb < VB; ++vb) { f0[k * VB + vb] = vb * N + i; fm[k * VB + vb] = vb * N + mid; }
            ++k;
        }
        if ((rc = upload(n.m_f0, f0, st)) || (rc = upload(n.m_fm, fm, st))) return rc;
        // GRU: global step g = w*N + s reads state slot g and writes slot g+1 (slot 0 = carried state)
        std::vector<int> gf(VN), gr(VN);
        for (int vb = 0; vb < VB; ++vb) {
            const int w = vb / B, bb = vb % B;
            for (int i = 0; i < N; ++i) {
                gf[vb * N + i] = (w * N + i + 1) * 2 * B + bb;             // forward output for frame i = step i of window w
                gr[vb * N + i] = (w * N + (N - 1 - i) + 1) * 2 * B + B + bb; // reverse output for frame i = step N-1-i
            }
        }
        if ((rc = upload(n.m_gf_f, gf, st)) || (rc = upload(n.m_gf_r, gr, st))) return rc;
        for (int w = 0; w < Wn; ++w)
            for (int s = 0; s < N; ++s) {
                const int g = w * N + s;
                std::vector<int> gx(2 * B), gh(2 * B);
                for (int bb = 0; bb < B; ++bb) {
                    gx[bb] = (w * B + bb) * N + s; gx[B + bb] = (w * B + bb) * N + (N - 1 - s);
                    gh[bb] = g * 2 * B + bb; gh[B + bb] = g * 2 * B + B + bb;
                }
                if ((rc = upload(n.m_gx[g], gx, st)) || (rc = upload(n.m_gh[g], gh, st))) return rc;
            }
    }
    // ---------------- tensor-core launches
    ConvTCDesc d;
    // pred_map on the N+1 unique (frame, frame) pairs of every window
    d = mk(n, T_PM0, np, ACT_RELU); d.n_src = 2; d.src[0] = n.F; d.src[1] = n.F; d.src_img[0] = n.m_pairA; d.src_img[1] = n.m_pairB;
    d.out = n.t_pm0;
    if ((rc = conv_tc_prepare(d, &n.c_pm0))) return rc;
    d = mk(n, T_PM1, np, ACT_SIGMOID); d.src[0] = n.t_pm0; d.out_f32 = n.maps; d.out_f32_C = 1;
    if ((rc = conv_tc_prepare(d, &n.c_pm1))) return rc;
    // local_fusion: ResidualBlock(192) + conv 192->64, + feat1
    d = mk(n, T_LF1, VN, ACT_RELU); d.src[0] = n.t_cat; d.out = n.t_lf1;
    if ((rc = conv_tc_prepare(d, &n.c_lf1))) return rc;
    d = mk(n, T_LF2, VN, ACT_RELU); d.src[0] = n.t_lf1; d.res_mode = RES_PRE_ACT; d.res = n.t_cat; d.out = n.t_lf2;
    if ((rc = conv_tc_prepare(d, &n.c_lf2))) return rc;
    d = mk(n, T_LF3, VN, ACT_NONE); d.src[0] = n.t_lf2; d.res_mode = RES_POST_ACT; d.res = n.F; d.res_img = n.m_lf3res; d.out = n.ltc;
    if ((rc = conv_tc_prepare(d, &n.c_lf3))) return rc;
    // ConvGRU: x-side conv once for all window slots (same weights in both directions)
    d = mk(n, T_GX, VN, ACT_RELU); d.src[0] = n.ltc; d.out = n.xc;
    if ((rc = conv_tc_prepare(d, &n.c_gx))) return rc;
    const int nsteps = Wn * N;
    n.c_gzr.resize(nsteps); n.c_go.resize(nsteps);
    for (int g = 0; g < nsteps; ++g) {
        d = mk(n, T_GZR, 2 * B, ACT_NONE); d.n_src = 2; d.src[0] = n.xc; d.src_img[0] = n.m_gx[g]; d.src[1] = n.hs; d.src_img[1] = n.m_gh[g];
        d.epi_mode = EPI_GRU_ZR; d.h_prev = view_imgs(n.hs, g * 2 * B); d.z_buf = n.zbuf; d.out = n.rh;
        if ((rc = conv_tc_prepare(d, &n.c_gzr[g]))) return rc;
        d = mk(n, T_GO, 2 * B, ACT_NONE); d.n_src = 2; d.src[0] = n.xc; d.src_img[0] = n.m_gx[g]; d.src[1] = n.rh;
        d.epi_mode = EPI_GRU_OUT; d.h_prev = view_imgs(n.hs, g * 2 * B); d.z_buf = n.zbuf; d.out = view_imgs(n.hs, (g + 1) * 2 * B);
        if ((rc = conv_tc_prepare(d, &n.c_go[g]))) return rc;
    }
    d = mk(n, T_GF, VN, ACT_RELU); d.n_src = 2; d.src[0] = n.hs; d.src_img[0] = n.m_gf_f; d.src[1] = n.hs; d.src_img[1] = n.m_gf_r;
    d.res_mode = RES_POST_ACT; d.res = n.F; d.res_img = n.m_gfres; d.out = n.tp;
    if ((rc = conv_tc_prepare(d, &n.c_gf))) return rc;
    // STFusion.fuse on the N-1 non-middle frames of every window
    d = mk(n, T_OF0, nf, ACT_RELU); d.n_src = 2; d.src[0] = n.tp; d.src_img[0] = n.m_f0; d.src[1] = n.tp; d.src_img[1] = n.m_fm; d.out = n.t_of0;
    if ((rc = conv_tc_prepare(d, &n.c_of0))) return rc;
    d = mk(n, T_OF1, nf, ACT_NONE); d.src[0] = n.t_of0; d.out = n.t_off;
    if ((rc = conv_tc_prepare(d, &n.c_of1))) return rc;
    d = mk(n, T_COM, nf, ACT_SIGMOID); d.act_from = 144; d.src[0] = n.t_off; d.out_f32 = n.om; d.out_f32_C = 216;
    if ((rc = conv_tc_prepare(d, &n.c_com))) return rc;
    d = mk(n, T_DCN, nf, ACT_RELU); d.ntaps = 1; d.src[0] = n.cols; d.out = n.aligned;
    if ((rc = conv_tc_prepare(d, &n.c_dcn))) return rc;
    // default: the sampler writes the swizzled A tiles straight into shared memory (no columns tensor);
    // ESR_DCN_COLUMNS=1 keeps the two-kernel path (columns in HBM + 1x1 GEMM) for comparison
    const bool dcn_cols = getenv("ESR_DCN_COLUMNS") != nullptr;      // read per net, so a test can build both
    if (!dcn_cols) {
        if ((rc = dcn_fused_prepare(n.tp, n.m_f0, n.om, pw(n, T_DCN), pb(n, T_DCN), nf, ACT_RELU, n.aligned, &n.dcn_plan))) return rc;
    }
    d = mk(n, T_CB0, nf, ACT_RELU); d.n_src = 2; d.src[0] = n.aligned; d.src[1] = n.tp; d.src_img[1] = n.m_fm; d.out = n.t_cb0;
    if ((rc = conv_tc_prepare(d, &n.c_cb0))) return rc;
    d = mk(n, T_CB1, nf, ACT_NONE); d.src[0] = n.t_cb0; d.out = n.feat;
    if ((rc = conv_tc_prepare(d, &n.c_cb1))) return rc;
    d = mk(n, T_KER, nf, ACT_SIGMOID); d.src[0] = n.feat; d.out_f32 = n.sk; d.out_f32_C = 2;
    if ((rc = conv_tc_prepare(d, &n.c_ker))) return rc;
    d = mk(n, T_DF0, nf, ACT_RELU); d.src[0] = n.ycat; d.out = n.t_df0;
    if ((rc = conv_tc_prepare(d, &n.c_df0))) return rc;
    d = mk(n, T_DF1, nf, ACT_NONE); d.src[0] = n.t_df0; d.out = n.fused;
    if ((rc = conv_tc_prepare(d, &n.c_df1))) return rc;
    // dense_fusion.0 over cat(fused_0 .. fused_{N-2}, middle frame) without materialising the concatenation: `fused` holds the N-1
    // neighbours k-major (image k * VB + vb), so it is one source of N-1 chunks VB images apart; the first VB entries of m_fm
    // map window vb to its middle frame
    d = mk(n, T_DN0, VB, ACT_RELU); d.n_src = 2;
    d.src[0] = n.fused; d.src_chunks[0] = N - 1; d.chunk_img_step[0] = VB; d.src[1] = n.tp; d.src_img[1] = n.m_fm;
    d.out = n.t_dn0;
    if ((rc = conv_tc_prepare(d, &n.c_dn0))) return rc;
    d = mk(n, T_DN1, VB, ACT_NONE); d.src[0] = n.t_dn0; d.out = n.x0;
    if ((rc = conv_tc_prepare(d, &n.c_dn1))) return rc;
    d = mk(n, T_AT0, FR, ACT_SIGMOID); d.src[0] = n.F; d.out_f32 = n.att0; d.out_f32_C = 1;
    if ((rc = conv_tc_prepare(d, &n.c_at0))) return rc;
    // recons[0] (64 -> 32 at 2h x 2w) on the tensor cores: bilinear x2 is materialised once, then a plain 3x3 conv
    d = mk(n, T_RC0, VB, ACT_RELU); d.src[0] = n.up0; d.out = n.x1;
    if ((rc = conv_tc_prepare(d, &n.c_rc0))) return rc;

    // ---------------- direct launches
    const ParamLayout &Lp = n.P;
    auto base = [&](int i, int act) {
        DirectArgs a; a.w = (const float *)(n.params + Lp.dw[i]); a.bias = (const float *)(n.params + Lp.db[i]); a.act = act;
        a.w_mma = n.params + Lp.dm[i];
        return a;
    };
    auto in_split = [&](DirectArgs &a, const SplitTensor &t) { a.in_split = t.base; a.in_plane = t.plane(); a.Hin = t.H; a.Win = t.W; };
    auto out_split = [&](DirectArgs &a, const SplitTensor &t, int n_img) {
        a.out_split = t.base; a.out_plane = t.plane(); a.Hout = t.H; a.Wout = t.W; a.n_img = n_img;
    };
    // head (2->8 @HR) is fused into the first encoder layer (8->16, stride 2): its 8-channel full-resolution output is
    // recomputed per tile in shared memory instead of taking a round trip through HBM
    DirectArgs a = base(D_ENC0, ACT_RELU);
    a.w0 = (const float *)(n.params + Lp.dw[D_HEAD]); a.b0 = (const float *)(n.params + Lp.db[D_HEAD]);
    a.Hin = n.H; a.Win = n.W; a.pad_top = n.pad_top; a.pad_bottom = n.pad_bottom; a.pad_left = n.pad_left; a.pad_right = n.pad_right;
    out_split(a, n.t_e0, FR); n.d[D_ENC0] = a;
    a = base(D_ENC1, ACT_RELU); in_split(a, n.t_e0); out_split(a, n.t_e1, FR); n.d[D_ENC1] = a;
    a = base(D_ENC2, ACT_RELU); in_split(a, n.t_e1); out_split(a, n.F, FR); n.d[D_ENC2] = a;
    a = base(D_AT1, ACT_SIGMOID); in_split(a, n.t_e1); a.out_f32 = n.att1; a.Hout = n.t_e1.H; a.Wout = n.t_e1.W; a.n_img = FR; n.d[D_AT1] = a;
    a = base(D_AT2, ACT_SIGMOID); in_split(a, n.t_e0); a.out_f32 = n.att2; a.Hout = n.t_e0.H; a.Wout = n.t_e0.W; a.n_img = FR; n.d[D_AT2] = a;
    a = base(D_RC0, ACT_RELU); in_split(a, n.pre0); out_split(a, n.x1, VB); n.d[D_RC0] = a;
    a = base(D_RC1, ACT_RELU); in_split(a, n.pre1); out_split(a, n.x2, VB); n.d[D_RC1] = a;
    a = base(D_RC2, ACT_RELU); in_split(a, n.pre2); out_split(a, n.x3, VB); n.d[D_RC2] = a;
    a = base(D_TAIL, ACT_RELU); in_split(a, n.x3); a.Hout = n.Hc; a.Wout = n.Wc; a.n_img = VB;
    a.crop_top = n.pad_top; a.crop_left = n.pad_left; a.out_H = n.H; a.out_W = n.W; n.d[D_TAIL] = a;
    return ESR_OK;
}

// Optional per-launch timing (bench.py roofline): CUDA events on the launching stream around every kernel.
struct Prof {
    struct Entry { cudaEvent_t e0, e1; int cls; double flops, bytes; const char *name; };
    std::vector<Entry> entries;
};
enum ProfClass : int { PC_TC = 0, PC_DIRECT = 1, PC_OTHER = 2 };

static double tc_flops(const ConvTCArgs &a) { return 2.0 * a.n_img * a.H * a.W * (double)a.cout * (double)a.nkb * 64.0; }
static double direct_flops(int dl, const DirectArgs &a)
{
    return 2.0 * a.n_img * a.Hout * a.Wout * (double)DLS[dl].cout * (double)DLS[dl].cin * 9.0;
}
// algorithmic bytes of a launch: every input and output element once at 4 bytes (fp32, or split bf16 = 2 x 2 bytes); weights
// (<= 1.3 MB per layer, L2-resident) are not counted
static double tc_bytes(const ConvTCArgs &a)
{
    return 4.0 * a.n_img * a.H * a.W * ((double)a.nkb * 64.0 / a.ntaps + (double)a.cout);
}
static double direct_bytes(int dl, const DirectArgs &a)
{
    const double in_px = a.Hin > 0 ? (double)a.Hin * a.Win : (double)a.Hout * a.Wout;
    return 4.0 * a.n_img * (in_px * DLS[dl].cin + (double)a.Hout * a.Wout * DLS[dl].cout);
}

static int forward(Net &n, const float *input, const int *in_img, float *output, cudaStream_t st, Prof *prof = nullptr)
{
    int rc;
#define RUNC(name_, cls_, flops_, bytes_, x)                                               \
    do {                                                                                   \
        Prof::Entry pe{};                                                                  \
        if (prof) {                                                                        \
            cudaEventCreate(&pe.e0); cudaEventCreate(&pe.e1);                              \
            pe.cls = (cls_); pe.flops = (flops_); pe.bytes = (bytes_); pe.name = (name_);  \
            cudaEventRecord(pe.e0, st);                                                    \
        }                                                                                  \
        rc = (x);                                                                          \
        if (prof) { cudaEventRecord(pe.e1, st); prof->entries.push_back(pe); }             \
        if (rc) return rc;                                                                 \
    } while (0)
#define RUN(name_, bytes_, x) RUNC(name_, PC_OTHER, 0.0, bytes_, x)
#define RUNT(name_, args) RUNC(name_, PC_TC, tc_flops(args), tc_bytes(args), conv_tc_launch(args, st))
#define RUND(name_, kind, dl, args) RUNC(name_, PC_DIRECT, direct_flops(dl, args), direct_bytes(dl, args), conv_direct(kind, args, st))
    const int B = n.B, N = n.N, VB = n.VB, VN = VB * N, nf = (N - 1) * VB, nsteps = n.Wn * N;
    const ParamLayout &L = n.P;
    // ---- per-frame work, once per bank frame: head + encoder (models/model.py:329-331) and the three attention maps
    //      of scale_aggre (model.py:259-262), which depend on the encoder features only
    const double px = (double)n.h * n.w;             // feature-resolution pixels per image
    DirectArgs a = n.d[D_ENC0]; a.in_f32 = input; a.in_img = in_img;
    RUNC("head+enc0", PC_DIRECT, direct_flops(D_ENC0, a) + 2.0 * a.n_img * n.Hc * n.Wc * 8.0 * 2.0 * 9.0,
         4.0 * a.n_img * ((double)n.H * n.W * 2.0 + (double)a.Hout * a.Wout * 16.0), conv_direct(DK_HEAD_ENC0, a, st));
    RUND("enc1", DK_ENC1, D_ENC1, n.d[D_ENC1]);
    RUND("enc2", DK_ENC2, D_ENC2, n.d[D_ENC2]);
    RUNT("atten0", n.c_at0);
    RUND("atten1", DK_ATT32, D_AT1, n.d[D_AT1]);
    RUND("atten2", DK_ATT16, D_AT2, n.d[D_AT2]);
    // ---- TimePropagation.local_time_corre for every window (model.py:77-89,133-146)
    RUNT("pred_map0", n.c_pm0);
    RUNT("pred_map1", n.c_pm1);
    RUN("ltc_cat", 4.0 * VN * px * (192.0 + 192.0 + 2.0), ltc_cat(n.F, n.maps, n.m_ltc5, VN, n.t_cat, st));
    RUNT("local_fusion.res.conv1", n.c_lf1);
    RUNT("local_fusion.res.conv2", n.c_lf2);
    RUNT("local_fusion.conv", n.c_lf3);
    // ---- TimePropagation.global_time_corre: bidirectional ConvGRU (model.py:91-124); the only serial part:
    //      window after window, step after step, both directions batched as 2B images
    RUNT("gru.xconv", n.c_gx);
    for (int g = 0; g < nsteps; ++g) {
        RUNT("gru.zr", n.c_gzr[g]);
        RUNT("gru.out", n.c_go[g]);
    }
    RUNT("global_fusion", n.c_gf);
    // carried states: the last slot becomes slot 0 of the next call
    RUN("state_carry", 4.0 * 2 * B * px * 128.0, copy_split(view_imgs(n.hs, nsteps * 2 * B), nullptr, 2 * B, view_imgs(n.hs, 0), st));
    // ---- STFusion.fuse for the non-middle frames (model.py:208-231)
    RUNT("offset0", n.c_of0);
    RUNT("offset1", n.c_of1);
    RUNT("conv_offset_mask", n.c_com);
    if (n.dcn_plan) {
        RUNC("dcn_fused", PC_TC, 2.0 * 64 * 576 * (double)nf * px, 4.0 * nf * px * (64.0 + 216.0 + 64.0), dcn_fused_launch(n.dcn_plan, st));
    } else {
        RUN("dcn_columns", 4.0 * nf * px * (64.0 + 216.0 + 576.0), dcn_columns(n.tp, n.m_f0, n.om, nf, n.cols, st));
        RUNT("dcn_gemm", n.c_dcn);
    }
    RUNT("convblock0", n.c_cb0);
    RUNT("convblock1", n.c_cb1);
    RUNC("spatial_kernel", PC_OTHER, 0.0, tc_bytes(n.c_ker), conv_narrow(n.feat, nullptr, (const float *)(n.params + L.nw_ker), pb(n, T_KER), 2, 1, nf, n.sk, st));
    RUN("chan_max", 4.0 * nf * px * 64.0, chan_max(n.feat, nf, n.mx, st));
    RUN("attn_mlp", 4.0 * nf * 192.0, attn_mlp(n.mx, nf, (const float *)(n.params + L.fc0w), (const float *)(n.params + L.fc0b),
                 (const float *)(n.params + L.fc1w), (const float *)(n.params + L.fc1b), n.ck, st));
    RUN("attn_apply", 4.0 * nf * px * (64.0 + 64.0 + 2.0 + 128.0), attn_apply(n.aligned, n.tp, n.m_fm, n.sk, n.ck, nf, n.ycat, st));
    RUNT("dcn_fusion0", n.c_df0);
    RUNT("dcn_fusion1", n.c_df1);
    // ---- dense fusion (model.py:233-251)
    RUNT("dense_fusion0", n.c_dn0);
    RUNT("dense_fusion1", n.c_dn1);
    // ---- scale aggregation + reconstruction x3 (model.py:253-291), tail (model.py:337)
    RUN("scale_aggre0", 4.0 * VB * px * (64.0 * (2 + N) + N), scale_aggregate(n.x0, n.F, n.att0, n.m_fr, VB, N, n.pre0, st));
    RUN("upsample2x", 4.0 * VB * px * 64.0 * 5.0, upsample2x(n.pre0, VB, n.up0, st));
    RUNT("recons0", n.c_rc0);
    RUN("scale_aggre1", 4.0 * VB * 4.0 * px * (32.0 * (2 + N) + N), scale_aggregate(n.x1, n.t_e1, n.att1, n.m_fr, VB, N, n.pre1, st));
    RUND("recons1", DK_RECON1, D_RC1, n.d[D_RC1]);
    RUN("scale_aggre2", 4.0 * VB * 16.0 * px * (16.0 * (2 + N) + N), scale_aggregate(n.x2, n.t_e0, n.att2, n.m_fr, VB, N, n.pre2, st));
    RUND("recons2", DK_RECON2, D_RC2, n.d[D_RC2]);
    a = n.d[D_TAIL]; a.out_f32 = output;
    RUNC("tail", PC_DIRECT, direct_flops(D_TAIL, a), 4.0 * a.n_img * ((double)n.Hc * n.Wc * 8.0 + (double)n.H * n.W * 2.0),
         conv_direct(DK_TAIL, a, st));
#undef RUN
#undef RUNT
#undef RUND
#undef RUNC
    return ESR_OK;
}

} // namespace esr

// =================================================================================================
// C ABI
// =================================================================================================
using namespace esr;

static void net_dims(Net &n, int B, int N, int L, int H, int W)
{
    n.B = B; n.N = N; n.L = L; n.Wn = L - N + 1; n.VB = n.Wn * B; n.FR = B * L; n.H = H; n.W = W;
    n.Hc = (H + 7) / 8 * 8; n.Wc = (W + 7) / 8 * 8; n.h = n.Hc / 8; n.w = n.Wc / 8;
    // CropSize (models/model_util.py:148-151): ceil on top/left, floor on bottom/right
    n.pad_top = (n.Hc - H + 1) / 2; n.pad_bottom = (n.Hc - H) / 2;
    n.pad_left = (n.Wc - W + 1) / 2; n.pad_right = (n.Wc - W) / 2;
}

extern "C" size_t esr_net_param_bytes_n(int num_frame) { return num_frame_ok(num_frame) ? param_layout(num_frame).total : 0; }
extern "C" size_t esr_net_param_bytes(void) { return esr_net_param_bytes_n(3); }

extern "C" int esr_net_pack_params_n(int num_frame, const float *const *p, void *blob, esr_stream_t stream)
{
    ESR_REQUIRE(p && blob, "esr_net_pack_params: null pointer");
    ESR_REQUIRE(num_frame_ok(num_frame), "esr_net_pack_params: num_frame=%d (odd, >= 3)", num_frame);
    cudaStream_t st = (cudaStream_t)stream;
    const ParamLayout L = param_layout(num_frame);
    char *out = (char *)blob;
    int rc;
    ESR_CUDA_CHECK(cudaMemsetAsync(blob, 0, L.total, st));
    for (int i = 0; i < T_COUNT; ++i) {
        const TLInfo &t = TLS[i];
        const int co_each = t.w2 >= 0 ? t.cout / 2 : t.cout;
        if ((rc = pack_conv_weight2(p[t.w], t.w2 >= 0 ? p[t.w2] : nullptr, co_each, tl_cin(i, num_frame), t.k, out + L.tw[i], st)))
            return rc;
        ESR_CUDA_CHECK(cudaMemcpyAsync(out + L.tb[i], p[t.b], sizeof(float) * co_each, cudaMemcpyDeviceToDevice, st));
        if (t.b2 >= 0)
            ESR_CUDA_CHECK(cudaMemcpyAsync(out + L.tb[i] + sizeof(float) * co_each, p[t.b2], sizeof(float) * co_each,
                                           cudaMemcpyDeviceToDevice, st));
    }
    for (int i = 0; i < D_COUNT; ++i) {
        const DLInfo &d = DLS[i];
        if ((rc = pack_direct_weight(p[d.w], d.cout, d.cin, (float *)(out + L.dw[i]), st))) return rc;
        if ((rc = pack_mma_weight(p[d.w], d.cout, d.cin, out + L.dm[i], st))) return rc;
        ESR_CUDA_CHECK(cudaMemcpyAsync(out + L.db[i], p[d.b], sizeof(float) * d.cout, cudaMemcpyDeviceToDevice, st));
    }
    ESR_CUDA_CHECK(cudaMemcpyAsync(out + L.fc0w, p[P_FC0_W], sizeof(float) * 32 * 64, cudaMemcpyDeviceToDevice, st));
    ESR_CUDA_CHECK(cudaMemcpyAsync(out + L.fc0b, p[P_FC0_B], sizeof(float) * 32, cudaMemcpyDeviceToDevice, st));
    ESR_CUDA_CHECK(cudaMemcpyAsync(out + L.fc1w, p[P_FC1_W], sizeof(float) * 128 * 32, cudaMemcpyDeviceToDevice, st));
    ESR_CUDA_CHECK(cudaMemcpyAsync(out + L.fc1b, p[P_FC1_B], sizeof(float) * 128, cudaMemcpyDeviceToDevice, st));
    if ((rc = pack_narrow_weight(p[P_KER_W], 2, 1, (float *)(out + L.nw_ker), st))) return rc;
    return ESR_OK;
}
extern "C" int esr_net_pack_params(const float *const *p, void *blob, esr_stream_t stream) { return esr_net_pack_params_n(3, p, blob, stream); }

// bytes from `p` to the end of the device allocation holding it (0 = unknown): a blob packed for a smaller num_frame is too short
static size_t bytes_to_allocation_end(const void *p)
{
    typedef CUresult (*PFN_range)(CUdeviceptr *, size_t *, CUdeviceptr);
    static PFN_range fn = [] {
        void *f = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuMemGetAddressRange", &f, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess)
            f = nullptr;
        return (PFN_range)f;
    }();
    CUdeviceptr base = 0;
    size_t size = 0;
    if (!fn || fn(&base, &size, (CUdeviceptr)p) != CUDA_SUCCESS) return 0;
    return (size_t)(base + size - (CUdeviceptr)p);
}

extern "C" size_t esr_net_workspace_bytes(int B, int N, int L, int H, int W)
{
    if (L < N) return 0;
    Net n{};
    net_dims(n, B, N, L, H, W);
    n.ws = nullptr; n.ws_bytes = 0;
    return layout(n);
}

extern "C" int esr_net_create(esr_net_t *out, int B, int N, int L, int H, int W, void *params, void *workspace, size_t ws_bytes,
                              esr_stream_t stream)
{
    ESR_REQUIRE(out && params && workspace, "esr_net_create: null pointer");
    ESR_REQUIRE(B > 0 && H > 0 && W > 0 && L >= N, "esr_net_create: bad dims");
    ESR_REQUIRE(2 * B <= 65535 && (long long)B * L * ((H + 7) / 8) * ((W + 7) / 8) < (1ll << 28), "esr_net_create: batch too large");
    if (!num_frame_ok(N)) { set_error("esr_net_create: num_frame=%d (the reference needs an odd num_frame >= 3)", N); return ESR_EUNSUPPORTED; }
    const size_t blob_room = bytes_to_allocation_end(params);
    if (blob_room != 0 && blob_room < esr_net_param_bytes_n(N)) {
        set_error("esr_net_create: the parameter blob (%zu bytes to the end of its allocation) is smaller than the %zu bytes of "
                  "num_frame=%d; pack it with esr_net_pack_params_n(%d, ...)", blob_room, esr_net_param_bytes_n(N), N, N);
        return ESR_EINVAL;
    }
    Net *n = new Net();
    net_dims(*n, B, N, L, H, W);
    n->P = param_layout(N);
    n->params = (char *)params; n->ws = (char *)workspace; n->ws_bytes = ws_bytes;
    const size_t need = layout(*n);
    if (need > ws_bytes) { set_error("esr_net_create: workspace %zu < %zu", ws_bytes, need); delete n; return ESR_EWORKSPACE; }
    cudaStream_t st = (cudaStream_t)stream;
    int rc = build(*n, st);
    if (rc) { delete n; return rc; }
    cudaError_t e = cudaMemsetAsync(n->hs.base, 0, n->hs.bytes(), st);
    if (e != cudaSuccess) { set_error("memset failed: %s", cudaGetErrorString(e)); delete n; return ESR_ECUDA; }
    *out = n;
    return ESR_OK;
}

extern "C" int esr_net_destroy(esr_net_t net)
{
    if (net && ((Net *)net)->dcn_plan) dcn_fused_destroy(((Net *)net)->dcn_plan);
    delete (Net *)net;
    return ESR_OK;
}

extern "C" int esr_net_reset_states(esr_net_t net, esr_stream_t stream)
{
    ESR_REQUIRE(net, "esr_net_reset_states: null net");
    Net &n = *(Net *)net;
    // a None state is replaced by zeros in the reference (models/submodules.py:503-505)
    SplitTensor s0 = view_imgs(n.hs, 0);
    const size_t cnt = (size_t)2 * n.B * n.h * n.w * 64 * sizeof(__nv_bfloat16);
    ESR_CUDA_CHECK(cudaMemsetAsync(s0.base, 0, cnt, (cudaStream_t)stream));
    ESR_CUDA_CHECK(cudaMemsetAsync(s0.base + n.hs.plane(), 0, cnt, (cudaStream_t)stream));
    return ESR_OK;
}

extern "C" int esr_net_reset_sample_states(esr_net_t net, int b, esr_stream_t stream)
{
    ESR_REQUIRE(net, "esr_net_reset_sample_states: null net");
    Net &n = *(Net *)net;
    ESR_REQUIRE(b >= 0 && b < n.B, "esr_net_reset_sample_states: sample %d out of [0, %d)", b, n.B);
    // slot 0 holds the forward-direction state of sample b in image b and the reverse-direction one in image B + b
    const size_t img = (size_t)n.h * n.w * 64;
    const size_t cnt = img * sizeof(__nv_bfloat16);
    __nv_bfloat16 *s0 = view_imgs(n.hs, 0).base;
    for (int i : {b, n.B + b}) {
        ESR_CUDA_CHECK(cudaMemsetAsync(s0 + (size_t)i * img, 0, cnt, (cudaStream_t)stream));
        ESR_CUDA_CHECK(cudaMemsetAsync(s0 + n.hs.plane() + (size_t)i * img, 0, cnt, (cudaStream_t)stream));
    }
    return ESR_OK;
}

extern "C" int esr_net_forward(esr_net_t net, const float *input, const int32_t *in_img, float *output, esr_stream_t stream)
{
    ESR_REQUIRE(net && input && output, "esr_net_forward: null pointer");
    return forward(*(Net *)net, input, in_img, output, (cudaStream_t)stream);
}

extern "C" int esr_net_forward_profiled(esr_net_t net, const float *input, const int32_t *in_img, float *output,
                                        int max_entries, int *n_entries_host, int *cls_host, float *ms_host,
                                        double *flops_host, double *bytes_host, char *names_host, esr_stream_t stream)
{
    ESR_REQUIRE(net && input && output && n_entries_host && cls_host && ms_host && flops_host, "esr_net_forward_profiled: null pointer");
    Prof prof;
    cudaStream_t st = (cudaStream_t)stream;
    int rc = forward(*(Net *)net, input, in_img, output, st, &prof);
    cudaError_t e = cudaStreamSynchronize(st);
    int k = 0;
    for (auto &pe : prof.entries) {
        float ms = 0.0f;
        if (e == cudaSuccess) cudaEventElapsedTime(&ms, pe.e0, pe.e1);
        if (k < max_entries) {
            cls_host[k] = pe.cls; ms_host[k] = ms; flops_host[k] = pe.flops;
            if (bytes_host) bytes_host[k] = pe.bytes;
            if (names_host) { snprintf(names_host + 32 * k, 32, "%s", pe.name ? pe.name : ""); }
            ++k;
        }
        cudaEventDestroy(pe.e0); cudaEventDestroy(pe.e1);
    }
    *n_entries_host = k;
    if (rc) return rc;
    if (e != cudaSuccess) { set_error("esr_net_forward_profiled: %s", cudaGetErrorString(e)); return ESR_ECUDA; }
    return ESR_OK;
}

extern "C" int esr_net_get_states(esr_net_t net, float *states, esr_stream_t stream)
{
    ESR_REQUIRE(net && states, "esr_net_get_states: null pointer");
    Net &n = *(Net *)net;
    // [2, B, 64, h, w] fp32: forward-direction then reverse-direction state; slot 0 holds images [0,B) fwd, [B,2B) rev
    SplitTensor s0 = view_imgs(n.hs, 0);
    return split_to_nchw_planes(s0.base, n.hs.plane(), 2 * n.B, 64, n.h, n.w, states, (cudaStream_t)stream);
}

extern "C" int esr_net_set_states(esr_net_t net, const float *states, esr_stream_t stream)
{
    ESR_REQUIRE(net && states, "esr_net_set_states: null pointer");
    Net &n = *(Net *)net;
    SplitTensor s0 = view_imgs(n.hs, 0);
    return split_from_nchw_planes(states, 2 * n.B, 64, n.h, n.w, s0.base, n.hs.plane(), (cudaStream_t)stream);
}

// ---- state rows: one sample's carried state outside any plan -----------------------------------------------------------
// Row layout (private to this file): [direction 2][plane 2][h][w][64] bf16 -- forward then reverse direction, hi then lo
// split plane, each an image of slot 0 as the plan keeps it, so a row moves in and out of a plan as raw bf16 words.
static size_t state_img8(int H, int W) { return (size_t)((H + 7) / 8) * ((W + 7) / 8) * 64 / 8; }

extern "C" size_t esr_net_state_bytes(int H, int W)
{
    return H > 0 && W > 0 ? 4 * state_img8(H, W) * 8 * sizeof(__nv_bfloat16) : 0;
}

namespace esr {
// one thread per 16 bytes: i -> (slot b, part k = direction * 2 + plane, element e); consecutive threads, consecutive e
template <bool GATHER>
__global__ void __launch_bounds__(256)
k_state_rows(__nv_bfloat16 *__restrict__ slot0, size_t plane, int B, size_t img8, uint4 *__restrict__ pool,
             const int32_t *__restrict__ row_of_slot)
{
    const size_t total = (size_t)B * 4 * img8;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int b = (int)(i / (4 * img8));
        const size_t r = i % (4 * img8), k = r / img8, e = r % img8;
        const int row = row_of_slot[b];
        uint4 *s = reinterpret_cast<uint4 *>(slot0 + (k & 1) * plane) + ((k >> 1) * B + b) * img8 + e;
        if (GATHER)
            *s = row < 0 ? make_uint4(0, 0, 0, 0) : pool[(size_t)row * 4 * img8 + r];
        else if (row >= 0)
            pool[(size_t)row * 4 * img8 + r] = *s;
    }
}
} // namespace esr

static int state_rows(esr_net_t net, void *pool, const int32_t *row_of_slot, bool gather, esr_stream_t stream)
{
    ESR_REQUIRE(net && pool && row_of_slot, "esr_net_%s_states: null pointer", gather ? "gather" : "scatter");
    Net &n = *(Net *)net;
    ESR_REQUIRE(((uintptr_t)pool & 15) == 0, "esr_net_%s_states: the pool must be 16-byte aligned", gather ? "gather" : "scatter");
    const size_t img8 = state_img8(n.H, n.W), total = (size_t)n.B * 4 * img8;
    const unsigned grid = (unsigned)std::min<int64_t>(ceil_div64((int64_t)total, 256), (int64_t)dev_info().sm_count * 16);
    __nv_bfloat16 *s0 = view_imgs(n.hs, 0).base;
    if (gather)
        k_state_rows<true><<<grid, 256, 0, (cudaStream_t)stream>>>(s0, n.hs.plane(), n.B, img8, (uint4 *)pool, row_of_slot);
    else
        k_state_rows<false><<<grid, 256, 0, (cudaStream_t)stream>>>(s0, n.hs.plane(), n.B, img8, (uint4 *)pool, row_of_slot);
    ESR_LAUNCH_CHECK();
    return ESR_OK;
}

extern "C" int esr_net_gather_states(esr_net_t net, const void *pool, const int32_t *row_of_slot, esr_stream_t stream)
{
    return state_rows(net, const_cast<void *>(pool), row_of_slot, true, stream);
}

extern "C" int esr_net_scatter_states(esr_net_t net, void *pool, const int32_t *row_of_slot, esr_stream_t stream)
{
    return state_rows(net, pool, row_of_slot, false, stream);
}
