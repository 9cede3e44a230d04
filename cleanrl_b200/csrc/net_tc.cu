// NatureCNN on the Hopper tensor cores (wgmma, accumulators in registers), bf16 operands,
// fp32 accumulation.  Reference network: cleanrl/ppo_atari_envpool.py:123-139.
//
// Data layout in HBM (all activations are LINEAR PIXEL GRIDS: row = grid position, 128 bytes = 64 channels)
//   frames   bf16 [n, 21x21, 64]   space-to-depth(4) of the uint8 frames: channel = c*16 + sy*4 + sx of source
//                                  pixel (4Y+sy, 4X+sx); written once per env step (tc_frames_to_s2d), 0..255 is
//                                  exact in bf16 and the /255 of ppo_atari_envpool.py:144 is applied to the fp32
//                                  accumulator.  conv1 (8x8 s4) = 2x2 stride-1 conv on this grid.
//   act1     bf16 [n, 10x10, 128]  conv1 output as 2x2 cells (space-to-depth(2)): conv2 (4x4 s2) = 2x2 stride-1.
//   act2     bf16 [n,  9x9,  64]   act3 bf16 [n, 7x7, 64]   hidden bf16 [n, 512]
//   gradients of act3 / act2 are written twice by their producer: on the consumer-weight-gradient's grid
//   (zeros at positions that are not valid outputs) and zero-padded for the data-gradient's "full" correlation;
//   d(act1) lives on the 21x21 grid with 32 channels.  Never-written positions rely on a zero-initialised
//   workspace.  The minibatch gather b_obs[mb_inds] (ppo.py:250, 3.7 GB fp32 per minibatch in the reference)
//   is an image-index indirection inside the conv1 kernels.
//
// Kernels
//   tc_conv_win<BN,CPR,STAGES,NTAPS>   stride-1 "window" convolution (conv1 forward, conv2 data gradient; with the channels
//       on the MMA's M side, tc_conv_win_t, the conv3 data gradient):
//       GEMM rows enumerate grid positions, so tap (dy,dx) of row r is row r + dy*Wp + dx.  A persistent CTA
//       stages ONE window of 128+maxshift rows per tile as a TMA box (cp.async.bulk.tensor; for conv1 a 3-D box
//       whose image coordinate is the minibatch gather) and every tap is a wgmma descriptor whose start address is
//       shifted by whole 128-byte rows (legal for SWIZZLE_128B: the pattern is a function of the smem address
//       bits).  Weights stay resident in smem.  Warp 0 = TMA producer, two warpgroups run wgmma on 64 rows each and
//       the epilogue; ReLU masks are exchanged between forward and backward as bits.
//   tc_conv23_fwd                conv2 -> conv3 forward in one persistent kernel, one image per tile: conv2's epilogue
//       writes act2 into a shared-memory operand image that conv3's MMAs read (and to HBM for the backward).
//   tc_wgrad_rows / tc_wgrad_win conv weight gradients: dW^T[(tap,c), co] = sum_r X[r+shift_tap, c] * dY[r, co]; the same
//       row images are read as MN-major operands (rows = reduction index), taps again by row shifts; the bias
//       gradient (column sums of dY) is accumulated by the four dY warps from the staged tiles.  tc_wgrad_rows (conv2,
//       conv3) puts dY^T on the M side and a whole kernel row of taps on N; tc_wgrad_win (conv1 on bf16 frames) takes
//       image-aligned steps through the minibatch gather.
//   tc_gemm_tma<BN,STAGES>       fc forward / data-gradient: both operands are TMA boxes of row-major matrices.
//   tc_wgrad_tma                 fc weight gradient (MN-major views of TMA-loaded dhid / act3 row boxes).
//   tc_heads_*                   the A+1 head outputs in fp32 on CUDA cores (A+1 <= kMaxHeads).
//   wide heads (kMaxHeads < A+1 <= kMaxWideHeads, e.g. C51 logits): forward = tc_gemm_tma with an fp32 + bias epilogue
//       over hidden; backward = a bf16 copy of dhead feeding tc_wgrad_tma (dWh, folded over row splits in order) and
//       tc_gemm_tma (dhid, ReLU-masked, into the slot the fc kernels read); dbh = fp32 column sums of dhead.
#include <cuda.h>            // CUtensorMap types only; the encoder is resolved at run time (no libcuda link)
#include <algorithm>
#include "tc_base.cuh"
#include "tc_conv_win.cuh"
#include "tc_conv23.cuh"
#include "tc_conv1_u8.cuh"
#include "tc_gemm_tma.cuh"
#include "tc_wgrad_win.cuh"
#include "tc_reduce.cuh"
#include "tc_aux.cuh"
#include "tc_heads.cuh"
#include "tc_heads_wide.cuh"
#include "tc_lstm.cuh"

// =====================================================================================
// Host side: NatureCNN plan over the kernels above (C-ABI entry points, include/b200rl.h)
// =====================================================================================
namespace b200rl {

struct NatureLayout {
    int A;
    // flat fp32 parameter offsets (libb200rl order: trunk, then both head weights, then both head biases)
    int64_t c1w, c1b, c2w, c2b, c3w, c3b, fcw, fcb, hw, hb, total;
    // packed bf16 operand offsets (elements)
    int64_t w1f, w2f, w2dg, w3f, w3dg, wfcf, wfcdg, w1l, w1sc, packed_total;
    // wide heads only: G = A+1 padded to kWideHeadPad; whf bf16 [G,512], whdg bf16 [512,G], hbp f32 [G]
    bool wide; int G; int64_t whf, whdg, hbp;
    // recurrent agent only (-1 otherwise): LSTM tensors (params) and the packed bf16 W_hh [512][128]
    int64_t wih, whh, bih, bhh, whhp;
    explicit NatureLayout(int A_) : A(A_), wih(-1), whh(-1), bih(-1), bhh(-1), whhp(-1) {
        int64_t o = 0;
        c1w = o; o += 32 * 4 * 8 * 8;  c1b = o; o += 32;
        c2w = o; o += 64 * 32 * 4 * 4; c2b = o; o += 64;
        c3w = o; o += 64 * 64 * 3 * 3; c3b = o; o += 64;
        fcw = o; o += 512 * 3136;      fcb = o; o += 512;
        hw = o;  o += (int64_t)(A + 1) * 512;
        hb = o;  o += A + 1;
        total = o;
        int64_t q = 0;
        w1f = q; q += 32 * 256;
        w2f = q; q += 64 * 512;
        w2dg = q; q += 4 * 32 * 256;
        w3f = q; q += 64 * 576;
        w3dg = q; q += 64 * 576;
        wfcf = q; q += 512 * 3136;
        wfcdg = q; q += 3136 * 512;
        w1l = q; q += 64 * 256 / 2;          // conv1 weight limbs: s8 [64][256] (16 KB)
        w1sc = q; q += 64 * 2;               // conv1 column scales: f32 [64]
        wide = A + 1 > kMaxHeads;
        G = wide ? (int)ceil_div(A + 1, kWideHeadPad) * kWideHeadPad : 0;
        whf = whdg = hbp = 0;
        if (wide) {
            whf = q; q += (int64_t)G * 512;
            whdg = q; q += (int64_t)G * 512;
            hbp = q; q += (int64_t)G * 2;
        }
        packed_total = q;
    }
    // LSTMAgent._param_order: the trunk with conv1.w [32,1,8,8], then weight_ih [512,512], weight_hh [512,128], bias_ih,
    // bias_hh, then the heads over the 128 hidden units.  The input projection W_ih is packed as a wide head (G = 512
    // outputs over the 512 features: whf, whdg, hbp = b_ih); conv1 is packed for the single-frame kernel (w1f [32][64]).
    struct Lstm {};
    NatureLayout(int A_, Lstm) : A(A_) {
        int64_t o = 0;
        c1w = o; o += 32 * 8 * 8;      c1b = o; o += 32;
        c2w = o; o += 64 * 32 * 4 * 4; c2b = o; o += 64;
        c3w = o; o += 64 * 64 * 3 * 3; c3b = o; o += 64;
        fcw = o; o += 512 * 3136;      fcb = o; o += 512;
        wih = o; o += 512 * 512;       whh = o; o += 512 * 128;
        bih = o; o += 512;             bhh = o; o += 512;
        hw = o;  o += (int64_t)(A + 1) * 128;
        hb = o;  o += A + 1;
        total = o;
        int64_t q = 0;
        w1f = q; q += 32 * 64;
        w2f = q; q += 64 * 512;
        w2dg = q; q += 4 * 32 * 256;
        w3f = q; q += 64 * 576;
        w3dg = q; q += 64 * 576;
        wfcf = q; q += 512 * 3136;
        wfcdg = q; q += 3136 * 512;
        w1l = w1sc = -1;
        wide = true; G = 512;
        whf = q; q += 512 * 512;
        whdg = q; q += 512 * 512;
        hbp = q; q += 512 * 2;
        whhp = q; q += 512 * 128;
        packed_total = q;
    }
};

struct NatureActs {   // bf16 element offsets inside the (zero-initialised) activation workspace for batch n
    int64_t x0, act1, act2, act3, hid, dhid, dact3a, dact3b, dact2a, dact2b, dact1, m1, m2, m3, m4, total;
    explicit NatureActs(int64_t n, bool with_x0 = true) {
        int64_t o = 0;
        x0 = o; if (with_x0) o += n * 28224;     // space-to-depth frames [n,441,64] (only for uint8 input)
        act1 = o; o += n * 12800;                // conv1 out as 2x2 cells   [n,100,128]
        act2 = o; o += n * 5184;                 // conv2 out               [n, 81, 64]
        act3 = o; o += n * 3136;                 // conv3 out               [n, 49, 64]
        hid = o;  o += n * 512;
        dhid = o; o += n * 512;
        dact3a = o; o += n * 5184;               // d(act3) on the 9x9 linear grid (zeros outside 7x7)
        dact3b = o; o += n * 7744;               // d(act3) zero-padded to 11x11 (interior at +2,+2)
        dact2a = o; o += n * 6400;               // d(act2) on the 10x10 linear grid (zeros at row/col 9)
        dact2b = o; o += n * 7744;               // d(act2) zero-padded to 11x11 (interior at +1,+1)
        dact1 = o; o += n * 14112;               // d(act1) on the 21x21 linear grid, 32 channels
        // ReLU masks as bits (uint32 words; offsets stay in bf16 elements = 2 words per 4 elements)
        auto pad8 = [](int64_t v) { return (v + 7) & ~int64_t(7); };
        m1 = o; o += pad8(n * 100 * 4 * 2);      // act1 > 0: [n,100 cells] x 4 words (128 channels)
        m2 = o; o += pad8(n * 81 * 2 * 2);       // act2 > 0: [n,81] x 2 words
        m3 = o; o += pad8(n * 49 * 2 * 2);       // act3 > 0: [n,49] x 2 words (= dense [n,3136] / 32)
        m4 = o; o += pad8(n * 16 * 2);           // hid  > 0: [n] x 16 words
        total = o;
    }
};

static void gemm_rowmajor(KGemmParams& p, const bf16* x, int64_t n, int nchunks) {   // x [n, 64*nchunks]
    memset(&p, 0, sizeof(p));
    p.scale = 1.f;
    p.A = x; p.M = n; p.nchunks = nchunks;
}


// ---- window-convolution descriptions of the three conv layers
static void win_defaults(WinParams& p) { memset(&p, 0, sizeof(p)); p.scale = 1.f; }
static int round8(int v) { return (v + 7) & ~7; }
static void win_conv1(WinParams& p, const bf16* x0, const int64_t* rows, int64_t n) {     // 2x2 taps on the 21x21 s2d grid
    p.A = x0; p.rows = rows; p.n = (int)n; p.G = 441; p.Wp = 21; p.M = n * 441;
    p.tpi_shift = 2;                             // 4 tiles of 128 grid rows per image (441 used)
    p.n_images = rows ? (int64_t)1 << 24 : n;    // gather indices are the caller's contract (never range-checked)
    p.ntaps = 4; p.shift[0] = 0; p.shift[1] = 1; p.shift[2] = 21; p.shift[3] = 22; p.WR = round8(128 + 22);
}
static void wgw_defaults(WGradWinParams& w) { memset(&w, 0, sizeof(w)); }

// row splits of the window weight gradients: one or two waves of CTAs on the 132 SMs of an H100
static const int kC1Ctas = 264, kC2Ctas = 132, kC3Ctas = 132;
static WPlan conv1_wgrad_plan(int64_t n, bool u8) {          // the uint8 kernel takes whole images (512 rows) per CTA
    return u8 ? wgrad_plan(n * 512, kC2Ctas, 512) : wgrad_plan(n * 512, kC1Ctas, 128);
}
static WPlan conv2_wgrad_plan(int64_t n) { return wgrad_plan(n * 100, kC2Ctas, 128); }
static WPlan conv3_wgrad_plan(int64_t n) { return wgrad_plan(n * 81, kC3Ctas, 128); }

// scratch of the window weight gradients (launch_wgrad_win, launch_wgrad_rows and the uint8 conv1 weight gradient):
// dW partials ws[splits][nslots*64][64] in the big region, bias partials wsb[splits][64] in the small one
static size_t wgrad_win_bytes(int splits, int nslots) { return (size_t)splits * nslots * 64 * 64 * sizeof(float); }
static size_t wgrad_win_bias_bytes(int splits) { return (size_t)splits * 64 * sizeof(float); }
static int check_splits(int64_t M, int64_t rows_per_cta, int ctas, const char* what) {
    if (rows_per_cta % 128 != 0) return fail(B200RL_ERR_INVALID_ARGUMENT, "%s: rows per CTA must be a multiple of 128", what);
    if (ctas < 1 || (int64_t)(ctas - 1) * rows_per_cta >= M)
        return fail(B200RL_ERR_INVALID_ARGUMENT, "%s: every row split must own at least one row", what);
    return B200RL_OK;
}
// conv1 on bf16 frames: image-aligned steps (3-D TMA for X, cp.async for the 64-byte dY rows), one CTA per row split
static int launch_wgrad_win(const WGradWinParams& p, int ctas, cudaStream_t s, const char* what) {
    const size_t smem = (size_t)kWgradWinStages * ((size_t)p.WRX * 128 * p.cpr + 128 * 128) + 4096 + 1024;
    static SmemAttrCache attr;
    int rc;
    if ((rc = attr.ensure(tc_wgrad_win, smem, what))) return rc;
    if ((rc = check_splits(p.M, p.rows_per_cta, ctas, what))) return rc;
    if (p.nslots != 4) return fail(B200RL_ERR_INVALID_ARGUMENT, "%s: the wgmma warpgroups take 2 output tiles of 2 slots", what);
    if ((128 << p.tpi_shift) < p.G) return fail(B200RL_ERR_INVALID_ARGUMENT, "%s: steps per image too small", what);
    CUtensorMap tmX;
    memset(&tmX, 0, sizeof(tmX));
    if ((rc = make_tmap_3d(&tmX, p.X, p.n_images, p.G, (int64_t)p.cpr * 64, p.WRX, what))) return rc;
    tc_wgrad_win<<<ctas, kWgradWinThreads, smem, s>>>(tmX, p);
    return check_launch(what);
}
// conv2 / conv3 on the linear grid: X [M, 64 CPR] and dY [M, 64] (bf16), one CTA per split of plan `pl`
template <int CPR, int KROWS, int TPR, int WP, int NCW>
static int launch_wgrad_rows(const bf16* X, const bf16* Y, int64_t M, const WPlan& pl, float* ws, float* wsb, cudaStream_t s,
                             const char* what) {
    using C = WgradRowsCfg<CPR, KROWS, TPR, WP, NCW>;
    static SmemAttrCache attr;
    int rc;
    if ((rc = attr.ensure(tc_wgrad_rows<CPR, KROWS, TPR, WP, NCW>, C::kSmem, what))) return rc;
    if ((rc = check_splits(M, pl.rows_per_cta, pl.splits, what))) return rc;
    CUtensorMap tmX, tmY;
    memset(&tmX, 0, sizeof(tmX)); memset(&tmY, 0, sizeof(tmY));
    if ((rc = make_tmap_2d(&tmX, X, M, (int64_t)CPR * 64, C::kWRX, what))) return rc;
    if ((rc = make_tmap_2d(&tmY, Y, M, 64, 128, what))) return rc;
    WGradRowsParams p;
    p.M = M; p.rows_per_cta = pl.rows_per_cta; p.ws = ws; p.wsb = wsb;
    tc_wgrad_rows<CPR, KROWS, TPR, WP, NCW><<<pl.splits, C::kThreads, C::kSmem, s>>>(tmX, tmY, p);
    return check_launch(what);
}

}  // namespace b200rl

using namespace b200rl;

namespace b200rl {
// head widths the bf16 NatureCNN accepts: narrow (CUDA-core heads) or wide (wgmma heads)
static bool head_ok(int A) { return A >= 1 && A < kMaxWideHeads; }
// wide-head backward scratch over A1 outputs: dWh partials wgrad_tma_bytes(n, G, 512) (big part) and dhead bf16 +
// bias-sum partials (small part)
static size_t wide_dhead_bytes(int64_t n, const NatureLayout& L) { return ((size_t)n * L.G * 2 + 255) & ~(size_t)255; }
static size_t wide_small_bytes(int64_t n, const NatureLayout& L, int A1) {
    return wide_dhead_bytes(n, L) + colsum_f32_ws(n, A1);
}

// ---- the parts of the NatureCNN plan that the recurrent agent shares (same kernels, same launches)
// conv2 -> conv3 -> fc: act1 (2x2 cells) -> hid [n,512] (ReLU bits in m4)
static int trunk_fwd(const NatureLayout& L, const NatureActs& Q, const float* params, const bf16* P, bf16* act, int64_t n,
                     cudaStream_t s) {
    int rc;
    KGemmParams p;
    // conv2 (2x2 window conv on the 128-channel cells) -> act2 [n,9,9,64] -> conv3 (3x3) -> act3 [n,7,7,64], one kernel:
    // act2 reaches HBM for the backward but is not read back
    Conv23Params cp;
    cp.n = (int)n; cp.b2 = params + L.c2b; cp.b3 = params + L.c3b; cp.act2 = act + Q.act2; cp.act3 = act + Q.act3;
    cp.m2 = reinterpret_cast<uint32_t*>(act + Q.m2); cp.m3 = reinterpret_cast<uint32_t*>(act + Q.m3);
    { ProfScope ps(s, "conv23_fwd", 2.0 * n * 81 * 64 * 512 + 2.0 * n * 49 * 64 * 576,
                   (double)n * (12800 * 2 + 5184 * 2 + 648 + 3136 * 2 + 392));
      if ((rc = launch_conv23_fwd(act + Q.act1, P + L.w2f, P + L.w3f, cp, s, "naturecnn/conv23"))) return rc; }
    // fc -> hidden [n,512]
    gemm_rowmajor(p, act + Q.act3, n, 49);
    p.Bw = P + L.wfcf; p.N = 512; p.out = act + Q.hid; p.ldo = 512; p.bias = params + L.fcb; p.relu = 1;
    p.mask_out = reinterpret_cast<uint32_t*>(act + Q.m4);
    { ProfScope ps(s, "fc_fwd", 2.0 * n * 512 * 3136, (double)n * (3136 + 512) * 2 + 512.0 * 3136 * 2);
      // small batches (rollout step): narrower N tiles => 4x more CTAs for the same work
      if (n <= 8192) { if ((rc = launch_gemm_tma<64, 6>(p, s, "naturecnn/fc"))) return rc; }
      else if ((rc = launch_gemm_tma<128, 3>(p, s, "naturecnn/fc"))) return rc; }
    return B200RL_OK;
}

// fc -> conv2 backward: dhid (ReLU-masked) -> fc, conv3, conv2 weight gradients and, unless `dact1_fused` (the uint8
// rollout: tc_conv21_bwd_u8 computes it inside the conv1 weight gradient), d(act1) on the 21x21 grid in bf16.
// `tail_ready_event` is recorded when grads[fcw ..) is final.
static int trunk_bwd(const NatureLayout& L, const NatureActs& Q, const bf16* P, bf16* act, float* grads, int64_t n,
                     float* wsbig, float* wssmall, void* tail_ready_event, bool dact1_fused, cudaStream_t s) {
    int rc;
    KGemmParams p;
    // ---- fc: dW[o][c*49+p] = sum_m dhid[m][o] * act3[m][p*64+c]
    {
        int splits;
        // X = dhid (512 columns), Y = act3 (3136 columns, the last Y group partly past the end: zero-filled by TMA)
        { ProfScope ps(s, "fc_wgrad", 2.0 * n * 512 * 3136, (double)n * (3136 + 512) * 2 + 512.0 * 3136 * 4);
          if ((splits = launch_wgrad_tma(act + Q.dhid, 512, act + Q.act3, 3136, n, wsbig, s, "naturecnn/fc_wgrad")) < 0) return splits; }
        { ProfScope ps(s, "wgrad_fold_bias", 0, 0);
          note_launches(1); tc_fold_fc<<<(unsigned)ceil_div((int64_t)512 * 3136, 256), 256, 0, s>>>(wsbig, splits, 512, 13 * 256, 512, 3136, 64, 49, 1.f, grads + L.fcw);
          if ((rc = colsum(act + Q.dhid, n, 512, 512, wssmall, grads + L.fcb, s))) return rc; }
        // grads[fcw .. total) (fc weight + bias, both heads) are final: the caller may start exchanging them now
        if (tail_ready_event) {
            cudaError_t e = cudaEventRecord(reinterpret_cast<cudaEvent_t>(tail_ready_event), s);
            if (e != cudaSuccess) return fail(B200RL_ERR_CUDA, "naturecnn_backward: cudaEventRecord: %s", cudaGetErrorString(e));
        }
        // dact3_pre = (dhid . Wfc) * (act3 > 0), written on the 9x9 linear grid and the zero-padded 11x11 grid
        gemm_rowmajor(p, act + Q.dhid, n, 8);
        p.Bw = P + L.wfcdg; p.N = 3136; p.out = act + Q.dact3a; p.out2 = act + Q.dact3b; p.dual_dact3 = 1;
        p.ldo = 3136; p.mask_bits = reinterpret_cast<const uint32_t*>(act + Q.m3);
        { ProfScope ps(s, "fc_dgrad", 2.0 * n * 512 * 3136, (double)n * ((3136 + 512) * 2 + 392) + 512.0 * 3136 * 2);
          if ((rc = launch_gemm_tma<128, 3>(p, s, "naturecnn/fc_dgrad"))) return rc; }
    }
    WinParams wp;
    FoldWin fw;
    // ---- conv3: dW from act2 windows x dact3 (9x9 grid), then dact2 = full correlation of padded dact3 with W3
    {
        // 3 kernel rows of 3 taps (shifts 9 ky + kx) on one 64-channel chunk; one wgmma warpgroup per kernel row
        const WPlan pl = conv3_wgrad_plan(n);
        { ProfScope ps(s, "conv3_wgrad", 2.0 * n * 49 * 64 * 576, (double)n * (5184 + 5184) * 2);
          if ((rc = launch_wgrad_rows<1, 3, 3, 9, 3>(act + Q.act2, act + Q.dact3a, n * 81, pl, wsbig, wssmall, s,
                                                      "naturecnn/conv3_wgrad"))) return rc; }
        memset(&fw, 0, sizeof(fw));
        fw.layer = 3; fw.S = pl.splits; fw.nslots = 9; fw.Cout = 64; fw.scale = 1.f; fw.bscale = 1.f;
        for (int k = 0; k < 9; ++k) fw.slot_tap[k] = k;
        { ProfScope ps(s, "wgrad_fold_bias", 0, 0);
          fw.wsb = wssmall; fw.db = grads + L.c3b;
          tc_fold_win<<<(unsigned)ceil_div(576 * 64 + 64, 32), 256, 0, s>>>(wsbig, fw, grads + L.c3w);
          if ((rc = check_launch("naturecnn/conv3_fold"))) return rc; }
        win_defaults(wp);
        wp.A = act + Q.dact3b; wp.n = (int)n; wp.G = 121; wp.Wp = 11; wp.M = n * 121; wp.ntaps = 9;
        for (int ky = 0; ky < 3; ++ky) for (int kx = 0; kx < 3; ++kx) wp.shift[ky * 3 + kx] = (2 - ky) * 11 + (2 - kx);
        wp.WR = round8(128 + 24);
        wp.Bw = P + L.w3dg; wp.N = 64; wp.vH = 9; wp.vW = 9; wp.out_mode = WOUT_DACT2;
        wp.out = act + Q.dact2a; wp.out2 = act + Q.dact2b; wp.mask_bits = reinterpret_cast<const uint32_t*>(act + Q.m2);
        { ProfScope ps(s, "conv3_dgrad", 2.0 * n * 81 * 64 * 576, (double)n * ((7744 + 6400 + 7744) * 2 + 648));
          if ((rc = launch_conv_win_t<128, 1, 4, 9>(wp, s, "naturecnn/conv3_dgrad"))) return rc; }
    }
    // ---- conv2: dW from act1 cell windows x dact2 (10x10 grid); dact1 = one N=128 GEMM over the 4 stride-parity
    //      classes (the 4 channel groups of a cell)
    {
        // 2 kernel rows of 2 taps (shifts 10 a + b) on each of the 2 channel chunks of a cell; one wgmma warpgroup per
        // kernel row, both chunks
        const WPlan pl = conv2_wgrad_plan(n);
        { ProfScope ps(s, "conv2_wgrad", 2.0 * n * 81 * 64 * 512, (double)n * (12800 + 6400) * 2);
          if ((rc = launch_wgrad_rows<2, 2, 2, 10, 2>(act + Q.act1, act + Q.dact2a, n * 100, pl, wsbig, wssmall, s,
                                                       "naturecnn/conv2_wgrad"))) return rc; }
        memset(&fw, 0, sizeof(fw));
        fw.layer = 2; fw.S = pl.splits; fw.nslots = 8; fw.Cout = 64; fw.scale = 1.f; fw.bscale = 1.f;
        for (int k = 0; k < 8; ++k) { fw.slot_tap[k] = k >> 1; fw.slot_cc[k] = k & 1; }
        { ProfScope ps(s, "wgrad_fold_bias", 0, 0);
          fw.wsb = wssmall; fw.db = grads + L.c2b;
          tc_fold_win<<<(unsigned)ceil_div(512 * 64 + 64, 32), 256, 0, s>>>(wsbig, fw, grads + L.c2w);
          if ((rc = check_launch("naturecnn/conv2_fold"))) return rc; }
        if (dact1_fused) return B200RL_OK;
        win_defaults(wp);
        wp.A = act + Q.dact2b; wp.n = (int)n; wp.G = 121; wp.Wp = 11; wp.M = n * 121; wp.ntaps = 4;
        for (int a = 0; a < 2; ++a) for (int b = 0; b < 2; ++b) wp.shift[a * 2 + b] = (1 - a) * 11 + (1 - b);
        wp.WR = round8(128 + 12);
        wp.Bw = P + L.w2dg; wp.N = 128; wp.vH = 10; wp.vW = 10; wp.out_mode = WOUT_DACT1;
        wp.out = act + Q.dact1; wp.mask_bits = reinterpret_cast<const uint32_t*>(act + Q.m1);
        { ProfScope ps(s, "conv2_dgrad", 2.0 * n * 400 * 32 * 256, (double)n * ((7744 + 14112) * 2 + 1600));
          if ((rc = launch_conv_win<128, 1, 4, 4>(wp, s, "naturecnn/conv2_dgrad"))) return rc; }
    }
    return B200RL_OK;
}
// scratch of trunk_bwd: the fc, conv3 and conv2 weight-gradient partials (big part); the fc bias column sums and the
// conv bias partials (small part)
static size_t trunk_big_bytes(int64_t n) {
    // conv3 writes 9 slots; 10 stay reserved so that the workspace size reported to callers (and allocated by them, at
    // small n this term is the largest) is the one earlier releases reported
    return std::max({wgrad_tma_bytes(n, 512, 3136), wgrad_win_bytes(conv3_wgrad_plan(n).splits, 10),
                     wgrad_win_bytes(conv2_wgrad_plan(n).splits, 8)});
}
static size_t trunk_small_bytes(int64_t n) {
    return std::max({colsum_ws(n, 512), wgrad_win_bias_bytes(conv3_wgrad_plan(n).splits),
                     wgrad_win_bias_bytes(conv2_wgrad_plan(n).splits)});
}

// wide head forward: out [n, A1] (fp32, row stride A1) = hid . Wh^T + bh over the zero-padded [G, 512] operands
static int wide_head_fwd(const NatureLayout& L, const bf16* P, const bf16* hid, int64_t n, int A1, float* out, cudaStream_t s) {
    KGemmParams p;
    gemm_rowmajor(p, hid, n, 8);
    p.Bw = P + L.whf; p.N = L.G; p.bias = reinterpret_cast<const float*>(P + L.hbp);
    p.out_f32 = out; p.ldo = A1; p.ncols_f32 = A1;
    return launch_gemm_tma<128, 3>(p, s, "wide_heads");
}

// wide head backward: dhead [n, A1] fp32 -> bf16 [n, G] (left at the start of wssmall); dW = dhead_bf16^T . hid on wgmma
// (row splits folded in order), db = fp32 column sums of dhead; dhid = (dhead_bf16 . Wh) * (hid > 0) on wgmma
static int wide_head_bwd(const NatureLayout& L, const bf16* P, const float* dhead, int64_t n, int A1, const bf16* hid, bf16* dhid,
                         const uint32_t* hid_bits, float* dW, float* db, float* wsbig, float* wssmall, cudaStream_t s) {
    int rc;
    KGemmParams p;
    bf16* dh16 = reinterpret_cast<bf16*>(wssmall);
    float* dbpart = reinterpret_cast<float*>(reinterpret_cast<char*>(wssmall) + wide_dhead_bytes(n, L));
    int cb = (int)ceil_div(n * L.G, 256); if (cb > num_sms() * 8) cb = num_sms() * 8;
    tc_head_dhead_bf16<<<cb, 256, 0, s>>>(dhead, n, A1, L.G, dh16);
    if ((rc = check_launch("wide_heads_dhead"))) return rc;
    if ((rc = colsum_f32(dhead, n, A1, dbpart, db, s))) return rc;
    const int splits = launch_wgrad_tma(dh16, L.G, hid, 512, n, wsbig, s, "wide_heads_wgrad");
    if (splits < 0) return splits;
    tc_fold_fc<<<(unsigned)ceil_div((int64_t)A1 * 512, 256), 256, 0, s>>>(wsbig, splits, L.G, 512, A1, 512, 512, 1, 1.f, dW);
    if ((rc = check_launch("wide_heads_wgrad"))) return rc;
    gemm_rowmajor(p, dh16, n, L.G / 64);
    p.Bw = P + L.whdg; p.N = 512; p.out = dhid; p.ldo = 512;
    p.mask_bits = hid_bits;
    if (n <= 8192) { if ((rc = launch_gemm_tma<64, 6>(p, s, "wide_heads_dgrad"))) return rc; }
    else if ((rc = launch_gemm_tma<128, 3>(p, s, "wide_heads_dgrad"))) return rc;
    return B200RL_OK;
}
}  // namespace b200rl

extern "C" int64_t b200rl_naturecnn_param_count(int A) { return A >= 1 ? NatureLayout(A).total : -1; }
extern "C" int64_t b200rl_naturecnn_grad_tail_offset(int A) { return A >= 1 ? NatureLayout(A).fcw : -1; }
extern "C" size_t b200rl_naturecnn_bf16_packed_bytes(int A) { return head_ok(A) ? (size_t)NatureLayout(A).packed_total * 2 : 0; }
extern "C" size_t b200rl_naturecnn_bf16_acts_bytes(int64_t n, int obs_format) {
    return n >= 0 ? (size_t)NatureActs(n, obs_format == B200RL_OBS_U8_NCHW).total * 2 + 256 : 0;
}

extern "C" int b200rl_frames_to_s2d_bf16(const uint8_t* obs, const int64_t* rows, int64_t n, void* out, void* stream) {
    B200RL_REQUIRE(n >= 0, "frames_to_s2d: negative n");
    if (n == 0) return B200RL_OK;
    B200RL_REQUIRE(obs && out, "frames_to_s2d: null pointer");
    B200RL_REQUIRE(aligned(obs, 4) && aligned(out, 16), "frames_to_s2d: misaligned buffer");
    cudaStream_t s = (cudaStream_t)stream;
    ProfScope ps(s, "frames_to_s2d", 0, (double)n * 28224 * 3);
    tc_frames_to_s2d<<<(unsigned)ceil_div(n * 1764, 256), 256, 0, s>>>(obs, rows, n, reinterpret_cast<bf16*>(out));
    return check_launch("frames_to_s2d");
}

extern "C" int b200rl_frames_to_s2d_u8(const uint8_t* obs, const int64_t* rows, int64_t n, uint8_t* out_rm, uint8_t* out_cm, void* stream) {
    B200RL_REQUIRE(n >= 0, "frames_to_s2d_u8: negative n");
    if (n == 0) return B200RL_OK;
    B200RL_REQUIRE(obs && out_rm && out_cm, "frames_to_s2d_u8: null pointer");
    B200RL_REQUIRE(aligned(obs, 16) && aligned(out_rm, 16) && aligned(out_cm, 16), "frames_to_s2d_u8: misaligned buffer");
    B200RL_REQUIRE(n <= (int64_t)1 << 28, "frames_to_s2d_u8: n too large");
    cudaStream_t s = (cudaStream_t)stream;
    ProfScope ps(s, "frames_to_s2d", 0, (double)n * (28224 + 28224 + 28672));
    tc_frames_to_s2d_u8<<<(unsigned)n, kS2dThreads, 0, s>>>(obs, rows, n, out_rm, out_cm);
    return check_launch("frames_to_s2d_u8");
}

// the backward workspace = [big part: weight-gradient partials | small part, 256-B aligned], each the largest its launches
// need: heads, trunk, and conv1 on either kind of input (bf16 window kernel or uint8 kernel)
static size_t naturecnn_big_bytes(int64_t n, const NatureLayout& L) {
    return std::max({trunk_big_bytes(n), L.wide ? wgrad_tma_bytes(n, L.G, 512) : 0,
                     wgrad_win_bytes(conv1_wgrad_plan(n, false).splits, 4), wgrad_win_bytes(conv1_wgrad_plan(n, true).splits, 4)});
}

extern "C" size_t b200rl_naturecnn_bf16_workspace_bytes(int64_t n, int A) {
    if (n < 1 || !head_ok(A)) return 0;
    const NatureLayout L(A);
    const size_t small = std::max({trunk_small_bytes(n), L.wide ? wide_small_bytes(n, L, A + 1) : heads_partial_bytes(n, A + 1, 512),
                                   wgrad_win_bias_bytes(conv1_wgrad_plan(n, false).splits),
                                   wgrad_win_bias_bytes(conv1_wgrad_plan(n, true).splits)});
    return naturecnn_big_bytes(n, L) + small + 512;
}

extern "C" int b200rl_naturecnn_bf16_pack(const float* params, int A, void* packed, void* stream) {
    B200RL_REQUIRE(params && packed && head_ok(A), "naturecnn_pack: bad arguments (A must be in [1,%d])", kMaxWideHeads - 1);
    B200RL_REQUIRE(aligned(packed, 16), "naturecnn_pack: packed buffer must be 16-B aligned");
    const NatureLayout L(A);
    bf16* P = reinterpret_cast<bf16*>(packed);
    cudaStream_t s = (cudaStream_t)stream;
    ProfScope ps(s, "pack_weights", 0, (double)L.total * 4 + (double)L.packed_total * 2);
    tc_pack_conv1_s2d<<<32, 256, 0, s>>>(params + L.c1w, P + L.w1f);
    tc_pack_conv1_i8<<<32, 256, 0, s>>>(params + L.c1w, reinterpret_cast<int8_t*>(P + L.w1l), reinterpret_cast<float*>(P + L.w1sc));
    tc_pack_conv2_cells<<<128, 256, 0, s>>>(params + L.c2w, P + L.w2f);
    tc_pack_conv_s2_classes<<<(unsigned)ceil_div(32768, 256), 256, 0, s>>>(params + L.c2w, 64, 32, P + L.w2dg);
    tc_pack_conv<<<(unsigned)ceil_div(36864, 256), 256, 0, s>>>(params + L.c3w, 64, 64, 3, 3, 0, P + L.w3f, P + L.w3dg);
    tc_pack_fc<<<dim3(512 / 8, 49 / 7), 256, 0, s>>>(params + L.fcw, 512, 49, P + L.wfcf, P + L.wfcdg);
    if (L.wide) {
        tc_pack_head_wide<<<(unsigned)ceil_div((int64_t)L.G * 512, 256), 256, 0, s>>>(params + L.hw, params + L.hb, A + 1, L.G,
                                                                                    P + L.whf, P + L.whdg, reinterpret_cast<float*>(P + L.hbp));
        return check_launch("naturecnn_pack", 7);
    }
    return check_launch("naturecnn_pack", 6);
}

extern "C" int b200rl_naturecnn_bf16_forward(const void* obs, int obs_format, const int64_t* rows, int64_t n, int A,
                                             const float* params, const void* packed, void* acts,
                                             float* head_out, void* stream) {
    B200RL_REQUIRE(n >= 0, "naturecnn_forward: negative n");
    if (n == 0) return B200RL_OK;
    B200RL_REQUIRE(obs && params && packed && acts && head_out, "naturecnn_forward: null pointer");
    B200RL_REQUIRE(head_ok(A), "naturecnn_forward: A=%d outside [1,%d]", A, kMaxWideHeads - 1);
    B200RL_REQUIRE(obs_format == B200RL_OBS_U8_NCHW || obs_format == B200RL_OBS_S2D_BF16 || obs_format == B200RL_OBS_S2D_U8,
                   "naturecnn_forward: bad obs_format %d", obs_format);
    B200RL_REQUIRE(aligned(obs, 16) && aligned(acts, 16) && aligned(packed, 16), "naturecnn_forward: misaligned buffer");
    B200RL_REQUIRE(n <= (int64_t)1 << 22, "naturecnn_forward: n too large");
    const NatureLayout L(A);
    const NatureActs Q(n, obs_format == B200RL_OBS_U8_NCHW);
    const bf16* P = reinterpret_cast<const bf16*>(packed);
    bf16* act = reinterpret_cast<bf16*>(acts);
    cudaStream_t s = (cudaStream_t)stream;
    int rc;
    WinParams wp;
    // conv1: 2x2 window conv on space-to-depth frames -> act1 as 2x2 cells [n,10,10,128]
    const bf16* x0 = reinterpret_cast<const bf16*>(obs);
    const int64_t* x0rows = rows;
    if (obs_format == B200RL_OBS_U8_NCHW) {
        if ((rc = b200rl_frames_to_s2d_bf16(reinterpret_cast<const uint8_t*>(obs), rows, n, act + Q.x0, stream))) return rc;
        x0 = act + Q.x0; x0rows = nullptr;
    }
    if (obs_format == B200RL_OBS_S2D_U8) {
        // uint8 space-to-depth frames straight into the integer tensor cores (tc_conv1_u8.cuh)
        Conv1U8Params cp;
        memset(&cp, 0, sizeof(cp));
        cp.rows = rows; cp.n = (int)n; cp.n_images = rows ? (int64_t)1 << 24 : n;
        cp.limbs = reinterpret_cast<const int8_t*>(P + L.w1l); cp.sc = reinterpret_cast<const float*>(P + L.w1sc);
        cp.bias = params + L.c1b; cp.out = act + Q.act1; cp.mask_out = reinterpret_cast<uint32_t*>(act + Q.m1);
        ProfScope ps(s, "conv1_fwd", 2.0 * n * 400 * 32 * 256, (double)n * (28224 + 12800 * 2 + 1600));
        if ((rc = launch_conv1_i8(cp, obs, s, "naturecnn/conv1_i8"))) return rc;
    } else {
    win_defaults(wp); win_conv1(wp, x0, x0rows, n);
    wp.Bw = P + L.w1f; wp.N = 32; wp.vH = 20; wp.vW = 20; wp.out_mode = WOUT_S2D2; wp.out = act + Q.act1;
    wp.bias = params + L.c1b; wp.scale = 1.0f / 255.0f; wp.relu = 1; wp.mask_out = reinterpret_cast<uint32_t*>(act + Q.m1);
    { ProfScope ps(s, "conv1_fwd", 2.0 * n * 400 * 32 * 256, (double)n * ((28224 + 12800) * 2 + 1600));
      if ((rc = launch_conv_win<32, 1, 9, 4>(wp, s, "naturecnn/conv1"))) return rc; }
    }
    if ((rc = trunk_fwd(L, Q, params, P, act, n, s))) return rc;
    if (L.wide) {
        // wide heads on wgmma: head_out [n, A+1] (fp32) = hidden . Wh^T + bh, over the zero-padded [G, 512] weights
        ProfScope ps(s, "heads_fwd", 2.0 * n * 512 * (A + 1), (double)n * (1024 + 4 * (A + 1)) + (double)L.G * 1024);
        return wide_head_fwd(L, P, act + Q.hid, n, A + 1, head_out, s);
    }
    // heads (fp32 math on CUDA cores): head_out [n, A+1] = [logits | value]
    ProfScope ps(s, "heads_fwd", 2.0 * n * 512 * (A + 1), (double)n * (1024 + 4 * (A + 1)));
    return heads_fwd<512>(act + Q.hid, params + L.hw, params + L.hb, n, A + 1, head_out, s, "naturecnn/heads");
}

extern "C" int b200rl_naturecnn_bf16_backward(const void* obs, const void* obs_aux, int obs_format, const int64_t* rows, int64_t n, int A,
                                              const float* params, const void* packed, void* acts,
                                              const float* dhead, float* grads,
                                              void* workspace, size_t workspace_bytes, void* tail_ready_event, void* stream) {
    B200RL_REQUIRE(n >= 1, "naturecnn_backward: n must be >= 1");
    B200RL_REQUIRE(obs && params && packed && acts && dhead && grads && workspace, "naturecnn_backward: null pointer");
    B200RL_REQUIRE(head_ok(A), "naturecnn_backward: A=%d outside [1,%d]", A, kMaxWideHeads - 1);
    B200RL_REQUIRE(aligned(workspace, 16), "naturecnn_backward: workspace misaligned");
    const size_t need = b200rl_naturecnn_bf16_workspace_bytes(n, A);
    if (workspace_bytes < need) return fail(B200RL_ERR_WORKSPACE, "naturecnn_backward: workspace %zu < %zu", workspace_bytes, need);
    B200RL_REQUIRE(obs_format == B200RL_OBS_U8_NCHW || obs_format == B200RL_OBS_S2D_BF16 || obs_format == B200RL_OBS_S2D_U8,
                   "naturecnn_backward: bad obs_format %d", obs_format);
    B200RL_REQUIRE(obs_format != B200RL_OBS_S2D_U8 || (obs_aux && aligned(obs_aux, 16)), "naturecnn_backward: the uint8 rollout needs obs_aux");
    const NatureLayout L(A);
    const NatureActs Q(n, obs_format == B200RL_OBS_U8_NCHW);
    const bf16* P = reinterpret_cast<const bf16*>(packed);
    bf16* act = reinterpret_cast<bf16*>(acts);
    cudaStream_t s = (cudaStream_t)stream;
    // uint8 input: forward left the space-to-depth frames of this minibatch in the workspace
    const bf16* x0 = obs_format == B200RL_OBS_U8_NCHW ? act + Q.x0 : reinterpret_cast<const bf16*>(obs);   // unused for S2D_U8
    const int64_t* x0rows = obs_format == B200RL_OBS_U8_NCHW ? nullptr : rows;
    // workspace split: [wgrad partials | small partials]
    const size_t big = (naturecnn_big_bytes(n, L) + 255) & ~(size_t)255;
    float* wsbig = reinterpret_cast<float*>(workspace);
    float* wssmall = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + big);
    int rc;
    const int A1 = A + 1;
    if (L.wide) {
        // ---- wide heads: dhead -> bf16 [n, G]; dbh = fp32 column sums; dWh = dhead_bf16^T . hid on wgmma (row splits
        //      folded in order); dhid_pre = (dhead_bf16 . Wh) * (hid > 0) on wgmma
        ProfScope ps(s, "heads_bwd", 4.0 * n * 512 * A1, (double)n * (2048 + 64 + 8 * A1));
        if ((rc = wide_head_bwd(L, P, dhead, n, A1, act + Q.hid, act + Q.dhid, reinterpret_cast<const uint32_t*>(act + Q.m4),
                                grads + L.hw, grads + L.hb, wsbig, wssmall, s))) return rc;
    } else
    // ---- heads: dW, db, then dhid_pre = (dhead . Wh) * (hid > 0)
    {
        ProfScope ps(s, "heads_bwd", 4.0 * n * 512 * A1, (double)n * (2048 + 64 + 8 * A1));
        if ((rc = heads_bwd_weight<512>(dhead, act + Q.hid, n, A1, wssmall, grads + L.hw, grads + L.hb, s, "naturecnn/heads_bwd"))) return rc;
        if ((rc = heads_bwd_data<512>(dhead, params + L.hw, reinterpret_cast<const uint8_t*>(act + Q.m4), n, A1, act + Q.dhid, s,
                                      "naturecnn/heads_bwd"))) return rc;
    }
    if ((rc = trunk_bwd(L, Q, P, act, grads, n, wsbig, wssmall, tail_ready_event, obs_format == B200RL_OBS_S2D_U8, s))) return rc;
    // ---- conv1 (no data gradient: the input is the observation)
    const bool u8 = obs_format == B200RL_OBS_S2D_U8;
    const WPlan pl = conv1_wgrad_plan(n, u8);
    if (u8) {
        // conv2 data gradient (fp16 x kDact1Scale) + the row-major uint8 frames expanded to an fp16 wgmma operand in
        // shared memory (tc_conv1_u8.cuh); 1 CTA per SM.  obs_aux (the channel-major copy) is not read.
        Conv21BwdU8Params cw;
        memset(&cw, 0, sizeof(cw));
        cw.rows = rows; cw.n = (int)n; cw.rows_per_cta = pl.rows_per_cta; cw.ws = wsbig; cw.wsb = wssmall;
        cw.w2dg = P + L.w2dg; cw.m1 = reinterpret_cast<const uint32_t*>(act + Q.m1);
        { ProfScope ps(s, "conv21_bwd", 2.0 * 2.0 * n * 400 * 32 * 256, (double)n * (7744 * 2 + 1600 + 28224 + 14112 * 2));
          if ((rc = launch_conv21_bwd_u8(cw, obs, rows ? (int64_t)1 << 24 : n, act + Q.dact2b, act + Q.dact1, pl.splits, s,
                                         "naturecnn/conv21_bwd_u8"))) return rc; }
    } else {
        WGradWinParams gw;
        wgw_defaults(gw);
        gw.X = x0; gw.rows = x0rows; gw.M = n * 512; gw.n = (int)n; gw.G = 441; gw.cpr = 1; gw.nslots = 4; gw.WRX = round8(128 + 22);
        gw.tpi_shift = 2; gw.n_images = x0rows ? (int64_t)1 << 24 : n;       // 4 steps of 128 grid rows per image
        gw.shift[0] = 0; gw.shift[1] = 1; gw.shift[2] = 21; gw.shift[3] = 22;
        for (int k = 0; k < 4; ++k) { gw.slot_tap[k] = k; gw.slot_cc[k] = 0; }
        gw.Y = act + Q.dact1; gw.ldy = 32; gw.ncolsY = 32;
        gw.rows_per_cta = pl.rows_per_cta; gw.ws = wsbig; gw.wsb = wssmall;
        { ProfScope ps(s, "conv1_wgrad", 2.0 * n * 400 * 32 * 256, (double)n * (28224 + 14112) * 2);
          if ((rc = launch_wgrad_win(gw, pl.splits, s, "naturecnn/conv1_wgrad"))) return rc; }
    }
    // both kernels leave ws rows in tap order (uint8: tile b, lane m -> tap 2 b + (m >> 6)); the uint8 one scaled dY by
    // kDact1Scale
    FoldWin fw;
    memset(&fw, 0, sizeof(fw));
    fw.layer = 1; fw.S = pl.splits; fw.nslots = 4; fw.Cout = 32;
    fw.scale = u8 ? 1.0f / 255.0f / kDact1Scale : 1.0f / 255.0f;
    fw.bscale = u8 ? 1.0f / kDact1Scale : 1.f;
    for (int k = 0; k < 4; ++k) fw.slot_tap[k] = k;
    { ProfScope ps(s, "wgrad_fold_bias", 0, 0);
      fw.wsb = wssmall; fw.db = grads + L.c1b;
      tc_fold_win<<<(unsigned)ceil_div(256 * 32 + 32, 32), 256, 0, s>>>(wsbig, fw, grads + L.c1w);
      if ((rc = check_launch("naturecnn/conv1_fold"))) return rc; }
    return B200RL_OK;
}

// =====================================================================================
// Recurrent agent (LSTMAgent, cleanrl/ppo_atari_lstm.py:117-160): single-frame conv1 (tc_lstm.cuh), the shared trunk,
// W_ih as a 512-output wide head, the persistent recurrence kernels, CUDA-core heads over the 128 hidden units
// =====================================================================================
namespace b200rl {
constexpr int64_t kLstmMaxRows = (int64_t)1 << 17;     // S * n

struct LstmActs {           // the trunk (NatureActs, bf16 element offsets, at byte 0), then byte offsets of the LSTM tensors
    NatureActs T;
    int64_t gx, hseq, hm, save, cm, dgates, total;
    explicit LstmActs(int64_t M) : T(M, false) {
        int64_t o = (T.total * 2 + 255) & ~int64_t(255);
        auto take = [&](int64_t bytes) { const int64_t r = o; o += (bytes + 255) & ~int64_t(255); return r; };
        gx = take(M * 512 * 4);
        hseq = take(M * 128 * 2);
        hm = take(M * 128 * 2);
        save = take(M * 640 * 4);
        cm = take(M * 128 * 4);
        dgates = take(M * 512 * 4);
        total = o;
    }
};

static bool lstm_heads_ok(int A) { return A >= 1 && A + 1 <= lstm::kMaxA1; }
static bool lstm_sizes_ok(int64_t S, int64_t n) { return S >= 1 && n >= 1 && S <= kLstmMaxRows && n <= kLstmMaxRows && S * n <= kLstmMaxRows; }

struct C1Plan { int64_t per_cta; int ctas; };
static C1Plan lstm_conv1_plan(int64_t M) {           // whole frames per CTA, one or two waves
    C1Plan c;
    const int64_t want = M < kC1Ctas ? M : kC1Ctas;
    c.per_cta = ceil_div(M, want);
    c.ctas = (int)ceil_div(M, c.per_cta);
    return c;
}
// backward workspace = [big part (256-B aligned) | small part], each the largest its launches need: heads, W_ih as a wide
// head, W_hh, trunk, conv1
static size_t lstm_big_bytes(int64_t M, const NatureLayout& L) {
    const size_t a = std::max({wgrad_tma_bytes(M, L.G, 512), wgrad_tma_bytes(M, 512, 128), trunk_big_bytes(M),
                               (size_t)lstm_conv1_plan(M).ctas * 32 * 64 * 4});
    return (a + 255) & ~(size_t)255;
}
static size_t lstm_small_bytes(int64_t M, const NatureLayout& L) {
    return std::max({heads_partial_bytes(M, L.A + 1, 128), wide_small_bytes(M, L, 512), trunk_small_bytes(M),
                     (size_t)lstm_conv1_plan(M).ctas * 32 * 4});
}
}  // namespace b200rl

extern "C" int64_t b200rl_lstm_agent_param_count(int A) { return A >= 1 ? NatureLayout(A, NatureLayout::Lstm{}).total : -1; }
extern "C" size_t b200rl_lstm_agent_bf16_packed_bytes(int A) {
    return lstm_heads_ok(A) ? (size_t)NatureLayout(A, NatureLayout::Lstm{}).packed_total * 2 : 0;
}
extern "C" size_t b200rl_lstm_agent_bf16_acts_bytes(int64_t S, int64_t n) {
    return lstm_sizes_ok(S, n) ? (size_t)LstmActs(S * n).total : 0;
}
extern "C" int b200rl_lstm_agent_bf16_acts_layout(int64_t S, int64_t n, int64_t* offsets) {
    B200RL_REQUIRE(offsets, "lstm_acts_layout: null pointer");
    B200RL_REQUIRE(lstm_sizes_ok(S, n), "lstm_acts_layout: S=%lld n=%lld out of range", (long long)S, (long long)n);
    const LstmActs Q(S * n);
    const int64_t v[B200RL_LSTM_ACTS_TENSORS] = {Q.T.act1 * 2, Q.T.m1 * 2, Q.T.act2 * 2, Q.T.act3 * 2, Q.T.hid * 2, Q.T.m4 * 2,
                                                 Q.gx, Q.hseq, Q.hm, Q.save, Q.cm, Q.dgates, Q.T.dhid * 2};
    for (int k = 0; k < B200RL_LSTM_ACTS_TENSORS; ++k) offsets[k] = v[k];
    return B200RL_OK;
}
extern "C" size_t b200rl_lstm_agent_bf16_workspace_bytes(int64_t S, int64_t n, int A) {
    if (!lstm_sizes_ok(S, n) || !lstm_heads_ok(A)) return 0;
    const NatureLayout L(A, NatureLayout::Lstm{});
    return lstm_big_bytes(S * n, L) + lstm_small_bytes(S * n, L) + 512;
}

extern "C" int b200rl_lstm_agent_bf16_pack(const float* params, int A, void* packed, void* stream) {
    B200RL_REQUIRE(params && packed, "lstm_pack: null pointer");
    B200RL_REQUIRE(lstm_heads_ok(A), "lstm_pack: A=%d outside [1,%d]", A, lstm::kMaxA1 - 1);
    B200RL_REQUIRE(aligned(params, 16) && aligned(packed, 16), "lstm_pack: misaligned buffer");
    const NatureLayout L(A, NatureLayout::Lstm{});
    bf16* P = reinterpret_cast<bf16*>(packed);
    cudaStream_t s = (cudaStream_t)stream;
    ProfScope ps(s, "pack_weights", 0, (double)L.total * 4 + (double)L.packed_total * 2);
    lstm::lstm_pack_conv1<<<8, 256, 0, s>>>(params + L.c1w, P + L.w1f);
    tc_pack_conv2_cells<<<128, 256, 0, s>>>(params + L.c2w, P + L.w2f);
    tc_pack_conv_s2_classes<<<(unsigned)ceil_div(32768, 256), 256, 0, s>>>(params + L.c2w, 64, 32, P + L.w2dg);
    tc_pack_conv<<<(unsigned)ceil_div(36864, 256), 256, 0, s>>>(params + L.c3w, 64, 64, 3, 3, 0, P + L.w3f, P + L.w3dg);
    tc_pack_fc<<<dim3(512 / 8, 49 / 7), 256, 0, s>>>(params + L.fcw, 512, 49, P + L.wfcf, P + L.wfcdg);
    tc_pack_head_wide<<<(unsigned)ceil_div((int64_t)L.G * 512, 256), 256, 0, s>>>(params + L.wih, params + L.bih, 512, L.G,
                                                                                P + L.whf, P + L.whdg, reinterpret_cast<float*>(P + L.hbp));
    tc_head_dhead_bf16<<<256, 256, 0, s>>>(params + L.whh, 512, 128, 128, P + L.whhp);     // W_hh -> bf16 [512][128]
    return check_launch("lstm_pack", 7);
}

extern "C" int b200rl_lstm_agent_bf16_forward(const uint8_t* obs, const int64_t* rows, int64_t S, int64_t n, int A,
                                              const float* params, const void* packed, const float* h0, const float* c0,
                                              const float* done, void* acts, float* head_out, float* h_out, float* c_out,
                                              void* stream) {
    B200RL_REQUIRE(obs && params && packed && h0 && c0 && done && acts && head_out && h_out && c_out, "lstm_forward: null pointer");
    B200RL_REQUIRE(lstm_heads_ok(A), "lstm_forward: A=%d outside [1,%d]", A, lstm::kMaxA1 - 1);
    B200RL_REQUIRE(lstm_sizes_ok(S, n), "lstm_forward: S=%lld n=%lld (S*n at most %lld)", (long long)S, (long long)n,
                   (long long)kLstmMaxRows);
    B200RL_REQUIRE(aligned(obs, 16) && aligned(rows, 8) && aligned(params, 16) && aligned(packed, 16) && aligned(acts, 256) &&
                   aligned(h0, 16) && aligned(c0, 16) && aligned(done, 4) && aligned(head_out, 4) && aligned(h_out, 16) &&
                   aligned(c_out, 16), "lstm_forward: misaligned buffer");
    const int64_t M = S * n;
    const NatureLayout L(A, NatureLayout::Lstm{});
    const LstmActs Q(M);
    const bf16* P = reinterpret_cast<const bf16*>(packed);
    uint8_t* ab = reinterpret_cast<uint8_t*>(acts);
    bf16* act = reinterpret_cast<bf16*>(acts);
    cudaStream_t s = (cudaStream_t)stream;
    int rc;
    {   // conv1 on the uint8 frames -> act1 (2x2 cells) + ReLU bits
        lstm::Conv1P cp;
        cp.obs = obs; cp.rows = rows; cp.n = M; cp.w = P + L.w1f; cp.bias = params + L.c1b; cp.out = act + Q.T.act1;
        cp.mask_out = reinterpret_cast<uint32_t*>(act + Q.T.m1);
        ProfScope ps(s, "conv1_fwd", 2.0 * M * 400 * 32 * 64, (double)M * (7056 + 12800 * 2 + 1600));
        const int64_t grid = M < (int64_t)num_sms() * 8 ? M : (int64_t)num_sms() * 8;
        lstm::lstm_conv1_fwd<<<(unsigned)grid, lstm::kThreads, lstm::conv1_fwd_smem(), s>>>(cp);
        if ((rc = check_launch("lstm/conv1"))) return rc;
    }
    if ((rc = trunk_fwd(L, Q.T, params, P, act, M, s))) return rc;
    float* gx = reinterpret_cast<float*>(ab + Q.gx);
    { ProfScope ps(s, "lstm_ih_fwd", 2.0 * M * 512 * 512, (double)M * (1024 + 2048) + 512.0 * 1024);
      if ((rc = wide_head_fwd(L, P, act + Q.T.hid, M, 512, gx, s))) return rc; }
    {
        lstm::RecFwdP rp;
        rp.S = (int)S; rp.n = n; rp.whh = P + L.whhp; rp.bhh = params + L.bhh; rp.gx = gx; rp.done = done; rp.h0 = h0; rp.c0 = c0;
        rp.hseq = reinterpret_cast<bf16*>(ab + Q.hseq); rp.hm = reinterpret_cast<bf16*>(ab + Q.hm);
        rp.save = reinterpret_cast<float*>(ab + Q.save); rp.cm = reinterpret_cast<float*>(ab + Q.cm);
        rp.h_out = h_out; rp.c_out = c_out;
        static SmemAttrCache attr;
        if ((rc = attr.ensure(lstm::lstm_rec_fwd, lstm::rec_fwd_smem(), "lstm/recurrence"))) return rc;
        ProfScope ps(s, "lstm_rec_fwd", 2.0 * M * 512 * 128, (double)M * (2048 + 4 + 512 + 3840) + 131072.0);
        lstm::lstm_rec_fwd<<<(unsigned)ceil_div(n, lstm::kRows), lstm::kThreads, lstm::rec_fwd_smem(), s>>>(rp);
        if ((rc = check_launch("lstm/recurrence"))) return rc;
    }
    ProfScope ps(s, "heads_fwd", 2.0 * M * 128 * (A + 1), (double)M * (256 + 4 * (A + 1)));
    return heads_fwd<128>(reinterpret_cast<const bf16*>(ab + Q.hseq), params + L.hw, params + L.hb, M, A + 1, head_out, s, "lstm/heads");
}

extern "C" int b200rl_lstm_agent_bf16_backward(const uint8_t* obs, const int64_t* rows, int64_t S, int64_t n, int A,
                                               const float* params, const void* packed, const float* done, void* acts,
                                               const float* dhead, float* grads, void* workspace, size_t workspace_bytes,
                                               void* stream) {
    B200RL_REQUIRE(obs && params && packed && done && acts && dhead && grads && workspace, "lstm_backward: null pointer");
    B200RL_REQUIRE(lstm_heads_ok(A), "lstm_backward: A=%d outside [1,%d]", A, lstm::kMaxA1 - 1);
    B200RL_REQUIRE(lstm_sizes_ok(S, n), "lstm_backward: S=%lld n=%lld (S*n at most %lld)", (long long)S, (long long)n,
                   (long long)kLstmMaxRows);
    B200RL_REQUIRE(aligned(obs, 16) && aligned(rows, 8) && aligned(params, 16) && aligned(packed, 16) && aligned(acts, 256) &&
                   aligned(done, 4) && aligned(dhead, 4) && aligned(grads, 16) && aligned(workspace, 256),
                   "lstm_backward: misaligned buffer");
    const size_t need = b200rl_lstm_agent_bf16_workspace_bytes(S, n, A);
    if (workspace_bytes < need) return fail(B200RL_ERR_WORKSPACE, "lstm_backward: workspace %zu < %zu", workspace_bytes, need);
    const int64_t M = S * n;
    const int A1 = A + 1;
    const NatureLayout L(A, NatureLayout::Lstm{});
    const LstmActs Q(M);
    const bf16* P = reinterpret_cast<const bf16*>(packed);
    uint8_t* ab = reinterpret_cast<uint8_t*>(acts);
    bf16* act = reinterpret_cast<bf16*>(acts);
    cudaStream_t s = (cudaStream_t)stream;
    float* wsbig = reinterpret_cast<float*>(workspace);
    float* wssmall = reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + lstm_big_bytes(M, L));
    const bf16* hseq = reinterpret_cast<const bf16*>(ab + Q.hseq);
    float* dgates = reinterpret_cast<float*>(ab + Q.dgates);
    int rc;
    {   // heads weight gradient (the data gradient is folded into the recurrence backward)
        ProfScope ps(s, "heads_bwd", 2.0 * M * 128 * A1, (double)M * (256 + 4 * A1));
        if ((rc = heads_bwd_weight<128>(dhead, hseq, M, A1, wssmall, grads + L.hw, grads + L.hb, s, "lstm/heads_bwd"))) return rc;
    }
    {
        lstm::RecBwdP bp;
        bp.S = (int)S; bp.n = n; bp.A1 = A1; bp.whh = P + L.whhp; bp.wh = params + L.hw; bp.dhead = dhead; bp.done = done;
        bp.save = reinterpret_cast<const float*>(ab + Q.save); bp.cm = reinterpret_cast<const float*>(ab + Q.cm);
        bp.dgates = dgates;
        static SmemAttrCache attr;
        if ((rc = attr.ensure(lstm::lstm_rec_bwd, lstm::rec_bwd_smem(), "lstm/recurrence_bwd"))) return rc;
        ProfScope ps(s, "lstm_rec_bwd", 2.0 * M * 512 * 128 + 2.0 * M * 128 * A1, (double)M * (4 * A1 + 3072 + 2048));
        lstm::lstm_rec_bwd<<<(unsigned)ceil_div(n, lstm::kRows), lstm::kThreads, lstm::rec_bwd_smem(), s>>>(bp);
        if ((rc = check_launch("lstm/recurrence_bwd"))) return rc;
    }
    {   // W_ih, b_ih and d(feats) through the wide-head backward; it leaves dgates in bf16 at the start of wssmall
        ProfScope ps(s, "lstm_ih_bwd", 4.0 * M * 512 * 512, (double)M * (2048 + 1024 * 3 + 64));
        if ((rc = wide_head_bwd(L, P, dgates, M, 512, act + Q.T.hid, act + Q.T.dhid, reinterpret_cast<const uint32_t*>(act + Q.T.m4),
                                grads + L.wih, grads + L.bih, wsbig, wssmall, s))) return rc;
    }
    {   // dW_hh = dgates^T . h' over all S*n rows (row splits folded in order); db_hh = db_ih
        ProfScope ps(s, "lstm_hh_wgrad", 2.0 * M * 512 * 128, (double)M * (1024 + 256) + 512.0 * 128 * 4);
        // X = dgates (512 columns), Y = h' (128 columns: the rest of the 256-column Y group is zero-filled by TMA)
        const int splits = launch_wgrad_tma(wssmall, 512, ab + Q.hm, 128, M, wsbig, s, "lstm/hh_wgrad");
        if (splits < 0) return splits;
        tc_fold_fc<<<(unsigned)ceil_div((int64_t)512 * 128, 256), 256, 0, s>>>(wsbig, splits, 512, 64 * kFcWgradYChunks, 512, 128,
                                                                            128, 1, 1.f, grads + L.whh);
        if ((rc = check_launch("lstm/hh_wgrad"))) return rc;
        const cudaError_t e = cudaMemcpyAsync(grads + L.bhh, grads + L.bih, 512 * sizeof(float), cudaMemcpyDeviceToDevice, s);
        if (e != cudaSuccess) return fail(B200RL_ERR_CUDA, "lstm_backward: bias copy: %s", cudaGetErrorString(e));
    }
    if ((rc = trunk_bwd(L, Q.T, P, act, grads, M, wsbig, wssmall, nullptr, false, s))) return rc;
    {   // conv1 weight gradient from the frames and d(act1) on the 21x21 grid
        const C1Plan pl = lstm_conv1_plan(M);
        lstm::Conv1WgradP wp;
        wp.obs = obs; wp.rows = rows; wp.n = M; wp.dy = act + Q.T.dact1; wp.imgs_per_cta = pl.per_cta; wp.ws = wsbig; wp.wsb = wssmall;
        static SmemAttrCache attr;
        if ((rc = attr.ensure(lstm::lstm_conv1_wgrad, lstm::conv1_wgrad_smem(), "lstm/conv1_wgrad"))) return rc;
        ProfScope ps(s, "conv1_wgrad", 2.0 * M * 400 * 32 * 64, (double)M * (7056 + 14112 * 2));
        lstm::lstm_conv1_wgrad<<<pl.ctas, lstm::kThreads, lstm::conv1_wgrad_smem(), s>>>(wp);
        lstm::lstm_conv1_fold<<<(unsigned)ceil_div(32 * 64 + 32, 256), 256, 0, s>>>(wsbig, wssmall, pl.ctas, grads + L.c1w, grads + L.c1b);
        if ((rc = check_launch("lstm/conv1_wgrad", 2))) return rc;
    }
    return B200RL_OK;
}
