// Exact-arithmetic (fp32 FMA on CUDA cores) network layers in the reference's
// own NCHW / [out,in] layouts: conv2d and linear, forward / data-grad /
// weight-grad, all as ONE register-tiled implicit-GEMM kernel
//     C[i,j] = sum_r A(i,r) * B(j,r)
// parameterised by a "problem" functor that maps (i,r)/(j,r) to global
// addresses (im2col gather, minibatch row gather, uint8 -> f32 decode) and
// stores C with the fused epilogue (bias, activation, activation derivative).
//
// This is the fp32 validation path of the NatureCNN (reference:
// cleanrl/ppo_atari_envpool.py:123-139) and the production path of the 64-wide
// MLPs of ppo.py / ppo_continuous_action.py, which are launch-latency bound.
// The bf16 wgmma path (net_tc.cu) is the throughput path for the CNN.
//
// Tile: 64x64 outputs per CTA, K-step 16, 256 threads, 4x4 outputs/thread.
// Weight-grad problems split the (huge) reduction over grid.z into a partial
// buffer that a second kernel folds in fixed order => deterministic.
#include "common.cuh"

namespace b200rl {

constexpr int BM = 64, BN = 64, BK = 16, PAD = 4;

__device__ __forceinline__ float act_fwd(float v, int act) {
    if (act == B200RL_ACT_RELU) return fmaxf(v, 0.f);
    if (act == B200RL_ACT_TANH) return tanhf(v);
    return v;
}
__device__ __forceinline__ float act_bwd(float y, int act) {   // derivative from the POST-activation value
    if (act == B200RL_ACT_RELU) return y > 0.f ? 1.f : 0.f;
    if (act == B200RL_ACT_TANH) return 1.f - y * y;
    return 1.f;
}

struct Geo {            // conv geometry (linear layers use H=W=KH=KW=1)
    int64_t n;
    int Cin, H, W, Cout, KH, KW, s, OH, OW;
    int pad;             // zero padding on every side (IMPALA-CNN 3x3 convolutions, cleanrl/ppo_procgen.py:92-93)
};

template <typename XT>
__device__ __forceinline__ float decode(const XT* p, int64_t off, float div) {
    const float v = (float)p[off];
    return div != 1.f ? v / div : v;    // x / 255.0 exactly as the reference (ppo_atari_envpool.py:144)
}

// ---------------------------------------------------------------- problems
template <typename XT>
struct ConvFwd {
    static constexpr bool A_I_FAST = true, B_J_FAST = false;
    Geo g; const XT* x; const int64_t* rows; float div; const float* w; const float* b; float* y; int act;
    __device__ int64_t M() const { return g.n * g.OH * g.OW; }
    __device__ int64_t N() const { return g.Cout; }
    __device__ int64_t R() const { return (int64_t)g.Cin * g.KH * g.KW; }
    __device__ float A(int64_t i, int64_t r) const {
        const int ohw = g.OH * g.OW;
        const int64_t n_ = i / ohw; const int rem = (int)(i - n_ * ohw);
        const int oy = rem / g.OW, ox = rem - oy * g.OW;
        const int khw = g.KH * g.KW;
        const int c = (int)(r / khw); const int rr = (int)(r - (int64_t)c * khw);
        const int ky = rr / g.KW, kx = rr - ky * g.KW;
        const int64_t sn = rows ? rows[n_] : n_;
        const int iy = oy * g.s + ky - g.pad, ix = ox * g.s + kx - g.pad;
        if (iy < 0 || ix < 0 || iy >= g.H || ix >= g.W) return 0.f;
        return decode(x, ((sn * g.Cin + c) * g.H + iy) * g.W + ix, div);
    }
    __device__ float B(int64_t j, int64_t r) const { return w[j * R() + r]; }
    __device__ void store(int64_t i, int64_t j, float acc, int) const {
        const int ohw = g.OH * g.OW;
        const int64_t n_ = i / ohw; const int rem = (int)(i - n_ * ohw);
        y[(n_ * g.Cout + j) * ohw + rem] = act_fwd(acc + (b ? b[j] : 0.f), act);
    }
};

struct ConvBwdData {
    static constexpr bool A_I_FAST = true, B_J_FAST = false;
    Geo g; const float* dy; const float* w; const float* xpost; int prev_act; float* dx;
    __device__ int64_t M() const { return g.n * g.H * g.W; }
    __device__ int64_t N() const { return g.Cin; }
    __device__ int64_t R() const { return (int64_t)g.Cout * g.KH * g.KW; }
    __device__ float A(int64_t i, int64_t r) const {
        const int hw = g.H * g.W;
        const int64_t n_ = i / hw; const int rem = (int)(i - n_ * hw);
        const int iy = rem / g.W, ix = rem - iy * g.W;
        const int khw = g.KH * g.KW;
        const int co = (int)(r / khw); const int rr = (int)(r - (int64_t)co * khw);
        const int ky = rr / g.KW, kx = rr - ky * g.KW;
        const int ty = iy + g.pad - ky, tx = ix + g.pad - kx;
        if (ty < 0 || tx < 0) return 0.f;
        const int oy = ty / g.s, ox = tx / g.s;
        if (oy * g.s != ty || ox * g.s != tx || oy >= g.OH || ox >= g.OW) return 0.f;
        return dy[((n_ * g.Cout + co) * g.OH + oy) * g.OW + ox];
    }
    __device__ float B(int64_t j, int64_t r) const {
        const int khw = g.KH * g.KW;
        const int co = (int)(r / khw); const int rr = (int)(r - (int64_t)co * khw);
        return w[((int64_t)co * g.Cin + j) * khw + rr];
    }
    __device__ void store(int64_t i, int64_t j, float acc, int) const {
        const int hw = g.H * g.W;
        const int64_t n_ = i / hw; const int rem = (int)(i - n_ * hw);
        const int64_t o = (n_ * g.Cin + j) * hw + rem;
        dx[o] = acc * act_bwd(xpost[o], prev_act);
    }
};

// dw[co, (c,ky,kx)] and db[co] (extra virtual column j == Cin*KH*KW with B == 1)
template <typename XT>
struct ConvBwdWeight {
    static constexpr bool A_I_FAST = false, B_J_FAST = false;
    Geo g; const XT* x; const int64_t* rows; float div; const float* dy; float* partial;  // [S][Cout*(K+1)]
    __device__ int64_t M() const { return g.Cout; }
    __device__ int64_t N() const { return (int64_t)g.Cin * g.KH * g.KW + 1; }
    __device__ int64_t R() const { return g.n * g.OH * g.OW; }
    __device__ float A(int64_t i, int64_t r) const {
        const int ohw = g.OH * g.OW;
        const int64_t n_ = r / ohw; const int rem = (int)(r - n_ * ohw);
        return dy[(n_ * g.Cout + i) * ohw + rem];
    }
    __device__ float B(int64_t j, int64_t r) const {
        if (j == N() - 1) return 1.f;
        const int ohw = g.OH * g.OW;
        const int64_t n_ = r / ohw; const int rem = (int)(r - n_ * ohw);
        const int oy = rem / g.OW, ox = rem - oy * g.OW;
        const int khw = g.KH * g.KW;
        const int c = (int)(j / khw); const int rr = (int)(j - (int64_t)c * khw);
        const int ky = rr / g.KW, kx = rr - ky * g.KW;
        const int64_t sn = rows ? rows[n_] : n_;
        const int iy = oy * g.s + ky - g.pad, ix = ox * g.s + kx - g.pad;
        if (iy < 0 || ix < 0 || iy >= g.H || ix >= g.W) return 0.f;
        return decode(x, ((sn * g.Cin + c) * g.H + iy) * g.W + ix, div);
    }
    __device__ void store(int64_t i, int64_t j, float acc, int z) const {
        partial[((int64_t)z * M() + i) * N() + j] = acc;
    }
};

struct LinFwd {
    static constexpr bool A_I_FAST = false, B_J_FAST = false;
    int64_t n; int in, out; const float* x; const int64_t* rows; const float* w; const float* b; float* y; int act;
    __device__ int64_t M() const { return n; }
    __device__ int64_t N() const { return out; }
    __device__ int64_t R() const { return in; }
    __device__ float A(int64_t i, int64_t r) const { return x[(rows ? rows[i] : i) * in + r]; }
    __device__ float B(int64_t j, int64_t r) const { return w[j * in + r]; }
    __device__ void store(int64_t i, int64_t j, float acc, int) const {
        y[i * out + j] = act_fwd(acc + (b ? b[j] : 0.f), act);
    }
};

struct LinBwdData {
    static constexpr bool A_I_FAST = false, B_J_FAST = true;
    int64_t n; int in, out; const float* dy; const float* w; const float* xpost; int prev_act; float* dx;
    __device__ int64_t M() const { return n; }
    __device__ int64_t N() const { return in; }
    __device__ int64_t R() const { return out; }
    __device__ float A(int64_t i, int64_t r) const { return dy[i * out + r]; }
    __device__ float B(int64_t j, int64_t r) const { return w[r * in + j]; }
    __device__ void store(int64_t i, int64_t j, float acc, int) const {
        const int64_t o = i * in + j;
        dx[o] = acc * (xpost ? act_bwd(xpost[o], prev_act) : 1.f);
    }
};

struct LinBwdWeight {
    static constexpr bool A_I_FAST = true, B_J_FAST = true;
    int64_t n; int in, out; const float* x; const int64_t* rows; const float* dy; float* partial;
    __device__ int64_t M() const { return out; }
    __device__ int64_t N() const { return in + 1; }
    __device__ int64_t R() const { return n; }
    __device__ float A(int64_t i, int64_t r) const { return dy[r * out + i]; }
    __device__ float B(int64_t j, int64_t r) const {
        if (j == in) return 1.f;
        return x[(rows ? rows[r] : r) * in + j];
    }
    __device__ void store(int64_t i, int64_t j, float acc, int z) const {
        partial[((int64_t)z * M() + i) * N() + j] = acc;
    }
};

// ------------------------------------------------------------------ kernel
template <class P>
__global__ void __launch_bounds__(256) sgemm_generic(P p, int64_t r_chunk) {
    __shared__ __align__(16) float As[BK][BM + PAD];
    __shared__ __align__(16) float Bs[BK][BN + PAD];
    const int tid = threadIdx.x;
    const int tx = tid & 15, ty = tid >> 4;
    const int64_t i0 = (int64_t)blockIdx.x * BM, j0 = (int64_t)blockIdx.y * BN;
    const int64_t M = p.M(), N = p.N(), R = p.R();
    const int64_t r_begin = (int64_t)blockIdx.z * r_chunk;
    int64_t r_end = r_begin + r_chunk;
    if (r_end > R) r_end = R;
    float acc[4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[a][b] = 0.f;

    for (int64_t r0 = r_begin; r0 < r_end; r0 += BK) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int idx = tid + 256 * e;
            int ii, rr;
            if (P::A_I_FAST) { ii = idx & (BM - 1); rr = idx >> 6; } else { rr = idx & (BK - 1); ii = idx >> 4; }
            const int64_t gi = i0 + ii, gr = r0 + rr;
            As[rr][ii] = (gi < M && gr < r_end) ? p.A(gi, gr) : 0.f;
            int jj, rb;
            if (P::B_J_FAST) { jj = idx & (BN - 1); rb = idx >> 6; } else { rb = idx & (BK - 1); jj = idx >> 4; }
            const int64_t gj = j0 + jj, grb = r0 + rb;
            Bs[rb][jj] = (gj < N && grb < r_end) ? p.B(gj, grb) : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            const float4 a4 = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
            const float4 b4 = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
            const float a[4] = {a4.x, a4.y, a4.z, a4.w};
            const float b[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
            for (int u = 0; u < 4; ++u)
#pragma unroll
                for (int v = 0; v < 4; ++v) acc[u][v] = fmaf(a[u], b[v], acc[u][v]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
        const int64_t gi = i0 + ty * 4 + u;
        if (gi >= M) continue;
#pragma unroll
        for (int v = 0; v < 4; ++v) {
            const int64_t gj = j0 + tx * 4 + v;
            if (gj < N) p.store(gi, gj, acc[u][v], blockIdx.z);
        }
    }
}

// fold S partial slabs [S][rows][cols+1] into dw [rows][cols] and db [rows] (fixed order)
__global__ void fold_partials_kernel(const float* __restrict__ partial, int S, int64_t rows, int64_t cols1,
                                     float scale_unused, float* __restrict__ dw, float* __restrict__ db) {
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t total = rows * cols1;
    if (idx >= total) return;
    float s = 0.f;
    for (int z = 0; z < S; ++z) s += partial[(int64_t)z * total + idx];
    const int64_t i = idx / cols1, j = idx - i * cols1;
    if (j == cols1 - 1) { if (db) db[i] = s; }
    else dw[i * (cols1 - 1) + j] = s;
}

template <class P>
static int launch(const P& p, int64_t M, int64_t N, int64_t R, int splits, cudaStream_t s, const char* what) {
    if (M == 0 || N == 0) return B200RL_OK;
    dim3 grid((unsigned)ceil_div(M, BM), (unsigned)ceil_div(N, BN), (unsigned)splits);
    if (grid.y > 65535 || grid.z > 65535) return fail(B200RL_ERR_UNSUPPORTED, "%s: grid too large", what);
    int64_t r_chunk = ceil_div(ceil_div(R, splits), BK) * BK;
    if (r_chunk < BK) r_chunk = BK;
    sgemm_generic<P><<<grid, 256, 0, s>>>(p, r_chunk);
    return check_launch(what);
}

static int split_count(int64_t tiles, int64_t R) {
    int64_t want = ceil_div(132 * 4, tiles > 0 ? tiles : 1);
    int64_t maxs = ceil_div(R, 256);     // keep >= 256 reduction steps per split
    if (want > maxs) want = maxs;
    if (want < 1) want = 1;
    if (want > 1024) want = 1024;
    return (int)want;
}

static bool make_geo(Geo& g, int64_t n, int Cin, int H, int W, int Cout, int KH, int KW, int stride, int pad = 0) {
    if (n < 0 || Cin < 1 || H < 1 || W < 1 || Cout < 1 || KH < 1 || KW < 1 || stride < 1 || pad < 0 || pad >= KH || pad >= KW ||
        KH > H + 2 * pad || KW > W + 2 * pad)
        return false;
    g.n = n; g.Cin = Cin; g.H = H; g.W = W; g.Cout = Cout; g.KH = KH; g.KW = KW; g.s = stride; g.pad = pad;
    g.OH = (H + 2 * pad - KH) / stride + 1; g.OW = (W + 2 * pad - KW) / stride + 1;
    return true;
}

}  // namespace b200rl

using namespace b200rl;

extern "C" int b200rl_conv2d_fwd_f32(const void* x, int x_dtype, const int64_t* rows, double in_div,
                                     const float* w, const float* b, float* y,
                                     int64_t n, int Cin, int H, int W, int Cout, int KH, int KW, int stride,
                                     int act, void* stream) {
    return b200rl_conv2d_fwd_pad_f32(x, x_dtype, rows, in_div, w, b, y, n, Cin, H, W, Cout, KH, KW, stride, 0, act, stream);
}
extern "C" int b200rl_conv2d_fwd_pad_f32(const void* x, int x_dtype, const int64_t* rows, double in_div,
                                         const float* w, const float* b, float* y,
                                         int64_t n, int Cin, int H, int W, int Cout, int KH, int KW, int stride, int pad,
                                         int act, void* stream) {
    Geo g;
    B200RL_REQUIRE(make_geo(g, n, Cin, H, W, Cout, KH, KW, stride, pad), "conv2d_fwd: bad geometry");
    if (n == 0) return B200RL_OK;
    B200RL_REQUIRE(x && w && y, "conv2d_fwd: null pointer");
    B200RL_REQUIRE(act >= 0 && act <= 2, "conv2d_fwd: bad act %d", act);
    B200RL_REQUIRE(in_div != 0.0, "conv2d_fwd: in_div == 0");
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t M = n * g.OH * g.OW, R = (int64_t)Cin * KH * KW;
    if (x_dtype == B200RL_DT_U8) {
        ConvFwd<uint8_t> p{g, (const uint8_t*)x, rows, (float)in_div, w, b, y, act};
        return launch(p, M, Cout, R, 1, s, "conv2d_fwd");
    } else if (x_dtype == B200RL_DT_F32) {
        ConvFwd<float> p{g, (const float*)x, rows, (float)in_div, w, b, y, act};
        return launch(p, M, Cout, R, 1, s, "conv2d_fwd");
    }
    return fail(B200RL_ERR_INVALID_ARGUMENT, "conv2d_fwd: unknown x_dtype %d", x_dtype);
}

extern "C" int b200rl_conv2d_bwd_data_f32(const float* dy, const float* w, const float* x_post, int prev_act,
                                          float* dx,
                                          int64_t n, int Cin, int H, int W, int Cout, int KH, int KW, int stride,
                                          void* stream) {
    return b200rl_conv2d_bwd_data_pad_f32(dy, w, x_post, prev_act, dx, n, Cin, H, W, Cout, KH, KW, stride, 0, stream);
}
extern "C" int b200rl_conv2d_bwd_data_pad_f32(const float* dy, const float* w, const float* x_post, int prev_act,
                                              float* dx,
                                              int64_t n, int Cin, int H, int W, int Cout, int KH, int KW, int stride, int pad,
                                              void* stream) {
    Geo g;
    B200RL_REQUIRE(make_geo(g, n, Cin, H, W, Cout, KH, KW, stride, pad), "conv2d_bwd_data: bad geometry");
    if (n == 0) return B200RL_OK;
    B200RL_REQUIRE(dy && w && dx, "conv2d_bwd_data: null pointer");
    B200RL_REQUIRE(prev_act == 0 || x_post, "conv2d_bwd_data: x_post required when prev_act != none");
    ConvBwdData p{g, dy, w, x_post ? x_post : dx, x_post ? prev_act : 0, dx};
    return launch(p, n * H * W, Cin, (int64_t)Cout * KH * KW, 1, (cudaStream_t)stream, "conv2d_bwd_data");
}

extern "C" size_t b200rl_conv2d_bwd_weight_workspace_bytes(int64_t n, int Cin, int H, int W, int Cout, int KH, int KW,
                                                           int stride) {
    return b200rl_conv2d_bwd_weight_pad_workspace_bytes(n, Cin, H, W, Cout, KH, KW, stride, 0);
}
extern "C" size_t b200rl_conv2d_bwd_weight_pad_workspace_bytes(int64_t n, int Cin, int H, int W, int Cout, int KH, int KW,
                                                               int stride, int pad) {
    Geo g;
    if (!make_geo(g, n, Cin, H, W, Cout, KH, KW, stride, pad)) return 0;
    const int64_t cols1 = (int64_t)Cin * KH * KW + 1;
    const int64_t tiles = ceil_div(Cout, BM) * ceil_div(cols1, BN);
    const int S = split_count(tiles, n * g.OH * g.OW);
    return (size_t)S * Cout * cols1 * sizeof(float);
}

extern "C" int b200rl_conv2d_bwd_weight_f32(const void* x, int x_dtype, const int64_t* rows, double in_div,
                                            const float* dy, float* dw, float* db,
                                            int64_t n, int Cin, int H, int W, int Cout, int KH, int KW, int stride,
                                            void* workspace, size_t workspace_bytes, void* stream) {
    return b200rl_conv2d_bwd_weight_pad_f32(x, x_dtype, rows, in_div, dy, dw, db, n, Cin, H, W, Cout, KH, KW, stride, 0, workspace,
                                            workspace_bytes, stream);
}
extern "C" int b200rl_conv2d_bwd_weight_pad_f32(const void* x, int x_dtype, const int64_t* rows, double in_div,
                                                const float* dy, float* dw, float* db,
                                                int64_t n, int Cin, int H, int W, int Cout, int KH, int KW, int stride, int pad,
                                                void* workspace, size_t workspace_bytes, void* stream) {
    Geo g;
    B200RL_REQUIRE(make_geo(g, n, Cin, H, W, Cout, KH, KW, stride, pad), "conv2d_bwd_weight: bad geometry");
    B200RL_REQUIRE(x && dy && dw && workspace, "conv2d_bwd_weight: null pointer");
    B200RL_REQUIRE(in_div != 0.0, "conv2d_bwd_weight: in_div == 0");
    const size_t need = b200rl_conv2d_bwd_weight_pad_workspace_bytes(n, Cin, H, W, Cout, KH, KW, stride, pad);
    if (workspace_bytes < need) return fail(B200RL_ERR_WORKSPACE, "conv2d_bwd_weight: workspace %zu < %zu", workspace_bytes, need);
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t cols1 = (int64_t)Cin * KH * KW + 1;
    const int64_t R = n * g.OH * g.OW;
    const int64_t tiles = ceil_div(Cout, BM) * ceil_div(cols1, BN);
    const int S = split_count(tiles, R);
    int rc;
    if (x_dtype == B200RL_DT_U8) {
        ConvBwdWeight<uint8_t> p{g, (const uint8_t*)x, rows, (float)in_div, dy, (float*)workspace};
        rc = launch(p, Cout, cols1, R, S, s, "conv2d_bwd_weight");
    } else if (x_dtype == B200RL_DT_F32) {
        ConvBwdWeight<float> p{g, (const float*)x, rows, (float)in_div, dy, (float*)workspace};
        rc = launch(p, Cout, cols1, R, S, s, "conv2d_bwd_weight");
    } else {
        return fail(B200RL_ERR_INVALID_ARGUMENT, "conv2d_bwd_weight: unknown x_dtype %d", x_dtype);
    }
    if (rc) return rc;
    const int64_t total = (int64_t)Cout * cols1;
    fold_partials_kernel<<<(unsigned)ceil_div(total, 256), 256, 0, s>>>((const float*)workspace, S, Cout, cols1, 1.f, dw, db);
    return check_launch("conv2d_bwd_weight/fold");
}

extern "C" int b200rl_linear_fwd_f32(const float* x, const int64_t* rows, const float* w, const float* b, float* y,
                                     int64_t n, int in_features, int out_features, int act, void* stream) {
    B200RL_REQUIRE(n >= 0 && in_features >= 1 && out_features >= 1, "linear_fwd: bad shape");
    if (n == 0) return B200RL_OK;
    B200RL_REQUIRE(x && w && y, "linear_fwd: null pointer");
    B200RL_REQUIRE(act >= 0 && act <= 2, "linear_fwd: bad act %d", act);
    LinFwd p{n, in_features, out_features, x, rows, w, b, y, act};
    return launch(p, n, out_features, in_features, 1, (cudaStream_t)stream, "linear_fwd");
}

extern "C" int b200rl_linear_bwd_data_f32(const float* dy, const float* w, const float* x_post, int prev_act, float* dx,
                                          int64_t n, int in_features, int out_features, void* stream) {
    B200RL_REQUIRE(n >= 0 && in_features >= 1 && out_features >= 1, "linear_bwd_data: bad shape");
    if (n == 0) return B200RL_OK;
    B200RL_REQUIRE(dy && w && dx, "linear_bwd_data: null pointer");
    B200RL_REQUIRE(prev_act == 0 || x_post, "linear_bwd_data: x_post required when prev_act != none");
    LinBwdData p{n, in_features, out_features, dy, w, x_post, prev_act, dx};
    return launch(p, n, in_features, out_features, 1, (cudaStream_t)stream, "linear_bwd_data");
}

extern "C" size_t b200rl_linear_bwd_weight_workspace_bytes(int64_t n, int in_features, int out_features) {
    if (n < 0 || in_features < 1 || out_features < 1) return 0;
    const int64_t cols1 = (int64_t)in_features + 1;
    const int64_t tiles = ceil_div(out_features, BM) * ceil_div(cols1, BN);
    const int S = split_count(tiles, n);
    return (size_t)S * out_features * cols1 * sizeof(float);
}

extern "C" int b200rl_linear_bwd_weight_f32(const float* x, const int64_t* rows, const float* dy, float* dw, float* db,
                                            int64_t n, int in_features, int out_features,
                                            void* workspace, size_t workspace_bytes, void* stream) {
    B200RL_REQUIRE(n >= 0 && in_features >= 1 && out_features >= 1, "linear_bwd_weight: bad shape");
    B200RL_REQUIRE(x && dy && dw && workspace, "linear_bwd_weight: null pointer");
    const size_t need = b200rl_linear_bwd_weight_workspace_bytes(n, in_features, out_features);
    if (workspace_bytes < need) return fail(B200RL_ERR_WORKSPACE, "linear_bwd_weight: workspace %zu < %zu", workspace_bytes, need);
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t cols1 = (int64_t)in_features + 1;
    const int64_t tiles = ceil_div(out_features, BM) * ceil_div(cols1, BN);
    const int S = split_count(tiles, n);
    LinBwdWeight p{n, in_features, out_features, x, rows, dy, (float*)workspace};
    int rc = launch(p, out_features, cols1, n, S, s, "linear_bwd_weight");
    if (rc) return rc;
    const int64_t total = (int64_t)out_features * cols1;
    fold_partials_kernel<<<(unsigned)ceil_div(total, 256), 256, 0, s>>>((const float*)workspace, S, out_features, cols1, 1.f, dw, db);
    return check_launch("linear_bwd_weight/fold");
}
