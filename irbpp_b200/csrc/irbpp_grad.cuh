// irbpp_grad.cuh -- the candidate-row network of the location level and its backward pass: log p(s, a_t, .) of
// Agent.learn's gradient pass (agent.py:85-86 on model.py:316-352, 386-404 with args.bufferSize == 1) and the
// gradients of -sum(m . log p) through it (agent.py:117-119), for irbpp_dqn_log_prob / irbpp_dqn_log_prob_backward.
//
// The split with torch: torch computes shape_feature [B, 128] (shapeEncoder, max over the points) and map_feature
// [B, 256] (heightEncoder) with autograd and builds the NoisyLinear effective weights; these kernels take them as plain
// inputs and return their gradients.  Everything whose cost scales with batch x rows runs here:
// init_candidate_embed, project_layer, the zeroing of invalid rows and the row mean, fc_h_v / fc_z_v, fc_h_a / fc_z_a,
// the dueling combine and the log-softmax of row a_t.
//
// Layout.  The valid rows (mask == 1) of the whole batch are compacted into one row space, transition by transition
// in ascending row order: transition b's valid rows are rows B + off_b .. B + off_b + n_b - 1.  Rows 0 .. B - 1 are
// one stand-in per transition for all of its invalid rows: its embedding is zero (model.py:347-349), so its advantage
// is a0 = fc_z_a(relu(fc_h_a.bias)), and in the backward pass it carries the summed upstream gradient of those rows.
// The layers are row-parallel GEMMs over that space (FP32 SIMT, __fmaf_rn in a fixed k order); the per-transition
// parts (value head, means, log-softmax) run one CTA per transition.
//
// Reformulations (each exact in real arithmetic):
//   * project_layer.0 split by concat order (shape 0:128 | map 128:384 | candidate 384:512): u_b = W0[:, 0:384] .
//     [sf_b; mf_b] + b0 once per transition, W0[:, 384:512] . e_r per row.  Backward: S_b = sum_r dpre0_{b,r} (one
//     vector per transition), d[sf_b; mf_b] = W0[:, 0:384]^T S_b, dW0[:, 0:384] = sum_b S_b (x) [sf_b; mf_b],
//     db0 = sum_b S_b; per row only dW0[:, 384:512] += dpre0_r (x) e_r and de_r = W0[:, 384:512]^T dpre0_r.
//   * log p = q - max - log sum exp(q - max) (finite where p underflows).  Backward with g = dL/dlog p:
//     dq = g - softmax(q) sum(g); dv = dq; every row r gets da_r = -dq / sel, row a_t additionally + dq.
//   * invalid rows have x_r = 0, so no gradient reaches project_layer or init_candidate_embed through them; their
//     contribution to fc_z_a and fc_h_a.bias is that of the stand-in row with da = (sel - n_b) (-dq / sel), plus dq
//     when a_t itself is invalid: no per-row work.
//   * xGlobal = sum_valid x_r / sel: dxGlobal / sel (value head) is added to every valid row's dx_r.
// Determinism: no atomics.  A weight gradient is summed over its rows in GR_CHUNKS fixed slices (each slice by one
// thread per output in row order), then over the slices in order; per-transition sums run in row order.
#pragma once
#include <stdint.h>

#include "irbpp_actor.cuh"

namespace irbpp {

constexpr int GR_THREADS = 256;
constexpr int GR_TILE = 64;          // a GEMM tile is 64 x 64 outputs, 4 x 4 per thread
constexpr int GR_KT = 16;            // reduction step of a tile
constexpr int GR_CHUNKS = 32;        // fixed row slices of every weight gradient
constexpr int GR_MAX_WGRAD = 256 * 384;   // largest weight-gradient block: project_layer.0's per-transition columns

// gradients of the effective row-section tensors (include/irbpp.h irbpp_dqn_grads)
struct GradOut {
    float *cand1_w, *cand1_b, *cand2_w, *cand2_b, *proj1_w, *proj1_b, *proj2_w, *proj2_b;
    float *fc_h_v_w, *fc_h_v_b, *fc_z_v_w, *fc_z_v_b, *fc_h_a_w, *fc_h_a_b, *fc_z_a_w, *fc_z_a_b;
};

struct GradParams {
    ActorWeights w;
    const float* obs; int64_t obs_stride;
    int32_t B, sel, atoms;
    const float* shape_feature;          // [B][128]
    const float* map_feature;            // [B][256]
    const int64_t* actions;              // [B], clamped to [0, sel)
    float* log_p;                        // [B][atoms] or NULL
    const float* grad_log_p;             // [B][atoms], backward only
    // scratch (grad_scratch_layout); rows = B + B * sel
    float* xcat;                         // [B][384] [sf; mf]
    float* u;                            // [B][256] u_b
    int32_t* pos;                        // [B][sel] index of a valid row among its transition's valid rows, -1 if invalid
    int32_t* n_valid;                    // [B]
    int32_t* off;                        // [B] valid rows before transition b
    int32_t* count;                      // [1] valid rows of the batch (R)
    int32_t* owner;                      // [rows] transition of a row
    float* cand;                         // [rows][4]   [rot, x, y, H]
    float* h1;                           // [rows][32]  leaky(init_candidate_embed.0); backward: its pre-activation gradient
    float* ec;                           // [rows][128] candidate embedding;            backward: its gradient
    float* p0;                           // [rows][256] leaky(project_layer.0);          backward: its pre-activation gradient
    float* emb;                          // [rows][128] row embedding (0 on stand-ins);  backward: its gradient
    float* ha;                           // [rows][128] relu(fc_h_a);                    backward: its pre-activation gradient
    float* adv;                          // [rows][32]  advantages
    float* dadv;                         // [rows][32]  their gradients
    float* gv;                           // [B][128] xGlobal
    float* hv;                           // [B][128] relu(fc_h_v(xGlobal))
    float* dq;                           // [B][32]
    float* dhv;                          // [B][128] pre-activation gradient of fc_h_v
    float* dg;                           // [B][128] dxGlobal / sel
    float* S;                            // [B][256] sum over the transition's rows of dpre0
    float* part;                         // [GR_CHUNKS][GR_MAX_WGRAD + 256] weight-gradient slices
};

__host__ __device__ inline int64_t grad_scratch_bytes(int64_t B, int64_t sel) {
    const int64_t rows = B + B * sel;
    return actor_align(B * 384 * 4) + actor_align(B * 256 * 4) + actor_align(B * sel * 4) + 2 * actor_align(B * 4) +
           actor_align(4) + actor_align(rows * 4) + actor_align(rows * (4 + 32 + 128 + 256 + 128 + 128 + 32 + 32) * 4) +
           4 * actor_align(B * 128 * 4) + actor_align(B * 32 * 4) + actor_align(B * 256 * 4) +
           actor_align((int64_t)GR_CHUNKS * (GR_MAX_WGRAD + 256) * 4);
}

__host__ __device__ inline void grad_scratch_layout(GradParams& P, void* scratch) {
    char* p = static_cast<char*>(scratch);
    const int64_t B = P.B, sel = P.sel, rows = B + B * sel;
    auto take = [&](int64_t bytes) { char* q = p; p += actor_align(bytes); return q; };
    P.xcat = reinterpret_cast<float*>(take(B * 384 * 4));
    P.u = reinterpret_cast<float*>(take(B * 256 * 4));
    P.pos = reinterpret_cast<int32_t*>(take(B * sel * 4));
    P.n_valid = reinterpret_cast<int32_t*>(take(B * 4));
    P.off = reinterpret_cast<int32_t*>(take(B * 4));
    P.count = reinterpret_cast<int32_t*>(take(4));
    P.owner = reinterpret_cast<int32_t*>(take(rows * 4));
    float* a = reinterpret_cast<float*>(take(rows * (4 + 32 + 128 + 256 + 128 + 128 + 32 + 32) * 4));
    P.cand = a; a += rows * 4;
    P.h1 = a; a += rows * 32;
    P.ec = a; a += rows * 128;
    P.p0 = a; a += rows * 256;
    P.emb = a; a += rows * 128;
    P.ha = a; a += rows * 128;
    P.adv = a; a += rows * 32;
    P.dadv = a;
    P.gv = reinterpret_cast<float*>(take(B * 128 * 4));
    P.hv = reinterpret_cast<float*>(take(B * 128 * 4));
    P.dhv = reinterpret_cast<float*>(take(B * 128 * 4));
    P.dg = reinterpret_cast<float*>(take(B * 128 * 4));
    P.dq = reinterpret_cast<float*>(take(B * 32 * 4));
    P.S = reinterpret_cast<float*>(take(B * 256 * 4));
    P.part = reinterpret_cast<float*>(take((int64_t)GR_CHUNKS * (GR_MAX_WGRAD + 256) * 4));
}

// ---- row-parallel GEMMs ------------------------------------------------------------------------------------------
// C[i][j] = sum_t a(i, t) b(t, j) in one of three forms (W in nn.Linear layout [n][k], rows of the row space):
//   GR_FWD    i = row, j = n, t = k:   out[r][n] = act(sum_k in[r][k] W[n][k] + bias[n] + add[owner[r]][n])
//   GR_DGRAD  i = row, j = k, t = n:   out[r][k] = (sum_n dy[r][n] W[n][k] + add[owner[r]][k]) * act'(out[r][k]);
//             out holds the layer's activation on entry (its sign gives the derivative) and is overwritten
//   GR_WGRAD  i = n, j = k, t = row:   slice c of part: sum over the rows of slice c of dy[r][n] x[r][k], and of dy[r][n]
// Rows are [row0, row0 + rows_host + *rows_dev).
constexpr int GR_FWD = 0, GR_DGRAD = 1, GR_WGRAD = 2;

struct GemmArgs {
    const float* a; int lda;             // FWD: in; DGRAD, WGRAD: dy
    const float* b; int ldb;             // FWD, DGRAD: W; WGRAD: x
    float* c; int ldc;                   // FWD, DGRAD: out; WGRAD: part (slices of M * ldc + M floats)
    const float* bias;                   // FWD
    const float* add; int ld_add;        // FWD, DGRAD: per-transition vector added to every row of the transition
    const int32_t* owner;
    int act; float slope;
    int M, N, T;                         // FWD, DGRAD: M unused (rows), N columns, T reduction; WGRAD: M x N, T unused
    int row0, rows_host; const int32_t* rows_dev;
};

template <int MODE>
__device__ __forceinline__ void grad_gemm(const GemmArgs& g) {
    __shared__ __align__(16) float As[GR_KT][GR_TILE + 4];
    __shared__ __align__(16) float Bs[GR_KT][GR_TILE + 4];
    const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
    const int rows = g.rows_host + (g.rows_dev ? *g.rows_dev : 0);
    const int Mi = MODE == GR_WGRAD ? g.M : rows;                 // extent of i
    const int T = MODE == GR_WGRAD ? rows : g.T;                  // extent of t (WGRAD: all rows; sliced below)
    const int ti = (Mi + GR_TILE - 1) / GR_TILE, tj = (g.N + GR_TILE - 1) / GR_TILE;
    const int tiles = ti * tj * (MODE == GR_WGRAD ? GR_CHUNKS : 1);
    for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const int i0 = (tile % ti) * GR_TILE, j0 = ((tile / ti) % tj) * GR_TILE, chunk = tile / (ti * tj);
        int t_lo = 0, t_hi = T;
        if (MODE == GR_WGRAD) {
            t_lo = (int)((int64_t)T * chunk / GR_CHUNKS);
            t_hi = (int)((int64_t)T * (chunk + 1) / GR_CHUNKS);
        }
        float acc[4][4];
#pragma unroll
        for (int x = 0; x < 4; ++x)
#pragma unroll
            for (int y = 0; y < 4; ++y) acc[x][y] = 0.0f;
        float bacc = 0.0f;                                        // WGRAD, j-tile 0: sum over t of a(i0 + tid, t)
        for (int t0 = t_lo; t0 < t_hi; t0 += GR_KT) {
            __syncthreads();                                      // the previous step's readers are done
            for (int e = tid; e < GR_KT * GR_TILE; e += GR_THREADS) {
                int tt, ii;
                if (MODE == GR_WGRAD) { ii = e % GR_TILE; tt = e / GR_TILE; }        // a(i, t) = dy[t][i]
                else { tt = e % GR_KT; ii = e / GR_KT; }                            // a(i, t) = in / dy [i][t]
                const int i = i0 + ii, t = t0 + tt;
                float v = 0.0f;
                if (i < Mi && t < t_hi) {
                    if (MODE == GR_WGRAD) v = g.a[(int64_t)(g.row0 + t) * g.lda + i];
                    else v = g.a[(int64_t)(g.row0 + i) * g.lda + t];
                }
                As[tt][ii] = v;
                int jj;
                if (MODE == GR_FWD) { tt = e % GR_KT; jj = e / GR_KT; }            // b(t, j) = W[j][t]
                else { jj = e % GR_TILE; tt = e / GR_TILE; }                        // b(t, j) = W[t][j] / x[t][j]
                const int j = j0 + jj, t2 = t0 + tt;
                float w = 0.0f;
                if (j < g.N && t2 < t_hi) {
                    if (MODE == GR_FWD) w = g.b[(int64_t)j * g.ldb + t2];
                    else if (MODE == GR_DGRAD) w = g.b[(int64_t)t2 * g.ldb + j];
                    else w = g.b[(int64_t)(g.row0 + t2) * g.ldb + j];
                }
                Bs[tt][jj] = w;
            }
            __syncthreads();
#pragma unroll
            for (int tt = 0; tt < GR_KT; ++tt) {
                float av[4], bv[4];
#pragma unroll
                for (int x = 0; x < 4; ++x) av[x] = As[tt][ty * 4 + x];
#pragma unroll
                for (int y = 0; y < 4; ++y) bv[y] = Bs[tt][tx * 4 + y];
#pragma unroll
                for (int x = 0; x < 4; ++x)
#pragma unroll
                    for (int y = 0; y < 4; ++y) acc[x][y] = __fmaf_rn(av[x], bv[y], acc[x][y]);
            }
            if (MODE == GR_WGRAD && j0 == 0 && tid < GR_TILE)
                for (int tt = 0; tt < GR_KT; ++tt) bacc += As[tt][tid];
        }
#pragma unroll
        for (int x = 0; x < 4; ++x) {
            const int i = i0 + ty * 4 + x;
            if (i >= Mi) continue;
#pragma unroll
            for (int y = 0; y < 4; ++y) {
                const int j = j0 + tx * 4 + y;
                if (j >= g.N) continue;
                float v = acc[x][y];
                if (MODE == GR_WGRAD) {
                    g.c[(int64_t)chunk * (g.M * g.ldc + g.M) + (int64_t)i * g.ldc + j] = v;
                    continue;
                }
                const int64_t r = g.row0 + i;
                if (MODE == GR_FWD && g.bias) v += g.bias[j];
                if (g.add) v += g.add[(int64_t)g.owner[r] * g.ld_add + j];
                float* o = g.c + r * g.ldc + j;
                if (MODE == GR_FWD) {
                    if (g.act == ACT_LEAKY) v = ac_leaky(v, g.slope);
                    if (g.act == ACT_RELU) v = v > 0.0f ? v : 0.0f;
                } else {                                          // torch: leaky_relu_backward (input > 0), relu (output > 0)
                    if (g.act == ACT_LEAKY) v = *o > 0.0f ? v : v * g.slope;
                    if (g.act == ACT_RELU) v = *o > 0.0f ? v : 0.0f;
                }
                *o = v;
            }
        }
        if (MODE == GR_WGRAD && j0 == 0 && tid < GR_TILE && i0 + tid < Mi)
            g.c[(int64_t)chunk * (g.M * g.ldc + g.M) + (int64_t)g.M * g.ldc + i0 + tid] = bacc;
    }
}

__global__ void __launch_bounds__(GR_THREADS) irbpp_grad_fwd_kernel(const GemmArgs g) { grad_gemm<GR_FWD>(g); }
__global__ void __launch_bounds__(GR_THREADS) irbpp_grad_dgrad_kernel(const GemmArgs g) { grad_gemm<GR_DGRAD>(g); }
__global__ void __launch_bounds__(GR_THREADS) irbpp_grad_wgrad_kernel(const GemmArgs g) { grad_gemm<GR_WGRAD>(g); }

// dW[i][j] (row stride ldo) = sum over the slices in order; db[i] likewise (db may be NULL)
__global__ void __launch_bounds__(GR_THREADS) irbpp_grad_reduce_kernel(const float* part, int M, int N, int ldc,
                                                                       float* dw, int ldo, float* db) {
    const int64_t total = (int64_t)M * N + (db ? M : 0), stride = (int64_t)M * ldc + M;
    for (int64_t e = (int64_t)blockIdx.x * GR_THREADS + threadIdx.x; e < total; e += (int64_t)gridDim.x * GR_THREADS) {
        const bool bias = e >= (int64_t)M * N;
        const int64_t src = bias ? (int64_t)M * ldc + (e - (int64_t)M * N) : (e / N) * ldc + e % N;
        float s = 0.0f;
        for (int c = 0; c < GR_CHUNKS; ++c) s += part[c * stride + src];
        if (bias) db[e - (int64_t)M * N] = s;
        else dw[(e / N) * ldo + e % N] = s;
    }
}

// ---- per-transition kernels --------------------------------------------------------------------------------------
// [sf; mf] and the valid rows (mask == 1, model.py:347-349) of transition b: pos and n_valid.
__global__ void __launch_bounds__(GR_THREADS) irbpp_grad_prep_kernel(const GradParams P) {
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31;
    for (int k = tid; k < 384; k += GR_THREADS)
        P.xcat[(int64_t)b * 384 + k] = k < AC_EMB ? P.shape_feature[(int64_t)b * AC_EMB + k]
                                                  : P.map_feature[(int64_t)b * 256 + k - AC_EMB];
    if (tid >= 32) return;
    const float* ob = P.obs + (int64_t)b * P.obs_stride;
    int n = 0;
    for (int r0 = 0; r0 < P.sel; r0 += 32) {
        const int r = r0 + lane;
        const bool v = r < P.sel && ob[(int64_t)r * 5 + 4] == 1.0f;
        const unsigned bal = __ballot_sync(0xffffffffu, v);
        if (r < P.sel) P.pos[(int64_t)b * P.sel + r] = v ? n + __popc(bal & ((1u << lane) - 1u)) : -1;
        n += __popc(bal);
    }
    if (lane == 0) P.n_valid[b] = n;
}

// off_b, R, and transition b's rows of the row space: owners, candidate inputs, the stand-in's zero embedding
__global__ void __launch_bounds__(GR_THREADS) irbpp_grad_scatter_kernel(const GradParams P) {
    __shared__ int part[GR_THREADS / 32];
    const int b = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, B = P.B;
    int s = 0;
    for (int i = tid; i < b; i += GR_THREADS) s += P.n_valid[i];
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) s += __shfl_xor_sync(0xffffffffu, s, d);
    if (lane == 0) part[warp] = s;
    __syncthreads();
    int off = 0;
    for (int w = 0; w < GR_THREADS / 32; ++w) off += part[w];
    const int n = P.n_valid[b];
    if (tid == 0) {
        P.off[b] = off;
        if (b == B - 1) *P.count = off + n;
    }
    if (tid < AC_EMB) P.emb[(int64_t)b * AC_EMB + tid] = 0.0f;
    if (tid == 0) P.owner[b] = b;
    const float* ob = P.obs + (int64_t)b * P.obs_stride;
    for (int r = tid; r < P.sel; r += GR_THREADS) {
        const int j = P.pos[(int64_t)b * P.sel + r];
        if (j < 0) continue;
        const int64_t c = (int64_t)B + off + j;
        P.owner[c] = b;
        for (int q = 0; q < 4; ++q) P.cand[c * 4 + q] = ob[(int64_t)r * 5 + q];
    }
}

// The value head, both means, q of row a_t and its log-softmax; BACKWARD: dq and everything the weight gradients of the
// value head and of the advantage stream need from it (dadv of every row, dhv, dg).
template <bool BACKWARD>
__device__ __forceinline__ void grad_head(const GradParams& P) {
    __shared__ float gv[AC_EMB], hv[AC_EMB], dhv[AC_EMB], v[AC_MAXATOMS], mean[AC_MAXATOMS], a0[AC_MAXATOMS], dq[AC_MAXATOMS];
    __shared__ int at_pos;
    const int b = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int B = P.B, sel = P.sel, atoms = P.atoms, n = P.n_valid[b];
    const int64_t base = (int64_t)B + P.off[b];
    if (tid < AC_EMB) {                                           // mean over all sel rows, zeros included (model.py:350)
        float s = 0.0f;
        for (int j = 0; j < n; ++j) s += P.emb[(base + j) * AC_EMB + tid];
        gv[tid] = s / (float)sel;
    } else if (tid < AC_EMB + AC_MAXATOMS) {                      // mean(a) = (sum_valid a + (sel - n) a0) / sel
        const int z = tid - AC_EMB;
        float s = 0.0f;
        for (int j = 0; j < n; ++j) s += P.adv[(base + j) * AC_MAXATOMS + z];
        a0[z] = P.adv[(int64_t)b * AC_MAXATOMS + z];
        mean[z] = (s + (float)(sel - n) * a0[z]) / (float)sel;
    }
    __syncthreads();
    if (tid < AC_EMB) {                                           // fc_h_v, ReLU
        const float* wr = P.w.fc_h_v_w + tid * AC_EMB;
        float acc = 0.0f;
        for (int k = 0; k < AC_EMB; ++k) acc = __fmaf_rn(wr[k], gv[k], acc);
        acc += P.w.fc_h_v_b[tid];
        hv[tid] = acc > 0.0f ? acc : 0.0f;
    }
    __syncthreads();
    if (tid < AC_MAXATOMS) {                                      // fc_z_v
        float acc = 0.0f;
        if (tid < atoms) {
            const float* wr = P.w.fc_z_v_w + tid * AC_EMB;
            for (int k = 0; k < AC_EMB; ++k) acc = __fmaf_rn(wr[k], hv[k], acc);
            acc += P.w.fc_z_v_b[tid];
        }
        v[tid] = acc;
    }
    __syncthreads();
    if (warp == 0) {                                              // row a_t: lane = atom
        int64_t r = P.actions[b];
        r = r < 0 ? 0 : (r >= sel ? sel - 1 : r);
        const int j = P.pos[(int64_t)b * sel + r];
        const float az = j >= 0 ? P.adv[(base + j) * AC_MAXATOMS + lane] : a0[lane];
        const float qz = lane < atoms ? (v[lane] + az) - mean[lane] : -INFINITY;
        float m = qz;
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, s));
        const float e = lane < atoms ? expf(qz - m) : 0.0f;
        float se = e;
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) se += __shfl_xor_sync(0xffffffffu, se, s);
        if (!BACKWARD && P.log_p && lane < atoms) P.log_p[(int64_t)b * atoms + lane] = (qz - m) - logf(se);
        if (BACKWARD) {                                           // dq = g - softmax(q) sum(g)
            const float gz = lane < atoms ? P.grad_log_p[(int64_t)b * atoms + lane] : 0.0f;
            float sg = gz;
#pragma unroll
            for (int s = 16; s > 0; s >>= 1) sg += __shfl_xor_sync(0xffffffffu, sg, s);
            const float d = lane < atoms ? gz - (e / se) * sg : 0.0f;
            dq[lane] = d;
            P.dq[(int64_t)b * AC_MAXATOMS + lane] = d;
            if (lane == 0) at_pos = j;
        }
    }
    if (!BACKWARD) return;
    __syncthreads();
    const int jt = at_pos;
    // da_r = -dq / sel for every row, + dq on row a_t; the stand-in carries the (sel - n) invalid rows
    for (int e = tid; e < (n + 1) * AC_MAXATOMS; e += GR_THREADS) {
        const int j = e / AC_MAXATOMS - 1, z = e % AC_MAXATOMS;   // j = -1: the stand-in
        const float one = -dq[z] / (float)sel;
        float d;
        if (j < 0) d = (float)(sel - n) * one + (jt < 0 ? dq[z] : 0.0f);
        else d = one + (j == jt ? dq[z] : 0.0f);
        P.dadv[(j < 0 ? (int64_t)b : base + j) * AC_MAXATOMS + z] = d;
    }
    if (tid < AC_EMB) {                                           // dhv = fc_z_v^T dq where hv > 0
        float acc = 0.0f;
        for (int z = 0; z < atoms; ++z) acc = __fmaf_rn(P.w.fc_z_v_w[z * AC_EMB + tid], dq[z], acc);
        dhv[tid] = hv[tid] > 0.0f ? acc : 0.0f;
        P.dhv[(int64_t)b * AC_EMB + tid] = dhv[tid];
        P.gv[(int64_t)b * AC_EMB + tid] = gv[tid];
        P.hv[(int64_t)b * AC_EMB + tid] = hv[tid];
    }
    __syncthreads();
    if (tid < AC_EMB) {                                           // dxGlobal / sel = fc_h_v^T dhv / sel
        float acc = 0.0f;
        for (int k = 0; k < AC_EMB; ++k) acc = __fmaf_rn(P.w.fc_h_v_w[k * AC_EMB + tid], dhv[k], acc);
        P.dg[(int64_t)b * AC_EMB + tid] = acc / (float)sel;
    }
}

__global__ void __launch_bounds__(GR_THREADS) irbpp_grad_logp_kernel(const GradParams P) { grad_head<false>(P); }
__global__ void __launch_bounds__(GR_THREADS) irbpp_grad_head_backward_kernel(const GradParams P) { grad_head<true>(P); }

// S_b = sum over transition b's valid rows of dpre0 (in row order)
__global__ void __launch_bounds__(GR_THREADS) irbpp_grad_rowsum_kernel(const GradParams P) {
    const int b = blockIdx.x, k = threadIdx.x;
    const int n = P.n_valid[b];
    const int64_t base = (int64_t)P.B + P.off[b];
    float s = 0.0f;
    for (int j = 0; j < n; ++j) s += P.p0[(base + j) * AC_PROJ + k];
    P.S[(int64_t)b * AC_PROJ + k] = s;
}

}  // namespace irbpp
