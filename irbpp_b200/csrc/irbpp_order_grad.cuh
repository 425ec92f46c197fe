// irbpp_order_grad.cuh -- the order network and its backward pass: log p(s, a_t, .) of Agent.learn's gradient pass at
// the order level (agent.py:85-86 on model.py:355-383, 386-404 with args.level == 'order' and bufferSize k > 1) and the
// gradients of -sum(m . log p) through it (agent.py:117-119), for irbpp_dqn_order_log_prob /
// irbpp_dqn_order_log_prob_backward.
//
// The split with torch is the location level's (irbpp_grad.cuh): torch computes shape_features [S, 128] (shapeEncoder
// on every library shape, max over the points) and map_feature [B, 256] (heightEncoder) with autograd and builds the
// NoisyLinear effective weights; these kernels take them as plain inputs and return their gradients.  Everything per
// slot and per bin runs here: gat_project_layer, W_query / W_key / W_val, the k x k attention of each bin (nothing
// masked, model.py:377), W_out and its residual, the feed-forward block and its residual, the slot mean, the value head
// on it, the advantage stream per slot, the dueling combine and the log-softmax of slot a_t.
//
// Layout.  The row space is the B * k slots, bin-major (row r = b * k + j); every slot is a row, so there is no
// compaction.  The per-slot layers are the row-parallel GEMMs of irbpp_grad.cuh (their add[owner[r]] carries the
// per-bin terms); the per-bin parts (attention, value head, means, log-softmax) run one CTA per bin.
//
// Reformulations (each exact in real arithmetic):
//   * gat_project_layer.0 split by concat order (shape 0:128 | map 128:384), as irbpp_order_actor.cuh does:
//     pre0 = W0[:, 0:128] . f_id + u_b with u_b = W0[:, 128:384] . mf_b + b0 once per bin.  Backward: with per-shape
//     sums Sid_s = sum over the slots holding shape s of dpre0 and per-bin sums Sb_b = sum_j dpre0_bj,
//     d f_s = W0[:, 0:128]^T Sid_s, d mf_b = W0[:, 128:384]^T Sb_b, dW0[:, 0:128] = sum_s Sid_s (x) f_s,
//     dW0[:, 128:384] = sum_b Sb_b (x) mf_b, db0 = sum_b Sb_b.
//   * log p = q - max - log sum exp(q - max).  Backward with g = dL/dlog p: dq = g - softmax(q) sum(g); dv = dq; every
//     slot gets da_j = -dq / k, slot a_t additionally + dq.
//   * graph embedding = sum_j h2_j / k: dxGlobal / k (value head) is added to every slot's dh2.
//   * attention: dV = attn^T dheads, dattn = dheads V^T, dcompat = attn (.) (dattn - rowsum(dattn (.) attn)),
//     dQ = s dcompat K, dK = s dcompat^T Q with s = 1 / sqrt(128).
// Determinism: no atomics.  Weight gradients are the GEMMs' fixed slices (irbpp_grad.cuh).  The per-shape sums run over
// the slots in slot order: a stable rank of every slot by (id, slot) gives each shape its slots as one contiguous run.
#pragma once
#include <stdint.h>

#include "irbpp_grad.cuh"
#include "irbpp_order_actor.cuh"

namespace irbpp {

// gradients of the effective tensors after the six convolutions (include/irbpp.h irbpp_dqn_order_grads)
struct OrderGradOut {
    float *gat1_w, *gat1_b, *gat2_w, *gat2_b, *wq, *wk, *wv, *wo_w, *wo_b, *ff1_w, *ff1_b, *ff2_w, *ff2_b;
    float *fc_h_v_w, *fc_h_v_b, *fc_z_v_w, *fc_z_v_b, *fc_h_a_w, *fc_h_a_b, *fc_z_a_w, *fc_z_a_b;
};

struct OrderGradParams {
    OrderWeights w;
    const float* obs; int64_t obs_stride;
    int32_t B, k, S, atoms;
    const float* shape_features;         // [S][128]
    const float* map_feature;            // [B][256]
    const int64_t* actions;              // [B], clamped to [0, k)
    float* log_p;                        // [B][atoms] or NULL
    const float* grad_log_p;             // [B][atoms], backward only
    // scratch (order_grad_scratch_layout); rows = B * k
    float* wqkv;                         // [384][128] W_query; W_key; W_val
    int32_t* ids;                        // [rows] item id of a slot, clamped to [0, S)
    int32_t* owner;                      // [rows] bin of a slot
    int32_t* perm;                       // [rows] slots ordered by (id, slot)
    int32_t* sorted;                     // [rows] their ids
    float* xs;                           // [rows][128] f_id of each slot
    float* p0;                           // [rows][256] leaky(gat_project_layer.0); backward: its pre-activation gradient
    float* h;                            // [rows][128] h;                          backward: its gradient
    float* qkv;                          // [rows][384] Q | K | V
    float* dqkv;                         // [rows][384] their gradients
    float* attn;                         // [rows][k]   softmax(compat) row of each slot
    float* heads;                        // [rows][128] attn V;                     backward: its gradient
    float* h1;                           // [rows][128] h + W_out(heads);           backward: its gradient
    float* f1;                           // [rows][128] relu(ff1(h1));              backward: its pre-activation gradient
    float* h2;                           // [rows][128] h1 + ff2(f1);               backward: its gradient
    float* ha;                           // [rows][128] relu(fc_h_a(h2));           backward: its pre-activation gradient
    float* adv;                          // [rows][32]  advantages
    float* dadv;                         // [rows][32]  their gradients
    float* u;                            // [B][256] u_b
    float* gv;                           // [B][128] graph embedding
    float* hv;                           // [B][128] relu(fc_h_v(gv))
    float* dhv;                          // [B][128] pre-activation gradient of fc_h_v
    float* dg;                           // [B][128] dxGlobal / k
    float* dq;                           // [B][32]
    float* Sb;                           // [B][256] per-bin sums of dpre0
    float* Sid;                          // [S][256] per-shape sums of dpre0
    float* part;                         // [GR_CHUNKS][GR_MAX_WGRAD + 256] weight-gradient slices
};

__host__ __device__ inline int64_t order_grad_scratch_bytes(int64_t B, int64_t k, int64_t S) {
    const int64_t rows = B * k;
    return actor_align(384 * AC_EMB * 4) + 4 * actor_align(rows * 4) +
           actor_align(rows * (128 + 256 + 128 + 384 + 384 + OA_MAXK + 128 + 128 + 128 + 128 + 128 + 32 + 32) * 4) +
           actor_align(B * (256 + 4 * 128 + 32 + 256) * 4) + actor_align(S * 256 * 4) +
           actor_align((int64_t)GR_CHUNKS * (GR_MAX_WGRAD + 256) * 4);
}

__host__ __device__ inline void order_grad_scratch_layout(OrderGradParams& P, void* scratch) {
    char* p = static_cast<char*>(scratch);
    const int64_t B = P.B, rows = B * P.k, S = P.S;
    auto take = [&](int64_t bytes) { char* q = p; p += actor_align(bytes); return q; };
    P.wqkv = reinterpret_cast<float*>(take(384 * AC_EMB * 4));
    P.ids = reinterpret_cast<int32_t*>(take(rows * 4));
    P.owner = reinterpret_cast<int32_t*>(take(rows * 4));
    P.perm = reinterpret_cast<int32_t*>(take(rows * 4));
    P.sorted = reinterpret_cast<int32_t*>(take(rows * 4));
    float* a = reinterpret_cast<float*>(
        take(rows * (128 + 256 + 128 + 384 + 384 + OA_MAXK + 128 + 128 + 128 + 128 + 128 + 32 + 32) * 4));
    P.xs = a; a += rows * 128;
    P.p0 = a; a += rows * 256;
    P.h = a; a += rows * 128;
    P.qkv = a; a += rows * 384;
    P.dqkv = a; a += rows * 384;
    P.attn = a; a += rows * OA_MAXK;
    P.heads = a; a += rows * 128;
    P.h1 = a; a += rows * 128;
    P.f1 = a; a += rows * 128;
    P.h2 = a; a += rows * 128;
    P.ha = a; a += rows * 128;
    P.adv = a; a += rows * 32;
    P.dadv = a;
    float* c = reinterpret_cast<float*>(take(B * (256 + 4 * 128 + 32 + 256) * 4));
    P.u = c; c += B * 256;
    P.gv = c; c += B * 128;
    P.hv = c; c += B * 128;
    P.dhv = c; c += B * 128;
    P.dg = c; c += B * 128;
    P.dq = c; c += B * 32;
    P.Sb = c;
    P.Sid = reinterpret_cast<float*>(take(S * 256 * 4));
    P.part = reinterpret_cast<float*>(take((int64_t)GR_CHUNKS * (GR_MAX_WGRAD + 256) * 4));
}

// Bin b's slots: clamped ids, owners and the gathered shape features; the CTAs together copy W_query, W_key and W_val
// into one [384][128] matrix, so that Q | K | V is one GEMM.
__global__ void __launch_bounds__(GR_THREADS) irbpp_order_grad_prep_kernel(const OrderGradParams P) {
    __shared__ int sid[OA_MAXK];
    const int b = blockIdx.x, tid = threadIdx.x, k = P.k;
    const int64_t base = (int64_t)b * k;
    if (tid < k) {
        int id = (int)P.obs[(int64_t)b * P.obs_stride + tid];            // the act's rule (irbpp_order_actor.cuh)
        id = id < 0 ? 0 : (id >= P.S ? P.S - 1 : id);
        sid[tid] = id;
        P.ids[base + tid] = id;
        P.owner[base + tid] = b;
    }
    __syncthreads();
    for (int e = tid; e < k * AC_EMB; e += GR_THREADS)
        P.xs[base * AC_EMB + e] = P.shape_features[(int64_t)sid[e >> 7] * AC_EMB + (e & 127)];
    for (int64_t e = (int64_t)b * GR_THREADS + tid; e < 3 * AC_EMB * AC_EMB; e += (int64_t)P.B * GR_THREADS) {
        const int m = (int)(e / (AC_EMB * AC_EMB)), o = (int)(e % (AC_EMB * AC_EMB));
        P.wqkv[e] = (m == 0 ? P.w.wq : (m == 1 ? P.w.wk : P.w.wv))[o];
    }
}

// The attention of bin b (model.py:94-117): compat = s (Q K^T), attn = softmax over the slots, heads = attn V; the
// arithmetic of irbpp_order_actor.cuh's slots kernel.
__global__ void __launch_bounds__(GR_THREADS) irbpp_order_grad_attn_kernel(const OrderGradParams P) {
    __shared__ float S[OA_MAXK][OA_LD_S];
    const int b = blockIdx.x, tid = threadIdx.x, k = P.k;
    const int64_t base = (int64_t)b * k;
    const float* qkv = P.qkv + base * 384;
    const float norm = 1.0f / sqrtf((float)AC_EMB);
    for (int o = tid; o < k * k; o += GR_THREADS) {
        const int i = o / k, j = o - i * k;
        const float* q = qkv + i * 384;
        const float* kk = qkv + j * 384 + AC_EMB;
        float acc = 0.0f;
        for (int c = 0; c < AC_EMB; ++c) acc = __fmaf_rn(q[c], kk[c], acc);
        S[i][j] = norm * acc;
    }
    __syncthreads();
    if (tid < k) {
        float* s = S[tid];
        float m = -INFINITY;
        for (int j = 0; j < k; ++j) m = fmaxf(m, s[j]);
        float se = 0.0f;
        for (int j = 0; j < k; ++j) { s[j] = expf(s[j] - m); se += s[j]; }
        for (int j = 0; j < k; ++j) s[j] = s[j] / se;
    }
    __syncthreads();
    for (int o = tid; o < k * k; o += GR_THREADS) P.attn[base * k + o] = S[o / k][o % k];
    for (int o = tid; o < k * AC_EMB; o += GR_THREADS) {
        const int i = o >> 7, c = o & 127;
        const float* v = qkv + 2 * AC_EMB + c;
        float acc = 0.0f;
        for (int j = 0; j < k; ++j) acc = __fmaf_rn(S[i][j], v[j * 384], acc);
        P.heads[(base + i) * AC_EMB + c] = acc;
    }
}

// The attention's backward pass for bin b: dQ | dK | dV from dheads (in P.heads) into P.dqkv.
__global__ void __launch_bounds__(GR_THREADS) irbpp_order_grad_attn_backward_kernel(const OrderGradParams P) {
    __shared__ float A[OA_MAXK][OA_LD_S], D[OA_MAXK][OA_LD_S];
    const int b = blockIdx.x, tid = threadIdx.x, k = P.k;
    const int64_t base = (int64_t)b * k;
    const float* qkv = P.qkv + base * 384;
    const float* dh = P.heads + base * AC_EMB;
    const float norm = 1.0f / sqrtf((float)AC_EMB);
    for (int o = tid; o < k * k; o += GR_THREADS) {               // attn, and dattn = dheads V^T
        const int i = o / k, j = o - i * k;
        A[i][j] = P.attn[base * k + o];
        const float* d = dh + i * AC_EMB;
        const float* v = qkv + j * 384 + 2 * AC_EMB;
        float acc = 0.0f;
        for (int c = 0; c < AC_EMB; ++c) acc = __fmaf_rn(d[c], v[c], acc);
        D[i][j] = acc;
    }
    __syncthreads();
    if (tid < k) {                                                // dcompat = attn (dattn - sum_j dattn attn)
        float r = 0.0f;
        for (int j = 0; j < k; ++j) r = __fmaf_rn(D[tid][j], A[tid][j], r);
        for (int j = 0; j < k; ++j) D[tid][j] = A[tid][j] * (D[tid][j] - r);
    }
    __syncthreads();
    for (int o = tid; o < k * AC_EMB; o += GR_THREADS) {
        const int i = o >> 7, c = o & 127;
        float dq = 0.0f, dk = 0.0f, dv = 0.0f;
        for (int j = 0; j < k; ++j) {
            dq = __fmaf_rn(D[i][j], qkv[j * 384 + AC_EMB + c], dq);   // dQ_i = s sum_j dcompat_ij K_j
            dk = __fmaf_rn(D[j][i], qkv[j * 384 + c], dk);            // dK_i = s sum_j dcompat_ji Q_j
            dv = __fmaf_rn(A[j][i], dh[j * AC_EMB + c], dv);          // dV_i = sum_j attn_ji dheads_j
        }
        float* out = P.dqkv + (base + i) * 384 + c;
        out[0] = norm * dq;
        out[AC_EMB] = norm * dk;
        out[2 * AC_EMB] = dv;
    }
}

// y += x over n floats (the two residuals and their gradients)
__global__ void __launch_bounds__(GR_THREADS) irbpp_order_grad_add_kernel(float* y, const float* x, int64_t n) {
    for (int64_t e = (int64_t)blockIdx.x * GR_THREADS + threadIdx.x; e < n; e += (int64_t)gridDim.x * GR_THREADS)
        y[e] += x[e];
}

// The graph embedding and value head, the slot mean of the advantages, q of slot a_t and its log-softmax; BACKWARD: dq
// and what the weight gradients of the value head and of the advantage stream need from it (dadv of every slot, dhv,
// dg).  The formulas of grad_head (irbpp_grad.cuh) with every slot a row.
template <bool BACKWARD>
__device__ __forceinline__ void order_grad_head(const OrderGradParams& P) {
    __shared__ float gv[AC_EMB], hv[AC_EMB], dhv[AC_EMB], v[AC_MAXATOMS], mean[AC_MAXATOMS], dq[AC_MAXATOMS];
    __shared__ int at_slot;
    const int b = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int k = P.k, atoms = P.atoms;
    const int64_t base = (int64_t)b * k;
    if (tid < AC_EMB) {                                           // mean over the slots (model.py:381-382)
        float s = 0.0f;
        for (int j = 0; j < k; ++j) s += P.h2[(base + j) * AC_EMB + tid];
        gv[tid] = s / (float)k;
    } else if (tid < AC_EMB + AC_MAXATOMS) {                      // mean_j a (model.py:396)
        const int z = tid - AC_EMB;
        float s = 0.0f;
        for (int j = 0; j < k; ++j) s += P.adv[(base + j) * AC_MAXATOMS + z];
        mean[z] = s / (float)k;
    }
    __syncthreads();
    if (tid < AC_EMB) {                                           // fc_h_v, ReLU
        const float* wr = P.w.fc_h_v_w + tid * AC_EMB;
        float acc = 0.0f;
        for (int c = 0; c < AC_EMB; ++c) acc = __fmaf_rn(wr[c], gv[c], acc);
        acc += P.w.fc_h_v_b[tid];
        hv[tid] = acc > 0.0f ? acc : 0.0f;
    }
    __syncthreads();
    if (tid < AC_MAXATOMS) {                                      // fc_z_v
        float acc = 0.0f;
        if (tid < atoms) {
            const float* wr = P.w.fc_z_v_w + tid * AC_EMB;
            for (int c = 0; c < AC_EMB; ++c) acc = __fmaf_rn(wr[c], hv[c], acc);
            acc += P.w.fc_z_v_b[tid];
        }
        v[tid] = acc;
    }
    __syncthreads();
    if (warp == 0) {                                              // slot a_t: lane = atom
        int64_t j = P.actions[b];
        j = j < 0 ? 0 : (j >= k ? k - 1 : j);
        const float az = P.adv[(base + j) * AC_MAXATOMS + lane];
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
            if (lane == 0) at_slot = (int)j;
        }
    }
    if (!BACKWARD) return;
    __syncthreads();
    const int jt = at_slot;
    for (int e = tid; e < k * AC_MAXATOMS; e += GR_THREADS) {    // da_j = -dq / k, + dq on slot a_t
        const int j = e / AC_MAXATOMS, z = e % AC_MAXATOMS;
        P.dadv[(base + j) * AC_MAXATOMS + z] = -dq[z] / (float)k + (j == jt ? dq[z] : 0.0f);
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
    if (tid < AC_EMB) {                                           // dxGlobal / k = fc_h_v^T dhv / k
        float acc = 0.0f;
        for (int c = 0; c < AC_EMB; ++c) acc = __fmaf_rn(P.w.fc_h_v_w[c * AC_EMB + tid], dhv[c], acc);
        P.dg[(int64_t)b * AC_EMB + tid] = acc / (float)k;
    }
}

__global__ void __launch_bounds__(GR_THREADS) irbpp_order_grad_logp_kernel(const OrderGradParams P) { order_grad_head<false>(P); }
__global__ void __launch_bounds__(GR_THREADS) irbpp_order_grad_head_backward_kernel(const OrderGradParams P) {
    order_grad_head<true>(P);
}

// The stable rank of slot r by (id, r): perm[rank] = r, sorted[rank] = id, so the slots of one shape form one run in
// slot order.  One thread per slot compares its id with every slot's.
__global__ void __launch_bounds__(GR_THREADS) irbpp_order_grad_rank_kernel(const OrderGradParams P) {
    __shared__ int tile[GR_THREADS];
    const int R = P.B * P.k, tid = threadIdx.x, r = blockIdx.x * GR_THREADS + tid;
    const int my = r < R ? P.ids[r] : 0;
    int rank = 0;
    for (int t0 = 0; t0 < R; t0 += GR_THREADS) {
        __syncthreads();
        tile[tid] = t0 + tid < R ? P.ids[t0 + tid] : 0;
        __syncthreads();
        const int n = min(GR_THREADS, R - t0);
        for (int t = 0; t < n; ++t) rank += (tile[t] < my) | ((tile[t] == my) & (t0 + t < r));
    }
    if (r < R) {
        P.perm[rank] = r;
        P.sorted[rank] = my;
    }
}

static_assert(AC_PROJ == GR_THREADS, "the segment sums take one thread per column of dpre0");

// CTA s < S: Sid_s = sum of dpre0 over the slots holding shape s, in slot order; CTA S + b: Sb_b = sum_j dpre0_bj.
// One thread per column.
__global__ void __launch_bounds__(GR_THREADS) irbpp_order_grad_segsum_kernel(const OrderGradParams P) {
    const int c = threadIdx.x, R = P.B * P.k;
    float acc = 0.0f;
    if ((int)blockIdx.x < P.S) {
        const int s = blockIdx.x;
        int lo = 0, hi = R;                                       // first rank with id >= s
        while (lo < hi) { const int mid = (lo + hi) >> 1; if (P.sorted[mid] < s) lo = mid + 1; else hi = mid; }
        for (int t = lo; t < R && P.sorted[t] == s; ++t) acc += P.p0[(int64_t)P.perm[t] * AC_PROJ + c];
        P.Sid[(int64_t)s * AC_PROJ + c] = acc;
    } else {
        const int b = blockIdx.x - P.S;
        for (int j = 0; j < P.k; ++j) acc += P.p0[((int64_t)b * P.k + j) * AC_PROJ + c];
        P.Sb[(int64_t)b * AC_PROJ + c] = acc;
    }
}

}  // namespace irbpp
