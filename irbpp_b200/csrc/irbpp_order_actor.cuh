// irbpp_order_actor.cuh -- the order network's forward pass and Agent.act for every bin (reference model.py:355-383,
// 386-404 with args.level == 'order' and bufferSize k > 1; agent.py:51-58).
//
// The observation of a bin is [k item ids | 32 x 32 heightmap] (binPhy.py:229-230); the network embeds each of the
// k buffer slots, mixes them with one graph-attention layer and scores them with the dueling heads.  Three kernels:
//   irbpp_order_table_kernel  T_s = W0[:, 0:128] . f_s for every library shape s (W0 = gat_project_layer.0.weight,
//                             f_s the shape feature): one CTA per shape;
//   irbpp_order_bin_kernel    heightEncoder (shared with the location level) and u_b = W0[:, 128:384] . map_b + b0:
//                             one CTA per bin;
//   irbpp_order_slots_kernel  everything per slot and per bin, on tiles of AC_TM rows (slots) that hold whole bins.
// gat_project_layer.0 is split by its concat order (model.py:374-375, shape 0:128 | map 128:384), exact in real
// arithmetic: the first layer of slot (b, j) is leaky(T[id_bj] + u_b), so it costs a gather per slot.
// Per tile the slots kernel runs 256 -> 128 (h), W_query, W_key, W_val, W_out, the two FFN layers, fc_h_a and fc_z_a
// with ac_layer (mma.sync TF32, 3xTF32 split, irbpp_actor.cuh), and the bins' value heads as a second 64-row matrix
// (one row per bin) through the same layers; the k x k attention of each bin, the residuals, the slot means, the atom
// softmax, the expectation over the support, the mask and the argmax are float32 SIMT.
// Item ids are read as (int) obs[b, j] and clamped to [0, S) (the rule of irbpp_pointnet.cuh); the reference would
// raise IndexError on an id outside its shapeArray.
#pragma once
#include <stdint.h>

#include "irbpp_actor.cuh"

namespace irbpp {

constexpr int OA_MAXK = 32;                 // buffer slots per bin (graph size)
// slots kernel shared memory: H [AC_TM][132] (h, h1, h2), X [AC_TM][132], P [AC_TM][260], S [AC_TM][OA_MAXK + 1]
// (attention weights, then the per-bin mean advantage), zero bias [128], expected values [AC_TM]
constexpr int OA_LD_S = OA_MAXK + 1;
constexpr int OA_SLOTS_SMEM_FLOATS = 2 * AC_TM * AC_LD_Q + AC_TM * AC_LD_P + AC_TM * OA_LD_S + AC_EMB + AC_TM;
constexpr int OA_SLOTS_SMEM_BYTES = OA_SLOTS_SMEM_FLOATS * (int)sizeof(float);
static_assert(OA_SLOTS_SMEM_BYTES <= 227 * 1024, "the slots kernel's shared memory must fit one SM");
static_assert(AC_TM / 2 * AC_MAXATOMS <= AC_TM * OA_LD_S, "the per-bin mean advantages reuse the attention buffer");

// Weights in nn.Linear / nn.Conv2d layouts (out x in), float32, device memory (include/irbpp.h irbpp_dqn_order_weights).
struct OrderWeights {
    const float *conv1_w, *conv1_b, *conv2_w, *conv2_b, *conv3_w, *conv3_b;
    const float *gat1_w, *gat1_b, *gat2_w, *gat2_b;         // gat_project_layer.0 [256, 384], .2 [128, 256]
    const float *wq, *wk, *wv, *wo_w, *wo_b;                // embedder attention: W_query, W_key, W_val [128, 128], W_out
    const float *ff1_w, *ff1_b, *ff2_w, *ff2_b;             // embedder feed-forward: Linear(128,128), ReLU, Linear(128,128)
    const float *fc_h_v_w, *fc_h_v_b, *fc_z_v_w, *fc_z_v_b, *fc_h_a_w, *fc_h_a_b, *fc_z_a_w, *fc_z_a_b;
    float slope;                       // LeakyReLU negative slope (0.01)
};

struct OrderParams {
    OrderWeights w;
    const float* obs; int64_t obs_stride;       // [N][>= k + 1024]
    int32_t N, k, S, atoms;
    const float* shape_features;                // [S][128]
    const float* support;                       // [atoms]
    const float* mask; int64_t mask_row, mask_elem;   // mask[b*mask_row + j*mask_elem], NULL: no masking
    int64_t* actions;                           // [N]
    float* sum_q;                               // [N][k] or NULL
    // scratch (order_scratch_layout)
    float* u;                                   // [N][256]
    float* table;                               // [S][256]
};

__host__ __device__ inline int64_t order_scratch_bytes(int64_t N, int64_t S) {
    return actor_align(N * AC_PROJ * 4) + actor_align(S * AC_PROJ * 4);
}
__host__ __device__ inline void order_scratch_layout(OrderParams& A, void* scratch) {
    char* p = static_cast<char*>(scratch);
    A.u = reinterpret_cast<float*>(p); p += actor_align((int64_t)A.N * AC_PROJ * 4);
    A.table = reinterpret_cast<float*>(p);
}

// ---- per-shape table -------------------------------------------------------------------------------------------------
// T_s[j] = gat1_w[j, 0:128] . f_s: one warp per output, lanes over k (coalesced rows of the weight)
__global__ void __launch_bounds__(AC_THREADS) irbpp_order_table_kernel(const OrderParams A) {
    __shared__ __align__(16) float f[AC_EMB];
    const int s = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid < AC_EMB) f[tid] = A.shape_features[(int64_t)s * AC_EMB + tid];
    __syncthreads();
    for (int j = warp; j < AC_PROJ; j += AC_THREADS / 32) {
        const float* wr = A.w.gat1_w + (int64_t)j * 384;
        float acc = 0.0f;
        for (int c = lane; c < AC_EMB; c += 32) acc = __fmaf_rn(wr[c], f[c], acc);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (lane == 0) A.table[(int64_t)s * AC_PROJ + j] = acc;
    }
}

// ---- per-bin kernel ----------------------------------------------------------------------------------------------
// heightEncoder of the bin's heightmap (model.py:361-363, from column k on) and u_b = gat1_w[:, 128:384] . map + gat1_b
__global__ void __launch_bounds__(AC_THREADS) irbpp_order_bin_kernel(const OrderParams A) {
    __shared__ __align__(16) float hm[AC_HM * AC_HM];
    __shared__ __align__(16) float c1[16 * 16 * 16];
    __shared__ __align__(16) float c2[32 * 8 * 8];
    __shared__ __align__(16) float map[256];
    const int b = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const float* hsrc = A.obs + (int64_t)b * A.obs_stride + A.k;
    for (int i = tid; i < AC_HM * AC_HM; i += AC_THREADS) hm[i] = hsrc[i];
    ac_height_encoder(A.w, hm, c1, c2, map);
    for (int j = warp; j < AC_PROJ; j += AC_THREADS / 32) {
        const float* wr = A.w.gat1_w + (int64_t)j * 384 + AC_EMB;
        float acc = 0.0f;
        for (int c = lane; c < 256; c += 32) acc = __fmaf_rn(wr[c], map[c], acc);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (lane == 0) A.u[(int64_t)b * AC_PROJ + j] = acc + A.w.gat1_b[j];
    }
}

// ---- slots kernel ------------------------------------------------------------------------------------------------
// One CTA per tile of nb = AC_TM / k whole bins (rows r = lb * k + j, lb the bin within the tile, j the slot):
//   P[:, 0:256] = leaky(T[id] + u_b)            -> gat_project_layer.2 -> H = h
//   X = H Wq^T, P[:, 0:128] = H Wk^T, P[:, 128:256] = H Wv^T
//   per bin: S = softmax_j(X_i . K_j / sqrt(128)); X = S V          (model.py:94-117, nothing masked: :377)
//   P[:, 0:128] = W_out(X) + b; H += P (h1);  X = relu(ff1(H)); P[:, 0:128] = ff2(X); H += P (h2)  (model.py:16, 24)
//   X[lb] = mean_j H[lb * k + j] (g, model.py:381-382); P[:, 0:128] = relu(fc_h_v(X)); P[:, 128:160] = fc_z_v(...) = v
//   X = relu(fc_h_a(H)); P[:, 160:192] = fc_z_a(X) = a;  S[lb] = mean_j a
//   q = v + a - mean(a), softmax over the atoms, expectation over the support, mask, argmax over the k slots.
// TARGET (irbpp_order_target_kernel): the final phase instead builds p = softmax(q) of slot a* = T.next_actions[b] of
// each bin only, one warp per bin, and projects it (learn_project, irbpp_learn.cuh); no expectation, argmax or sum_q.
template <bool TARGET>
__device__ __forceinline__ void order_slots(const OrderParams A, const LearnTarget& T) {
    extern __shared__ __align__(16) float oa_smem[];
    float* H = oa_smem;                               // [AC_TM][AC_LD_Q]
    float* X = H + AC_TM * AC_LD_Q;                   // [AC_TM][AC_LD_Q]
    float* P = X + AC_TM * AC_LD_Q;                   // [AC_TM][AC_LD_P]
    float* S = P + AC_TM * AC_LD_P;                   // [AC_TM][OA_LD_S]
    float* zero = S + AC_TM * OA_LD_S;                // [128] the bias of W_query / W_key / W_val (none)
    float* sq = zero + AC_EMB;                        // [AC_TM] expected value of each row
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int k = A.k, atoms = A.atoms;
    const float slope = A.w.slope;
    const int per = AC_TM / k;                        // bins per tile
    const int b0 = blockIdx.x * per;
    const int nb = min(per, A.N - b0), nr = nb * k;   // bins and rows of this tile
    if (tid < AC_EMB) zero[tid] = 0.0f;
    // gat_project_layer.0 as leaky(T[id] + u_b) into P[:, 0:256]; rows >= nr are zero
    for (int o = tid; o < AC_TM * AC_PROJ; o += AC_THREADS) {
        const int r = o >> 8, c = o & 255;
        float v = 0.0f;
        if (r < nr) {
            const int b = b0 + r / k, j = r - (r / k) * k;
            int id = (int)A.obs[(int64_t)b * A.obs_stride + j];
            id = id < 0 ? 0 : (id >= A.S ? A.S - 1 : id);
            v = ac_leaky(A.table[(int64_t)id * AC_PROJ + c] + A.u[(int64_t)b * AC_PROJ + c], slope);
        }
        P[r * AC_LD_P + c] = v;
    }
    __syncthreads();
    ac_layer<256, 128, 2, ACT_NONE>(P, AC_LD_P, A.w.gat2_w, 256, 128, A.w.gat2_b, H, AC_LD_Q, slope);     // h
    __syncthreads();
    ac_layer<128, 128, 2, ACT_NONE>(H, AC_LD_Q, A.w.wq, 128, 128, zero, X, AC_LD_Q, slope);                // Q
    ac_layer<128, 128, 2, ACT_NONE>(H, AC_LD_Q, A.w.wk, 128, 128, zero, P, AC_LD_P, slope);                // K
    ac_layer<128, 128, 2, ACT_NONE>(H, AC_LD_Q, A.w.wv, 128, 128, zero, P + AC_EMB, AC_LD_P, slope);       // V
    __syncthreads();
    // compatibility = norm_factor * (Q K^T) over the slots of the row's bin (model.py:49, 99)
    const float norm = 1.0f / sqrtf((float)AC_EMB);
    for (int o = tid; o < nr * k; o += AC_THREADS) {
        const int r = o / k, j = o - r * k, rk = (r / k) * k + j;
        const float* q = X + r * AC_LD_Q;
        const float* kk = P + rk * AC_LD_P;
        float acc = 0.0f;
        for (int c = 0; c < AC_EMB; ++c) acc = __fmaf_rn(q[c], kk[c], acc);
        S[r * OA_LD_S + j] = norm * acc;
    }
    __syncthreads();
    if (tid < nr) {                                   // softmax over the slots (model.py:109)
        float* s = S + tid * OA_LD_S;
        float m = -INFINITY;
        for (int j = 0; j < k; ++j) m = fmaxf(m, s[j]);
        float se = 0.0f;
        for (int j = 0; j < k; ++j) { s[j] = expf(s[j] - m); se += s[j]; }
        for (int j = 0; j < k; ++j) s[j] = s[j] / se;
    }
    __syncthreads();
    for (int o = tid; o < AC_TM * AC_EMB; o += AC_THREADS) {      // heads = attn V (model.py:117) into X
        const int r = o >> 7, c = o & 127;
        float acc = 0.0f;
        if (r < nr) {
            const float* s = S + r * OA_LD_S;
            const float* v = P + (r / k) * k * AC_LD_P + AC_EMB + c;
            for (int j = 0; j < k; ++j) acc = __fmaf_rn(s[j], v[j * AC_LD_P], acc);
        }
        X[r * AC_LD_Q + c] = acc;
    }
    __syncthreads();
    ac_layer<128, 128, 2, ACT_NONE>(X, AC_LD_Q, A.w.wo_w, 128, 128, A.w.wo_b, P, AC_LD_P, slope);          // W_out
    __syncthreads();
    for (int o = tid; o < AC_TM * AC_EMB; o += AC_THREADS) H[(o >> 7) * AC_LD_Q + (o & 127)] += P[(o >> 7) * AC_LD_P + (o & 127)];
    __syncthreads();
    ac_layer<128, 128, 2, ACT_RELU>(H, AC_LD_Q, A.w.ff1_w, 128, 128, A.w.ff1_b, X, AC_LD_Q, slope);        // FFN
    __syncthreads();
    ac_layer<128, 128, 2, ACT_NONE>(X, AC_LD_Q, A.w.ff2_w, 128, 128, A.w.ff2_b, P, AC_LD_P, slope);
    __syncthreads();
    for (int o = tid; o < AC_TM * AC_EMB; o += AC_THREADS) H[(o >> 7) * AC_LD_Q + (o & 127)] += P[(o >> 7) * AC_LD_P + (o & 127)];
    __syncthreads();
    for (int o = tid; o < AC_TM * AC_EMB; o += AC_THREADS) {      // g = mean over the slots, one row per bin
        const int lb = o >> 7, c = o & 127;
        float acc = 0.0f;
        if (lb < nb) {
            for (int j = 0; j < k; ++j) acc += H[(lb * k + j) * AC_LD_Q + c];
            acc = acc / (float)k;
        }
        X[lb * AC_LD_Q + c] = acc;
    }
    __syncthreads();
    ac_layer<128, 128, 2, ACT_RELU>(X, AC_LD_Q, A.w.fc_h_v_w, 128, 128, A.w.fc_h_v_b, P, AC_LD_P, slope);   // value head
    __syncthreads();
    ac_layer<128, 32, 4, ACT_NONE>(P, AC_LD_P, A.w.fc_z_v_w, 128, atoms, A.w.fc_z_v_b, P + AC_EMB, AC_LD_P, slope);
    __syncthreads();
    ac_layer<128, 128, 2, ACT_RELU>(H, AC_LD_Q, A.w.fc_h_a_w, 128, 128, A.w.fc_h_a_b, X, AC_LD_Q, slope);   // advantage
    __syncthreads();
    ac_layer<128, 32, 4, ACT_NONE>(X, AC_LD_Q, A.w.fc_z_a_w, 128, atoms, A.w.fc_z_a_b, P + AC_EMB + 32, AC_LD_P, slope);
    __syncthreads();
    for (int o = tid; o < nb * AC_MAXATOMS; o += AC_THREADS) {    // mean_j a (model.py:396)
        const int lb = o >> 5, z = o & 31;
        float acc = 0.0f;
        for (int j = 0; j < k; ++j) acc += P[(lb * k + j) * AC_LD_P + AC_EMB + 32 + z];
        S[o] = acc / (float)k;
    }
    __syncthreads();
    // one warp per row, lane = atom
    const float sup = lane < atoms ? A.support[lane] : 0.0f;
    if constexpr (TARGET) {                                     // one warp per bin, slot a*
        for (int lb = warp; lb < nb; lb += AC_THREADS / 32) {
            const int64_t b = b0 + lb;
            int64_t j = T.next_actions[b];
            j = j < 0 ? 0 : (j >= k ? k - 1 : j);
            const int r = lb * k + (int)j;
            const float qz = lane < atoms ? (P[lb * AC_LD_P + AC_EMB + lane] + P[r * AC_LD_P + AC_EMB + 32 + lane]) - S[lb * 32 + lane]
                                          : -INFINITY;
            float m = qz;
#pragma unroll
            for (int s = 16; s > 0; s >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, s));
            const float e = lane < atoms ? expf(qz - m) : 0.0f;
            float se = e;
#pragma unroll
            for (int s = 16; s > 0; s >>= 1) se += __shfl_xor_sync(0xffffffffu, se, s);
            const float p = e / se;
            if (T.p_next && lane < atoms) T.p_next[b * atoms + lane] = p;
            learn_project(T, b, atoms, p, sup, lane);
        }
        return;
    }
    for (int r = warp; r < nr; r += AC_THREADS / 32) {
        const int lb = r / k, j = r - lb * k, b = b0 + lb;
        const float qz = lane < atoms ? (P[lb * AC_LD_P + AC_EMB + lane] + P[r * AC_LD_P + AC_EMB + 32 + lane]) - S[lb * 32 + lane]
                                      : -INFINITY;
        float m = qz;
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, s));
        const float e = lane < atoms ? expf(qz - m) : 0.0f;
        float se = e;
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) se += __shfl_xor_sync(0xffffffffu, se, s);
        float sqz = (e / se) * sup;
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) sqz += __shfl_xor_sync(0xffffffffu, sqz, s);
        if (A.mask && A.mask[(int64_t)b * A.mask_row + (int64_t)j * A.mask_elem] != 1.0f) sqz = -INFINITY;   // agent.py:56-57
        if (lane == 0) {
            sq[r] = sqz;
            if (A.sum_q) A.sum_q[(int64_t)b * k + j] = sqz;
        }
    }
    __syncthreads();
    if (tid < nb) {                                   // torch.argmax: the first slot of the maximum, 0 if all are -inf
        float best = -INFINITY;
        int bi = 0;
        for (int j = 0; j < k; ++j)
            if (sq[tid * k + j] > best) { best = sq[tid * k + j]; bi = j; }
        A.actions[b0 + tid] = bi;
    }
}

__global__ void __launch_bounds__(AC_THREADS, 1) irbpp_order_slots_kernel(const OrderParams A) {
    order_slots<false>(A, LearnTarget{});
}

// Agent.learn's target pass (agent.py:94-115) over the order-level target net: irbpp_dqn_order_target
__global__ void __launch_bounds__(AC_THREADS, 1) irbpp_order_target_kernel(const OrderParams A, const LearnTarget T) {
    order_slots<true>(A, T);
}

}  // namespace irbpp
