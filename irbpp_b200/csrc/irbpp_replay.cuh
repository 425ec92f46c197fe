// irbpp_replay.cuh -- the reference's prioritized n-step replay (memory.py) for M memories on the device.
//
// Reference (memory.py:15-208): one ReplayMemory per environment (main.py:61-63), each a float32 sum tree
// `sum_tree[2C-1]` in heap layout (leaf j = node C-1+j, parent (i-1)//2) over a ring of C transitions, kept on the
// host and appended to one bin at a time (trainer.py:184-186).  Here the M rings, their trees and the small state
// block {index, full, t, max} live in caller-owned device memory, memory-major, and three launches cover one
// actor / learner iteration:
//   append           one CTA per memory: the row copy (the observation is the bandwidth), then thread 0 stores the
//                    scalars, sets the leaf to `max` and recomputes its ancestors as left + right (memory.py:45-69)
//   sample           one CTA per listed memory: stratified float32 descents with at most A attempts per stratum
//                    (memory.py:163-170, which loops until it succeeds), the n-step gather and the importance weights
//                    normalised by this memory's batch maximum (memory.py:191-203)
//   update           one warp per memory: the batch rows of that memory applied in batch order (a duplicated leaf
//                    takes the last value), each followed by its ancestor recompute, and `max` raised
// Every parent is recomputed as left + right, so the tree is a pure function of its leaves and the sequence of
// float32 adds is the reference's: the trees match bit for bit.  The library is built -fmad=false.
#pragma once
#include <stdint.h>

namespace irbpp {

constexpr int RP_APPEND_THREADS = 256;
constexpr int RP_SAMPLE_THREADS = 128;
constexpr int RP_UPDATE_WARPS = 4;
constexpr int RP_MAX_N = 64;               // multi-step limit (the discount vector travels in the launch parameters)

struct ReplayAppendArgs {
    irbpp_replay_memory mem;
    const float* obs; int64_t obs_stride;  // [M] rows of the step's observation
    const int64_t* action; const float* reward; const uint8_t* done; const uint8_t* valid;   // [M]; valid may be NULL
    float reward_clip;                     // > 0: reward clamped to [-clip, clip] (trainer.py:181-182)
};

struct ReplaySampleArgs {
    irbpp_replay_memory mem;
    const int32_t* mem_ids;                // [G] memories to sample, k strata each
    int32_t G, k, n, attempts;
    float scale[RP_MAX_N];                 // float32(discount ** i), i < n (memory.py:107)
    double neg_beta;                       // -priority_weight, rounded to float32 as torch's pow does
    uint64_t seed, call;                   // counter-based uniforms when `uniforms` is NULL
    const double* uniforms;                // [G * k][attempts] caller-supplied uniforms in [0, 1), or NULL
    irbpp_replay_batch out;
    uint32_t* error_flags;                 // bit c set when some sample reported code c (may be NULL)
};

struct ReplayUpdateArgs {
    irbpp_replay_memory mem;
    const int32_t* mem_ids; const int64_t* tree_idxs; const float* loss;   // [B]
    int32_t B;
    double omega;                          // priority_exponent, rounded to float32 as numpy's float32 power does
    uint32_t* error_flags;
};

__host__ __device__ __forceinline__ uint64_t rp_mix(uint64_t z) {       // splitmix64 finaliser
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

// Uniform in [0, 1) with 53 random bits for (seed, sample call, batch row, attempt < 2^16).
__host__ __device__ __forceinline__ double rp_uniform(uint64_t seed, uint64_t call, uint64_t row, uint32_t attempt) {
    uint64_t z = rp_mix(seed + 0x9E3779B97F4A7C15ull * (call + 1));
    z = rp_mix(z + 0x9E3779B97F4A7C15ull * ((row << 16) + attempt + 1));
    return (double)(z >> 11) * (1.0 / 9007199254740992.0);
}

// memory.py:45-50: every ancestor of node i recomputed as left + right, bottom-up.
__device__ __forceinline__ void rp_propagate(float* tree, int i) {
    while (i > 0) {
        const int p = (i - 1) >> 1;
        tree[p] = tree[2 * p + 1] + tree[2 * p + 2];
        i = p;
    }
}

__global__ void irbpp_replay_init_kernel(const irbpp_replay_memory mem) {
    const int64_t nodes = (int64_t)mem.num_memories * (2 * mem.capacity - 1);
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nodes; i += (int64_t)gridDim.x * blockDim.x) {
        mem.tree[i] = 0.0f;
        if (i < mem.num_memories) {
            mem.state[i].index = 0; mem.state[i].full = 0; mem.state[i].t = 0; mem.state[i].max = 1.0f;   // memory.py:27
        }
    }
}

// memory.py:58-69 + :110-113 for every memory whose valid byte is set (trainer.py:184-186 skips the others).
__global__ void __launch_bounds__(RP_APPEND_THREADS) irbpp_replay_append_kernel(const ReplayAppendArgs A) {
    const int m = blockIdx.x;
    if (A.valid && !A.valid[m]) return;
    irbpp_replay_state* st = A.mem.state + m;
    const int C = A.mem.capacity, L = A.mem.obs_len;
    const int idx = st->index;
    const int64_t row = (int64_t)m * C + idx;
    const float* src = A.obs + (int64_t)m * A.obs_stride;
    float* dst = A.mem.states + row * L;
    for (int j = threadIdx.x; j < L; j += blockDim.x) dst[j] = src[j];
    __syncthreads();                                        // every thread has read st->index
    if (threadIdx.x == 0) {
        const bool terminal = A.done[m] != 0;
        float r = A.reward[m];
        if (A.reward_clip > 0.0f) r = fmaxf(fminf(r, A.reward_clip), -A.reward_clip);
        A.mem.timesteps[row] = st->t;
        A.mem.actions[row] = A.action[m];
        A.mem.rewards[row] = r;
        A.mem.nonterminals[row] = terminal ? 0 : 1;
        float* tree = A.mem.tree + (int64_t)m * (2 * C - 1);
        tree[C - 1 + idx] = st->max;                        // new transitions enter with the running max priority
        rp_propagate(tree, C - 1 + idx);
        const int next = idx + 1 == C ? 0 : idx + 1;
        st->index = next;
        st->full = st->full || next == 0;
        st->t = terminal ? 0 : st->t + 1;
    }
}

// memory.py:163-203 for memory mem_ids[g]: strata i = 0..k-1 of one CTA, batch rows g * k + i.
__global__ void __launch_bounds__(RP_SAMPLE_THREADS) irbpp_replay_sample_kernel(const ReplaySampleArgs A) {
    __shared__ int s_row[RP_SAMPLE_THREADS][2];            // ring slot of the state / of the n-th next state (-1 blank)
    __shared__ int s_wmax;                                  // batch max of the positive weights, as float bits
    const int g = blockIdx.x, tid = threadIdx.x;
    const int m = A.mem_ids[g];
    const bool bad = m < 0 || m >= A.mem.num_memories;
    const int C = A.mem.capacity, L = A.mem.obs_len, n = A.n;
    const float* tree = bad ? nullptr : A.mem.tree + (int64_t)m * (2 * C - 1);
    if (tid == 0) s_wmax = 0;
    int index = 0;
    float total = 0.0f, capf = 0.0f;
    if (!bad) {
        const irbpp_replay_state st = A.mem.state[m];
        index = st.index;
        total = tree[0];
        capf = (float)(st.full ? C : st.index);             // memory.py:200
    }
    const float seg = total / (float)A.k;                   // memory.py:193, float32
    __syncthreads();                                        // s_wmax is cleared before any sample raises it
    for (int base = 0; base < A.k; base += RP_SAMPLE_THREADS) {
        const int i = base + tid;
        int r0 = -1, rn = -1;
        if (i < A.k) {
            const int64_t b = (int64_t)g * A.k + i;
            int code = bad ? IRBPP_REPLAY_ERR_MEMORY : IRBPP_REPLAY_ERR_STARVED;
            int node = -1, tries = 0;
            if (!bad) {
                const float lo = (float)i * seg, hi = (float)(i + 1) * seg;
                for (int a = 0; a < A.attempts; ++a) {
                    const double u = A.uniforms ? A.uniforms[b * A.attempts + a] : rp_uniform(A.seed, A.call, (uint64_t)b, (uint32_t)a);
                    // np.random.uniform(lo, hi) = lo + (hi - lo) * U in float64; the descent then compares and
                    // subtracts in float32 (memory.py:72-79 goes through torch), so the draw is rounded once here
                    float v = (float)((double)lo + ((double)hi - (double)lo) * u);
                    int x = 0;
                    while (2 * x + 1 < 2 * C - 1) {
                        const float left = tree[2 * x + 1];
                        if (v <= left) x = 2 * x + 1;
                        else { v = v - left; x = 2 * x + 2; }
                    }
                    const int idx = x - (C - 1);
                    const int behind = ((index - idx) % C + C) % C, ahead = ((idx - index) % C + C) % C;
                    tries = a + 1;
                    if (behind > n && ahead >= 1 && tree[x] != 0.0f) { node = x; code = 0; break; }
                }
            }
            if (A.out.attempts) A.out.attempts[b] = tries;
            if (A.out.error) A.out.error[b] = code;
            if (code) {
                if (A.error_flags) atomicOr(A.error_flags, 1u << code);
                A.out.tree_idx[b] = -1; A.out.actions[b] = 0; A.out.returns[b] = 0.0f;
                A.out.nonterminals[b] = 0.0f; A.out.weights[b] = 0.0f;
            } else {
                const int idx = node - (C - 1);
                const int64_t ring = (int64_t)m * C;
                // memory.py:115-130: entries idx + t, t = 0..n; after the first fetched terminal everything is blank
                float R = 0.0f, nt = 0.0f;
                bool fetch = true;
                for (int t = 0; t <= n; ++t) {
                    const int slot = (idx + t) % C;
                    float rw = 0.0f;
                    nt = 0.0f;
                    if (fetch) {
                        rw = A.mem.rewards[ring + slot];
                        nt = A.mem.nonterminals[ring + slot] ? 1.0f : 0.0f;
                        if (t == n) rn = slot;
                    }
                    if (t < n) R = R + rw * A.scale[t];     // memory.py:181-182, summed in order
                    fetch = nt != 0.0f;
                }
                r0 = idx;
                const float prob = tree[node];
                const float w = (float)pow((double)(capf * (prob / total)), A.neg_beta);   // memory.py:199-201
                A.out.tree_idx[b] = node;
                A.out.actions[b] = A.mem.actions[ring + idx];
                A.out.returns[b] = R;
                A.out.nonterminals[b] = nt;
                A.out.weights[b] = w;
                atomicMax(&s_wmax, __float_as_int(w));
            }
        }
        s_row[tid][0] = r0; s_row[tid][1] = rn;
        __syncthreads();
        const int cnt = min(RP_SAMPLE_THREADS, A.k - base);
        for (int s = 0; s < cnt; ++s) {                     // the CTA copies state and n-th next state of each sample
            const int64_t b = (int64_t)g * A.k + base + s;
            const int a0 = s_row[s][0], an = s_row[s][1];
            const float* p0 = a0 >= 0 ? A.mem.states + ((int64_t)m * C + a0) * L : nullptr;
            const float* pn = an >= 0 ? A.mem.states + ((int64_t)m * C + an) * L : nullptr;
            float* o0 = A.out.states + b * L;
            float* on = A.out.next_states + b * L;
            for (int j = tid; j < L; j += RP_SAMPLE_THREADS) {
                o0[j] = p0 ? p0[j] : 0.0f;
                on[j] = pn ? pn[j] : 0.0f;
            }
        }
        __syncthreads();
    }
    const float wmax = __int_as_float(s_wmax);
    for (int i = tid; i < A.k; i += RP_SAMPLE_THREADS) {    // memory.py:202: normalised by this memory's batch max
        const int64_t b = (int64_t)g * A.k + i;
        if (A.out.tree_idx[b] >= 0) A.out.weights[b] = A.out.weights[b] / wmax;
    }
}

// memory.py:206-208 for the rows of memory m, in batch order: leaf = float32 priority ** omega, then its ancestors.
__global__ void __launch_bounds__(32 * RP_UPDATE_WARPS) irbpp_replay_update_kernel(const ReplayUpdateArgs A) {
    const int lane = threadIdx.x & 31;
    const int m = blockIdx.x * RP_UPDATE_WARPS + (threadIdx.x >> 5);
    if (m >= A.mem.num_memories) return;                    // whole warps
    const int C = A.mem.capacity;
    float* tree = A.mem.tree + (int64_t)m * (2 * C - 1);
    float mx = A.mem.state[m].max;
    bool touched = false;
    for (int base = 0; base < A.B; base += 32) {
        const int r = base + lane;
        const int mid = r < A.B ? A.mem_ids[r] : -1;
        if (m == 0 && r < A.B && (mid < 0 || mid >= A.mem.num_memories) && A.error_flags)
            atomicOr(A.error_flags, 1u << IRBPP_REPLAY_ERR_INDEX);
        int node = -1;                                      // -1: tree index out of range
        float v = 0.0f;
        if (mid == m) {
            const int64_t raw = A.tree_idxs[r];
            node = raw >= C - 1 && raw < 2 * (int64_t)C - 1 ? (int)raw : -1;
            v = A.loss[r];
        }
        unsigned hit = __ballot_sync(0xffffffffu, mid == m);
        while (hit) {
            const int src = __ffs((int)hit) - 1;
            hit &= hit - 1;
            const int x = __shfl_sync(0xffffffffu, node, src);
            const float loss = __shfl_sync(0xffffffffu, v, src);
            if (lane == 0) {
                const float val = (float)pow((double)loss, A.omega);
                if (x < 0) {
                    if (A.error_flags) atomicOr(A.error_flags, 1u << IRBPP_REPLAY_ERR_INDEX);
                } else {
                    tree[x] = val;
                    rp_propagate(tree, x);
                    mx = mx > val ? mx : val;               // Python max(value, self.max), memory.py:56
                    touched = true;
                }
            }
        }
    }
    if (lane == 0 && touched) A.mem.state[m].max = mx;
}

}  // namespace irbpp
