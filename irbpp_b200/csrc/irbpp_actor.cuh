// irbpp_actor.cuh -- the location network's forward pass and Agent.act for every bin (reference model.py:316-352,
// 386-404 with args.bufferSize == 1; agent.py:51-58).
//
// Two kernels per act, one CTA per bin in both:
//   irbpp_actor_bin_kernel   the height encoder (model.py:258-264), the bin's half of project_layer.0 and the list of
//                            the bin's valid rows;
//   irbpp_actor_rows_kernel  the candidate chain over the valid rows only, both row means, the value head, softmax,
//                            expectation over the support, mask and argmax.
// Two reformulations make the work proportional to the valid rows (both exact in real arithmetic):
//   * project_layer.0 is split by the concat order of model.py:339-341 (shape 0:128 | map 128:384 | candidate
//     384:512): W[:, 0:384] . [shape_b; map_b] + b depends on the bin only and is computed once per bin (u_b); per
//     row only W[:, 384:512] . e_c remains.
//   * model.py:347-349 zeroes the embedding of every row with mask != 1, in place, so the advantage stream sees zeros
//     there too: every such row's advantage is a0 = fc_z_a(relu(fc_h_a.bias)) (0 . W + b is exactly b).  Those rows
//     need no GEMM; they enter both means as (sel - n_valid) copies of a0.
// The three wide layers (128->256, 256->128, 128->128) and the two narrower ones (32->128, 128->atoms) run on tensor
// cores as mma.sync m16n8k8 TF32 with the 3xTF32 split (a_hi.b_hi + a_hi.b_lo + a_lo.b_hi, fp32 accumulate), which
// keeps float32-level accuracy; everything else is float32 SIMT with explicit __fmaf_rn (the library is built
// -fmad=false).  Weights stay in global memory (L2-resident across the grid) and are split per fragment.
#pragma once
#include <stdint.h>

#include "irbpp_learn.cuh"

namespace irbpp {

constexpr int AC_THREADS = 256;            // both kernels
constexpr int AC_TM = 64;                  // valid rows per tile of the rows kernel
constexpr int AC_EMB = 128;                // embedding_dim / hidden_size (model.py:276, arguments hidden_size)
constexpr int AC_PROJ = 256;               // project_layer hidden width
constexpr int AC_MAXATOMS = 32;
constexpr int AC_HM = 32;                  // heightmap side (model.py:257)
// activation buffers of the rows kernel (row strides = width + 4: the A-fragment reads of 8 rows x 4 columns hit 32
// distinct banks)
constexpr int AC_LD_P = AC_PROJ + 4;       // buffer P: [AC_TM][260] (inputs, 4->32 output, 128->256 output, fc_h_a output)
constexpr int AC_LD_Q = AC_EMB + 4;        // buffer Q: [AC_TM][132] (32->128 output, embeddings, advantages)
constexpr int AC_ROWS_SMEM_FLOATS = AC_TM * AC_LD_P + AC_TM * AC_LD_Q + AC_PROJ /*u_b*/ + 3 * AC_EMB /*g, value head, a0*/ +
                                    4 * AC_MAXATOMS + AC_TM /*row ids*/ + 2 * 8 /*argmax*/;
constexpr int AC_ROWS_SMEM_BYTES = AC_ROWS_SMEM_FLOATS * (int)sizeof(float);
static_assert(AC_ROWS_SMEM_BYTES * 2 <= 227 * 1024, "two rows CTAs per SM must fit the 227 KB of shared memory");
static_assert(AC_LD_P % 32 == 4 && AC_LD_Q % 32 == 4, "conflict-free A-fragment reads need strides of 4 mod 32");

// Weights in nn.Linear / nn.Conv2d layouts (out x in), float32, device memory (include/irbpp.h irbpp_dqn_weights).
struct ActorWeights {
    const float *conv1_w, *conv1_b, *conv2_w, *conv2_b, *conv3_w, *conv3_b;
    const float *cand1_w, *cand1_b, *cand2_w, *cand2_b, *proj1_w, *proj1_b, *proj2_w, *proj2_b;
    const float *fc_h_v_w, *fc_h_v_b, *fc_z_v_w, *fc_z_v_b, *fc_h_a_w, *fc_h_a_b, *fc_z_a_w, *fc_z_a_b;
    float slope;                       // LeakyReLU negative slope (0.01)
};

struct ActorParams {
    ActorWeights w;
    const float* obs; int64_t obs_stride;       // [N][>= sel*5 + 9 + 1024]
    int32_t N, sel, atoms;
    const float* shape_feature;                 // [N][128]
    const float* support;                       // [atoms]
    const float* mask; int64_t mask_row, mask_elem;   // mask[b*mask_row + r*mask_elem], NULL: no masking
    int64_t* actions;                           // [N]
    float* sum_q;                               // [N][sel] or NULL
    // scratch (actor_scratch_layout)
    float* u;                                   // [N][256]
    int32_t* list;                              // [N][sel] valid rows, ascending
    int32_t* n_valid;                           // [N]
    float* adv;                                 // [N][sel][32] advantages of the valid rows (by row index)
};

__host__ __device__ inline int64_t actor_align(int64_t b) { return (b + 255) & ~(int64_t)255; }
__host__ __device__ inline int64_t actor_scratch_bytes(int64_t N, int64_t sel) {
    return actor_align(N * AC_PROJ * 4) + actor_align(N * sel * 4) + actor_align(N * 4) + actor_align(N * sel * AC_MAXATOMS * 4);
}
__host__ __device__ inline void actor_scratch_layout(ActorParams& A, void* scratch) {
    char* p = static_cast<char*>(scratch);
    const int64_t N = A.N, sel = A.sel;
    A.u = reinterpret_cast<float*>(p); p += actor_align(N * AC_PROJ * 4);
    A.list = reinterpret_cast<int32_t*>(p); p += actor_align(N * sel * 4);
    A.n_valid = reinterpret_cast<int32_t*>(p); p += actor_align(N * 4);
    A.adv = reinterpret_cast<float*>(p);
}

__device__ __forceinline__ float ac_leaky(float v, float slope) { return v > 0.0f ? v : v * slope; }

// ---- tensor-core primitives --------------------------------------------------------------------------------------
// Under the test-only host emulation (tests/host_harness/cuda_emu.h defines IRBPP_HOST_EMULATION) the two PTX
// instructions are restated on the host: cvt.rna rounds as the hardware does, and the mma is a warp collective over
// the emulator's lane exchange in the PTX fragment layouts, so fragment-layout mistakes show up without a GPU.
#ifdef IRBPP_HOST_EMULATION
static inline float __fmaf_rn(float a, float b, float c) { return fmaf(a, b, c); }

// cvt.rna.tf32.f32: round to the 10-bit mantissa of TF32, ties away from zero (float32 layout, 13 low bits cleared)
static inline uint32_t ac_tf32(float x) {
    uint32_t u;
    memcpy(&u, &x, 4);
    if ((u & 0x7f800000u) == 0x7f800000u) return u;            // inf, NaN unchanged
    return (u + 0x1000u) & 0xffffe000u;
}

// mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 (g = lane / 4, t = lane % 4):
//   A 16 x 8: a0 (g, t), a1 (g + 8, t), a2 (g, t + 4), a3 (g + 8, t + 4);  B 8 x 8: b0 (k = t, n = g), b1 (k = t + 4, n = g);
//   C 16 x 8: c0 (g, 2t), c1 (g, 2t + 1), c2 (g + 8, 2t), c3 (g + 8, 2t + 1).
// Operands are read as TF32 (the 13 low bits ignored); the products are exact in float32 and are accumulated in
// float32 in k order.
static inline void ac_mma(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
    uint64_t x01[32], x23[32], xb[32];
    cuda_emu::exchange((uint64_t)a[0] | ((uint64_t)a[1] << 32), x01);
    cuda_emu::exchange((uint64_t)a[2] | ((uint64_t)a[3] << 32), x23);
    cuda_emu::exchange((uint64_t)b[0] | ((uint64_t)b[1] << 32), xb);
    auto f = [](uint32_t u) { u &= 0xffffe000u; float v; memcpy(&v, &u, 4); return v; };
    float A[16][8], B[8][8];
    for (int l = 0; l < 32; ++l) {
        const int g = l >> 2, t = l & 3;
        A[g][t] = f((uint32_t)x01[l]); A[g + 8][t] = f((uint32_t)(x01[l] >> 32));
        A[g][t + 4] = f((uint32_t)x23[l]); A[g + 8][t + 4] = f((uint32_t)(x23[l] >> 32));
        B[t][g] = f((uint32_t)xb[l]); B[t + 4][g] = f((uint32_t)(xb[l] >> 32));
    }
    const int g = cuda_emu::lane() >> 2, t = cuda_emu::lane() & 3;
    for (int h = 0; h < 4; ++h) {
        const int r = g + (h >> 1) * 8, n = 2 * t + (h & 1);
        float s = c[h];
        for (int k = 0; k < 8; ++k) s += A[r][k] * B[k][n];
        c[h] = s;
    }
}
#else
__device__ __forceinline__ uint32_t ac_tf32(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ void ac_mma(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
#endif

// x = hi + lo with hi, lo TF32 values (lo carries the bits hi drops)
__device__ __forceinline__ void ac_split(float x, uint32_t& hi, uint32_t& lo) {
    hi = ac_tf32(x);
    lo = ac_tf32(x - __int_as_float((int)hi));
}

constexpr int ACT_NONE = 0, ACT_LEAKY = 1, ACT_RELU = 2;

// out[r][n] = act(sum_k in[r][k] * W[n][k] + bias[n]) for the AC_TM rows of a tile, n < N (columns n >= n_out read
// zero weights and are stored as zero).  8 warps as WM x (8 / WM); each warp owns MT m-tiles x NT n-tiles of 16 x 8.
template <int K, int N, int WM, int ACT>
__device__ __forceinline__ void ac_layer(const float* in, int ld_in, const float* __restrict__ W, int ldw, int n_out,
                                         const float* bias, float* out, int ld_out, float slope) {
    constexpr int WN = 8 / WM, MT = AC_TM / 16 / WM, NT = N / 8 / WN;
    static_assert(MT * WM * 16 == AC_TM && NT * WN * 8 == N && K % 8 == 0, "tile split");
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const int row0 = (warp / WN) * MT * 16, col0 = (warp % WN) * NT * 8;
    float acc[MT][NT][4];
#pragma unroll
    for (int i = 0; i < MT; ++i)
#pragma unroll
        for (int j = 0; j < NT; ++j) acc[i][j][0] = acc[i][j][1] = acc[i][j][2] = acc[i][j][3] = 0.0f;
#pragma unroll 1
    for (int k0 = 0; k0 < K; k0 += 8) {
        uint32_t ah[MT][4], al[MT][4];
#pragma unroll
        for (int i = 0; i < MT; ++i) {
            const float* p = in + (row0 + i * 16 + g) * ld_in + k0 + t;
            ac_split(p[0], ah[i][0], al[i][0]);
            ac_split(p[8 * ld_in], ah[i][1], al[i][1]);
            ac_split(p[4], ah[i][2], al[i][2]);
            ac_split(p[8 * ld_in + 4], ah[i][3], al[i][3]);
        }
#pragma unroll
        for (int j = 0; j < NT; ++j) {
            const int n = col0 + j * 8 + g;
            float w0 = 0.0f, w1 = 0.0f;
            if (n < n_out) { w0 = W[(int64_t)n * ldw + k0 + t]; w1 = W[(int64_t)n * ldw + k0 + t + 4]; }
            uint32_t bh[2], bl[2];
            ac_split(w0, bh[0], bl[0]);
            ac_split(w1, bh[1], bl[1]);
#pragma unroll
            for (int i = 0; i < MT; ++i) {      // small products first, then the big one
                ac_mma(acc[i][j], al[i], bh);
                ac_mma(acc[i][j], ah[i], bl);
                ac_mma(acc[i][j], ah[i], bh);
            }
        }
    }
#pragma unroll
    for (int i = 0; i < MT; ++i)
#pragma unroll
        for (int j = 0; j < NT; ++j)
#pragma unroll
            for (int h = 0; h < 4; ++h) {
                const int r = row0 + i * 16 + g + (h >> 1) * 8, n = col0 + j * 8 + 2 * t + (h & 1);
                float v = 0.0f;
                if (n < n_out) {
                    v = acc[i][j][h] + bias[n];
                    if (ACT == ACT_LEAKY) v = ac_leaky(v, slope);
                    if (ACT == ACT_RELU) v = v > 0.0f ? v : 0.0f;
                }
                out[r * ld_out + n] = v;
            }
}

// ---- heightEncoder ---------------------------------------------------------------------------------------------------
// heightEncoder (model.py:258-264, LeakyReLU after every conv) of the 32 x 32 heightmap the CTA's threads have stored
// in hm (the barrier is here), by the AC_THREADS threads of a CTA; the 256 map features, flattened in C, H, W order,
// go to map[0:256].  hm, c1 and c2 are the CTA's shared buffers.  Shared by the location and order levels (W:
// ActorWeights or OrderWeights, same conv fields).
template <class W>
__device__ __forceinline__ void ac_height_encoder(const W& w, float* hm, float* c1, float* c2, float* map) {
    const int tid = threadIdx.x;
    const float slope = w.slope;
    __syncthreads();
    // conv1: 1 -> 16, k4, stride 2, pad 1: 32 -> 16
    for (int o = tid; o < 16 * 16 * 16; o += AC_THREADS) {
        const int co = o >> 8, y = (o >> 4) & 15, xx = o & 15;
        float acc = w.conv1_b[co];
        const float* wk = w.conv1_w + co * 16;
        for (int ky = 0; ky < 4; ++ky) {
            const int iy = 2 * y - 1 + ky;
            if (iy < 0 || iy >= AC_HM) continue;
            for (int kx = 0; kx < 4; ++kx) {
                const int ix = 2 * xx - 1 + kx;
                if (ix < 0 || ix >= AC_HM) continue;
                acc = __fmaf_rn(hm[iy * AC_HM + ix], wk[ky * 4 + kx], acc);
            }
        }
        c1[o] = ac_leaky(acc, slope);
    }
    __syncthreads();
    // conv2: 16 -> 32, k4, stride 2, pad 1: 16 -> 8
    for (int o = tid; o < 32 * 8 * 8; o += AC_THREADS) {
        const int co = o >> 6, y = (o >> 3) & 7, xx = o & 7;
        float acc = w.conv2_b[co];
        for (int ci = 0; ci < 16; ++ci) {
            const float* wk = w.conv2_w + (co * 16 + ci) * 16;
            const float* in = c1 + ci * 256;
            for (int ky = 0; ky < 4; ++ky) {
                const int iy = 2 * y - 1 + ky;
                if (iy < 0 || iy >= 16) continue;
                for (int kx = 0; kx < 4; ++kx) {
                    const int ix = 2 * xx - 1 + kx;
                    if (ix < 0 || ix >= 16) continue;
                    acc = __fmaf_rn(in[iy * 16 + ix], wk[ky * 4 + kx], acc);
                }
            }
        }
        c2[o] = ac_leaky(acc, slope);
    }
    __syncthreads();
    // conv3: 32 -> 4, k3, stride 1, pad 1: 8 -> 8; flattened (C, H, W)
    {
        const int o = tid, co = o >> 6, y = (o >> 3) & 7, xx = o & 7;
        float acc = w.conv3_b[co];
        for (int ci = 0; ci < 32; ++ci) {
            const float* wk = w.conv3_w + (co * 32 + ci) * 9;
            const float* in = c2 + ci * 64;
            for (int ky = 0; ky < 3; ++ky) {
                const int iy = y - 1 + ky;
                if (iy < 0 || iy >= 8) continue;
                for (int kx = 0; kx < 3; ++kx) {
                    const int ix = xx - 1 + kx;
                    if (ix < 0 || ix >= 8) continue;
                    acc = __fmaf_rn(in[iy * 8 + ix], wk[ky * 3 + kx], acc);
                }
            }
        }
        map[o] = ac_leaky(acc, slope);
    }
    __syncthreads();
}

// ---- per-bin kernel ------------------------------------------------------------------------------------------------
// One CTA per bin: heightEncoder, u_b and the list of rows with mask == 1 (model.py:321-322, 347-349: every other
// row's embedding is zeroed).
__global__ void __launch_bounds__(AC_THREADS) irbpp_actor_bin_kernel(const ActorParams A) {
    __shared__ __align__(16) float hm[AC_HM * AC_HM];          // [1][32][32]
    __shared__ __align__(16) float c1[16 * 16 * 16];            // [16][16][16]
    __shared__ __align__(16) float c2[32 * 8 * 8];              // [32][8][8]
    __shared__ __align__(16) float x[384];                      // shape_feature | map_feature
    const int b = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const float* ob = A.obs + (int64_t)b * A.obs_stride;
    const float* hsrc = ob + (int64_t)A.sel * 5 + 9;            // model.py:181
    for (int i = tid; i < AC_HM * AC_HM; i += AC_THREADS) hm[i] = hsrc[i];
    if (tid < AC_EMB) x[tid] = A.shape_feature[(int64_t)b * AC_EMB + tid];
    ac_height_encoder(A.w, hm, c1, c2, x + AC_EMB);
    // u_b = proj1_w[:, 0:384] . x + proj1_b: one warp per output, lanes over k (coalesced rows of the weight)
    for (int j = warp; j < AC_PROJ; j += AC_THREADS / 32) {
        const float* wr = A.w.proj1_w + (int64_t)j * 512;
        float acc = 0.0f;
        for (int k = lane; k < 384; k += 32) acc = __fmaf_rn(wr[k], x[k], acc);
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, s);
        if (lane == 0) A.u[(int64_t)b * AC_PROJ + j] = acc + A.w.proj1_b[j];
    }
    // the valid rows in ascending order (warp 0, ballot compaction)
    if (warp == 0) {
        int n = 0;
        int32_t* list = A.list + (int64_t)b * A.sel;
        for (int r0 = 0; r0 < A.sel; r0 += 32) {
            const int r = r0 + lane;
            const bool v = r < A.sel && ob[(int64_t)r * 5 + 4] == 1.0f;
            const unsigned bal = __ballot_sync(0xffffffffu, v);
            if (v) list[n + __popc(bal & ((1u << lane) - 1u))] = r;
            n += __popc(bal);
        }
        if (lane == 0) A.n_valid[b] = n;
    }
}

// ---- rows kernel -------------------------------------------------------------------------------------------------
// One CTA per bin (both means are over the bin's rows).  Tiles of AC_TM valid rows run
//   [rot, x, y, H] -> 32 (LeakyReLU) -> 128 -> (+ u_b) 256 (LeakyReLU) -> 128 = embedding (summed for g)
//   -> fc_h_a 128 (ReLU) -> fc_z_a atoms = advantages (stored by row index in the scratch, summed for mean(a)),
// then the final phase: value head on g = sum / sel, mean(a) = (sum_valid a + (sel - n_valid) a0) / sel,
// q = v + a - mean(a) (a0 for invalid rows), softmax over the atoms, expectation over the support, mask, argmax.
// TARGET (irbpp_actor_target_kernel): the final phase instead builds p = softmax(q) of row a* = T.next_actions[b] only
// and projects it (learn_project); no expectation, argmax or sum_q.
template <bool TARGET>
__device__ __forceinline__ void actor_rows(const ActorParams A, const LearnTarget& T) {
    extern __shared__ __align__(16) float ac_smem[];
    float* P = ac_smem;                               // [AC_TM][AC_LD_P]
    float* Q = P + AC_TM * AC_LD_P;                   // [AC_TM][AC_LD_Q]
    float* u = Q + AC_TM * AC_LD_Q;                   // [256] u_b
    float* gv = u + AC_PROJ;                          // [128] g
    float* hv = gv + AC_EMB;                          // [128] relu(fc_h_v(g))
    float* ha = hv + AC_EMB;                          // [128] relu(fc_h_a.bias)
    float* v = ha + AC_EMB;                           // [32] value logits
    float* a0 = v + AC_MAXATOMS;                      // [32] advantage of an invalid row
    float* asum = a0 + AC_MAXATOMS;                   // [32] sum of the valid rows' advantages
    float* base = asum + AC_MAXATOMS;                 // [32] mean(a)
    int32_t* rows = reinterpret_cast<int32_t*>(base + AC_MAXATOMS);  // [AC_TM]
    float* wbest = reinterpret_cast<float*>(rows + AC_TM);           // [8]
    int32_t* wbidx = reinterpret_cast<int32_t*>(wbest + 8);          // [8]
    const int b = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int sel = A.sel, atoms = A.atoms;
    const float slope = A.w.slope;
    const float* ob = A.obs + (int64_t)b * A.obs_stride;
    const int nv = A.n_valid[b];
    const int32_t* list = A.list + (int64_t)b * sel;
    float* adv = A.adv + (int64_t)b * sel * AC_MAXATOMS;
    u[tid] = A.u[(int64_t)b * AC_PROJ + tid];
    float gacc = 0.0f, aacc = 0.0f;                   // thread c < 128: column sum of the embeddings; c < 32: of a
    for (int j0 = 0; j0 < nv; j0 += AC_TM) {
        const int nr = min(AC_TM, nv - j0);
        __syncthreads();                              // the previous tile's readers of P, Q and rows are done
        if (tid < AC_TM) rows[tid] = tid < nr ? list[j0 + tid] : -1;
        __syncthreads();
        // init_candidate_embed.0: 4 -> 32, LeakyReLU (SIMT) into P[:, 0:32]
        for (int o = tid; o < AC_TM * 32; o += AC_THREADS) {
            const int i = o >> 5, c = o & 31, r = rows[i];
            float acc = 0.0f;
            if (r >= 0) {
                const float* cr = ob + (int64_t)r * 5;
                const float* wr = A.w.cand1_w + c * 4;
                acc = A.w.cand1_b[c];
                acc = __fmaf_rn(cr[0], wr[0], acc);
                acc = __fmaf_rn(cr[1], wr[1], acc);
                acc = __fmaf_rn(cr[2], wr[2], acc);
                acc = __fmaf_rn(cr[3], wr[3], acc);
                acc = ac_leaky(acc, slope);
            }
            P[i * AC_LD_P + c] = acc;
        }
        __syncthreads();
        ac_layer<32, 128, 2, ACT_NONE>(P, AC_LD_P, A.w.cand2_w, 32, 128, A.w.cand2_b, Q, AC_LD_Q, slope);      // init_candidate_embed.2
        __syncthreads();
        ac_layer<128, 256, 2, ACT_LEAKY>(Q, AC_LD_Q, A.w.proj1_w + 384, 512, 256, u, P, AC_LD_P, slope);     // project_layer.0 (row part)
        __syncthreads();
        ac_layer<256, 128, 2, ACT_NONE>(P, AC_LD_P, A.w.proj2_w, 256, 128, A.w.proj2_b, Q, AC_LD_Q, slope);    // project_layer.2
        __syncthreads();
        if (tid < AC_EMB)
            for (int i = 0; i < nr; ++i) gacc += Q[i * AC_LD_Q + tid];
        ac_layer<128, 128, 2, ACT_RELU>(Q, AC_LD_Q, A.w.fc_h_a_w, 128, 128, A.w.fc_h_a_b, P, AC_LD_P, slope);  // fc_h_a
        __syncthreads();
        ac_layer<128, 32, 4, ACT_NONE>(P, AC_LD_P, A.w.fc_z_a_w, 128, atoms, A.w.fc_z_a_b, Q, AC_LD_Q, slope); // fc_z_a
        __syncthreads();
        if (tid < AC_MAXATOMS)
            for (int i = 0; i < nr; ++i) aacc += Q[i * AC_LD_Q + tid];
        for (int o = tid; o < nr * AC_MAXATOMS; o += AC_THREADS) {
            const int i = o >> 5, z = o & 31;
            adv[(int64_t)rows[i] * AC_MAXATOMS + z] = Q[i * AC_LD_Q + z];
        }
    }
    // ---- final phase ----
    if (tid < AC_EMB) {
        gv[tid] = gacc / (float)sel;                              // mean over all sel rows, zeros included (model.py:350)
        const float hb = A.w.fc_h_a_b[tid];
        ha[tid] = hb > 0.0f ? hb : 0.0f;                          // fc_h_a of a zeroed embedding is exactly its bias
    }
    if (tid < AC_MAXATOMS) asum[tid] = aacc;
    __syncthreads();
    if (tid < AC_EMB) {                                           // fc_h_v, ReLU
        const float* wr = A.w.fc_h_v_w + tid * AC_EMB;
        float acc = 0.0f;
        for (int k = 0; k < AC_EMB; ++k) acc = __fmaf_rn(wr[k], gv[k], acc);
        acc += A.w.fc_h_v_b[tid];
        hv[tid] = acc > 0.0f ? acc : 0.0f;
    }
    __syncthreads();
    if (tid < 2 * AC_MAXATOMS) {                                  // fc_z_v (threads 0-31), a0 = fc_z_a(relu(fc_h_a.bias)) (32-63)
        const int z = tid & 31;
        const bool val = tid < AC_MAXATOMS;
        float acc = 0.0f;
        if (z < atoms) {
            const float* wr = (val ? A.w.fc_z_v_w : A.w.fc_z_a_w) + z * AC_EMB;
            const float* in = val ? hv : ha;
            for (int k = 0; k < AC_EMB; ++k) acc = __fmaf_rn(wr[k], in[k], acc);
            acc += (val ? A.w.fc_z_v_b : A.w.fc_z_a_b)[z];
        }
        (val ? v : a0)[z] = acc;
    }
    __syncthreads();
    if (tid < AC_MAXATOMS) base[tid] = (asum[tid] + (float)(sel - nv) * a0[tid]) / (float)sel;   // mean(a) over all rows
    __syncthreads();
    if constexpr (TARGET) {                                                 // warp 0, lane = atom, row a*
        if (warp != 0) return;
        int64_t r = T.next_actions[b];
        r = r < 0 ? 0 : (r >= sel ? sel - 1 : r);
        const bool valid = ob[r * 5 + 4] == 1.0f;
        const float az = valid ? adv[r * AC_MAXATOMS + lane] : a0[lane];
        const float qz = lane < atoms ? (v[lane] + az) - base[lane] : -INFINITY;
        float m = qz;
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, s));
        const float e = lane < atoms ? expf(qz - m) : 0.0f;
        float se = e;
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) se += __shfl_xor_sync(0xffffffffu, se, s);
        const float p = e / se;
        if (T.p_next && lane < atoms) T.p_next[(int64_t)b * atoms + lane] = p;
        learn_project(T, b, atoms, p, lane < atoms ? A.support[lane] : 0.0f, lane);
        return;
    }
    // one warp per row, lane = atom
    const float sup = lane < atoms ? A.support[lane] : 0.0f;
    const float vz = v[lane], mz = base[lane], a0z = a0[lane];      // lanes >= atoms hold zeros
    float best = -INFINITY;
    int bidx = 0x7fffffff;
    for (int r = warp; r < sel; r += AC_THREADS / 32) {
        const bool valid = ob[(int64_t)r * 5 + 4] == 1.0f;
        const float az = valid ? adv[(int64_t)r * AC_MAXATOMS + lane] : a0z;
        const float qz = lane < atoms ? (vz + az) - mz : -INFINITY;
        float m = qz;
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, s));
        const float e = lane < atoms ? expf(qz - m) : 0.0f;
        float se = e;
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) se += __shfl_xor_sync(0xffffffffu, se, s);
        float sq = (e / se) * sup;
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, s);
        if (A.mask && A.mask[(int64_t)b * A.mask_row + (int64_t)r * A.mask_elem] != 1.0f) sq = -INFINITY;   // agent.py:56-57
        if (lane == 0 && A.sum_q) A.sum_q[(int64_t)b * sel + r] = sq;
        if (sq > best || (sq == best && r < bidx)) { best = sq; bidx = r; }
    }
    if (lane == 0) { wbest[warp] = best; wbidx[warp] = bidx; }
    __syncthreads();
    if (tid == 0) {                                               // torch.argmax: the first index of the maximum
        float bb = wbest[0];
        int bi = wbidx[0];
        for (int w = 1; w < AC_THREADS / 32; ++w)
            if (wbest[w] > bb || (wbest[w] == bb && wbidx[w] < bi)) { bb = wbest[w]; bi = wbidx[w]; }
        A.actions[b] = bi < sel ? bi : 0;
    }
}

__global__ void __launch_bounds__(AC_THREADS, 2) irbpp_actor_rows_kernel(const ActorParams A) {
    actor_rows<false>(A, LearnTarget{});
}

// Agent.learn's target pass (agent.py:94-115) over the target net: irbpp_dqn_target
__global__ void __launch_bounds__(AC_THREADS, 2) irbpp_actor_target_kernel(const ActorParams A, const LearnTarget T) {
    actor_rows<true>(A, T);
}

}  // namespace irbpp
