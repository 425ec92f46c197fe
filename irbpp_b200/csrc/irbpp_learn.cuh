// irbpp_learn.cuh -- the no-grad half of Agent.learn (reference agent.py:94-115): the target mode of the last kernel
// of both network levels (irbpp_actor_rows_kernel, irbpp_order_slots_kernel) reads the double-Q action a* of every
// bin, builds p(s', a*) with the network's own softmax, and projects R + gamma^n z onto the support here.
//
// learn_project restates torch's float32 evaluation of agent.py:100-115 step by step, each operation rounded once
// (explicit __fmul_rn / __fadd_rn / __fsub_rn, nothing contracted into an FMA):
//   Tz = R + (nt * gamma^n) * z           returns.unsqueeze(1) + nonterminals * (discount ** n) * support, left to
//                                         right; the Python float gamma^n enters as float32 (torch's opmath for a
//                                         float32 tensor and a scalar)
//   Tz = min(max(Tz, Vmin), Vmax)         Tensor.clamp
//   b  = (Tz - Vmin) * (1 / dz)           torch's CUDA kernel divides a tensor by a Python scalar as a multiplication by
//                                         the float32 reciprocal (div_true_kernel_cuda, the is_cpu_scalar branch:
//                                         inv_b = opmath_t(1.0) / b); its CPU kernel divides.  The kernel mirrors the
//                                         CUDA behaviour: inv_dz = 1.0f / (float)dz is formed on the host.
//   b  = min(b, atoms - 1)                the one departure from torch: at Tz = Vmax the float32 b can exceed
//                                         atoms - 1 by an ulp (32 atoms on [-1, 8]: 9 * float32(31 / 9) = 31.000002),
//                                         and torch's index_add_ then adds p (b - l) at u = atoms, i.e. into the next
//                                         transition's atom 0 (past the tensor for the last one); here b = atoms - 1
//   l = floor(b), u = ceil(b); l -= 1 where u > 0 and l == u; then u += 1 where l < atoms - 1 and l == u
//   m[l] += p (u - b), then m[u] += p (b - l)
// torch's index_add_ adds with atomics in no fixed order; here lane j sums the l-contributions that land on atom j in
// atom order, then the u-contributions in atom order, starting from 0: the same m for the same p on every run.
#pragma once
#include <stdint.h>

namespace irbpp {

#ifdef IRBPP_HOST_EMULATION
static inline float __fmul_rn(float a, float b) { return a * b; }      // the harness builds with -ffp-contract=off
static inline float __fadd_rn(float a, float b) { return a + b; }
static inline float __fsub_rn(float a, float b) { return a - b; }
#endif

// The target-mode arguments (include/irbpp.h irbpp_dqn_target / irbpp_dqn_order_target).
struct LearnTarget {
    const int64_t* next_actions;       // [N] a* (clamped to the rows / slots of the level)
    const float* returns;              // [N] R
    const float* nonterminals;         // [N] 0 or 1
    float gamma_n, v_min, v_max, inv_dz;   // discount ** n, Vmin, Vmax as float32; 1.0f / (float)dz
    float* m;                          // [N][atoms] projected target distribution
    float* p_next;                     // [N][atoms] p(s', a*) or NULL
};

// Called by one whole warp for bin b, lane = atom: p = p(s', a*)[lane] and sup = z[lane] for lane < atoms (lanes
// >= atoms pass anything; they contribute nothing).  Writes m[b, 0:atoms].
__device__ __forceinline__ void learn_project(const LearnTarget& T, int64_t b, int atoms, float p, float sup, int lane) {
    const float R = T.returns[b], nt = T.nonterminals[b];
    float tz = __fadd_rn(R, __fmul_rn(__fmul_rn(nt, T.gamma_n), sup));
    tz = fminf(fmaxf(tz, T.v_min), T.v_max);
    const float bz = fminf(__fmul_rn(__fsub_rn(tz, T.v_min), T.inv_dz), (float)(atoms - 1));
    int l = (int)floorf(bz), u = (int)ceilf(bz);
    if (u > 0 && l == u) l -= 1;                      // agent.py:108
    if (l < atoms - 1 && l == u) u += 1;              // agent.py:109
    const bool live = lane < atoms;
    const float cl = live ? __fmul_rn(p, __fsub_rn((float)u, bz)) : 0.0f;
    const float cu = live ? __fmul_rn(p, __fsub_rn(bz, (float)l)) : 0.0f;
    float acc = 0.0f;
#pragma unroll 1
    for (int i = 0; i < atoms; ++i) {                 // agent.py:114, atom order
        const int li = __shfl_sync(0xffffffffu, l, i);
        const float ci = __shfl_sync(0xffffffffu, cl, i);
        if (li == lane) acc = __fadd_rn(acc, ci);
    }
#pragma unroll 1
    for (int i = 0; i < atoms; ++i) {                 // agent.py:115, atom order
        const int ui = __shfl_sync(0xffffffffu, u, i);
        const float ci = __shfl_sync(0xffffffffu, cu, i);
        if (ui == lane) acc = __fadd_rn(acc, ci);
    }
    if (live) T.m[b * atoms + lane] = acc;
}

}  // namespace irbpp
