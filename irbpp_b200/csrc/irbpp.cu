// irbpp.cu -- C-ABI (include/irbpp.h) host side: state ownership, table preprocessing, launches.
//
// No CPU fallback lives here: every entry point that computes anything launches the CUDA kernels of
// irbpp_kernels.cuh (irbpp_scan_kernel or irbpp_scan_warp_kernel -> irbpp_candidates_kernel).
#include <cuda_runtime.h>
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <functional>
#include <map>
#include <mutex>
#include <cmath>
#include <string>
#include <vector>

#include "../../include/irbpp.h"
#include "irbpp_kernels.cuh"
#include "irbpp_pointnet.cuh"
#include "irbpp_pack.cuh"
#include "irbpp_replay.cuh"
#include "irbpp_actor.cuh"
#include "irbpp_order_actor.cuh"
#include "irbpp_grad.cuh"
#include "irbpp_height_encoder.cuh"
#include "irbpp_order_grad.cuh"

using namespace irbpp;

static thread_local std::string g_create_error;     // error of the calling thread's last failed irbpp_create

struct irbpp_env {
    irbpp_config cfg;
    Params P;                      // device pointers + configuration (mode/inputs filled per launch)
    int scan_smem = 0;
    int scan_warp_smem = 0;        // > 0: the online step scans with irbpp_scan_warp_kernel (block-form library, 16x16 grid)
    uint32_t* ready_dev = nullptr;       // scan -> candidates hand-over flags (one per unit)
    uint32_t epoch = 0;                  // launch counter behind the flags
    int epc = ENVS_PER_CTA_NARROW;       // bins per CTA of the candidates kernel (envs_per_cta_for(R))
    int step = 2;                        // stepSize of the action grid (Grid<step>): 2 -> 16x16 actions, 1 -> 32x32
    int npose = Grid<2>::NPOSE;          // poses per rotation of that grid
    std::string err;
    bool shapes_loaded = false, sequences_set = false, was_reset = false, waiting_step = false;
    bool scan_current = false;        // the scan scratch holds the drop heights of every bin's cur_item
    int32_t* heur_pose_dev = nullptr; int64_t* heur_index_dev = nullptr;
    bool results_on_host = false;           // the pending step wrote its results straight to the host mirror
    cudaStream_t pending_stream = nullptr;
    int64_t launches = 0;
    // device allocations
    std::vector<void*> dev_allocs;
    void* results_dev = nullptr;   // the device result block (step_results)
    // two pinned host blocks, mapped: the steps with host actions alternate between them, so the views of step k stay
    // valid until step k + 2 is launched
    void* results_host[2] = {nullptr, nullptr};
    void* results_mapped[2] = {nullptr, nullptr};   // device addresses of results_host[]
    int res_turn = 0;                               // block of the current step
    int64_t* actions_dev = nullptr;
    int64_t* actions_pinned = nullptr;      // [2][N] pinned staging: step actions, order actions
    uint8_t* which_dev = nullptr;
    // shape pools
    ShapeRot* srot_dev = nullptr; double* Bs_dev = nullptr; double* Ts_dev = nullptr;
    double* vol_dev = nullptr; double* rew_dev = nullptr; int32_t* seq_dev = nullptr;
    int32_t* grp_off_dev = nullptr; int32_t* grp_mem_dev = nullptr;
    int32_t* traj_items_dev = nullptr; int64_t* traj_off_dev = nullptr;
    TileEntry* tiles_dev = nullptr;
    unsigned long long* phase_dev = nullptr;
};

// Every entry point runs on its handle's device and leaves the calling thread's current device as it found it: the
// host framework (torch) tracks the current device itself, and a library that changes it behind its back makes the
// caller's next `tensor.cuda()` land on another GPU (seen in a two-device test before this guard existed).
struct DeviceGuard {
    int prev = -1, cur = -1;
    explicit DeviceGuard(int dev) : cur(dev) {
        if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
        if (prev != dev) cudaSetDevice(dev);
    }
    ~DeviceGuard() { if (prev >= 0 && prev != cur) cudaSetDevice(prev); }
};

// device that owns a device pointer (the handle-free entry points run where their buffers live)
static int device_of(const void* p) {
#ifdef IRBPP_HOST_EMULATION
    (void)p; return 0;
#else
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) == cudaSuccess && at.type == cudaMemoryTypeDevice) return at.device;
    cudaGetLastError();
    int d = 0; cudaGetDevice(&d); return d;
#endif
}

static int fail(irbpp_env* h, int code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    if (h) h->err = buf; else g_create_error = buf;
    return code;
}

// The result block of N bins: ratio | ep_reward | reward | counter | ep_len | done | valid | error.  These two
// functions are the only place that knows its order and sizes.
static size_t step_results_bytes(size_t N) {
    return N * (2 * sizeof(double) + sizeof(float) + 2 * sizeof(int32_t) + 3 * sizeof(uint8_t));
}

static StepResults step_results(void* base, size_t N) {
    char* b = static_cast<char*>(base);
    StepResults r;
    r.ratio = reinterpret_cast<double*>(b); b += N * sizeof(double);
    r.ep_reward = reinterpret_cast<double*>(b); b += N * sizeof(double);
    r.reward = reinterpret_cast<float*>(b); b += N * sizeof(float);
    r.counter = reinterpret_cast<int32_t*>(b); b += N * sizeof(int32_t);
    r.ep_len = reinterpret_cast<int32_t*>(b); b += N * sizeof(int32_t);
    r.done = reinterpret_cast<uint8_t*>(b); b += N;
    r.valid = reinterpret_cast<uint8_t*>(b); b += N;
    r.error = reinterpret_cast<uint8_t*>(b);
    return r;
}

static void public_results(const StepResults& r, irbpp_step_result* out) {
    out->reward = r.reward; out->done = r.done; out->valid = r.valid; out->error = r.error;
    out->counter = r.counter; out->ep_len = r.ep_len; out->ratio = r.ratio; out->ep_reward = r.ep_reward;
}

// IRBPP_EDEVICE naming the first bin whose error code (host memory) is set
static int first_device_error(irbpp_env* h, const uint8_t* error) {
    for (int i = 0; i < h->P.N; ++i)
        if (error[i]) return fail(h, IRBPP_EDEVICE, "env %d reported device error code %d", i, (int)error[i]);
    return IRBPP_OK;
}

#define CUDA_TRY(h, expr)                                                                         \
    do {                                                                                          \
        cudaError_t e_ = (expr);                                                                  \
        if (e_ != cudaSuccess)                                                                    \
            return fail(h, IRBPP_ECUDA, "%s failed: %s", #expr, cudaGetErrorString(e_));          \
    } while (0)

template <class T>
static cudaError_t dev_alloc(irbpp_env* h, T** p, size_t count, bool zero = true) {
    void* q = nullptr;
    cudaError_t e = cudaMalloc(&q, count * sizeof(T) + 16);
    if (e != cudaSuccess) return e;
    if (zero) { e = cudaMemset(q, 0, count * sizeof(T) + 16); if (e != cudaSuccess) return e; }
    h->dev_allocs.push_back(q);
    *p = reinterpret_cast<T*>(q);
    return cudaSuccess;
}


static void free_dev(irbpp_env* h, void* p) {
    if (!p) return;
    auto it = std::find(h->dev_allocs.begin(), h->dev_allocs.end(), p);
    if (it != h->dev_allocs.end()) h->dev_allocs.erase(it);
    cudaFree(p);
}

// The kernels of a configuration: the action grid (stepSize `step`), `epc` bins per candidates CTA (envs_per_cta_for(R)),
// `traj`: the trajectory item source, and the candidates kernel's dynamic shared memory at R rotations.
struct StepKernels {
    void (*scan)(const Params);
    void (*scan_warp)(const Params);     // one warp per bin: online step of a block-form library (16x16 grid only, else null)
    void (*cand)(const Params);
    void (*levels)(const Params);
    void (*heur)(const Params);
    int cand_smem;
};

template <int EPC, class G>
static StepKernels step_kernels_epc(bool traj, int R) {
    void (*scan_warp)(const Params) = nullptr;
    if constexpr (G::STEP == 2) scan_warp = traj ? irbpp_scan_warp_kernel<true> : irbpp_scan_warp_kernel<false>;
    return {traj ? irbpp_scan_kernel<G, true> : irbpp_scan_kernel<G, false>, scan_warp,
            traj ? irbpp_candidates_kernel<EPC, G, true> : irbpp_candidates_kernel<EPC, G, false>,
            irbpp_levels_kernel<G>, irbpp_heuristic_kernel<G>, cand_smem_bytes<EPC, G>(R)};
}

template <class G>
static StepKernels step_kernels_grid(int epc, bool traj, int R) {
    return epc == ENVS_PER_CTA_WIDE ? step_kernels_epc<ENVS_PER_CTA_WIDE, G>(traj, R) : step_kernels_epc<ENVS_PER_CTA_NARROW, G>(traj, R);
}

static StepKernels step_kernels(int step, int epc, bool traj, int R) {
    return step == 1 ? step_kernels_grid<Grid<1>>(epc, traj, R) : step_kernels_grid<Grid<2>>(epc, traj, R);
}

// scratch sizes of the grid of stepSize `step`
static int grid_list_cap_ws(int step) { return step == 1 ? CandScratch<Grid<1>>::LIST_CAP_WS : CandScratch<Grid<2>>::LIST_CAP_WS; }

// cudaFuncAttributeMaxDynamicSharedMemorySize is a per-function, PER-DEVICE attribute: the largest value any
// handle needed is tracked per (device, kernel) and only ever raised (several handles may coexist on a device,
// and one process may hold handles on several devices).
static cudaError_t raise_dynamic_smem(int device, const void* kernel, int bytes) {
    static std::map<std::pair<int, const void*>, int> raised;
    static std::mutex mu;
    std::lock_guard<std::mutex> lk(mu);
    int& done = raised[{device, kernel}];
    if (bytes <= done) return cudaSuccess;
    const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e == cudaSuccess) done = bytes;
    return e;
}

extern "C" {

int irbpp_abi_version(void) { return IRBPP_ABI_VERSION; }

const char* irbpp_last_error(irbpp_handle h) { return h ? h->err.c_str() : g_create_error.c_str(); }

int irbpp_create(const irbpp_config* cfg, irbpp_handle* out) {
    if (!cfg || !out) return fail(nullptr, IRBPP_EINVAL, "null argument");
    *out = nullptr;
    if (cfg->num_envs <= 0) return fail(nullptr, IRBPP_EINVAL, "num_envs must be positive");
    if (cfg->num_rotations < 1 || cfg->num_rotations > 32)
        return fail(nullptr, IRBPP_EINVAL, "num_rotations must be in [1, 32]");
    if (cfg->buffer_size < 1 || cfg->buffer_size > MAX_QUEUE)
        return fail(nullptr, IRBPP_EINVAL, "buffer_size must be in [1, %d]", MAX_QUEUE);
    if (cfg->selected_action < 1 || cfg->selected_action > 4096)
        return fail(nullptr, IRBPP_EINVAL, "selected_action must be in [1, 4096]");
    // grid sizes exactly as Space.__init__ computes them (space.py:19-24); supported: the 32x32 heightmap with step 2
    // (16x16 actions) or step 1 (32x32 actions)
    const double stepf = cfg->resolution_act / cfg->resolution_h;
    const int step = (int)stepf;
    const int hx = (int)ceil(cfg->bin_dimension[0] / cfg->resolution_h), hy = (int)ceil(cfg->bin_dimension[1] / cfg->resolution_h);
    const int ax = (int)ceil(cfg->bin_dimension[0] / cfg->resolution_act), ay = (int)ceil(cfg->bin_dimension[1] / cfg->resolution_act);
    const bool grid2 = step == Grid<2>::STEP && ax == Grid<2>::AX && ay == Grid<2>::AY;
    const bool grid1 = step == Grid<1>::STEP && ax == Grid<1>::AX && ay == Grid<1>::AY;
    if ((double)step != stepf || hx != HX || hy != HY || !(grid2 || grid1))
        return fail(nullptr, IRBPP_EINVAL,
                    "unsupported grid: heightmap %dx%d, actions %dx%d, step %g (supported: heightmap %dx%d with actions %dx%d, "
                    "step %d, or actions %dx%d, step %d)",
                    hx, hy, ax, ay, stepf, HX, HY, Grid<2>::AX, Grid<2>::AY, Grid<2>::STEP, Grid<1>::AX, Grid<1>::AY, Grid<1>::STEP);
    const int npose = ax * ay;
    if (cfg->selected_action > cfg->num_rotations * npose)
        return fail(nullptr, IRBPP_EINVAL, "selected_action exceeds the number of poses (reference fallback "
                                           "binPhy.py:217-225 would return a short table)");
    if (!(cfg->resolution_z > 0) || ceil(cfg->bin_dimension[2] / cfg->resolution_z) + 1 >= LEVEL_OFFSET)
        return fail(nullptr, IRBPP_EINVAL, "bin height / resolution_z must stay below %d levels", LEVEL_OFFSET - 1);

    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        return fail(nullptr, IRBPP_ECUDA, "no CUDA device (%s); this library has no CPU path",
                    e == cudaSuccess ? "count 0" : cudaGetErrorString(e));
    if (cfg->device < 0 || cfg->device >= ndev) return fail(nullptr, IRBPP_EINVAL, "bad device ordinal %d", cfg->device);
    DeviceGuard guard(cfg->device);
    {
        int now = -1;
        if (cudaGetDevice(&now) != cudaSuccess || now != cfg->device) return fail(nullptr, IRBPP_ECUDA, "cudaSetDevice(%d) failed", cfg->device);
    }

    irbpp_env* h = new irbpp_env();
    h->cfg = *cfg;
    Params& P = h->P;
    memset(&P, 0, sizeof(P));
    const int N = cfg->num_envs;
    P.N = N; P.R = cfg->num_rotations; P.sel = cfg->selected_action; P.K = cfg->buffer_size;
    P.loc_len = P.sel * 5 + 9 + HX * HY;
    P.order_len = P.K + HX * HY;
    P.obs_stride = (P.K > 1) ? P.order_len : P.loc_len;
    P.legacy = cfg->approx_legacy;
    P.binz = cfg->bin_dimension[2];
    P.resZ = cfg->resolution_z;
    P.resA = cfg->resolution_act;
    P.binvol = (cfg->bin_dimension[0] * cfg->bin_dimension[1]) * cfg->bin_dimension[2];   // np.prod
    h->epc = envs_per_cta_for(P.R);                  // bins (= warps) per CTA of the candidates kernel
    h->step = step; h->npose = npose;
    const int bmw = npose / 32;

#define TRY_ALLOC(expr)                                                                          \
    do { cudaError_t e2_ = (expr); if (e2_ != cudaSuccess) {                                      \
        fail(nullptr, IRBPP_ECUDA, "%s: %s", #expr, cudaGetErrorString(e2_)); irbpp_destroy(h); return IRBPP_ECUDA; } } while (0)
    TRY_ALLOC(dev_alloc(h, &P.hm, (size_t)N * HX * HY));
    P.cand_stride = (P.sel + 7) & ~7;                 // rows of whole 16-byte units: the scan kernel bulk-copies them
    TRY_ALLOC(dev_alloc(h, &P.cand, (size_t)N * P.cand_stride));
    TRY_ALLOC(dev_alloc(h, &P.state, (size_t)N));
    TRY_ALLOC(dev_alloc(h, &h->actions_dev, N)); TRY_ALLOC(dev_alloc(h, &h->which_dev, N));
    // scan -> candidates hand-over scratch
    // (buffered: one slice per (bin, buffer slot) pair, get_all_possible_observation scans all of them at once)
    const size_t units = (size_t)N * (size_t)P.K;
    TRY_ALLOC(dev_alloc(h, &P.posz, units * P.R * npose));
    TRY_ALLOC(dev_alloc(h, &P.maskbits, units * P.R * bmw));
    TRY_ALLOC(dev_alloc(h, &P.bitmaps, units * P.R * MAX_LEVELS * bmw));
    TRY_ALLOC(dev_alloc(h, &P.nlevels, units * P.R));
    if (P.R * npose > grid_list_cap_ws(step)) TRY_ALLOC(dev_alloc(h, &P.dlist, units * 2 * P.R * npose));     // phase-D lists of bins that spill
    if (step == 1) {
        // contour overflow buffers, one per warp of every candidates CTA (a warp redoes one contour at a time).  Every warp
        // of a CTA takes contour tasks in phase C, the idle warps of a partial last CTA included, so the count is the
        // units rounded up to whole CTAs
        static_assert(CandScratch<Grid<1>>::OVF_GLOBAL, "32x32 grid: the overflow buffer lives in global memory");
        const size_t warps = (units + h->epc - 1) / h->epc * h->epc;
        TRY_ALLOC(dev_alloc(h, &P.ovf, warps * CandScratch<Grid<1>>::OVF_BYTES, false));
    }
    TRY_ALLOC(dev_alloc(h, &h->ready_dev, units));        // zeroed: no launch has epoch 0
    const size_t res_bytes = step_results_bytes(N) + 64;
    TRY_ALLOC(cudaMalloc(&h->results_dev, res_bytes));
    TRY_ALLOC(cudaMemset(h->results_dev, 0, res_bytes));
    for (int t = 0; t < 2; ++t) {
        TRY_ALLOC(cudaHostAlloc(&h->results_host[t], res_bytes, cudaHostAllocMapped));
        TRY_ALLOC(cudaHostGetDevicePointer(&h->results_mapped[t], h->results_host[t], 0));
        memset(h->results_host[t], 0, res_bytes);
    }
    TRY_ALLOC(cudaHostAlloc((void**)&h->actions_pinned, 2 * (size_t)N * sizeof(int64_t), cudaHostAllocMapped));
    P.res = step_results(h->results_dev, N);
    for (bool traj : {false, true}) {
        const StepKernels k = step_kernels(step, h->epc, traj, P.R);
        TRY_ALLOC(raise_dynamic_smem(cfg->device, (const void*)k.cand, k.cand_smem));
    }
#undef TRY_ALLOC
    *out = h;
    return IRBPP_OK;
}

int irbpp_destroy(irbpp_handle h) {
    if (!h) return IRBPP_OK;
    DeviceGuard guard(h->cfg.device);
    cudaDeviceSynchronize();
    for (void* p : h->dev_allocs) cudaFree(p);
    if (h->results_dev) cudaFree(h->results_dev);
    for (int t = 0; t < 2; ++t) if (h->results_host[t]) cudaFreeHost(h->results_host[t]);
    if (h->actions_pinned) cudaFreeHost(h->actions_pinned);
    delete h;
    return IRBPP_OK;
}

int irbpp_obs_len(irbpp_handle h, int32_t* obs_len, int32_t* loc_obs_len, int32_t* order_obs_len) {
    if (!h) return IRBPP_EINVAL;
    if (obs_len) *obs_len = h->P.obs_stride;
    if (loc_obs_len) *loc_obs_len = h->P.loc_len;
    if (order_obs_len) *order_obs_len = h->P.order_len;
    return IRBPP_OK;
}

int irbpp_load_shapes(irbpp_handle h, int32_t S, int32_t R, const int32_t* dims, const double* ext,
                      const double* vol, const double* maps, const int64_t* offsets, int64_t maps_len) {
    if (!h || !dims || !ext || !vol || !maps || !offsets) return fail(h, IRBPP_EINVAL, "null argument");
    if (R != h->P.R) return fail(h, IRBPP_EINVAL, "library has %d rotations, env configured for %d", R, h->P.R);
    if (S <= 0) return fail(h, IRBPP_EINVAL, "empty shape library");
    const irbpp_config& c = h->cfg;
    std::vector<ShapeRot> srot((size_t)S * R);
    std::vector<double> Bs, Ts;
    std::vector<TileEntry> tiles;
    std::vector<double> rew(S);
    int max_entries = 1;
    const int step = h->step, ax = HX / step, ay = HY / step;
    for (int s = 0; s < S; ++s) {
        rew[s] = (vol[s] / h->P.binvol) * 10;                        // binPhy.py:155-156,321-322
        for (int r = 0; r < R; ++r) {
            const int32_t* d = dims + ((size_t)s * R + r) * 4;
            const double* e = ext + ((size_t)s * R + r) * 3;
            const int w = d[0], hh = d[1], wA = d[2], hA = d[3];
            if (w <= 0 || hh <= 0 || w > HX || hh > HY || wA <= 0 || hA <= 0)
                return fail(h, IRBPP_EINVAL, "shape %d rot %d: bad window %dx%d / %dx%d", s, r, w, hh, wA, hA);
            // the reference's window slice would run off the heightmap (NumPy broadcast error, space.py:118)
            if (w > step * wA || hh > step * hA)
                return fail(h, IRBPP_EINVAL, "shape %d rot %d: window %dx%d exceeds action footprint %dx%d "
                            "(the reference fails on this table)", s, r, w, hh, wA, hA);
            const int64_t off = offsets[(size_t)s * R + r];
            const int64_t n = (int64_t)w * hh;
            if (off < 0 || off + 4 * n > maps_len) return fail(h, IRBPP_EINVAL, "shape %d rot %d: table out of range", s, r);
            ShapeRot& q = srot[(size_t)s * R + r];
            q.w = w; q.h = hh;
            q.nX = ax - wA + 1; q.nY = ay - hA + 1;                  // range(rangeX_A - rangeX_OA + 1)
            if (q.nX < 0) q.nX = 0; if (q.nY < 0) q.nY = 0;
            q.ez = np_round6(e[2]);
            // prejudge (binPhy.py:236,240-241): round(round(l*resA, 6) + extent - bin, 6) > 0 fails
            q.okx = 0; q.oky = 0;
            for (int l = 0; l < ax; ++l) {
                const double tx = np_round6((double)l * c.resolution_act);
                if (!(np_round6(tx + e[0] - c.bin_dimension[0]) > 0)) q.okx |= 1u << l;
            }
            for (int l = 0; l < ay; ++l) {
                const double ty = np_round6((double)l * c.resolution_act);
                if (!(np_round6(ty + e[1] - c.bin_dimension[1]) > 0)) q.oky |= 1u << l;
            }
            q.off = (int64_t)Bs.size();
            const double* T = maps + off; const double* B = T + n; const double* mT = B + n; const double* mB = mT + n;
            int any_zero = 0;
            for (int64_t i = 0; i < n; ++i) {
                if ((mB[i] != 0.0 && mB[i] != 1.0) || (mT[i] != 0.0 && mT[i] != 1.0))
                    return fail(h, IRBPP_EINVAL, "shape %d rot %d: masks must be 0/1", s, r);
                if (!isfinite(B[i]) || !isfinite(T[i])) return fail(h, IRBPP_EINVAL, "shape %d rot %d: non-finite height", s, r);
                if (mB[i] == 0.0) any_zero = 1;
                Bs.push_back(mB[i] != 0.0 ? B[i] : INFINITY);
                Ts.push_back(mT[i] != 0.0 ? T[i] : -INFINITY);
            }
            q.any_zero = any_zero;
            q.tile = 1; q.tile_off = 0; q.ntiles = 0;
        }
        // block structure of the bottom tables of shape s (all rotations must agree on the block size); step 2 only, where
        // every window starts on an even cell
        for (int t = 4; t >= 2 && step == 2; t >>= 1) {
            bool ok = true;
            std::vector<std::vector<TileEntry>> found(R);
            for (int r = 0; r < R && ok; ++r) {
                const ShapeRot& q = srot[(size_t)s * R + r];
                const double* Bq = Bs.data() + q.off;            // +inf where masked
                for (int bi = 0; bi * t < q.w && ok; ++bi)
                    for (int bj = 0; bj * t < q.h && ok; ++bj) {
                        const int i1 = std::min(bi * t + t, q.w), j1 = std::min(bj * t + t, q.h);
                        bool any_open = false, any_masked = false, same = true;
                        double b0 = 0.0; bool have = false;
                        for (int i = bi * t; i < i1; ++i)
                            for (int j = bj * t; j < j1; ++j) {
                                const double b = Bq[(size_t)i * q.h + j];
                                if (std::isinf(b)) any_masked = true;
                                else { any_open = true; if (!have) { b0 = b; have = true; } else if (b != b0) same = false; }
                            }
                        if (!any_open) continue;                  // fully masked block contributes nothing
                        if (any_masked || !same || i1 - bi * t != t || j1 - bj * t != t) { ok = false; break; }
                        TileEntry e; e.off = 8 * ((bi * t / 2) * 16 + (bj * t / 2)); e.off_odd = 0; e.b = b0;
                        found[r].push_back(e);
                    }
            }
            if (ok) {
                for (int r = 0; r < R; ++r) {
                    ShapeRot& q = srot[(size_t)s * R + r];
                    q.tile = t; q.tile_off = (int32_t)tiles.size(); q.ntiles = (int32_t)found[r].size();
                    tiles.insert(tiles.end(), found[r].begin(), found[r].end());
                }
                break;
            }
        }
        if (srot[(size_t)s * R].tile == 1) {
            // no block structure: one entry per unmasked cell, offset into the column-parity planes from a window origin in an
            // even row, and (step 1) from one in an odd row
            for (int r = 0; r < R; ++r) {
                ShapeRot& q = srot[(size_t)s * R + r];
                const double* Bq = Bs.data() + q.off;
                q.tile_off = (int32_t)tiles.size();
                for (int i = 0; i < q.w; ++i)
                    for (int j = 0; j < q.h; ++j) {
                        const double b = Bq[(size_t)i * q.h + j];
                        if (std::isinf(b)) continue;
                        TileEntry e; e.off = 8 * hm_index(i, j); e.b = b;
                        e.off_odd = step == 1 ? 8 * (hm_index(i, j + 1) - hm_index(0, 1)) : 0;
                        tiles.push_back(e);
                    }
                q.ntiles = (int32_t)tiles.size() - q.tile_off;
            }
        }
        for (int r = 0; r < R; ++r) max_entries = std::max(max_entries, (int)srot[(size_t)s * R + r].ntiles);
    }
    DeviceGuard guard(c.device);
    CUDA_TRY(h, cudaDeviceSynchronize());
    for (void* old : {(void*)h->srot_dev, (void*)h->Bs_dev, (void*)h->Ts_dev, (void*)h->vol_dev, (void*)h->rew_dev, (void*)h->tiles_dev})
        free_dev(h, old);                                                 // a reload replaces the previous pools
    CUDA_TRY(h, dev_alloc(h, &h->srot_dev, srot.size(), false));
    CUDA_TRY(h, dev_alloc(h, &h->Bs_dev, Bs.size() + 1, false));
    CUDA_TRY(h, dev_alloc(h, &h->Ts_dev, Ts.size() + 1, false));
    CUDA_TRY(h, dev_alloc(h, &h->vol_dev, (size_t)S, false));
    CUDA_TRY(h, dev_alloc(h, &h->rew_dev, (size_t)S, false));
    CUDA_TRY(h, dev_alloc(h, &h->tiles_dev, tiles.size() + 1, false));
    if (!tiles.empty()) CUDA_TRY(h, cudaMemcpy(h->tiles_dev, tiles.data(), tiles.size() * sizeof(TileEntry), cudaMemcpyHostToDevice));
    h->P.tiles = h->tiles_dev;
    CUDA_TRY(h, cudaMemcpy(h->srot_dev, srot.data(), srot.size() * sizeof(ShapeRot), cudaMemcpyHostToDevice));
    CUDA_TRY(h, cudaMemcpy(h->Bs_dev, Bs.data(), Bs.size() * 8, cudaMemcpyHostToDevice));
    CUDA_TRY(h, cudaMemcpy(h->Ts_dev, Ts.data(), Ts.size() * 8, cudaMemcpyHostToDevice));
    CUDA_TRY(h, cudaMemcpy(h->vol_dev, vol, (size_t)S * 8, cudaMemcpyHostToDevice));
    CUDA_TRY(h, cudaMemcpy(h->rew_dev, rew.data(), (size_t)S * 8, cudaMemcpyHostToDevice));
    h->P.S = S; h->P.srot = h->srot_dev; h->P.Bs = h->Bs_dev; h->P.Ts = h->Ts_dev;
    h->P.vol = h->vol_dev; h->P.reward_tab = h->rew_dev;
    h->P.maxwh = max_entries;
    // per-warp staging lists, then the bin's candidate table row (bulk-copied by the scan kernel)
    h->scan_smem = CTA_WARPS * h->P.maxwh * (int)sizeof(TileEntry) + ((h->P.cand_stride * 2 + 15) & ~15);
    // the one-warp-per-bin scan serves the online step when every table is in block form and its per-warp staging (headers of
    // the placed item + the largest scan list) fits what the kernel's residency is built for
    bool block_form = step == 2;
    for (size_t i = 0; i < srot.size(); ++i) block_form = block_form && srot[i].tile > 1;
    const int warp_bytes = scanw_warp_bytes(R, max_entries);
    h->scan_warp_smem = (block_form && h->P.K == 1 && warp_bytes <= SCANW_WARP_DYN_MAX) ? CTA_WARPS * warp_bytes : 0;
    for (bool traj : {false, true}) {
        const StepKernels k = step_kernels(step, h->epc, traj, h->P.R);
        CUDA_TRY(h, raise_dynamic_smem(c.device, (const void*)k.scan, h->scan_smem));
        if (h->scan_warp_smem) CUDA_TRY(h, raise_dynamic_smem(c.device, (const void*)k.scan_warp, h->scan_warp_smem));
    }
    h->shapes_loaded = true;
    return IRBPP_OK;
}

// fresh per-bin state: cursors restart, `init(e, state)` stages what the bin's first draw needs
static int restart_items(irbpp_env* h, const std::function<void(int, EnvState&)>& init) {
    std::vector<EnvState> st((size_t)h->P.N);
    memset(st.data(), 0, st.size() * sizeof(EnvState));
    for (int e = 0; e < h->P.N; ++e) init(e, st[e]);
    CUDA_TRY(h, cudaDeviceSynchronize());
    CUDA_TRY(h, cudaMemcpy(h->P.state, st.data(), st.size() * sizeof(EnvState), cudaMemcpyHostToDevice));
    h->was_reset = false;
    h->scan_current = false;
    return IRBPP_OK;
}

// a new item source replaces the previous one and its device pools
static int drop_item_pools(irbpp_env* h) {
    CUDA_TRY(h, cudaDeviceSynchronize());
    for (void* old : {(void*)h->seq_dev, (void*)h->grp_off_dev, (void*)h->grp_mem_dev, (void*)h->traj_items_dev, (void*)h->traj_off_dev})
        free_dev(h, old);
    h->seq_dev = nullptr; h->grp_off_dev = nullptr; h->grp_mem_dev = nullptr; h->traj_items_dev = nullptr; h->traj_off_dev = nullptr;
    Params& P = h->P;
    P.seq = nullptr; P.L = 0; P.grp_off = nullptr; P.grp_mem = nullptr; P.G = 0;
    P.traj_items = nullptr; P.traj_off = nullptr; P.traj_end = 0;
    h->sequences_set = false;
    return IRBPP_OK;
}

static int upload(irbpp_env* h, void** dst, const void* src, size_t bytes) {
    char* p = nullptr;
    CUDA_TRY(h, dev_alloc(h, &p, bytes, false));
    *dst = p;
    if (bytes) CUDA_TRY(h, cudaMemcpy(p, src, bytes, cudaMemcpyHostToDevice));
    return IRBPP_OK;
}

int irbpp_set_sequences(irbpp_handle h, const int32_t* ids, int32_t length) {
    if (!h || !ids || length <= 0) return fail(h, IRBPP_EINVAL, "bad sequences");
    if (!h->shapes_loaded) return fail(h, IRBPP_ESTATE, "load shapes before sequences");
    const size_t n = (size_t)h->P.N * length;
    for (size_t i = 0; i < n; ++i)
        if (ids[i] < 0 || ids[i] >= h->P.S) return fail(h, IRBPP_EINVAL, "item id %d out of range at %zu", ids[i], i);
    DeviceGuard guard(h->cfg.device);
    int rc = drop_item_pools(h); if (rc) return rc;
    rc = upload(h, (void**)&h->seq_dev, ids, n * 4); if (rc) return rc;
    rc = restart_items(h, [&](int e, EnvState& s) { s.next_seq = ids[(size_t)e * length]; }); if (rc) return rc;
    h->P.item_src = ITEMS_SEQ; h->P.seq = h->seq_dev; h->P.L = length;
    h->sequences_set = true;
    return IRBPP_OK;
}

int irbpp_set_item_rng(irbpp_handle h, uint64_t seed) {
    if (!h) return IRBPP_EINVAL;
    if (!h->shapes_loaded) return fail(h, IRBPP_ESTATE, "load shapes before the item generator");
    DeviceGuard guard(h->cfg.device);
    int rc = drop_item_pools(h); if (rc) return rc;
    rc = restart_items(h, [](int, EnvState&) {}); if (rc) return rc;
    h->P.item_src = ITEMS_RNG; h->P.rng_seed = seed;
    h->sequences_set = true;
    return IRBPP_OK;
}

int irbpp_set_item_groups(irbpp_handle h, uint64_t seed, int32_t num_groups, const int32_t* group_offsets,
                          const int32_t* members) {
    if (!h) return IRBPP_EINVAL;
    if (!group_offsets || !members || num_groups <= 0) return fail(h, IRBPP_EINVAL, "bad item groups");
    if (!h->shapes_loaded) return fail(h, IRBPP_ESTATE, "load shapes before the item groups");
    if (group_offsets[0] != 0) return fail(h, IRBPP_EINVAL, "group_offsets[0] must be 0");
    for (int g = 0; g < num_groups; ++g)
        if (group_offsets[g + 1] <= group_offsets[g])
            return fail(h, IRBPP_EINVAL, "group %d is empty or its offsets are not increasing", g);
    const int32_t M = group_offsets[num_groups];
    for (int32_t i = 0; i < M; ++i)
        if (members[i] < 0 || members[i] >= h->P.S) return fail(h, IRBPP_EINVAL, "item id %d out of range at %d", members[i], i);
    DeviceGuard guard(h->cfg.device);
    int rc = drop_item_pools(h); if (rc) return rc;
    if ((rc = upload(h, (void**)&h->grp_off_dev, group_offsets, ((size_t)num_groups + 1) * 4))) return rc;
    if ((rc = upload(h, (void**)&h->grp_mem_dev, members, (size_t)M * 4))) return rc;
    rc = restart_items(h, [&](int e, EnvState& s) {     // draw 0 of every bin, staged as sequence mode stages its first entry
        s.next_seq = group_item(group_offsets, members, num_groups, seed, (uint32_t)e, 0u);
    });
    if (rc) return rc;
    Params& P = h->P;
    P.item_src = ITEMS_GROUPS; P.rng_seed = seed; P.G = num_groups; P.grp_off = h->grp_off_dev; P.grp_mem = h->grp_mem_dev;
    h->sequences_set = true;
    return IRBPP_OK;
}

int irbpp_set_trajectories(irbpp_handle h, const int32_t* items, const int64_t* offsets, int32_t num_trajectories,
                           int32_t first, int32_t count) {
    if (!h) return IRBPP_EINVAL;
    if (!items || !offsets || num_trajectories <= 0) return fail(h, IRBPP_EINVAL, "bad trajectories");
    if (!h->shapes_loaded) return fail(h, IRBPP_ESTATE, "load shapes before the trajectories");
    if (first < 0 || count < 0 || (int64_t)first + count > num_trajectories)
        return fail(h, IRBPP_EINVAL, "window [%d, %d + %d) outside the %d trajectories", first, first, count, num_trajectories);
    if (offsets[0] != 0) return fail(h, IRBPP_EINVAL, "offsets[0] must be 0");
    for (int t = 0; t < num_trajectories; ++t)
        if (offsets[t + 1] < offsets[t]) return fail(h, IRBPP_EINVAL, "offsets decrease at trajectory %d", t);
    const int64_t M = offsets[num_trajectories];
    for (int64_t i = 0; i < M; ++i)
        if (items[i] < 0 || items[i] >= h->P.S) return fail(h, IRBPP_EINVAL, "item id %d out of range at %lld", items[i], (long long)i);
    const int nfill = queue_len(h->P.K);             // what reset() previews
    for (int t = first; t < first + count; ++t)
        if (offsets[t + 1] - offsets[t] < nfill)
            return fail(h, IRBPP_EINVAL, "trajectory %d has %lld items, a reset takes %d", t, (long long)(offsets[t + 1] - offsets[t]), nfill);
    DeviceGuard guard(h->cfg.device);
    int rc = drop_item_pools(h); if (rc) return rc;
    if ((rc = upload(h, (void**)&h->traj_items_dev, items, (size_t)M * 4))) return rc;
    if ((rc = upload(h, (void**)&h->traj_off_dev, offsets, ((size_t)num_trajectories + 1) * 8))) return rc;
    const int32_t end = first + count;
    rc = restart_items(h, [&](int e, EnvState& s) {     // episode 0 of bin e plays trajectory first + e
        const int64_t t = (int64_t)first + e;
        s.traj_next = (int32_t)(t < end ? t : end);
    });
    if (rc) return rc;
    Params& P = h->P;
    P.item_src = ITEMS_TRAJ; P.traj_items = h->traj_items_dev; P.traj_off = h->traj_off_dev; P.traj_end = end;
    h->sequences_set = true;
    return IRBPP_OK;
}

// One pass of the pipeline: scan kernel (or the levels kernel for caller-supplied maps), then the
// candidates kernel when the observation carries candidate rows.  (Running bin ranges on separate
// streams so that one range's candidates kernel overlaps the next range's scan kernel was measured:
// no gain -- the scan kernel owns the whole register file, the two cannot co-reside.)

static int launch(irbpp_env* h, Params& P, cudaStream_t s) {
    // the units of a launch: bins, or (bin, buffer slot) pairs for get_all_possible_observation
    const int units = (P.mode == MODE_ALL_OBS) ? P.N * P.K : P.N;
    P.env_lo = 0;
    P.env_hi = units;
    const bool cand_follows = mode_emits_loc(P.mode, P.K);
    // per-unit hand-over flags instead of the grid-wide dependency wait, whenever a candidates grid follows.  Not for
    // caller-supplied maps (the levels kernel sets none) and not for the fused all-slot pass (the k scan CTAs of a bin
    // share its state and candidate table, which the candidates CTA of the last slot rewrites: that one must wait for all
    // of them)
    P.ready = (cand_follows && P.mode != MODE_DEBUG_HULLS && P.mode != MODE_ALL_OBS) ? h->ready_dev : nullptr;
    if (++h->epoch == 0) h->epoch = 1;
    P.epoch = h->epoch;
    const StepKernels k = step_kernels(h->step, h->epc, P.item_src == ITEMS_TRAJ, P.R);
    if (P.mode == MODE_DEBUG_HULLS) {
        void (*levels)(const Params) = k.levels;
        levels<<<P.N, CTA_THREADS, 0, s>>>(P);
    } else if (P.mode == MODE_STEP && h->scan_warp_smem) {
        void (*scan)(const Params) = k.scan_warp;
        scan<<<(units + CTA_WARPS - 1) / CTA_WARPS, CTA_THREADS, h->scan_warp_smem, s>>>(P);
    } else {
        void (*scan)(const Params) = k.scan;
        scan<<<units, CTA_THREADS, h->scan_smem, s>>>(P);
    }
    h->launches += 1;
    if (cand_follows) {
        // programmatic dependent launch: the candidates grid is scheduled while the scan grid's last
        // wave drains and waits at griddepcontrol.wait for the scan's completion
        cudaLaunchConfig_t lc = {};
        lc.gridDim = dim3((units + h->epc - 1) / h->epc); lc.blockDim = dim3(32 * h->epc);
        lc.dynamicSmemBytes = (size_t)k.cand_smem; lc.stream = s;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        at[0].val.programmaticStreamSerializationAllowed = (P.mode == MODE_DEBUG_HULLS) ? 0 : 1;
        lc.attrs = at; lc.numAttrs = 1;
        cudaLaunchKernelEx(&lc, k.cand, P);
        h->launches += 1;
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(h, IRBPP_ECUDA, "kernel launch: %s", cudaGetErrorString(e));
    // buffered step / reset change the heightmap without a scan; the debug modes scan foreign inputs
    // (get_all_possible_observation leaves its scans indexed by (bin, slot): not what the heuristic kernel reads)
    h->scan_current = (P.mode == MODE_CANDIDATES || ((P.mode == MODE_STEP || P.mode == MODE_RESET) && P.K == 1));
    return IRBPP_OK;
}

static int ready(irbpp_env* h) {
    if (!h) return IRBPP_EINVAL;
    if (!h->shapes_loaded || !h->sequences_set) return fail(h, IRBPP_ESTATE, "shapes / sequences not loaded");
    return IRBPP_OK;
}

int irbpp_reset(irbpp_handle h, const uint8_t* which, float* obs_out, void* stream) {
    int rc = ready(h); if (rc) return rc;
    DeviceGuard guard(h->cfg.device);
    if (!obs_out) return fail(h, IRBPP_EINVAL, "obs_out is null");
    cudaStream_t s = (cudaStream_t)stream;
    if (h->waiting_step) {         // "Called reset() while waiting for the step to complete" (shmem_vec_env.py:61-63)
        cudaStreamSynchronize(h->pending_stream);
        h->waiting_step = false;
    }
    Params P = h->P;
    P.mode = MODE_RESET; P.obs = obs_out; P.which = nullptr;
    if (which) {
        CUDA_TRY(h, cudaMemcpyAsync(h->which_dev, which, (size_t)P.N, cudaMemcpyHostToDevice, s));
        P.which = h->which_dev;
    }
    rc = launch(h, P, s); if (rc) return rc;
    h->was_reset = true;
    return IRBPP_OK;
}

static int step_async_impl(irbpp_env* h, const int64_t* actions, int32_t on_device, float* obs_out, void* stream,
                           int pose_actions) {
    int rc = ready(h); if (rc) return rc;
    DeviceGuard guard(h->cfg.device);
    if (!actions || !obs_out) return fail(h, IRBPP_EINVAL, "null argument");
    if (!h->was_reset) return fail(h, IRBPP_ESTATE, "step before reset");
    if (h->waiting_step) return fail(h, IRBPP_ESTATE, "already running an async step");   // vec_env.py:7-16
    cudaStream_t s = (cudaStream_t)stream;
    Params P = h->P;
    P.mode = MODE_STEP; P.obs = obs_out; P.pose_actions = pose_actions;
    h->results_on_host = !on_device;
    if (on_device) {
        P.actions = actions;
        rc = launch(h, P, s); if (rc) return rc;
    } else {
        // host actions: pinned staging + one H2D copy (measured faster end to end than letting the kernel read
        // them over PCIe); results: every bin's thread 0 also stores them into this step's pinned host block
        memcpy(h->actions_pinned, actions, (size_t)P.N * sizeof(int64_t));
        P.actions = h->actions_dev;
        h->res_turn ^= 1;                                   // this step's host block (the previous step's stays readable)
        P.res_host = step_results(h->results_mapped[h->res_turn], P.N);
        // (One CUDA graph per step -- H2D copy + both kernels, instantiated per observation buffer -- was measured:
        // a shorter submit, but the step's wait grew by as much; dropped.)
        CUDA_TRY(h, cudaMemcpyAsync(h->actions_dev, h->actions_pinned, (size_t)P.N * sizeof(int64_t), cudaMemcpyHostToDevice, s));
        rc = launch(h, P, s); if (rc) return rc;
    }
    h->waiting_step = true; h->pending_stream = s;
    return IRBPP_OK;
}

int irbpp_step_async(irbpp_handle h, const int64_t* actions, int32_t on_device, float* obs_out, void* stream) {
    return step_async_impl(h, actions, on_device, obs_out, stream, 0);
}

int irbpp_step_poses_async(irbpp_handle h, const int64_t* poses, int32_t on_device, float* obs_out, void* stream) {
    return step_async_impl(h, poses, on_device, obs_out, stream, 1);
}

int irbpp_step_wait(irbpp_handle h, irbpp_step_result* out) {
    int rc = ready(h); if (rc) return rc;
    DeviceGuard guard(h->cfg.device);
    if (!h->waiting_step) return fail(h, IRBPP_ESTATE, "not running an async step");   // vec_env.py:18-26
    cudaStream_t s = h->pending_stream;
    h->waiting_step = false;
    void* host = h->results_host[h->res_turn];
    if (out && !h->results_on_host)            // a device-resident step waited for with the host call: fetch the block
        CUDA_TRY(h, cudaMemcpyAsync(host, h->results_dev, step_results_bytes(h->P.N), cudaMemcpyDeviceToHost, s));
    CUDA_TRY(h, cudaStreamSynchronize(s));
    if (!out) return IRBPP_OK;
    public_results(step_results(host, h->P.N), out);
    return first_device_error(h, out->error);
}

int irbpp_step_wait_device(irbpp_handle h, irbpp_device_result* out) {
    int rc = ready(h); if (rc) return rc;
    DeviceGuard guard(h->cfg.device);
    if (!h->waiting_step) return fail(h, IRBPP_ESTATE, "not running an async step");
    h->waiting_step = false;
    if (out) public_results(h->P.res, out);
    return IRBPP_OK;
}

int irbpp_device_results(irbpp_handle h, irbpp_device_result* out) {
    if (!h || !out) return IRBPP_EINVAL;
    public_results(h->P.res, out);
    return IRBPP_OK;
}

int irbpp_get_action_candidates(irbpp_handle h, const int64_t* order_actions, int32_t on_device,
                                float* loc_obs_out, void* stream) {
    int rc = ready(h); if (rc) return rc;
    DeviceGuard guard(h->cfg.device);
    if (!order_actions || !loc_obs_out) return fail(h, IRBPP_EINVAL, "null argument");
    if (h->P.K <= 1) return fail(h, IRBPP_ESTATE, "get_action_candidates needs buffer_size > 1");
    if (!h->was_reset) return fail(h, IRBPP_ESTATE, "get_action_candidates before reset");
    cudaStream_t s = (cudaStream_t)stream;
    Params P = h->P;
    P.mode = MODE_CANDIDATES; P.obs = loc_obs_out; P.obs_stride = P.loc_len;
    if (on_device) P.actions = order_actions;
    else {
        // staged copy (not zero-copy): the caller may enqueue the following step before this kernel ran
        memcpy(h->actions_pinned + P.N, order_actions, (size_t)P.N * sizeof(int64_t));
        CUDA_TRY(h, cudaMemcpyAsync(h->actions_dev, h->actions_pinned + P.N, (size_t)P.N * sizeof(int64_t), cudaMemcpyHostToDevice, s));
        P.actions = h->actions_dev;
    }
    return launch(h, P, s);
}

int irbpp_get_all_possible_observation(irbpp_handle h, float* out, void* stream) {
    int rc = ready(h); if (rc) return rc;
    DeviceGuard guard(h->cfg.device);
    if (!out) return fail(h, IRBPP_EINVAL, "null argument");
    if (h->P.K <= 1) return fail(h, IRBPP_ESTATE, "get_all_possible_observation needs buffer_size > 1");
    if (!h->was_reset) return fail(h, IRBPP_ESTATE, "called before reset");
    Params P = h->P;
    // every (bin, buffered item) pair is one unit of ONE scan launch and ONE candidates launch (binPhy.py:175-179
    // loops over the k items): the K scans of a bin share its heightmap through L2 and the candidate extraction packs
    // the contour tasks of all pairs densely
    P.mode = MODE_ALL_OBS; P.obs = out; P.obs_stride = P.K * P.loc_len;
    return launch(h, P, (cudaStream_t)stream);
}

int irbpp_heuristic_actions(irbpp_handle h, int32_t method, int32_t dir_idx, int32_t* poses_out, int64_t* index_out,
                            int32_t on_device, void* stream) {
    int rc = ready(h); if (rc) return rc;
    DeviceGuard guard(h->cfg.device);
    if (method < 0 || method >= HEUR_COUNT) return fail(h, IRBPP_EINVAL, "unknown heuristic %d", method);
    if (dir_idx < 0 || dir_idx > 3) return fail(h, IRBPP_EINVAL, "dir_idx %d not in 0..3", dir_idx);   // space.py:167
    if (!h->was_reset || !h->scan_current)
        return fail(h, IRBPP_ESTATE, "no current scan (call after reset / step, or after get_action_candidates when buffer_size > 1)");
    if (h->waiting_step) return fail(h, IRBPP_ESTATE, "a step is pending");
    cudaStream_t s = (cudaStream_t)stream;
    const size_t N = h->P.N;
    if (!h->heur_pose_dev) {
        CUDA_TRY(h, dev_alloc(h, &h->heur_pose_dev, N * 3));
        CUDA_TRY(h, dev_alloc(h, &h->heur_index_dev, N));
    }
    Params P = h->P;
    P.heur_method = method; P.heur_dir = dir_idx;
    P.heur_pose = (on_device && poses_out) ? poses_out : h->heur_pose_dev;
    P.heur_index = (on_device && index_out) ? index_out : h->heur_index_dev;
    void (*heur)(const Params) = step_kernels(h->step, h->epc, false, P.R).heur;
    heur<<<P.N, CTA_THREADS, 0, s>>>(P);
    h->launches += 1;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(h, IRBPP_ECUDA, "kernel launch: %s", cudaGetErrorString(e));
    if (!on_device) {
        if (poses_out) CUDA_TRY(h, cudaMemcpyAsync(poses_out, h->heur_pose_dev, N * 3 * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
        if (index_out) CUDA_TRY(h, cudaMemcpyAsync(index_out, h->heur_index_dev, N * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
        CUDA_TRY(h, cudaStreamSynchronize(s));
    }
    return IRBPP_OK;
}

int irbpp_debug_state(irbpp_handle h, double* heightmap, int32_t* queue, int32_t* cursor, int32_t* packed_count) {
    int rc = ready(h); if (rc) return rc;
    DeviceGuard guard(h->cfg.device);
    CUDA_TRY(h, cudaDeviceSynchronize());
    const int N = h->P.N;
    if (heightmap) {
        std::vector<double> raw((size_t)N * HX * HY);
        CUDA_TRY(h, cudaMemcpy(raw.data(), h->P.hm, raw.size() * 8, cudaMemcpyDeviceToHost));
        for (int e = 0; e < N; ++e)
            for (int x = 0; x < HX; ++x)
                for (int y = 0; y < HY; ++y)
                    heightmap[((size_t)e * HX + x) * HY + y] = raw[(size_t)e * HX * HY + hm_index(x, y)];
    }
    if (queue || cursor || packed_count) {
        std::vector<EnvState> st((size_t)N);
        CUDA_TRY(h, cudaMemcpy(st.data(), h->P.state, st.size() * sizeof(EnvState), cudaMemcpyDeviceToHost));
        const int k = queue_len(h->P.K);
        for (int e = 0; e < N; ++e) {
            if (queue) for (int i = 0; i < k; ++i) queue[(size_t)e * k + i] = st[e].queue[i];
            if (cursor) cursor[e] = st[e].cursor;
            if (packed_count) packed_count[e] = st[e].packed;
        }
    }
    return IRBPP_OK;
}

int irbpp_debug_set_heightmap(irbpp_handle h, const double* heightmap) {
    int rc = ready(h); if (rc) return rc;
    DeviceGuard guard(h->cfg.device);
    if (!heightmap) return fail(h, IRBPP_EINVAL, "null argument");
    const int N = h->P.N;
    std::vector<double> raw((size_t)N * HX * HY);
    for (int e = 0; e < N; ++e)
        for (int x = 0; x < HX; ++x)
            for (int y = 0; y < HY; ++y)
                raw[(size_t)e * HX * HY + hm_index(x, y)] = heightmap[((size_t)e * HX + x) * HY + y];
    CUDA_TRY(h, cudaDeviceSynchronize());
    CUDA_TRY(h, cudaMemcpy(h->P.hm, raw.data(), raw.size() * 8, cudaMemcpyHostToDevice));
    return IRBPP_OK;
}

static int debug_run(irbpp_env* h, Params& P, double* posZmap, double* posZValid, double* naiveMask,
                     double* cand, int32_t* num_hull) {
    const size_t N = P.N, nm = N * P.R * h->npose, nc = N * P.sel * 5;
    double* d_cd = nullptr; int32_t* d_nh = nullptr; float* d_obs = nullptr;
    auto cleanup = [&]() { cudaFree(d_cd); cudaFree(d_nh); cudaFree(d_obs); };
#define DBG_TRY(expr) do { cudaError_t e_ = (expr); if (e_ != cudaSuccess) { cleanup(); return fail(h, IRBPP_ECUDA, "%s: %s", #expr, cudaGetErrorString(e_)); } } while (0)
    DBG_TRY(cudaMalloc(&d_cd, nc * 8)); DBG_TRY(cudaMalloc(&d_nh, N * 4));
    DBG_TRY(cudaMalloc(&d_obs, N * (size_t)P.loc_len * 4));
    P.dbg_cand = d_cd; P.dbg_nhull = d_nh; P.obs = d_obs; P.obs_stride = P.loc_len;
    int rc = launch(h, P, nullptr);
    if (rc) { cleanup(); return rc; }
    DBG_TRY(cudaDeviceSynchronize());
    if (posZmap || posZValid || naiveMask) {       // float64 views straight from the hand-over scratch
        std::vector<double> pz(nm);
        std::vector<uint32_t> mb(nm / 32);
        DBG_TRY(cudaMemcpy(pz.data(), P.posz, nm * 8, cudaMemcpyDeviceToHost));
        DBG_TRY(cudaMemcpy(mb.data(), P.maskbits, mb.size() * 4, cudaMemcpyDeviceToHost));
        for (size_t i = 0; i < nm; ++i) {
            const bool m = (mb[i >> 5] >> (i & 31)) & 1u;
            if (posZmap) posZmap[i] = pz[i];
            if (posZValid) posZValid[i] = m ? pz[i] : POSZ_INVALID;
            if (naiveMask) naiveMask[i] = m ? 1.0 : 0.0;
        }
    }
    if (cand) DBG_TRY(cudaMemcpy(cand, d_cd, nc * 8, cudaMemcpyDeviceToHost));
    if (num_hull) DBG_TRY(cudaMemcpy(num_hull, d_nh, N * 4, cudaMemcpyDeviceToHost));
    std::vector<uint8_t> errs(N);
    DBG_TRY(cudaMemcpy(errs.data(), P.res.error, N, cudaMemcpyDeviceToHost));
    cleanup();
#undef DBG_TRY
    return first_device_error(h, errs.data());
}

int irbpp_debug_scan(irbpp_handle h, const int32_t* item_ids, double* posZmap, double* posZValid,
                     double* naiveMask, double* cand, int32_t* num_hull) {
    int rc = ready(h); if (rc) return rc;
    DeviceGuard guard(h->cfg.device);
    if (!item_ids) return fail(h, IRBPP_EINVAL, "null argument");
    for (int i = 0; i < h->P.N; ++i)
        if (item_ids[i] < 0 || item_ids[i] >= h->P.S) return fail(h, IRBPP_EINVAL, "item id out of range");
    int32_t* d_items = nullptr;
    CUDA_TRY(h, cudaMalloc(&d_items, (size_t)h->P.N * 4));
    CUDA_TRY(h, cudaMemcpy(d_items, item_ids, (size_t)h->P.N * 4, cudaMemcpyHostToDevice));
    Params P = h->P;
    P.mode = MODE_DEBUG_SCAN; P.dbg_items = d_items;
    rc = debug_run(h, P, posZmap, posZValid, naiveMask, cand, num_hull);
    cudaFree(d_items);
    return rc;
}

int irbpp_debug_hulls(irbpp_handle h, const double* posZValid, const double* mask, double* cand, int32_t* num_hull) {
    int rc = ready(h); if (rc) return rc;
    DeviceGuard guard(h->cfg.device);
    if (!posZValid || !mask) return fail(h, IRBPP_EINVAL, "null argument");
    const size_t nm = (size_t)h->P.N * h->P.R * h->npose;
    std::vector<uint32_t> mb(nm / 32, 0u);
    for (size_t i = 0; i < nm; ++i) if (mask[i] != 0.0) mb[i >> 5] |= 1u << (i & 31);
    CUDA_TRY(h, cudaDeviceSynchronize());
    CUDA_TRY(h, cudaMemcpy(h->P.posz, posZValid, nm * 8, cudaMemcpyHostToDevice));
    CUDA_TRY(h, cudaMemcpy(h->P.maskbits, mb.data(), mb.size() * 4, cudaMemcpyHostToDevice));
    Params P = h->P;
    P.mode = MODE_DEBUG_HULLS;
    return debug_run(h, P, nullptr, nullptr, nullptr, cand, num_hull);
}

int64_t irbpp_launch_count(irbpp_handle h) { return h ? h->launches : 0; }

// ---- compact form of the location observation for the rollout gather (csrc/irbpp_pack.cuh) --------------------
int irbpp_packed_obs_bytes(int32_t selected_action) { return selected_action > 0 ? packed_words(selected_action) * 4 : -1; }

int irbpp_pack_observations(const float* obs, int64_t obs_stride, int32_t selected_action, int32_t n, void* packed, void* stream) {
    if (!obs || !packed || n <= 0 || selected_action <= 0 || obs_stride < selected_action * 5 + 9 + 1024)
        return fail(nullptr, IRBPP_EINVAL, "bad pack arguments");
    DeviceGuard guard(device_of(obs));
    irbpp_pack_obs_kernel<<<n, 128, 0, (cudaStream_t)stream>>>(obs, obs_stride, selected_action, reinterpret_cast<uint32_t*>(packed), n);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(nullptr, IRBPP_ECUDA, "kernel launch: %s", cudaGetErrorString(e));
    return IRBPP_OK;
}

int irbpp_unpack_observations(const void* packed, int32_t selected_action, int32_t n, float* obs, int64_t obs_stride, void* stream) {
    if (!obs || !packed || n <= 0 || selected_action <= 0 || obs_stride < selected_action * 5 + 9 + 1024)
        return fail(nullptr, IRBPP_EINVAL, "bad unpack arguments");
    DeviceGuard guard(device_of(obs));
    irbpp_unpack_obs_kernel<<<n, 128, 0, (cudaStream_t)stream>>>(reinterpret_cast<const uint32_t*>(packed), selected_action, obs, obs_stride, n);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(nullptr, IRBPP_ECUDA, "kernel launch: %s", cudaGetErrorString(e));
    return IRBPP_OK;
}

// ---- point clouds of the next items (SURVEY.md 8(f)3; csrc/irbpp_pointnet.cuh) ----------------------------------
// grid of the grid-stride gather kernels: 16 CTAs per SM of the device that runs them
static int64_t gather_grid_cap(int dev) {
    int sms = 0;
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 1;
    return (int64_t)sms * 16;
}

static int pn_common(PointNetParams& Q, const float* shape_array, int32_t S, int32_t P, const float* obs, int64_t obs_stride,
                     int32_t item_col, const int32_t* ids, int32_t B, uint64_t seed, uint64_t counter, int32_t n_points) {
    if (!shape_array || S <= 0 || P <= 0 || B <= 0 || n_points <= 0) return fail(nullptr, IRBPP_EINVAL, "bad point-cloud arguments");
    if (!obs && !ids) return fail(nullptr, IRBPP_EINVAL, "either the observations or explicit item ids are needed");
    if (obs && !ids && (obs_stride <= 0 || item_col < 0 || item_col >= obs_stride)) return fail(nullptr, IRBPP_EINVAL, "bad item column");
    memset(&Q, 0, sizeof(Q));
    Q.shape_array = shape_array; Q.S = S; Q.P = P; Q.n_points = n_points; Q.seed = seed; Q.counter = counter;
    Q.obs = obs; Q.obs_stride = obs_stride; Q.item_col = item_col; Q.ids = ids; Q.B = B;
    return IRBPP_OK;
}

int irbpp_sample_point_clouds(const float* shape_array, int32_t S, int32_t P, const float* obs, int64_t obs_stride,
                              int32_t item_col, const int32_t* ids, int32_t B, uint64_t seed, uint64_t counter,
                              int32_t n_points, float* out, int32_t* indices_out, void* stream) {
    PointNetParams Q;
    int rc = pn_common(Q, shape_array, S, P, obs, obs_stride, item_col, ids, B, seed, counter, n_points); if (rc) return rc;
    if (!out) return fail(nullptr, IRBPP_EINVAL, "null output");
    Q.out = out; Q.indices_out = indices_out;
    const int dev = device_of(shape_array);
    DeviceGuard guard(dev);
    const int64_t n = (int64_t)B * n_points;
    const int blocks = (int)std::min<int64_t>((n + 255) / 256, gather_grid_cap(dev));
    irbpp_cloud_gather_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(Q);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(nullptr, IRBPP_ECUDA, "kernel launch: %s", cudaGetErrorString(e));
    return IRBPP_OK;
}

int irbpp_shape_features(const float* shape_array, int32_t S, int32_t P, const float* obs, int64_t obs_stride,
                         int32_t item_col, const int32_t* ids, int32_t B, uint64_t seed, uint64_t counter,
                         int32_t n_points, const float* W1, const float* b1, const float* W2, const float* b2,
                         float negative_slope, int32_t* scratch_keys, float* out, void* stream) {
    PointNetParams Q;
    int rc = pn_common(Q, shape_array, S, P, obs, obs_stride, item_col, ids, B, seed, counter, n_points); if (rc) return rc;
    if (!W1 || !b1 || !W2 || !b2 || !scratch_keys || !out) return fail(nullptr, IRBPP_EINVAL, "null argument");
    Q.W1 = W1; Q.b1 = b1; Q.W2 = W2; Q.b2 = b2; Q.slope = negative_slope; Q.feat_keys = scratch_keys; Q.out = out;
    const int dev = device_of(shape_array);
    DeviceGuard guard(dev);
    cudaError_t e = raise_dynamic_smem(dev, (const void*)irbpp_shape_encode_kernel, PN_SMEM_BYTES);
    if (e != cudaSuccess) return fail(nullptr, IRBPP_ECUDA, "shape encoder set-up: %s", cudaGetErrorString(e));
    cudaStream_t s = (cudaStream_t)stream;
    irbpp_pn_init_kernel<<<(S * PN_H + 255) / 256, 256, 0, s>>>(scratch_keys, S * PN_H);
    const int tiles = (n_points + PN_TILE - 1) / PN_TILE;
    irbpp_shape_encode_kernel<<<S * tiles, PN_THREADS, PN_SMEM_BYTES, s>>>(Q);
    const int64_t n = (int64_t)B * PN_H;
    irbpp_feature_gather_kernel<<<(int)std::min<int64_t>((n + 255) / 256, gather_grid_cap(dev)), 256, 0, s>>>(Q);
    e = cudaGetLastError();
    if (e != cudaSuccess) return fail(nullptr, IRBPP_ECUDA, "kernel launch: %s", cudaGetErrorString(e));
    return IRBPP_OK;
}

// ---- prioritized n-step replay (csrc/irbpp_replay.cuh) ---------------------------------------------------------
static int replay_check(const irbpp_replay_memory* mem) {
    if (!mem) return fail(nullptr, IRBPP_EINVAL, "null replay memory");
    if (mem->num_memories <= 0 || mem->capacity < 2 || mem->obs_len <= 0)
        return fail(nullptr, IRBPP_EINVAL, "bad replay sizes (M %d, C %d, obs_len %d; need M > 0, C >= 2, obs_len > 0)",
                    mem->num_memories, mem->capacity, mem->obs_len);
    if ((int64_t)mem->capacity * 2 - 1 > INT32_MAX) return fail(nullptr, IRBPP_EINVAL, "replay capacity too large");
    if (!mem->states || !mem->timesteps || !mem->actions || !mem->rewards || !mem->nonterminals || !mem->tree || !mem->state)
        return fail(nullptr, IRBPP_EINVAL, "null replay array");
    return IRBPP_OK;
}

static int launch_status() {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(nullptr, IRBPP_ECUDA, "kernel launch: %s", cudaGetErrorString(e));
    return IRBPP_OK;
}

int irbpp_replay_init(const irbpp_replay_memory* mem, void* stream) {
    int rc = replay_check(mem); if (rc) return rc;
    const int dev = device_of(mem->tree);
    DeviceGuard guard(dev);
    const int64_t nodes = (int64_t)mem->num_memories * (2 * mem->capacity - 1);
    const int blocks = (int)std::min<int64_t>((nodes + 255) / 256, gather_grid_cap(dev));
    irbpp_replay_init_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(*mem);
    return launch_status();
}

int irbpp_replay_append(const irbpp_replay_memory* mem, const float* obs, int64_t obs_stride, const int64_t* action,
                        const float* reward, const uint8_t* done, const uint8_t* valid, float reward_clip, void* stream) {
    int rc = replay_check(mem); if (rc) return rc;
    if (!obs || !action || !reward || !done) return fail(nullptr, IRBPP_EINVAL, "null append input");
    if (obs_stride < mem->obs_len) return fail(nullptr, IRBPP_EINVAL, "observation stride %lld < obs_len %d", (long long)obs_stride, mem->obs_len);
    ReplayAppendArgs A;
    A.mem = *mem; A.obs = obs; A.obs_stride = obs_stride; A.action = action; A.reward = reward; A.done = done; A.valid = valid;
    A.reward_clip = reward_clip;
    DeviceGuard guard(device_of(mem->tree));
    irbpp_replay_append_kernel<<<mem->num_memories, RP_APPEND_THREADS, 0, (cudaStream_t)stream>>>(A);
    return launch_status();
}

int irbpp_replay_sample(const irbpp_replay_memory* mem, const int32_t* mem_ids, int32_t G, int32_t k, int32_t n,
                        double discount, double beta, int32_t max_attempts, uint64_t seed, uint64_t call,
                        const double* uniforms, const irbpp_replay_batch* out, uint32_t* error_flags, void* stream) {
    int rc = replay_check(mem); if (rc) return rc;
    if (!mem_ids || !out) return fail(nullptr, IRBPP_EINVAL, "null sample argument");
    if (G < 1 || k < 1) return fail(nullptr, IRBPP_EINVAL, "need G >= 1 memories and k >= 1 samples each (G %d, k %d)", G, k);
    if ((int64_t)G * k > INT32_MAX) return fail(nullptr, IRBPP_EINVAL, "batch too large");
    if (n < 0 || n >= mem->capacity || n > RP_MAX_N)
        return fail(nullptr, IRBPP_EINVAL, "multi_step %d outside [0, min(C - 1, %d)] (C %d)", n, RP_MAX_N, mem->capacity);
    if (max_attempts < 1 || max_attempts > 65536) return fail(nullptr, IRBPP_EINVAL, "max_attempts %d outside [1, 65536]", max_attempts);
    if (!out->tree_idx || !out->states || !out->actions || !out->returns || !out->next_states || !out->nonterminals || !out->weights)
        return fail(nullptr, IRBPP_EINVAL, "null sample output");
    ReplaySampleArgs A;
    memset(&A, 0, sizeof(A));
    A.mem = *mem; A.mem_ids = mem_ids; A.G = G; A.k = k; A.n = n; A.attempts = max_attempts;
    for (int i = 0; i < n; ++i) A.scale[i] = (float)std::pow(discount, (double)i);     // torch.tensor([γ ** i], float32)
    A.neg_beta = (double)(float)(-beta);
    A.seed = seed; A.call = call; A.uniforms = uniforms; A.out = *out; A.error_flags = error_flags;
    DeviceGuard guard(device_of(mem->tree));
    irbpp_replay_sample_kernel<<<G, RP_SAMPLE_THREADS, 0, (cudaStream_t)stream>>>(A);
    return launch_status();
}

int irbpp_replay_update_priorities(const irbpp_replay_memory* mem, const int32_t* mem_ids, const int64_t* tree_idxs,
                                   const float* loss, int32_t B, double omega, uint32_t* error_flags, void* stream) {
    int rc = replay_check(mem); if (rc) return rc;
    if (B < 1 || !mem_ids || !tree_idxs || !loss) return fail(nullptr, IRBPP_EINVAL, "bad update arguments (B %d)", B);
    ReplayUpdateArgs A;
    A.mem = *mem; A.mem_ids = mem_ids; A.tree_idxs = tree_idxs; A.loss = loss; A.B = B;
    A.omega = (double)(float)omega; A.error_flags = error_flags;
    DeviceGuard guard(device_of(mem->tree));
    const int blocks = (mem->num_memories + RP_UPDATE_WARPS - 1) / RP_UPDATE_WARPS;
    irbpp_replay_update_kernel<<<blocks, 32 * RP_UPDATE_WARPS, 0, (cudaStream_t)stream>>>(A);
    return launch_status();
}

// ---- the location network's forward pass and Agent.act (csrc/irbpp_actor.cuh) -------------------------------------
int64_t irbpp_dqn_scratch_bytes(int32_t N, int32_t selected_action) {
    if (N <= 0 || selected_action <= 0) return -1;
    return actor_scratch_bytes(N, selected_action);
}

// the arguments of Agent.learn's target pass beyond the act's (irbpp_dqn_target, irbpp_dqn_order_target)
static int learn_target_args(LearnTarget& T, int32_t atoms, const int64_t* next_actions, const float* returns,
                             const float* nonterminals, double discount_n, double v_min, double v_max, float* m,
                             float* p_next) {
    if (!next_actions || !returns || !nonterminals || !m) return fail(nullptr, IRBPP_EINVAL, "null target argument");
    if (atoms < 2 || atoms > AC_MAXATOMS) return fail(nullptr, IRBPP_EINVAL, "atoms %d outside [2, %d]", atoms, AC_MAXATOMS);
    if (!(v_max > v_min)) return fail(nullptr, IRBPP_EINVAL, "need v_max > v_min (v_min %g, v_max %g)", v_min, v_max);
    const double dz = (v_max - v_min) / (atoms - 1);           // agent.py:20, in double
    T.next_actions = next_actions; T.returns = returns; T.nonterminals = nonterminals;
    T.gamma_n = (float)discount_n; T.v_min = (float)v_min; T.v_max = (float)v_max;
    T.inv_dz = 1.0f / (float)dz;                                 // torch's CUDA tensor / scalar (irbpp_learn.cuh)
    T.m = m; T.p_next = p_next;
    return IRBPP_OK;
}

// irbpp_dqn_act (T == NULL) and irbpp_dqn_target (T: the target mode's arguments, checked)
static int dqn_forward(const irbpp_dqn_weights* weights, const float* obs, int64_t obs_stride, int32_t N,
                       int32_t selected_action, const float* shape_feature, const float* support, int32_t atoms,
                       const float* mask, int64_t mask_row_stride, int64_t mask_elem_stride, int64_t* actions,
                       float* sum_q_map, void* scratch, int64_t scratch_bytes, void* stream, const LearnTarget* T) {
    if (!weights || !obs || !shape_feature || !support || (!T && !actions) || !scratch) return fail(nullptr, IRBPP_EINVAL, "null act argument");
    if (N <= 0 || selected_action <= 0) return fail(nullptr, IRBPP_EINVAL, "need N >= 1 bins and selected_action >= 1 (N %d, sel %d)", N, selected_action);
    if (atoms < 1 || atoms > AC_MAXATOMS) return fail(nullptr, IRBPP_EINVAL, "atoms %d outside [1, %d]", atoms, AC_MAXATOMS);
    if (obs_stride < (int64_t)selected_action * 5 + 9 + AC_HM * AC_HM)
        return fail(nullptr, IRBPP_EINVAL, "observation stride %lld < selected_action * 5 + 9 + 1024", (long long)obs_stride);
    if (scratch_bytes < actor_scratch_bytes(N, selected_action))
        return fail(nullptr, IRBPP_EINVAL, "scratch of %lld bytes < %lld", (long long)scratch_bytes, (long long)actor_scratch_bytes(N, selected_action));
    if (reinterpret_cast<uintptr_t>(scratch) & 255) return fail(nullptr, IRBPP_EINVAL, "scratch not 256-byte aligned");
    const irbpp_dqn_weights& w = *weights;
    const float* ptrs[] = {w.conv1_w, w.conv1_b, w.conv2_w, w.conv2_b, w.conv3_w, w.conv3_b, w.cand1_w, w.cand1_b, w.cand2_w,
                           w.cand2_b, w.proj1_w, w.proj1_b, w.proj2_w, w.proj2_b, w.fc_h_v_w, w.fc_h_v_b, w.fc_z_v_w,
                           w.fc_z_v_b, w.fc_h_a_w, w.fc_h_a_b, w.fc_z_a_w, w.fc_z_a_b};
    for (const float* p : ptrs)
        if (!p) return fail(nullptr, IRBPP_EINVAL, "null weight pointer");
    ActorParams A;
    memset(&A, 0, sizeof(A));
    A.w = ActorWeights{w.conv1_w, w.conv1_b, w.conv2_w, w.conv2_b, w.conv3_w, w.conv3_b, w.cand1_w, w.cand1_b, w.cand2_w,
                       w.cand2_b, w.proj1_w, w.proj1_b, w.proj2_w, w.proj2_b, w.fc_h_v_w, w.fc_h_v_b, w.fc_z_v_w,
                       w.fc_z_v_b, w.fc_h_a_w, w.fc_h_a_b, w.fc_z_a_w, w.fc_z_a_b, w.negative_slope};
    A.obs = obs; A.obs_stride = obs_stride; A.N = N; A.sel = selected_action; A.atoms = atoms;
    A.shape_feature = shape_feature; A.support = support;
    A.mask = mask; A.mask_row = mask_row_stride; A.mask_elem = mask_elem_stride;
    A.actions = actions; A.sum_q = sum_q_map;
    actor_scratch_layout(A, scratch);
    const int dev = device_of(obs);
    DeviceGuard guard(dev);
    const void* rows = T ? (const void*)irbpp_actor_target_kernel : (const void*)irbpp_actor_rows_kernel;
    cudaError_t e = raise_dynamic_smem(dev, rows, AC_ROWS_SMEM_BYTES);
    if (e != cudaSuccess) return fail(nullptr, IRBPP_ECUDA, "rows kernel set-up: %s", cudaGetErrorString(e));
    cudaStream_t s = (cudaStream_t)stream;
    irbpp_actor_bin_kernel<<<N, AC_THREADS, 0, s>>>(A);
    if (T) irbpp_actor_target_kernel<<<N, AC_THREADS, AC_ROWS_SMEM_BYTES, s>>>(A, *T);
    else irbpp_actor_rows_kernel<<<N, AC_THREADS, AC_ROWS_SMEM_BYTES, s>>>(A);
    return launch_status();
}

int irbpp_dqn_act(const irbpp_dqn_weights* weights, const float* obs, int64_t obs_stride, int32_t N, int32_t selected_action,
                  const float* shape_feature, const float* support, int32_t atoms, const float* mask, int64_t mask_row_stride,
                  int64_t mask_elem_stride, int64_t* actions, float* sum_q_map, void* scratch, int64_t scratch_bytes,
                  void* stream) {
    return dqn_forward(weights, obs, obs_stride, N, selected_action, shape_feature, support, atoms, mask, mask_row_stride,
                       mask_elem_stride, actions, sum_q_map, scratch, scratch_bytes, stream, nullptr);
}

int irbpp_dqn_target(const irbpp_dqn_weights* target, const float* next_obs, int64_t obs_stride, int32_t B,
                     int32_t selected_action, const float* shape_feature, const float* support, int32_t atoms,
                     const int64_t* next_actions, const float* returns, const float* nonterminals, double discount_n,
                     double v_min, double v_max, float* m, float* p_next, void* scratch, int64_t scratch_bytes,
                     void* stream) {
    LearnTarget T;
    const int rc = learn_target_args(T, atoms, next_actions, returns, nonterminals, discount_n, v_min, v_max, m, p_next);
    if (rc) return rc;
    return dqn_forward(target, next_obs, obs_stride, B, selected_action, shape_feature, support, atoms, nullptr, 0, 0,
                       nullptr, nullptr, scratch, scratch_bytes, stream, &T);
}

// ---- the order network's forward pass and Agent.act (csrc/irbpp_order_actor.cuh) ---------------------------------
int64_t irbpp_dqn_order_scratch_bytes(int32_t N, int32_t k, int32_t S) {
    if (N <= 0 || k < 2 || k > OA_MAXK || S <= 0) return -1;
    return order_scratch_bytes(N, S);
}

// irbpp_dqn_order_act (T == NULL) and irbpp_dqn_order_target (T: the target mode's arguments, checked)
static int dqn_order_forward(const irbpp_dqn_order_weights* weights, const float* obs, int64_t obs_stride, int32_t N,
                             int32_t k, const float* shape_features, int32_t S, const float* support, int32_t atoms,
                             const float* mask, int64_t mask_row_stride, int64_t mask_elem_stride, int64_t* actions,
                             float* sum_q_map, void* scratch, int64_t scratch_bytes, void* stream, const LearnTarget* T) {
    if (!weights || !obs || !shape_features || !support || (!T && !actions) || !scratch) return fail(nullptr, IRBPP_EINVAL, "null order act argument");
    if (N <= 0 || S <= 0) return fail(nullptr, IRBPP_EINVAL, "need N >= 1 bins and S >= 1 shapes (N %d, S %d)", N, S);
    if (k < 2 || k > OA_MAXK) return fail(nullptr, IRBPP_EINVAL, "buffer size k %d outside [2, %d]", k, OA_MAXK);
    if (atoms < 1 || atoms > AC_MAXATOMS) return fail(nullptr, IRBPP_EINVAL, "atoms %d outside [1, %d]", atoms, AC_MAXATOMS);
    if (obs_stride < (int64_t)k + AC_HM * AC_HM)
        return fail(nullptr, IRBPP_EINVAL, "observation stride %lld < k + 1024", (long long)obs_stride);
    if (scratch_bytes < order_scratch_bytes(N, S))
        return fail(nullptr, IRBPP_EINVAL, "scratch of %lld bytes < %lld", (long long)scratch_bytes, (long long)order_scratch_bytes(N, S));
    if (reinterpret_cast<uintptr_t>(scratch) & 255) return fail(nullptr, IRBPP_EINVAL, "scratch not 256-byte aligned");
    const irbpp_dqn_order_weights& w = *weights;
    const float* ptrs[] = {w.conv1_w, w.conv1_b, w.conv2_w, w.conv2_b, w.conv3_w, w.conv3_b, w.gat1_w, w.gat1_b, w.gat2_w,
                           w.gat2_b, w.wq, w.wk, w.wv, w.wo_w, w.wo_b, w.ff1_w, w.ff1_b, w.ff2_w, w.ff2_b, w.fc_h_v_w,
                           w.fc_h_v_b, w.fc_z_v_w, w.fc_z_v_b, w.fc_h_a_w, w.fc_h_a_b, w.fc_z_a_w, w.fc_z_a_b};
    for (const float* p : ptrs)
        if (!p) return fail(nullptr, IRBPP_EINVAL, "null weight pointer");
    OrderParams A;
    memset(&A, 0, sizeof(A));
    A.w = OrderWeights{w.conv1_w, w.conv1_b, w.conv2_w, w.conv2_b, w.conv3_w, w.conv3_b, w.gat1_w, w.gat1_b, w.gat2_w,
                       w.gat2_b, w.wq, w.wk, w.wv, w.wo_w, w.wo_b, w.ff1_w, w.ff1_b, w.ff2_w, w.ff2_b, w.fc_h_v_w,
                       w.fc_h_v_b, w.fc_z_v_w, w.fc_z_v_b, w.fc_h_a_w, w.fc_h_a_b, w.fc_z_a_w, w.fc_z_a_b, w.negative_slope};
    A.obs = obs; A.obs_stride = obs_stride; A.N = N; A.k = k; A.S = S; A.atoms = atoms;
    A.shape_features = shape_features; A.support = support;
    A.mask = mask; A.mask_row = mask_row_stride; A.mask_elem = mask_elem_stride;
    A.actions = actions; A.sum_q = sum_q_map;
    order_scratch_layout(A, scratch);
    const int dev = device_of(obs);
    DeviceGuard guard(dev);
    const void* slots = T ? (const void*)irbpp_order_target_kernel : (const void*)irbpp_order_slots_kernel;
    cudaError_t e = raise_dynamic_smem(dev, slots, OA_SLOTS_SMEM_BYTES);
    if (e != cudaSuccess) return fail(nullptr, IRBPP_ECUDA, "slots kernel set-up: %s", cudaGetErrorString(e));
    cudaStream_t s = (cudaStream_t)stream;
    const int per = AC_TM / k;
    irbpp_order_table_kernel<<<S, AC_THREADS, 0, s>>>(A);
    irbpp_order_bin_kernel<<<N, AC_THREADS, 0, s>>>(A);
    if (T) irbpp_order_target_kernel<<<(N + per - 1) / per, AC_THREADS, OA_SLOTS_SMEM_BYTES, s>>>(A, *T);
    else irbpp_order_slots_kernel<<<(N + per - 1) / per, AC_THREADS, OA_SLOTS_SMEM_BYTES, s>>>(A);
    return launch_status();
}

int irbpp_dqn_order_act(const irbpp_dqn_order_weights* weights, const float* obs, int64_t obs_stride, int32_t N, int32_t k,
                        const float* shape_features, int32_t S, const float* support, int32_t atoms, const float* mask,
                        int64_t mask_row_stride, int64_t mask_elem_stride, int64_t* actions, float* sum_q_map, void* scratch,
                        int64_t scratch_bytes, void* stream) {
    return dqn_order_forward(weights, obs, obs_stride, N, k, shape_features, S, support, atoms, mask, mask_row_stride,
                             mask_elem_stride, actions, sum_q_map, scratch, scratch_bytes, stream, nullptr);
}

int irbpp_dqn_order_target(const irbpp_dqn_order_weights* target, const float* next_obs, int64_t obs_stride, int32_t B,
                           int32_t k, const float* shape_features, int32_t S, const float* support, int32_t atoms,
                           const int64_t* next_actions, const float* returns, const float* nonterminals,
                           double discount_n, double v_min, double v_max, float* m, float* p_next, void* scratch,
                           int64_t scratch_bytes, void* stream) {
    LearnTarget T;
    const int rc = learn_target_args(T, atoms, next_actions, returns, nonterminals, discount_n, v_min, v_max, m, p_next);
    if (rc) return rc;
    return dqn_order_forward(target, next_obs, obs_stride, B, k, shape_features, S, support, atoms, nullptr, 0, 0,
                             nullptr, nullptr, scratch, scratch_bytes, stream, &T);
}

// ---- the gradient pass of Agent.learn at the location level (csrc/irbpp_grad.cuh) ---------------------------------
int64_t irbpp_dqn_log_prob_scratch_bytes(int32_t B, int32_t selected_action) {
    if (B <= 0 || selected_action <= 0 || (int64_t)B * (selected_action + 1) >= INT32_MAX) return -1;
    return grad_scratch_bytes(B, selected_action);
}

// the argument checks both entry points share, and the parameter block
static int grad_params(GradParams& P, const irbpp_dqn_weights* weights, const float* obs, int64_t obs_stride, int32_t B,
                       int32_t sel, const float* shape_feature, const float* map_feature, const int64_t* actions,
                       int32_t atoms, void* scratch, int64_t scratch_bytes) {
    if (!weights || !obs || !shape_feature || !map_feature || !actions || !scratch)
        return fail(nullptr, IRBPP_EINVAL, "null log-prob argument");
    if (B <= 0 || sel <= 0) return fail(nullptr, IRBPP_EINVAL, "need B >= 1 transitions and selected_action >= 1 (B %d, sel %d)", B, sel);
    if ((int64_t)B * (sel + 1) >= INT32_MAX) return fail(nullptr, IRBPP_EINVAL, "B * (selected_action + 1) too large (B %d, sel %d)", B, sel);
    if (atoms < 1 || atoms > AC_MAXATOMS) return fail(nullptr, IRBPP_EINVAL, "atoms %d outside [1, %d]", atoms, AC_MAXATOMS);
    if (obs_stride < (int64_t)sel * 5 + 9 + AC_HM * AC_HM)
        return fail(nullptr, IRBPP_EINVAL, "observation stride %lld < selected_action * 5 + 9 + 1024", (long long)obs_stride);
    if (scratch_bytes < grad_scratch_bytes(B, sel))
        return fail(nullptr, IRBPP_EINVAL, "scratch of %lld bytes < %lld", (long long)scratch_bytes, (long long)grad_scratch_bytes(B, sel));
    if (reinterpret_cast<uintptr_t>(scratch) & 255) return fail(nullptr, IRBPP_EINVAL, "scratch not 256-byte aligned");
    const irbpp_dqn_weights& w = *weights;
    const float* ptrs[] = {w.cand1_w, w.cand1_b, w.cand2_w, w.cand2_b, w.proj1_w, w.proj1_b, w.proj2_w, w.proj2_b, w.fc_h_v_w,
                           w.fc_h_v_b, w.fc_z_v_w, w.fc_z_v_b, w.fc_h_a_w, w.fc_h_a_b, w.fc_z_a_w, w.fc_z_a_b};
    for (const float* p : ptrs)
        if (!p) return fail(nullptr, IRBPP_EINVAL, "null weight pointer");
    memset(&P, 0, sizeof(P));
    P.w = ActorWeights{w.conv1_w, w.conv1_b, w.conv2_w, w.conv2_b, w.conv3_w, w.conv3_b, w.cand1_w, w.cand1_b, w.cand2_w,
                       w.cand2_b, w.proj1_w, w.proj1_b, w.proj2_w, w.proj2_b, w.fc_h_v_w, w.fc_h_v_b, w.fc_z_v_w,
                       w.fc_z_v_b, w.fc_h_a_w, w.fc_h_a_b, w.fc_z_a_w, w.fc_z_a_b, w.negative_slope};
    P.obs = obs; P.obs_stride = obs_stride; P.B = B; P.sel = sel; P.atoms = atoms;
    P.shape_feature = shape_feature; P.map_feature = map_feature; P.actions = actions;
    grad_scratch_layout(P, scratch);
    return IRBPP_OK;
}

// one GEMM of csrc/irbpp_grad.cuh: rows [row0, row0 + rows_host + *rows_dev), at most rows_max of them.  owner, slope
// and the weight-gradient slices come from the caller's parameter block; dev_rows_max bounds *rows_dev.
struct GemmLauncher {
    cudaStream_t s;
    int64_t cap;
    const int32_t* owner;
    float slope;
    float* part;
    int64_t dev_rows_max;
    GemmArgs base() const {
        GemmArgs g;
        memset(&g, 0, sizeof(g));
        g.owner = owner; g.slope = slope;
        return g;
    }
    // the first n rows, a count known on the host
    void first(GemmArgs& g, int n) const { g.row0 = 0; g.rows_host = n; g.rows_dev = nullptr; }
    int64_t rows_max(const GemmArgs& g) const { return g.rows_host + (g.rows_dev ? dev_rows_max : 0); }
    int grid(int64_t tiles) const { return (int)std::max<int64_t>(1, std::min<int64_t>(tiles, cap)); }
    // out[r][n] = act(in[r][:] . W[n][:] + bias[n] (+ add[owner r][n]))
    void fwd(GemmArgs g, const float* in, int K, const float* W, int ldw, int N, const float* bias, float* out, int ldo,
             int act, const float* add = nullptr, int ld_add = 0) const {
        g.a = in; g.lda = K; g.b = W; g.ldb = ldw; g.c = out; g.ldc = ldo; g.bias = bias; g.add = add; g.ld_add = ld_add;
        g.act = act; g.N = N; g.T = K;
        irbpp_grad_fwd_kernel<<<grid((rows_max(g) + GR_TILE - 1) / GR_TILE * ((N + GR_TILE - 1) / GR_TILE)), GR_THREADS, 0, s>>>(g);
    }
    // out[r][k] = (dy[r][:] . W[:][k] (+ add[owner r][k])) * act'(out[r][k]) for k < K
    void dgrad(GemmArgs g, const float* dy, int ldy, int N, const float* W, int ldw, int K, float* out, int ldo, int act,
               const float* add = nullptr, int ld_add = 0) const {
        g.a = dy; g.lda = ldy; g.b = W; g.ldb = ldw; g.c = out; g.ldc = ldo; g.add = add; g.ld_add = ld_add;
        g.act = act; g.N = K; g.T = N;
        irbpp_grad_dgrad_kernel<<<grid((rows_max(g) + GR_TILE - 1) / GR_TILE * ((K + GR_TILE - 1) / GR_TILE)), GR_THREADS, 0, s>>>(g);
    }
    // dW[n][k] (row stride ldo) = sum_r dy[r][n] x[r][k], db[n] = sum_r dy[r][n] (db may be NULL)
    void wgrad(GemmArgs g, const float* dy, int ldy, int N, const float* x, int ldx, int K, float* dw, int ldo, float* db) const {
        g.a = dy; g.lda = ldy; g.b = x; g.ldb = ldx; g.c = part; g.ldc = K; g.M = N; g.N = K;
        const int64_t tiles = (int64_t)((N + GR_TILE - 1) / GR_TILE) * ((K + GR_TILE - 1) / GR_TILE) * GR_CHUNKS;
        irbpp_grad_wgrad_kernel<<<grid(tiles), GR_THREADS, 0, s>>>(g);
        irbpp_grad_reduce_kernel<<<grid(((int64_t)N * K + N + GR_THREADS - 1) / GR_THREADS), GR_THREADS, 0, s>>>(
            part, N, K, K, dw, ldo, db);
    }
};

// the location level's row spaces
struct GradLauncher : GemmLauncher {
    const GradParams& P;
    GradLauncher(const GradParams& P_, cudaStream_t s_, int64_t cap_)
        : GemmLauncher{s_, cap_, P_.owner, P_.w.slope, P_.part, (int64_t)P_.B * P_.sel}, P(P_) {}
    // all rows (stand-ins and valid rows), the valid rows, the B transitions
    void all(GemmArgs& g) const { g.row0 = 0; g.rows_host = P.B; g.rows_dev = P.count; }
    void valid(GemmArgs& g) const { g.row0 = P.B; g.rows_host = 0; g.rows_dev = P.count; }
    void per_transition(GemmArgs& g) const { first(g, P.B); }
};

// CTAs per GEMM launch: four per SM on the device.  The tile loop and the fixed row slices make the results independent
// of the grid, so the host emulator, which runs CTAs one after another on 256 host threads each, takes one CTA.
static int64_t grad_grid_cap(int dev) {
#ifdef IRBPP_HOST_EMULATION
    (void)dev; return 1;
#else
    return gather_grid_cap(dev) / 4;
#endif
}

// the forward pass into the scratch; log_p written by the head when P.log_p is set
static void grad_forward(const GradParams& P, const GradLauncher& L) {
    const ActorWeights& w = P.w;
    const int B = P.B;
    irbpp_grad_prep_kernel<<<B, GR_THREADS, 0, L.s>>>(P);
    GemmArgs g = L.base();
    L.per_transition(g);
    L.fwd(g, P.xcat, 384, w.proj1_w, 512, AC_PROJ, w.proj1_b, P.u, AC_PROJ, ACT_NONE);            // u_b
    irbpp_grad_scatter_kernel<<<B, GR_THREADS, 0, L.s>>>(P);
    L.valid(g);
    L.fwd(g, P.cand, 4, w.cand1_w, 4, 32, w.cand1_b, P.h1, 32, ACT_LEAKY);                            // init_candidate_embed.0
    L.fwd(g, P.h1, 32, w.cand2_w, 32, AC_EMB, w.cand2_b, P.ec, AC_EMB, ACT_NONE);                     // init_candidate_embed.2
    L.fwd(g, P.ec, AC_EMB, w.proj1_w + 384, 512, AC_PROJ, nullptr, P.p0, AC_PROJ, ACT_LEAKY, P.u, AC_PROJ);  // project_layer.0
    L.fwd(g, P.p0, AC_PROJ, w.proj2_w, AC_PROJ, AC_EMB, w.proj2_b, P.emb, AC_EMB, ACT_NONE);          // project_layer.2
    L.all(g);
    L.fwd(g, P.emb, AC_EMB, w.fc_h_a_w, AC_EMB, AC_EMB, w.fc_h_a_b, P.ha, AC_EMB, ACT_RELU);          // fc_h_a
    L.fwd(g, P.ha, AC_EMB, w.fc_z_a_w, AC_EMB, P.atoms, w.fc_z_a_b, P.adv, AC_MAXATOMS, ACT_NONE);   // fc_z_a
}

int irbpp_dqn_log_prob(const irbpp_dqn_weights* weights, const float* obs, int64_t obs_stride, int32_t B,
                       int32_t selected_action, const float* shape_feature, const float* map_feature,
                       const int64_t* actions, int32_t atoms, float* log_p, void* scratch, int64_t scratch_bytes,
                       void* stream) {
    GradParams P;
    int rc = grad_params(P, weights, obs, obs_stride, B, selected_action, shape_feature, map_feature, actions, atoms,
                         scratch, scratch_bytes);
    if (rc) return rc;
    if (!log_p) return fail(nullptr, IRBPP_EINVAL, "null log_p");
    P.log_p = log_p;
    const int dev = device_of(obs);
    DeviceGuard guard(dev);
    GradLauncher L{P, (cudaStream_t)stream, grad_grid_cap(dev)};
    grad_forward(P, L);
    irbpp_grad_logp_kernel<<<B, GR_THREADS, 0, L.s>>>(P);
    return launch_status();
}

int irbpp_dqn_log_prob_backward(const irbpp_dqn_weights* weights, const float* obs, int64_t obs_stride, int32_t B,
                                int32_t selected_action, const float* shape_feature, const float* map_feature,
                                const int64_t* actions, int32_t atoms, const float* grad_log_p,
                                const irbpp_dqn_grads* grads, float* d_shape_feature, float* d_map_feature,
                                void* scratch, int64_t scratch_bytes, void* stream) {
    GradParams P;
    int rc = grad_params(P, weights, obs, obs_stride, B, selected_action, shape_feature, map_feature, actions, atoms,
                         scratch, scratch_bytes);
    if (rc) return rc;
    if (!grad_log_p || !grads || !d_shape_feature || !d_map_feature) return fail(nullptr, IRBPP_EINVAL, "null backward argument");
    const irbpp_dqn_grads& d = *grads;
    float* outs[] = {d.cand1_w, d.cand1_b, d.cand2_w, d.cand2_b, d.proj1_w, d.proj1_b, d.proj2_w, d.proj2_b, d.fc_h_v_w,
                     d.fc_h_v_b, d.fc_z_v_w, d.fc_z_v_b, d.fc_h_a_w, d.fc_h_a_b, d.fc_z_a_w, d.fc_z_a_b};
    for (float* p : outs)
        if (!p) return fail(nullptr, IRBPP_EINVAL, "null gradient output");
    P.grad_log_p = grad_log_p;
    const ActorWeights& w = P.w;
    const int dev = device_of(obs);
    DeviceGuard guard(dev);
    GradLauncher L{P, (cudaStream_t)stream, grad_grid_cap(dev)};
    grad_forward(P, L);
    irbpp_grad_head_backward_kernel<<<B, GR_THREADS, 0, L.s>>>(P);
    // Each in-place DGRAD below overwrites an activation after the last GEMM that reads it.
    GemmArgs g = L.base();
    L.all(g);
    L.wgrad(g, P.dadv, AC_MAXATOMS, atoms, P.ha, AC_EMB, AC_EMB, d.fc_z_a_w, AC_EMB, d.fc_z_a_b);            // fc_z_a
    L.dgrad(g, P.dadv, AC_MAXATOMS, atoms, w.fc_z_a_w, AC_EMB, AC_EMB, P.ha, AC_EMB, ACT_RELU);             // ha <- d pre fc_h_a
    L.wgrad(g, P.ha, AC_EMB, AC_EMB, P.emb, AC_EMB, AC_EMB, d.fc_h_a_w, AC_EMB, d.fc_h_a_b);                // fc_h_a
    L.valid(g);
    L.dgrad(g, P.ha, AC_EMB, AC_EMB, w.fc_h_a_w, AC_EMB, AC_EMB, P.emb, AC_EMB, ACT_NONE, P.dg, AC_EMB);    // emb <- d emb
    L.wgrad(g, P.emb, AC_EMB, AC_EMB, P.p0, AC_PROJ, AC_PROJ, d.proj2_w, AC_PROJ, d.proj2_b);              // project_layer.2
    L.dgrad(g, P.emb, AC_EMB, AC_EMB, w.proj2_w, AC_PROJ, AC_PROJ, P.p0, AC_PROJ, ACT_LEAKY);              // p0 <- d pre0
    L.wgrad(g, P.p0, AC_PROJ, AC_PROJ, P.ec, AC_EMB, AC_EMB, d.proj1_w + 384, 512, nullptr);               // project_layer.0, rows
    irbpp_grad_rowsum_kernel<<<B, AC_PROJ, 0, L.s>>>(P);                                                   // S_b
    L.dgrad(g, P.p0, AC_PROJ, AC_PROJ, w.proj1_w + 384, 512, AC_EMB, P.ec, AC_EMB, ACT_NONE);              // ec <- d ec
    L.wgrad(g, P.ec, AC_EMB, AC_EMB, P.h1, 32, 32, d.cand2_w, 32, d.cand2_b);                              // init_candidate_embed.2
    L.dgrad(g, P.ec, AC_EMB, AC_EMB, w.cand2_w, 32, 32, P.h1, 32, ACT_LEAKY);                              // h1 <- d pre h1
    L.wgrad(g, P.h1, 32, 32, P.cand, 4, 4, d.cand1_w, 4, d.cand1_b);                                       // init_candidate_embed.0
    L.per_transition(g);
    L.wgrad(g, P.S, AC_PROJ, AC_PROJ, P.xcat, 384, 384, d.proj1_w, 512, d.proj1_b);                        // project_layer.0, [sf; mf]
    L.dgrad(g, P.S, AC_PROJ, AC_PROJ, w.proj1_w, 512, AC_EMB, d_shape_feature, AC_EMB, ACT_NONE);
    L.dgrad(g, P.S, AC_PROJ, AC_PROJ, w.proj1_w + AC_EMB, 512, 256, d_map_feature, 256, ACT_NONE);
    L.wgrad(g, P.dq, AC_MAXATOMS, atoms, P.hv, AC_EMB, AC_EMB, d.fc_z_v_w, AC_EMB, d.fc_z_v_b);            // fc_z_v
    L.wgrad(g, P.dhv, AC_EMB, AC_EMB, P.gv, AC_EMB, AC_EMB, d.fc_h_v_w, AC_EMB, d.fc_h_v_b);               // fc_h_v
    return launch_status();
}

// ---- the height encoder and its backward pass (csrc/irbpp_height_encoder.cuh) -----------------------------------------
int64_t irbpp_height_encoder_scratch_bytes(int32_t B) {
    if (B <= 0) return -1;
    return height_encoder_scratch_bytes(B);
}

// the argument checks both entry points share, and the parameter block
static int height_encoder_params(HeightEncoderParams& P, const irbpp_height_encoder_weights* weights, const float* hm,
                                 int64_t hm_stride, int32_t B) {
    if (!weights || !hm) return fail(nullptr, IRBPP_EINVAL, "null height-encoder argument");
    if (B <= 0) return fail(nullptr, IRBPP_EINVAL, "need B >= 1 samples (B %d)", B);
    if (hm_stride < AC_HM * AC_HM) return fail(nullptr, IRBPP_EINVAL, "heightmap stride %lld < 1024", (long long)hm_stride);
    const irbpp_height_encoder_weights& w = *weights;
    const float* ptrs[] = {w.conv1_w, w.conv1_b, w.conv2_w, w.conv2_b, w.conv3_w, w.conv3_b};
    for (const float* p : ptrs)
        if (!p) return fail(nullptr, IRBPP_EINVAL, "null weight pointer");
    if (!(w.negative_slope >= 0.0f) || !std::isfinite(w.negative_slope))
        return fail(nullptr, IRBPP_EINVAL, "negative_slope %g is not a finite value >= 0", (double)w.negative_slope);
    memset(&P, 0, sizeof(P));
    P.w = HeightEncoderWeights{w.conv1_w, w.conv1_b, w.conv2_w, w.conv2_b, w.conv3_w, w.conv3_b, w.negative_slope};
    P.hm = hm; P.hm_stride = hm_stride; P.B = B;
    return IRBPP_OK;
}

int irbpp_height_encoder_forward(const irbpp_height_encoder_weights* weights, const float* hm, int64_t hm_stride,
                                 int32_t B, float* map_feature, void* stream) {
    HeightEncoderParams P;
    int rc = height_encoder_params(P, weights, hm, hm_stride, B);
    if (rc) return rc;
    if (!map_feature) return fail(nullptr, IRBPP_EINVAL, "null map_feature");
    P.map = map_feature;
    DeviceGuard guard(device_of(hm));
    irbpp_height_encoder_kernel<<<B, AC_THREADS, 0, (cudaStream_t)stream>>>(P);
    return launch_status();
}

int irbpp_height_encoder_backward(const irbpp_height_encoder_weights* weights, const float* hm, int64_t hm_stride,
                                  int32_t B, const float* grad_map_feature, const irbpp_height_encoder_grads* grads,
                                  void* scratch, int64_t scratch_bytes, void* stream) {
    HeightEncoderParams P;
    int rc = height_encoder_params(P, weights, hm, hm_stride, B);
    if (rc) return rc;
    if (!grad_map_feature || !grads || !scratch) return fail(nullptr, IRBPP_EINVAL, "null backward argument");
    const irbpp_height_encoder_grads& d = *grads;
    float* outs[] = {d.conv1_w, d.conv1_b, d.conv2_w, d.conv2_b, d.conv3_w, d.conv3_b};
    for (float* p : outs)
        if (!p) return fail(nullptr, IRBPP_EINVAL, "null gradient output");
    if (scratch_bytes < height_encoder_scratch_bytes(B))
        return fail(nullptr, IRBPP_EINVAL, "scratch of %lld bytes < %lld", (long long)scratch_bytes, (long long)height_encoder_scratch_bytes(B));
    if (reinterpret_cast<uintptr_t>(scratch) & 255) return fail(nullptr, IRBPP_EINVAL, "scratch not 256-byte aligned");
    P.d_map = grad_map_feature;
    P.part = static_cast<float*>(scratch);
    const int dev = device_of(hm);
    DeviceGuard guard(dev);
    cudaStream_t s = (cudaStream_t)stream;
    irbpp_height_encoder_backward_kernel<<<B, AC_THREADS, 0, s>>>(P);
    const HeightEncoderGrads G{d.conv1_w, d.conv1_b, d.conv2_w, d.conv2_b, d.conv3_w, d.conv3_b};
    int64_t rows = B, stride = HE_GRADS;
    for (;;) {                                   // groups of HE_GROUP samples, in place, until one row is left
        const int64_t groups = (rows + HE_GROUP - 1) / HE_GROUP;
        const int64_t blocks = std::min<int64_t>((groups * HE_GRADS + AC_THREADS - 1) / AC_THREADS, gather_grid_cap(dev));
        irbpp_height_encoder_reduce_kernel<<<(int)blocks, AC_THREADS, 0, s>>>(P.part, stride, (int32_t)rows, G);
        if (groups == 1) break;
        rows = groups;
        stride *= HE_GROUP;
    }
    return launch_status();
}

// ---- the gradient pass of Agent.learn at the order level (csrc/irbpp_order_grad.cuh) ---------------------------------
int64_t irbpp_dqn_order_log_prob_scratch_bytes(int32_t B, int32_t k, int32_t S) {
    if (B <= 0 || k < 2 || k > OA_MAXK || S <= 0 || (int64_t)B * k * 384 >= INT32_MAX) return -1;
    return order_grad_scratch_bytes(B, k, S);
}

// the argument checks both entry points share, and the parameter block
static int order_grad_params(OrderGradParams& P, const irbpp_dqn_order_weights* weights, const float* obs,
                             int64_t obs_stride, int32_t B, int32_t k, const float* shape_features, int32_t S,
                             const float* map_feature, const int64_t* actions, int32_t atoms, void* scratch,
                             int64_t scratch_bytes) {
    if (!weights || !obs || !shape_features || !map_feature || !actions || !scratch)
        return fail(nullptr, IRBPP_EINVAL, "null order log-prob argument");
    if (B <= 0 || S <= 0) return fail(nullptr, IRBPP_EINVAL, "need B >= 1 transitions and S >= 1 shapes (B %d, S %d)", B, S);
    if (k < 2 || k > OA_MAXK) return fail(nullptr, IRBPP_EINVAL, "buffer size k %d outside [2, %d]", k, OA_MAXK);
    if ((int64_t)B * k * 384 >= INT32_MAX) return fail(nullptr, IRBPP_EINVAL, "B * k too large (B %d, k %d)", B, k);
    if (atoms < 1 || atoms > AC_MAXATOMS) return fail(nullptr, IRBPP_EINVAL, "atoms %d outside [1, %d]", atoms, AC_MAXATOMS);
    if (obs_stride < (int64_t)k + AC_HM * AC_HM)
        return fail(nullptr, IRBPP_EINVAL, "observation stride %lld < k + 1024", (long long)obs_stride);
    if (scratch_bytes < order_grad_scratch_bytes(B, k, S))
        return fail(nullptr, IRBPP_EINVAL, "scratch of %lld bytes < %lld", (long long)scratch_bytes, (long long)order_grad_scratch_bytes(B, k, S));
    if (reinterpret_cast<uintptr_t>(scratch) & 255) return fail(nullptr, IRBPP_EINVAL, "scratch not 256-byte aligned");
    const irbpp_dqn_order_weights& w = *weights;
    const float* ptrs[] = {w.gat1_w, w.gat1_b, w.gat2_w, w.gat2_b, w.wq, w.wk, w.wv, w.wo_w, w.wo_b, w.ff1_w, w.ff1_b,
                           w.ff2_w, w.ff2_b, w.fc_h_v_w, w.fc_h_v_b, w.fc_z_v_w, w.fc_z_v_b, w.fc_h_a_w, w.fc_h_a_b,
                           w.fc_z_a_w, w.fc_z_a_b};
    for (const float* p : ptrs)
        if (!p) return fail(nullptr, IRBPP_EINVAL, "null weight pointer");
    memset(&P, 0, sizeof(P));
    P.w = OrderWeights{w.conv1_w, w.conv1_b, w.conv2_w, w.conv2_b, w.conv3_w, w.conv3_b, w.gat1_w, w.gat1_b, w.gat2_w,
                       w.gat2_b, w.wq, w.wk, w.wv, w.wo_w, w.wo_b, w.ff1_w, w.ff1_b, w.ff2_w, w.ff2_b, w.fc_h_v_w,
                       w.fc_h_v_b, w.fc_z_v_w, w.fc_z_v_b, w.fc_h_a_w, w.fc_h_a_b, w.fc_z_a_w, w.fc_z_a_b, w.negative_slope};
    P.obs = obs; P.obs_stride = obs_stride; P.B = B; P.k = k; P.S = S; P.atoms = atoms;
    P.shape_features = shape_features; P.map_feature = map_feature; P.actions = actions;
    order_grad_scratch_layout(P, scratch);
    return IRBPP_OK;
}

static void order_grad_add(float* y, const float* x, int64_t n, const GemmLauncher& L) {
    irbpp_order_grad_add_kernel<<<L.grid((n + GR_THREADS - 1) / GR_THREADS), GR_THREADS, 0, L.s>>>(y, x, n);
}

// the forward pass into the scratch; log_p written by the head when P.log_p is set
static void order_grad_forward(const OrderGradParams& P, const GemmLauncher& L) {
    const OrderWeights& w = P.w;
    const int B = P.B, R = P.B * P.k;
    irbpp_order_grad_prep_kernel<<<B, GR_THREADS, 0, L.s>>>(P);
    GemmArgs g = L.base();
    L.first(g, B);
    L.fwd(g, P.map_feature, 256, w.gat1_w + AC_EMB, 384, AC_PROJ, w.gat1_b, P.u, AC_PROJ, ACT_NONE);     // u_b
    L.first(g, R);
    L.fwd(g, P.xs, AC_EMB, w.gat1_w, 384, AC_PROJ, nullptr, P.p0, AC_PROJ, ACT_LEAKY, P.u, AC_PROJ);      // gat_project_layer.0
    L.fwd(g, P.p0, AC_PROJ, w.gat2_w, AC_PROJ, AC_EMB, w.gat2_b, P.h, AC_EMB, ACT_NONE);                  // gat_project_layer.2
    L.fwd(g, P.h, AC_EMB, P.wqkv, AC_EMB, 384, nullptr, P.qkv, 384, ACT_NONE);                            // Q | K | V
    irbpp_order_grad_attn_kernel<<<B, GR_THREADS, 0, L.s>>>(P);
    L.fwd(g, P.heads, AC_EMB, w.wo_w, AC_EMB, AC_EMB, w.wo_b, P.h1, AC_EMB, ACT_NONE);                    // W_out
    order_grad_add(P.h1, P.h, (int64_t)R * AC_EMB, L);                                                    // h1
    L.fwd(g, P.h1, AC_EMB, w.ff1_w, AC_EMB, AC_EMB, w.ff1_b, P.f1, AC_EMB, ACT_RELU);                    // FFN
    L.fwd(g, P.f1, AC_EMB, w.ff2_w, AC_EMB, AC_EMB, w.ff2_b, P.h2, AC_EMB, ACT_NONE);
    order_grad_add(P.h2, P.h1, (int64_t)R * AC_EMB, L);                                                   // h2
    L.fwd(g, P.h2, AC_EMB, w.fc_h_a_w, AC_EMB, AC_EMB, w.fc_h_a_b, P.ha, AC_EMB, ACT_RELU);              // fc_h_a
    L.fwd(g, P.ha, AC_EMB, w.fc_z_a_w, AC_EMB, P.atoms, w.fc_z_a_b, P.adv, AC_MAXATOMS, ACT_NONE);       // fc_z_a
}

int irbpp_dqn_order_log_prob(const irbpp_dqn_order_weights* weights, const float* obs, int64_t obs_stride, int32_t B,
                             int32_t k, const float* shape_features, int32_t S, const float* map_feature,
                             const int64_t* actions, int32_t atoms, float* log_p, void* scratch, int64_t scratch_bytes,
                             void* stream) {
    OrderGradParams P;
    int rc = order_grad_params(P, weights, obs, obs_stride, B, k, shape_features, S, map_feature, actions, atoms, scratch,
                               scratch_bytes);
    if (rc) return rc;
    if (!log_p) return fail(nullptr, IRBPP_EINVAL, "null log_p");
    P.log_p = log_p;
    const int dev = device_of(obs);
    DeviceGuard guard(dev);
    const GemmLauncher L{(cudaStream_t)stream, grad_grid_cap(dev), P.owner, P.w.slope, P.part, 0};
    order_grad_forward(P, L);
    irbpp_order_grad_logp_kernel<<<B, GR_THREADS, 0, L.s>>>(P);
    return launch_status();
}

int irbpp_dqn_order_log_prob_backward(const irbpp_dqn_order_weights* weights, const float* obs, int64_t obs_stride,
                                      int32_t B, int32_t k, const float* shape_features, int32_t S,
                                      const float* map_feature, const int64_t* actions, int32_t atoms,
                                      const float* grad_log_p, const irbpp_dqn_order_grads* grads,
                                      float* d_shape_features, float* d_map_feature, void* scratch,
                                      int64_t scratch_bytes, void* stream) {
    OrderGradParams P;
    int rc = order_grad_params(P, weights, obs, obs_stride, B, k, shape_features, S, map_feature, actions, atoms, scratch,
                               scratch_bytes);
    if (rc) return rc;
    if (!grad_log_p || !grads || !d_shape_features || !d_map_feature)
        return fail(nullptr, IRBPP_EINVAL, "null backward argument");
    const irbpp_dqn_order_grads& d = *grads;
    float* outs[] = {d.gat1_w, d.gat1_b, d.gat2_w, d.gat2_b, d.wq, d.wk, d.wv, d.wo_w, d.wo_b, d.ff1_w, d.ff1_b, d.ff2_w,
                     d.ff2_b, d.fc_h_v_w, d.fc_h_v_b, d.fc_z_v_w, d.fc_z_v_b, d.fc_h_a_w, d.fc_h_a_b, d.fc_z_a_w, d.fc_z_a_b};
    for (float* p : outs)
        if (!p) return fail(nullptr, IRBPP_EINVAL, "null gradient output");
    P.grad_log_p = grad_log_p;
    const OrderWeights& w = P.w;
    const int R = B * k;
    const int dev = device_of(obs);
    DeviceGuard guard(dev);
    const GemmLauncher L{(cudaStream_t)stream, grad_grid_cap(dev), P.owner, P.w.slope, P.part, 0};
    order_grad_forward(P, L);
    irbpp_order_grad_head_backward_kernel<<<B, GR_THREADS, 0, L.s>>>(P);
    // Each in-place DGRAD below overwrites an activation after the last GEMM that reads it.
    GemmArgs g = L.base();
    L.first(g, R);
    L.wgrad(g, P.dadv, AC_MAXATOMS, atoms, P.ha, AC_EMB, AC_EMB, d.fc_z_a_w, AC_EMB, d.fc_z_a_b);             // fc_z_a
    L.dgrad(g, P.dadv, AC_MAXATOMS, atoms, w.fc_z_a_w, AC_EMB, AC_EMB, P.ha, AC_EMB, ACT_RELU);              // ha <- d pre fc_h_a
    L.wgrad(g, P.ha, AC_EMB, AC_EMB, P.h2, AC_EMB, AC_EMB, d.fc_h_a_w, AC_EMB, d.fc_h_a_b);                  // fc_h_a
    L.dgrad(g, P.ha, AC_EMB, AC_EMB, w.fc_h_a_w, AC_EMB, AC_EMB, P.h2, AC_EMB, ACT_NONE, P.dg, AC_EMB);      // h2 <- d h2
    L.wgrad(g, P.h2, AC_EMB, AC_EMB, P.f1, AC_EMB, AC_EMB, d.ff2_w, AC_EMB, d.ff2_b);                        // FFN.2
    L.dgrad(g, P.h2, AC_EMB, AC_EMB, w.ff2_w, AC_EMB, AC_EMB, P.f1, AC_EMB, ACT_RELU);                       // f1 <- d pre f1
    L.wgrad(g, P.f1, AC_EMB, AC_EMB, P.h1, AC_EMB, AC_EMB, d.ff1_w, AC_EMB, d.ff1_b);                        // FFN.0
    L.dgrad(g, P.f1, AC_EMB, AC_EMB, w.ff1_w, AC_EMB, AC_EMB, P.h1, AC_EMB, ACT_NONE);
    order_grad_add(P.h1, P.h2, (int64_t)R * AC_EMB, L);                                                      // h1 <- d h1
    L.wgrad(g, P.h1, AC_EMB, AC_EMB, P.heads, AC_EMB, AC_EMB, d.wo_w, AC_EMB, d.wo_b);                      // W_out
    L.dgrad(g, P.h1, AC_EMB, AC_EMB, w.wo_w, AC_EMB, AC_EMB, P.heads, AC_EMB, ACT_NONE);                    // heads <- d heads
    irbpp_order_grad_attn_backward_kernel<<<B, GR_THREADS, 0, L.s>>>(P);                                     // d Q | K | V
    float* dw[] = {d.wq, d.wk, d.wv};
    for (int m = 0; m < 3; ++m)
        L.wgrad(g, P.dqkv + m * AC_EMB, 384, AC_EMB, P.h, AC_EMB, AC_EMB, dw[m], AC_EMB, nullptr);         // W_query, W_key, W_val
    L.dgrad(g, P.dqkv, 384, 384, P.wqkv, AC_EMB, AC_EMB, P.h, AC_EMB, ACT_NONE);
    order_grad_add(P.h, P.h1, (int64_t)R * AC_EMB, L);                                                       // h <- d h
    L.wgrad(g, P.h, AC_EMB, AC_EMB, P.p0, AC_PROJ, AC_PROJ, d.gat2_w, AC_PROJ, d.gat2_b);                   // gat_project_layer.2
    L.dgrad(g, P.h, AC_EMB, AC_EMB, w.gat2_w, AC_PROJ, AC_PROJ, P.p0, AC_PROJ, ACT_LEAKY);                  // p0 <- d pre0
    irbpp_order_grad_rank_kernel<<<(R + GR_THREADS - 1) / GR_THREADS, GR_THREADS, 0, L.s>>>(P);
    irbpp_order_grad_segsum_kernel<<<S + B, GR_THREADS, 0, L.s>>>(P);                                       // Sid, Sb
    L.first(g, S);                                                                                           // gat_project_layer.0
    L.wgrad(g, P.Sid, AC_PROJ, AC_PROJ, P.shape_features, AC_EMB, AC_EMB, d.gat1_w, 384, nullptr);
    L.dgrad(g, P.Sid, AC_PROJ, AC_PROJ, w.gat1_w, 384, AC_EMB, d_shape_features, AC_EMB, ACT_NONE);
    L.first(g, B);
    L.wgrad(g, P.Sb, AC_PROJ, AC_PROJ, P.map_feature, 256, 256, d.gat1_w + AC_EMB, 384, d.gat1_b);
    L.dgrad(g, P.Sb, AC_PROJ, AC_PROJ, w.gat1_w + AC_EMB, 384, 256, d_map_feature, 256, ACT_NONE);
    L.wgrad(g, P.dq, AC_MAXATOMS, atoms, P.hv, AC_EMB, AC_EMB, d.fc_z_v_w, AC_EMB, d.fc_z_v_b);              // fc_z_v
    L.wgrad(g, P.dhv, AC_EMB, AC_EMB, P.gv, AC_EMB, AC_EMB, d.fc_h_v_w, AC_EMB, d.fc_h_v_b);                 // fc_h_v
    return launch_status();
}

int irbpp_debug_phase_cycles(irbpp_handle h, int32_t enable, uint64_t* out8) {
    if (!h) return IRBPP_EINVAL;
    DeviceGuard guard(h->cfg.device);
    if (!h->phase_dev) CUDA_TRY(h, dev_alloc(h, &h->phase_dev, 8));
    CUDA_TRY(h, cudaDeviceSynchronize());
    if (out8) CUDA_TRY(h, cudaMemcpy(out8, h->phase_dev, 8 * sizeof(uint64_t), cudaMemcpyDeviceToHost));
    CUDA_TRY(h, cudaMemset(h->phase_dev, 0, 8 * sizeof(uint64_t)));
    h->P.phase_cycles = enable ? h->phase_dev : nullptr;
    return IRBPP_OK;
}

}  // extern "C"
