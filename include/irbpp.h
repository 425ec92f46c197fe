/*
 * irbpp.h -- C ABI of the H100-native (sm_90a) IR-BPP packing-environment hot path.
 *
 * The reference (alexfrom0815/IR-BPP) has no FFI layer: its boundary is the Python VecEnv class
 * contract of envs.py:67-165 / wrapper/vec_env.py:29-108 / wrapper/shmem_vec_env.py:20-157.
 * Each entry point below states the reference interface it replaces (paths relative to the
 * reference root).  Host code (Python `irbpp_b200.vec_env.GpuVecEnv`) binds these with ctypes;
 * INTEGRATION.md shows the binding a reference maintainer would add.
 *
 * Conventions
 *   - plain pointers and sizes only; no C++ / torch types cross this boundary
 *   - every function returns 0 on success or a negative IRBPP_E* code; the message is available
 *     from irbpp_last_error(handle) (thread-unsafe per handle; one host thread per handle)
 *   - "dev" pointers are CUDA device pointers owned by the caller (e.g. torch tensors);
 *     "host" pointers are ordinary host memory owned by the caller
 *   - all GPU work is ordered on the `stream` argument (a cudaStream_t passed as void*, NULL =
 *     default stream); the library owns its internal state and result staging buffers
 *   - there is no CPU fallback: without a CUDA device irbpp_create fails with IRBPP_ECUDA
 */
#ifndef IRBPP_H_
#define IRBPP_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define IRBPP_ABI_VERSION 2

#define IRBPP_OK        0
#define IRBPP_EINVAL   -1   /* bad argument / unsupported configuration */
#define IRBPP_ECUDA    -2   /* CUDA runtime error */
#define IRBPP_ESTATE   -3   /* call order violated (e.g. step_async twice; vec_env.py:7-26) */
#define IRBPP_EDEVICE  -4   /* a kernel flagged an environment error (see irbpp_last_error) */

/* Per-env codes behind IRBPP_EDEVICE (irbpp_step_result.error, "env i reported device error code c"). */
#define IRBPP_ERR_ACTION    2   /* candidate row / pose out of range */
#define IRBPP_ERR_ORDER     3   /* get_action_candidates: order action not in [0, k) */
#define IRBPP_ERR_LEVEL     4   /* a drop height quantised outside the level range */
#define IRBPP_ERR_TRAJ_END  5   /* the bin drew past the end of its trajectory (irbpp_set_trajectories); the
                                 * reference appends None there and fails on it (IRcreator.py:94-101) */
#define IRBPP_ERR_CONTOUR   6   /* a contour longer than the overflow buffer (4 points per pose of the action grid:
                                 * no contour is that long, so the code is not expected) */

typedef struct irbpp_env* irbpp_handle;

/* PackingGame.__init__ / Space.__init__ settings that reach the hot path
 * (environment/physics0/binPhy.py:25-49, space.py:15-24, arguments.py:11-96,115). */
typedef struct irbpp_config {
    int32_t num_envs;          /* N bins resident on this GPU (args.num_processes) */
    int32_t num_rotations;     /* ZRotNum = --resolutionRot (arguments.py:85,117) */
    int32_t selected_action;   /* --selectedAction, candidate rows per observation (default 500) */
    int32_t buffer_size;       /* --bufferSize k; k > 1 selects the order->location protocol */
    double  bin_dimension[3];  /* [0.32, 0.32, 0.30] (arguments.py:115) */
    double  resolution_act;    /* --resolutionA: 0.02 (16x16 actions) or resolution_h (32x32 actions) */
    double  resolution_h;      /* --resolutionH 0.01 */
    double  resolution_z;      /* --resolutionZ 0.01 (cvTools.py:77 heightResolution) */
    int32_t device;            /* CUDA device ordinal */
    int32_t approx_legacy;     /* 0: approxPolyDP as cv2 4.13 (segment distance); 1: legacy line distance */
} irbpp_config;

/* Host views of the per-env results of the last step (library-owned pinned memory; two blocks alternate, so the
 * views stay valid until the SECOND next irbpp_step_async on the handle).  Replaces the (rews, dones, infos) tuple of
 * ShmemVecEnv.step_wait (wrapper/shmem_vec_env.py:76-81) and the Monitor episode info
 * (wrapper/monitor.py:58-75). */
typedef struct irbpp_step_result {
    const float*   reward;      /* [N]  10*volume/bin_volume on success, 0 otherwise (binPhy.py:299-322) */
    const uint8_t* done;        /* [N]  1 when the placement failed and the bin was auto-reset */
    const uint8_t* valid;       /* [N]  info['Valid'] (1 without the PyBullet settle; 0 for a bin with no
                                 *      trajectory left, see irbpp_set_trajectories) */
    const uint8_t* error;       /* [N]  non-zero: kernel-detected error for that env (IRBPP_ERR_*) */
    const int32_t* counter;     /* [N]  info['counter'] = items packed, meaningful where done */
    const int32_t* ep_len;      /* [N]  info['episode']['l'], meaningful where done */
    const double*  ratio;       /* [N]  info['ratio'] = packed volume / bin volume, where done */
    const double*  ep_reward;   /* [N]  unrounded sum of episode rewards (Monitor rounds to 6 dp) */
} irbpp_step_result;

/* The same struct pointing at the device-resident copies of the arrays (for callers that keep the loop on the GPU). */
typedef irbpp_step_result irbpp_device_result;

int irbpp_abi_version(void);

/* Replaces: make_vec_envs + N x PackingGame(args) construction (envs.py:67-99, binPhy.py:22-116). */
int irbpp_create(const irbpp_config* cfg, irbpp_handle* out);
int irbpp_destroy(irbpp_handle h);
const char* irbpp_last_error(irbpp_handle h);   /* h may be NULL: error of the last failed create */

/* Observation lengths: binPhy.py:87-98.  loc = selected_action*5 + 9 + Hx*Hy; order = k + Hx*Hy;
 * obs_len = (k > 1) ? order : loc. */
int irbpp_obs_len(irbpp_handle h, int32_t* obs_len, int32_t* loc_obs_len, int32_t* order_obs_len);

/* Replaces: args.shotInfo / args.shapeDict / args.infoDict (tools.py:248-279, binPhy.py:31-33).
 * Host arrays: dims[S,R,4] = (w, h, wA, hA) from space.py:104-106; ext[S,R,3] raw mesh extents;
 * vol[S]; maps = float64 pool with the four [w,h] row-major tables T | B | maskT | maskB of (s,r)
 * starting at offsets[s,r] (in doubles). */
int irbpp_load_shapes(irbpp_handle h, int32_t num_shapes, int32_t num_rotations,
                      const int32_t* dims, const double* ext, const double* vol,
                      const double* maps, const int64_t* offsets, int64_t maps_len);

/* Replaces: the item creators (environment/physics0/IRcreator.py:6-103).  ids[N,L] host int32; env e
 * draws ids[e, cursor % L] on every generate_item; the cursor persists across episodes.  Calling it again
 * replaces the sequences and restarts the cursors. */
int irbpp_set_sequences(irbpp_handle h, const int32_t* ids, int32_t length);

/* Alternative to explicit sequences: env e draws  id = mix(seed, e, draw counter) mod num_shapes  on the device
 * (splitmix64 finaliser, csrc/irbpp_kernels.cuh item_rng) -- i.i.d. uniform ids without a period, the stand-in
 * for RandomItemCreator (environment/physics0/IRcreator.py:26-33: np.random.choice on every generate_item). */
int irbpp_set_item_rng(irbpp_handle h, uint64_t seed);

/* Replaces: RandomInstanceCreator / RandomCateCreator (IRcreator.py:35-72; what arguments.py:109-112 selects for
 * training).  A CSR table of num_groups non-empty groups (host group_offsets int32[G + 1], offsets[0] = 0, strictly
 * increasing; members int32[offsets[G]] item ids).  Draw d of env e:  z = splitmix64(seed, e, d) (the value
 * irbpp_set_item_rng keeps the top half of),  g = hi32(z) mod G,  id = members[offsets[g] + lo32(z) mod n_g]:
 * a group uniformly, then a member uniformly.  The modulo bias is at most G / 2^32 and n_g / 2^32.
 * Like irbpp_set_sequences it replaces the item source and restarts every bin's item state.
 * IRBPP_EINVAL on an empty group, offsets that do not increase, or an id out of range. */
int irbpp_set_item_groups(irbpp_handle h, uint64_t seed, int32_t num_groups, const int32_t* group_offsets,
                          const int32_t* members);

/* Replaces: LoadItemCreator (IRcreator.py:74-101) over test_sequence.pt, the evaluation protocol of tools.test.
 * A pool of num_trajectories ragged trajectories (host items int32[offsets[T]], offsets int64[T + 1], offsets[0] = 0,
 * non-decreasing) and a window [first, first + count).  Episode j of env e (j counts the env's resets and
 * auto-resets since this call) plays trajectory t = first + e + j * N from its item 0; every draw (the reset's
 * preview of max(k, 1) items, the refill after each placement) takes the next item.  With N = 1 and first = 1
 * this is tools.test's sequence of trajectories.  A draw past the end of a trajectory is error code
 * IRBPP_ERR_TRAJ_END.  When t >= first + count the env is idle: every call leaves its state alone, its
 * observation rows are zero, its step reports reward 0, done 0, valid 0, error 0 whatever the action, and
 * irbpp_heuristic_actions returns index -1 for it.  Replaces the item source and restarts every bin's item state.
 * IRBPP_EINVAL on an id out of range, decreasing offsets, a window outside the pool or a trajectory of the window
 * shorter than the reset's preview. */
int irbpp_set_trajectories(irbpp_handle h, const int32_t* items, const int64_t* offsets, int32_t num_trajectories,
                           int32_t first, int32_t count);

/* Replaces: envs.reset() (envs.py:149-152 -> ShmemVecEnv.reset, shmem_vec_env.py:60-66; and
 * reset_specific, :113-118, when `which` (host uint8[N], 1 = reset) is not NULL).
 * obs_out: dev float32 [N, obs_len]; rows of envs not reset are left untouched. */
int irbpp_reset(irbpp_handle h, const uint8_t* which, float* obs_out, void* stream);

/* Replaces: envs.step_async (envs.py:154-159 -> shmem_vec_env.py:70-74).  actions: int64[N], a host
 * pointer (copied through pinned staging) or a device pointer when actions_on_device != 0.
 * obs_out: dev float32 [N, obs_len], written in stream order.  Returns IRBPP_ESTATE if a step is
 * already pending. */
int irbpp_step_async(irbpp_handle h, const int64_t* actions, int32_t actions_on_device,
                     float* obs_out, void* stream);

/* Replaces: envs.step_wait (envs.py:161-165 -> shmem_vec_env.py:76-81).  Copies the per-env results to
 * pinned host memory, synchronises the step's stream and fills *out.  out may be NULL (sync only). */
int irbpp_step_wait(irbpp_handle h, irbpp_step_result* out);

/* Device-side loop variant: marks the pending step as consumed without any host copy or sync and
 * returns device views of the result arrays (valid in stream order). */
int irbpp_step_wait_device(irbpp_handle h, irbpp_device_result* out);

/* The device copies of the per-env result arrays (fixed for the life of the handle; every step writes them in
 * stream order, also when its results are delivered to the host): what a device-resident replay buffer reads. */
int irbpp_device_results(irbpp_handle h, irbpp_device_result* out);

/* Replaces: envs.get_action_candidates(order_actions) (wrapper/shmem_vec_env.py:99-102 ->
 * binPhy.py:161-169), buffer_size > 1 only.  order_actions: int64[N] host or device.
 * loc_obs_out: dev float32 [N, loc_obs_len]. */
int irbpp_get_action_candidates(irbpp_handle h, const int64_t* order_actions, int32_t on_device,
                                float* loc_obs_out, void* stream);

/* Replaces: PackingGame.get_all_possible_observation (binPhy.py:171-180), buffer_size > 1 only.
 * out: dev float32 [N, k * loc_obs_len].  Leaves the candidate state of slot k-1 current. */
int irbpp_get_all_possible_observation(irbpp_handle h, float* out, void* stream);

/* Replaces: Space.get_heuristic_action(dirIdx, method, next_item_ID, next_item)
 * (environment/physics0/space.py:162-227) for every bin, over the drop heights / feasibility mask of
 * the bin's current item (the scan of the last reset / step (buffer_size 1) or
 * get_action_candidates).  method: IRBPP_HEUR_*; dir_idx 0..3 selects the X/Y flips (:163-166).
 * poses_out: int32[N,3] (rotIdx, lx, ly); index_out: int64[N] row of that pose in the bin's candidate
 * table (what envs.step takes), -1 if the pose is not a candidate; either may be NULL; both host
 * pointers, or device pointers when outputs_on_device != 0 (then nothing is synchronised).
 * The reference's RANDOM branch raises on every call and has no counterpart.
 * Returns IRBPP_ESTATE when no current scan exists (before reset, or buffer_size > 1 without
 * get_action_candidates). */
#define IRBPP_HEUR_MINZ      0
#define IRBPP_HEUR_DBLF      1
#define IRBPP_HEUR_FIRSTFIT  2
#define IRBPP_HEUR_HM        3
int irbpp_heuristic_actions(irbpp_handle h, int32_t method, int32_t dir_idx, int32_t* poses_out,
                            int64_t* index_out, int32_t outputs_on_device, void* stream);

/* irbpp_step_async with explicit poses instead of candidate rows: poses int64[N], each
 * (rotIdx * Ax + lx) * Ay + ly -- the (rotIdx, lx, ly) binPhy.action_to_position (binPhy.py:234-236)
 * would have read from candidates[action].  Everything after that line of PackingGame.step is
 * unchanged (prejudge, placement, reward, auto-reset); pair with irbpp_step_wait as usual. */
int irbpp_step_poses_async(irbpp_handle h, const int64_t* poses, int32_t poses_on_device,
                           float* obs_out, void* stream);

/* ---- parity / debugging views (float64, host destinations; any pointer may be NULL) ---- */

/* Current bin state: heightmap [N,Hx,Hy] row-major, the candidate table [N,selected_action,5]
 * (rot, x, y decoded from the packed state; H and V columns are 0), next item ids [N, max(k,1)]. */
int irbpp_debug_state(irbpp_handle h, double* heightmap, int32_t* queue, int32_t* cursor,
                      int32_t* packed_count);
int irbpp_debug_set_heightmap(irbpp_handle h, const double* heightmap /* host [N,Hx,Hy] */);

/* Run the scan + candidate extraction of space.py:98-129 / cvTools.py:61-103 / binPhy.py:205-225 for
 * item_ids[N] (host int32) on the CURRENT heightmaps without touching env state.  Host outputs:
 * posZmap, posZValid, naiveMask float64 [N,R,Ax,Ay]; cand float64 [N,selected_action,5];
 * num_hull int32 [N] = K before select/pad (0 = fallback path taken). */
int irbpp_debug_scan(irbpp_handle h, const int32_t* item_ids, double* posZmap, double* posZValid,
                     double* naiveMask, double* cand, int32_t* num_hull);

/* Candidate extraction alone on caller-supplied maps: posZValid, mask host float64 [N,R,Ax,Ay] ->
 * cand [N,selected_action,5], num_hull [N]  (cvTools.getConvexHullActions + binPhy.py:205-225). */
int irbpp_debug_hulls(irbpp_handle h, const double* posZValid, const double* mask, double* cand,
                      int32_t* num_hull);

/* Kernel launches issued by this handle so far (bench.py's gpu_launches). */
int64_t irbpp_launch_count(irbpp_handle h);

/* ---- compact observations for the rollout gather (SURVEY.md 8e) ----------------------------------------------
 * The float32 location observation [N, sel*5 + 9 + 1024] (binPhy.py:196-227) re-encoded without loss as u16 poses, f32
 * heights, one mask bit per row, the item id and the f32 heightmap: irbpp_packed_obs_bytes(sel) bytes per bin (7 184 at
 * sel = 500, 51 %).  What `sharding.CompactRolloutGather` sends between GPUs; device pointers, handle-free. */
int irbpp_packed_obs_bytes(int32_t selected_action);
int irbpp_pack_observations(const float* obs, int64_t obs_stride, int32_t selected_action, int32_t n, void* packed, void* stream);
int irbpp_unpack_observations(const void* packed, int32_t selected_action, int32_t n, float* obs, int64_t obs_stride, void* stream);

/* ---- point clouds of the next items (SURVEY.md 8(f)3) --------------------------------------------------------
 * Replaces model.py:328-335 / :366-372: `shapeArray[next_item_ID.cpu()]` (a HOST gather of [B, P, 3] float32 rows),
 * `np.random.randint(P, size=samplePointsNum)` (one index set shared by the batch) and the host-to-device copy
 * of [B, n, 3] on every forward pass.  Handle-free; every pointer is a DEVICE pointer owned by the caller;
 * errors are reported through irbpp_last_error(NULL).
 *   shape_array  float32 [S, P, 3], resident on the device (agent.py:26 `args.shapeArray`)
 *   item ids     ids int32 [B] when not NULL, else (int) obs[b * obs_stride + item_col]  (the next_item_vec slot of
 *                the observation: item_col = selected_action * 5, binPhy.py:191,227; model.py:327)
 *   index set    index j = mix(seed, counter, j) mod P  (counter-based, uniform with replacement like randint;
 *                csrc/irbpp_pointnet.cuh pn_index; pass a new counter per forward pass)
 * irbpp_sample_point_clouds: out float32 [B, n_points, 3] = shapeArray[item_b][indices] (drop-in for `nextShape`);
 *   indices_out int32 [n_points] or NULL.
 * irbpp_shape_features: the fused path -- shapeEncoder (model.py:266-270: Linear(3,128), LeakyReLU, Linear(128,128),
 *   LeakyReLU; weights in nn.Linear layout, float32) and the max over the points (model.py:335), evaluated once per
 *   library SHAPE (the index set is shared by the batch, so the feature depends on the shape only) and gathered per
 *   bin: out float32 [B, 128].  scratch_keys: int32 [S * 128] work space. */
int irbpp_sample_point_clouds(const float* shape_array, int32_t S, int32_t P, const float* obs, int64_t obs_stride,
                              int32_t item_col, const int32_t* ids, int32_t B, uint64_t seed, uint64_t counter,
                              int32_t n_points, float* out, int32_t* indices_out, void* stream);
int irbpp_shape_features(const float* shape_array, int32_t S, int32_t P, const float* obs, int64_t obs_stride,
                         int32_t item_col, const int32_t* ids, int32_t B, uint64_t seed, uint64_t counter,
                         int32_t n_points, const float* W1, const float* b1, const float* W2, const float* b2,
                         float negative_slope, int32_t* scratch_keys, float* out, void* stream);

/* ---- prioritized n-step replay (memory.py:15-208) -------------------------------------------------------------
 * Replaces: the N host ReplayMemory objects of main.py:61-63, their per-bin appends (trainer.py:184-186), the per-memory
 * sample of Agent.learn (agent.py:69-82) and its per-transition priority write-back (agent.py:123-124).  M memories of
 * capacity C share caller-owned DEVICE arrays, memory-major; handle-free; errors through irbpp_last_error(NULL).
 *   states float32 [M][C][obs_len], timesteps int32 [M][C], actions int64 [M][C], rewards float32 [M][C],
 *   nonterminals uint8 [M][C], tree float32 [M][2C-1] (heap layout: leaf j is node C-1+j), state [M] below.
 * The reference stores actions as float32 and returns them as int64, which is exact below 2^24; they are kept as
 * int64 here.  Every call issues one kernel on `stream`. */
typedef struct irbpp_replay_state {
    int32_t index;             /* next ring slot to write */
    int32_t full;              /* the ring has wrapped at least once */
    int32_t t;                 /* timestep within the current episode */
    float   max;               /* running maximum priority, starts at 1, never decreases */
} irbpp_replay_state;

typedef struct irbpp_replay_memory {
    int32_t num_memories, capacity, obs_len;   /* M, C >= 2, obs_len */
    float* states;
    int32_t* timesteps;
    int64_t* actions;
    float* rewards;
    uint8_t* nonterminals;
    float* tree;
    irbpp_replay_state* state;
} irbpp_replay_memory;

/* Outputs of one sample call, device arrays of B = G * k rows (row g * k + i is stratum i of memory mem_ids[g]):
 * tree_idx int64 [B] (-1 where the sample failed), states / next_states float32 [B][obs_len], actions int64 [B],
 * returns / nonterminals / weights float32 [B]; attempts int32 [B] (descents used) and error int32 [B]
 * (IRBPP_REPLAY_ERR_*) may be NULL. */
typedef struct irbpp_replay_batch {
    int64_t* tree_idx;
    float* states;
    int64_t* actions;
    float* returns;
    float* next_states;
    float* nonterminals;
    float* weights;
    int32_t* attempts;
    int32_t* error;
} irbpp_replay_batch;

/* Per-sample codes; a device error word (uint32, may be NULL) gets bit (1 << code) for every code reported. */
#define IRBPP_REPLAY_ERR_STARVED  1   /* no valid leaf in `max_attempts` descents of the stratum (the reference loops
                                       * forever there: memory.py:163-170) */
#define IRBPP_REPLAY_ERR_MEMORY   2   /* sample: memory id out of range */
#define IRBPP_REPLAY_ERR_INDEX    3   /* update: memory id or tree index out of range; the row is ignored */

/* Empty memories: tree zero, state {0, 0, 0, 1.0f} (memory.py:23-34).  The ring arrays need no initialisation. */
int irbpp_replay_init(const irbpp_replay_memory* mem, void* stream);

/* ReplayMemory.append (memory.py:110-113) for every memory m with valid[m] != 0 (valid may be NULL: all):
 * (t, obs[m * obs_stride ...], action[m], reward[m], !done[m]) at slot index with priority max, then index, full and t
 * advance.  obs float32, action int64, reward float32, done / valid uint8, all device, [M] rows.  reward_clip > 0 clamps
 * the reward to [-reward_clip, reward_clip] first (trainer.py:181-182). */
int irbpp_replay_append(const irbpp_replay_memory* mem, const float* obs, int64_t obs_stride, const int64_t* action,
                        const float* reward, const uint8_t* done, const uint8_t* valid, float reward_clip, void* stream);

/* ReplayMemory.sample(k) (memory.py:191-203) for each of the G memories of mem_ids (device int32 [G]), n = multi_step
 * (0 <= n < C, n <= 64), discount gamma, importance exponent beta.  Stratum i draws lo + (hi - lo) * U with
 * U = uniforms[row * max_attempts + a] (device float64, may be NULL) or, when uniforms is NULL, a counter-based
 * splitmix64 uniform of (seed, call, row, a) with 53 bits; at most max_attempts (1..65536) descents per stratum. */
int irbpp_replay_sample(const irbpp_replay_memory* mem, const int32_t* mem_ids, int32_t G, int32_t k, int32_t n,
                        double discount, double beta, int32_t max_attempts, uint64_t seed, uint64_t call,
                        const double* uniforms, const irbpp_replay_batch* out, uint32_t* error_flags, void* stream);

/* ReplayMemory.update_priorities for a whole batch (agent.py:123-124, memory.py:206-208): row r sets leaf tree_idxs[r]
 * of memory mem_ids[r] to float32 loss[r] ** omega; rows of one memory apply in batch order (a duplicated index keeps
 * the last value), each with its ancestors, and max rises to the largest value set.  Device int32 / int64 / float32 [B]. */
int irbpp_replay_update_priorities(const irbpp_replay_memory* mem, const int32_t* mem_ids, const int64_t* tree_idxs,
                                   const float* loss, int32_t B, double omega, uint32_t* error_flags, void* stream);

/* Profiling aid: when enabled, thread 0 of every CTA adds the SM cycles it spent in each kernel phase
 * (0 scan kernel: load + apply action, 1 scan kernel: observation heightmap + scan + level bitmaps,
 * 2 candidates kernel: contour tasks, 3 candidates kernel: select / pad) to counters 0-3; counters 4-7 count
 * level images, (image, start pixel) micro-tasks, rounds and >64-point overflow redos.  The call
 * returns the counters accumulated so far in out8 (may be NULL), clears them and sets the switch. */
int irbpp_debug_phase_cycles(irbpp_handle h, int32_t enable, uint64_t* out8);

#ifdef __cplusplus
}
#endif
#endif /* IRBPP_H_ */
