// locosim.cu -- CUDA engine + C-ABI (include/locosim.h) of the batched LocoEnv.step() hot path, sm_90a (H100).
//
// One fused kernel per control step: load state (HBM, env-major, coalesced per warp) -> n_substeps x
// [kinematics, CRB, collision, constraint assembly, Newton solve, integrate] entirely in shared memory ->
// observation gather + has_fallen + reward -> in-kernel auto-reset from the trajectory table -> store.
// Or (LOCOSIM_RESORT, default for UnitreeA1) the same step as several launches over ranges of sub-steps, with the envs
// regrouped by solver effort between launches (substep_kernel), or all of them in one persistent launch that regroups the
// envs between chunks of sub-steps from a device-side queue (persist_kernel, default for UnitreeA1).
// See locosim_core.cuh for the per-warp algorithm and DESIGN.md for the layout / roofline accounting.
#include <cuda_runtime.h>
#include <stdint.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/locosim.h"
#include "locosim_config.h"
#include "locosim_host.h"

// ----------------------------------------------------------------------------------------------------------
struct EngineState {
  float *qpos, *qvel, *ws, *goal;   // [N,nv] [N,nv] [N,nv] [N,4]
  int* episode;                     // [N] reset counter (drives the per-env random stream)
  int* counters;                    // [N,8]
  int* dr_row;                      // [N] row of the parameter pool used by the env's current episode
  int* perm;                        // [N] env handled by warp slot i (regrouped every step by solver effort)
  int* cursor;                      // [N] trajectory cursor traj * traj_len + sample (LS_REWARD_TRACKING, end_of_trajectory)
  int4* ep;                         // [N] episode statistics: x = control steps, y = sum of the written rewards (fp32 bits) since the
                                    // env's last reset; z, w = the same two of its last finished (absorbing or truncated) episode
  int max_episode_steps, end_of_trajectory;   // time limit (locosim_set_time_limit), 0 = off
  const float* rot_angle;           // [N] rotation angles pinned for the next reset (setup_random_rot, drop-in mode) or NULL
  const float* pool;                // [K, P] parameter pool (domain randomisation); K = 1: the model's own values
  int pool_K;
};

// reference outputs of a handle (locosim_set_reference_outputs): caller-owned [N, nb, LS_BODY_DIM] reference rows of the
// returned state (`ref`) and of the state to act on next (`next_ref`), NULL = not written; key [N] (engine-owned, NULL = the
// feature is off): what body_kernel last wrote the env's reference rows from, i.e. what the state to act on next is
// compared with: x = cursor, y = rotation angle (fp32 bits), z = parameter-pool row, w = the env's non-finite count
// (counters[4]). The step kernels never read it (a table of its own, like c_bodyout).
struct DevRefOut {
  float* ref;
  float* next_ref;
  int4* key;
};
__constant__ DevRefOut c_refout[LS_MAX_SLOTS];

__device__ __forceinline__ uint64_t mix64(uint64_t z) {
  z += 0x9E3779B97F4A7C15ULL;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
  return z ^ (z >> 31);
}
// counter-based draw of (trajectory, sample) for reset number `episode` of global env `genv`
__device__ __forceinline__ void draw_reset(uint64_t seed, int64_t genv, int episode, int n_traj, int traj_len, int* traj,
                                           int* step) {
  uint64_t r = mix64(seed ^ mix64((uint64_t)genv * 0x100000001B3ULL + (uint64_t)(uint32_t)episode));
  *traj = (int)((r & 0xffffffffULL) % (uint64_t)n_traj);
  *step = (int)((r >> 32) % (uint64_t)traj_len);
}

// setup_random_rot: rotation angle ~ U[0, 2 pi) of reset number `episode` of global env `genv`
__device__ __forceinline__ float draw_rot_angle(uint64_t seed, int64_t genv, int episode) {
  uint64_t r = mix64((seed + 0x2545F4914F6CDD1DULL) ^ mix64((uint64_t)genv * 0x100000001B3ULL + (uint64_t)(uint32_t)episode));
  return (float)(r >> 40) * (6.283185307179586f / 16777216.0f);
}

// rotation angle of the episode that reset number `episode` - 1 started (st.episode = `episode` while it runs): the one
// reset_kernel pinned (rot_pin: episode number, angle bits; locosim_set_reset_rotation), or the counter-based draw
__device__ __forceinline__ float episode_angle(const DevTask& t, const int2* rot_pin, uint64_t seed, int64_t genv, int env,
                                               int episode) {
  if (t.rot[0] < 0 || episode <= 0) return 0.0f;
  const int2 pin = rot_pin[env];
  return pin.x == episode ? __int_as_float(pin.y) : draw_rot_angle(seed, genv, episode - 1);
}

__device__ __forceinline__ int draw_pool_row(uint64_t seed, int64_t genv, int episode, int K) {
  if (K <= 1) return 0;
  uint64_t r = mix64((seed + 0x5DEECE66DULL) ^ mix64((uint64_t)genv * 0x100000001B3ULL + (uint64_t)(uint32_t)episode));
  return (int)(r % (uint64_t)K);
}

#ifndef LOCOSIM_EXTRA_CONFIGS_TU   // (locosim_configs31.cu: the second translation unit compiles the step kernels only)
// ----------------------------------------------------------------------------------------------------------
// reset kernel: one warp per env, no shared memory
// ----------------------------------------------------------------------------------------------------------
__global__ void reset_kernel(int ms, DevTask t, EngineState st, const uint8_t* mask, const int* traj_no,
                             const int* step_no, const int* pool_row, float* obs, int n_envs, uint64_t seed,
                             int64_t env_off, int2* rot_pin) {
  int env = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  int lane = threadIdx.x & 31;
  if (env >= n_envs) return;
  if (mask && !mask[env]) return;
  const DevModel& m = c_models[ms];
  const int nv = m.nv, ncol = 2 * nv + t.n_goal;
  int tr, sp;
  int ep = st.episode[env];
  draw_reset(seed, env_off + env, ep, t.n_traj, t.traj_len, &tr, &sp);
  if (traj_no) tr = min(max(traj_no[env], 0), t.n_traj - 1);       // (pinned rows are clamped into the table)
  if (step_no) sp = min(max(step_no[env], 0), t.traj_len - 1);
  const float* row = t.table + ((size_t)tr * t.traj_len + sp) * ncol;
  int prow = draw_pool_row(seed, env_off + env, ep, st.pool_K);     // the model of this episode (base.py:187-191)
  if (pool_row) prow = min(max(pool_row[env], 0), st.pool_K - 1);
  float angle = 0.0f;
  if (t.rot[0] >= 0) angle = st.rot_angle ? st.rot_angle[env] : draw_rot_angle(seed, env_off + env, ep);
  for (int i = lane; i < nv; i += 32) {
    st.qpos[(size_t)env * nv + i] = reset_value(t, row, nv, LS_OBS_QPOS, i, angle);
    st.qvel[(size_t)env * nv + i] = reset_value(t, row, nv, LS_OBS_QVEL, i, angle);
    st.ws[(size_t)env * nv + i] = 0;
  }
  for (int k = lane; k < t.n_goal; k += 32) st.goal[(size_t)env * 4 + k] = row[2 * nv + k];
  zero_applied(ms, env);
  if (obs) {
    for (int k = lane; k < t.obs_dim; k += 32) {
      int idx = t.obs_src_idx[k], ty = t.obs_src_type[k];
      float v;
      if (ty == LS_OBS_QPOS || ty == LS_OBS_QVEL) v = reset_value(t, row, nv, ty, idx, angle);
      else if (ty == LS_OBS_GRF) v = 0.0f;           // the running mean of the foot forces is reset with the episode
      else if (ty == LS_OBS_PARAM) v = st.pool[(size_t)prow * m.pool_P + t.po_user + idx];
      else v = row[2 * nv + idx];
      obs[(size_t)env * t.obs_dim + k] = v;
    }
  }
  if (lane == 0) {
    st.episode[env] = ep + 1; st.counters[(size_t)env * 8 + 1] += 1;
    st.dr_row[env] = prow;
    st.cursor[env] = tr * t.traj_len + sp;
    *reinterpret_cast<int2*>(&st.ep[env]) = make_int2(0, 0);
    if (st.rot_angle && t.rot[0] >= 0) rot_pin[env] = make_int2(ep + 1, __float_as_int(angle));   // (episode_angle)
  }
}

// ----------------------------------------------------------------------------------------------------------
// saved states (locosim_save_state / locosim_load_state, row layout LS_STATE_* of include/locosim.h): one warp per env, the
// row moved as 16-byte words. Words 0-15 are four int4: (tag, tag, episode, pool row), (cursor, angle, 0, 0), the episode
// statistics, the goal; from LS_STATE_QPOS on the per-dof arrays and the observation follow word by word.
// ----------------------------------------------------------------------------------------------------------
// word k (>= 0) of an env's row after LS_STATE_QPOS
__device__ __forceinline__ int state_array_word(const EngineState& st, const float* __restrict__ obs, int env, int nv, int D,
                                                int k) {
  if (k < nv) return __float_as_int(st.qpos[(size_t)env * nv + k]);
  if ((k -= nv) < nv) return __float_as_int(st.qvel[(size_t)env * nv + k]);
  if ((k -= nv) < nv) return __float_as_int(st.ws[(size_t)env * nv + k]);
  if ((k -= nv) < D) return __float_as_int(obs[(size_t)env * D + k]);
  return 0;
}
__device__ __forceinline__ void state_array_store(const EngineState& st, float* __restrict__ obs, int env, int nv, int D, int k,
                                                  int w) {
  if (k < nv) st.qpos[(size_t)env * nv + k] = __int_as_float(w);
  else if ((k -= nv) < nv) st.qvel[(size_t)env * nv + k] = __int_as_float(w);
  else if ((k -= nv) < nv) st.ws[(size_t)env * nv + k] = __int_as_float(w);
  else if ((k -= nv) < D) { if (obs) obs[(size_t)env * D + k] = __int_as_float(w); }
}

__global__ void save_state_kernel(DevTask t, EngineState st, const float* __restrict__ obs, int4* __restrict__ rows,
                                  int n_envs, int nv, int words, int fingerprint, uint64_t seed, int64_t env_off,
                                  const int2* __restrict__ rot_pin) {
  const int env = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (env >= n_envs) return;
  const int nc = words / 4, D = t.obs_dim;
  int4* row = rows + (size_t)env * nc;
  for (int c = lane; c < nc; c += 32) {
    int4 v;
    if (c == 0) v = make_int4(LS_STATE_VERSION, fingerprint, st.episode[env], st.dr_row[env]);
    else if (c == 1) {
      const float angle = episode_angle(t, rot_pin, seed, env_off + env, env, st.episode[env]);
      v = make_int4(st.cursor[env], __float_as_int(angle), 0, 0);
    } else if (c == 2) v = st.ep[env];
    else if (c == 3) v = reinterpret_cast<const int4*>(st.goal)[env];
    else {
      const int k = 4 * c - LS_STATE_QPOS(nv);
      v = make_int4(state_array_word(st, obs, env, nv, D, k), state_array_word(st, obs, env, nv, D, k + 1),
                    state_array_word(st, obs, env, nv, D, k + 2), state_array_word(st, obs, env, nv, D, k + 3));
    }
    row[c] = v;
  }
}

// env i <- row idx[i] (idx NULL: row i); loaded[i] = whether it was (the mask of the body / reference rows written next)
__global__ void load_state_kernel(DevTask t, EngineState st, const int4* __restrict__ rows, int n_rows,
                                  const int* __restrict__ idx, float* __restrict__ obs, int n_envs, int nv, int words,
                                  int fingerprint, int2* __restrict__ rot_pin, int* __restrict__ reset_mark,
                                  uint8_t* __restrict__ loaded) {
  const int env = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (env >= n_envs) return;
  const int nc = words / 4, D = t.obs_dim;
  const int r = idx ? idx[env] : env;
  bool ok = r >= 0 && r < n_rows;
  const int4* row = rows + (size_t)(ok ? r : 0) * nc;
  const int4 h0 = ok ? row[0] : make_int4(0, 0, 0, 0);
  ok = ok && h0.x == LS_STATE_VERSION && h0.y == fingerprint;
  if (lane == 0) loaded[env] = ok ? 1 : 0;
  if (!ok) return;
  for (int c = lane; c < nc; c += 32) {
    const int4 v = row[c];
    if (c == 0) {
      st.episode[env] = v.z;
      st.dr_row[env] = min(max(v.w, 0), st.pool_K - 1);
    } else if (c == 1) {
      st.cursor[env] = min(max(v.x, 0), t.n_traj * t.traj_len - 1);
      rot_pin[env] = make_int2(h0.z, v.y);          // (episode_angle: the saved angle, not the destination's draw)
    } else if (c == 2) st.ep[env] = v;
    else if (c == 3) reinterpret_cast<int4*>(st.goal)[env] = v;
    else {
      const int k = 4 * c - LS_STATE_QPOS(nv);
      state_array_store(st, obs, env, nv, D, k, v.x); state_array_store(st, obs, env, nv, D, k + 1, v.y);
      state_array_store(st, obs, env, nv, D, k + 2, v.z); state_array_store(st, obs, env, nv, D, k + 3, v.w);
    }
  }
  if (lane == 0 && reset_mark) reset_mark[env] = 0;
}
#endif

// ----------------------------------------------------------------------------------------------------------
// Sub-step launches (LOCOSIM_RESORT = S < n_substeps): the control step runs as ceil(n_substeps / S) launches of the step
// kernel, each over sub-steps [k0, k1), and the envs are regrouped by solver effort between launches. Consecutive sub-steps
// of an env cost alike (the lock-step cost of a block follows its hardest env sub-step by sub-step), the next control step
// under random actions much less so. What the fused kernel keeps in shared memory across sub-steps is carried in HBM
// (SplitState::carry); qpos / qvel / qacc_warmstart are stored as at the end of a step. Every launch appends its envs to
// per-key buckets and the next launch takes its envs from them, hardest first, so that regrouping needs no extra launch.
// ----------------------------------------------------------------------------------------------------------
#define LS_RANK_BUCKETS 128
#define LS_CARRY 32       // words per env: iter_sum, mpr_calls, sep_next, reward, sep_pair[4], sep_dir[4][3], grf[12]
struct SplitState {
  int* carry;             // [N, LS_CARRY]
  int* bcount;            // [2, LS_RANK_BUCKETS] envs per key bucket: read by one launch, appended to by the other
  int* benv;              // [2, LS_RANK_BUCKETS, N] the envs of every bucket (a permutation of all envs)
  int* seq;               // [2] buffer read by the current launch, blocks of the current launch that have finished
  int regroup, key_shift;
};

// env of position `pos` of the descending key order of the buckets (called by the whole warp)
__device__ __forceinline__ int bucket_env(const int* __restrict__ cnt, const int* __restrict__ benv, int n_envs, int pos) {
  const int lane = threadIdx.x & 31;
  int c[4], s = 0;
#pragma unroll
  for (int j = 0; j < 4; j++) { c[j] = cnt[LS_RANK_BUCKETS - 1 - 4 * lane - j]; s += c[j]; }
  int incl = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
  const int src = __ffs(__ballot_sync(0xffffffffu, incl > pos)) - 1;
  int b = 0, off = 0;
  if (lane == src) {
    int acc = incl - s;
    bool found = false;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      if (!found && pos < acc + c[j]) { b = LS_RANK_BUCKETS - 1 - 4 * lane - j; off = pos - acc; found = true; }
      acc += c[j];
    }
  }
  b = __shfl_sync(0xffffffffu, b, src); off = __shfl_sync(0xffffffffu, off, src);
  return benv[(size_t)b * n_envs + off];
}

// regrouping key of a sub-step launch: key mode 3 of the fused kernel with the counts of this launch's sub-steps scaled to a
// whole control step
template <class C>
__device__ __forceinline__ int launch_key(const DevTask& t, const EnvS<C>& e, int k0, int k1, int iter0, int mpr0,
                                          int key_mode_in) {
  const int ns = k1 - k0, mpr_w = (key_mode_in >> 8) & 255;
  return (e.iter_sum - iter0) * t.n_substeps / ns + (e.nefc >> 1) + mpr_w * min((e.mpr_calls - mpr0) * t.n_substeps / ns, 64);
}
__device__ __forceinline__ void append_env(const SplitState& split, int wr, int env, int n_envs, int key) {
  key >>= split.key_shift;
  const int b = key < LS_RANK_BUCKETS - 1 ? key : LS_RANK_BUCKETS - 1;
  const int pos = atomicAdd(&split.bcount[wr * LS_RANK_BUCKETS + b], 1);
  split.benv[((size_t)wr * LS_RANK_BUCKETS + b) * n_envs + pos] = env;
}

// ----------------------------------------------------------------------------------------------------------
// Per-env parts of a control step shared by the fused (step_kernel), sub-step (substep_kernel) and persistent
// (persist_kernel) kernels: the block's pair-table staging, the reward of the previous observation, the carry record
// between the launches or chunks of a split step, and the end of the step. Each kernel keeps only what differs: how a warp
// finds its env, which sub-steps it runs, and where the env goes next. tests/test_substep_launches.py and
// tests/test_persistent_kernel.py hold the three kernels to the same bits.
// ----------------------------------------------------------------------------------------------------------

// LOCOSIM_STAGE (default on where it fits): the table of the PRIMITIVE candidate pairs of the mid-phase (packed geom pair +
// bound; UnitreeA1: 357 entries read in every dynamics evaluation by every warp) is staged once per block into the shared
// memory behind the per-env working sets by ONE TMA bulk copy (cp.async.bulk global -> shared::cta, completion on an
// mbarrier); EnvS::pk_tab points to it, DevModel::pk_n is its entry count. Called by the whole block.
template <class C>
__device__ __forceinline__ void stage_pair_table(unsigned char* smem_raw, const unsigned char* __restrict__ stage_src,
                                                 int stage_bytes) {
  if (stage_bytes <= 0) return;
  unsigned char* dst = smem_raw + (size_t)(blockDim.x >> 5) * sizeof(EnvS<C>);
  const unsigned dst_a = (unsigned)__cvta_generic_to_shared(dst);
  const unsigned bar_a = dst_a + (unsigned)stage_bytes;
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar_a) : "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_a), "r"((unsigned)stage_bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_a),
                 "l"(stage_src), "r"((unsigned)stage_bytes), "r"(bar_a)
                 : "memory");
  }
  __syncthreads();                                    // (the barrier object is initialised before anybody polls it)
  unsigned ok = 0;
  while (!ok)
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(bar_a) : "memory");
}

// reward depends on the *previous* observation only (utils/reward.py via base.py:170-176): evaluated before the physics
// (the tracking reward, which compares the new observation with the mocap table, is step_epilogue's)
template <class C>
__device__ __forceinline__ float prev_obs_reward(const DevTask& t, const EnvS<C>& e) {
  float rew = 0;
  if (t.reward_type == LS_REWARD_TARGET_VELOCITY) { float d = obs_value(t, e, t.ri[0]) - t.rp[0]; rew = expf(-d * d); }
  else if (t.reward_type == LS_REWARD_VELOCITY_VECTOR) {
    float g = obs_value(t, e, t.ri[3]);
    float dx = obs_value(t, e, t.ri[0]) - g * obs_value(t, e, t.ri[2]);
    float dy = obs_value(t, e, t.ri[1]) - g * obs_value(t, e, t.ri[2] + 1);
    rew = expf(-5.0f * sqrtf(dx * dx + dy * dy));
  } else if (t.reward_type == LS_REWARD_POS) rew = obs_value(t, e, t.ri[0]);
  return rew;
}

// carry record of an env (LS_CARRY words): what the fused kernel keeps in shared memory across sub-steps and
// init_workspace clears, and the reward of the previous observation; stored by the whole warp after a launch or chunk that
// is not the last of the control step, loaded by the next one. CG: read past L1 (the persistent kernel: another SM of the
// same launch may have written the record).
template <class C>
__device__ __forceinline__ void save_carry(int* carry, const EnvS<C>& e, float rew) {
  static_assert(EnvS<C>::NSEP <= 4 && 3 * LS_MAX_GRF <= 12, "carry record layout");
  const int lane = threadIdx.x & 31;
  if (lane == 0) { carry[0] = e.iter_sum; carry[1] = e.mpr_calls; carry[2] = e.sep_next; carry[3] = __float_as_int(rew); }
  if (lane < EnvS<C>::NSEP) carry[4 + lane] = e.sep_pair[lane];
  if (lane < 3 * EnvS<C>::NSEP) carry[8 + lane] = __float_as_int((&e.sep_dir[0][0])[lane]);
  if (lane < 3 * LS_MAX_GRF) carry[20 + lane] = __float_as_int(e.grf[lane]);
}
template <bool CG>
__device__ __forceinline__ int ld_carry(const int* p) {
  if constexpr (CG) return __ldcg(p);
  else return *p;
}
// returns the carried reward (lane 0; 0 on the other lanes)
template <class C, bool CG>
__device__ __forceinline__ float load_carry(const int* carry, EnvS<C>& e) {
  const int lane = threadIdx.x & 31;
  float rew = 0;
  if (lane == 0) {
    e.iter_sum = ld_carry<CG>(&carry[0]); e.mpr_calls = ld_carry<CG>(&carry[1]); e.sep_next = ld_carry<CG>(&carry[2]);
    rew = __int_as_float(ld_carry<CG>(&carry[3]));
  }
  if (lane < EnvS<C>::NSEP) e.sep_pair[lane] = ld_carry<CG>(&carry[4 + lane]);
  if (lane < 3 * EnvS<C>::NSEP) (&e.sep_dir[0][0])[lane] = __int_as_float(ld_carry<CG>(&carry[8 + lane]));
  if (lane < 3 * LS_MAX_GRF) e.grf[lane] = __int_as_float(ld_carry<CG>(&carry[20 + lane]));
  __syncwarp();
  return rew;
}

// end of the control step of one (not ghost) env, by its warp: observation, termination, tracking reward and cursor, time
// limit, episode statistics, counters and regrouping key, auto-reset, state store. Returns whether the env was reset.
template <class C>
__device__ __forceinline__ bool step_epilogue(int ms, const DevTask& t, const EngineState& st, EnvS<C>& e, int env, float rew,
                                              float* __restrict__ obs, float* __restrict__ reward,
                                              uint8_t* __restrict__ done, float* __restrict__ next_obs, int auto_reset,
                                              uint64_t seed, int64_t env_off, int key_mode_in) {
  const int lane = threadIdx.x & 31;
  int key_mode = key_mode_in & 0xffff;
  const DevModel& m = c_models[ms];
  const int nv = m.nv, D = t.obs_dim;

  // ---- observation, termination, reward ----
  bool bad = false;
  for (int i = lane; i < nv; i += 32) bad |= !(isfinite(e.qpos[i]) && isfinite(e.qvel[i]));
  bool fallen = false;
  for (int k = lane; k < t.n_done; k += 32) {
    float v = obs_value(t, e, t.done_obs_idx[k]);
    fallen |= (v < t.done_lo[k]) || (v > t.done_hi[k]);
  }
  bad = __any_sync(0xffffffffu, bad);
  fallen = __any_sync(0xffffffffu, fallen) && t.use_absorbing;
  const bool is_done = fallen || bad;
  if (t.reward_type == LS_REWARD_TRACKING) {
    // mocap-tracking reward (include/locosim_task.h): the cursor advances one sample, the observation reached by this step
    // is compared with the table row at the advanced cursor
    int cur = st.cursor[env];
    const int tj = cur / t.traj_len;
    int sp = cur - tj * t.traj_len;
    sp = sp + 1 < t.traj_len ? sp + 1 : t.traj_len - 1;
    cur = tj * t.traj_len + sp;
    const float* ref = t.table + (size_t)cur * (2 * nv + t.n_goal);
    float ep = 0, ev = 0;
    for (int k = lane; k < D; k += 32) {
      const int ty = t.obs_src_type[k], idx = t.obs_src_idx[k];
      if (ty == LS_OBS_QPOS) { const float d = e.qpos[idx] - ref[idx]; ep += d * d; }
      else if (ty == LS_OBS_QVEL) { const float d = e.qvel[idx] - ref[nv + idx]; ev += d * d; }
    }
    ep = warp_sum(ep); ev = warp_sum(ev);
    rew = bad ? 0.0f : t.track[0] * expf(-t.track[1] * ep) + t.track[2] * expf(-t.track[3] * ev);
    if (lane == 0) st.cursor[env] = cur;
  }
  for (int k = lane; k < D; k += 32) {
    float v = obs_value(t, e, k);
    if (bad) v = 0.0f;
    obs[(size_t)env * D + k] = v;
  }
  bool truncated = false;
  if (lane == 0) {
    float r = rew;
    reward[env] = r;
    // episode statistics and time limit (include/locosim.h): length and return of the running episode, the two limits,
    // bit 1 of the done byte (absorbing wins), the finished episode's numbers
    int4 es = st.ep[env];
    es.x += 1; es.y = __float_as_int(__int_as_float(es.y) + r);
    truncated = st.max_episode_steps > 0 && es.x >= st.max_episode_steps;
    if (st.end_of_trajectory) {
      // one (clamped) advance of the cursor per step: the tracking reward above has made it already
      const int cur = st.cursor[env];
      int sp = cur % t.traj_len;
      if (t.reward_type != LS_REWARD_TRACKING && sp + 1 < t.traj_len) { sp += 1; st.cursor[env] = cur + 1; }
      truncated |= sp == t.traj_len - 1;
    }
    truncated = truncated && !is_done;
    done[env] = is_done ? 1 : (truncated ? 2 : 0);
    if (is_done || truncated) { es.z = es.x; es.w = es.y; }
    st.ep[env] = es;
    int* cnt = st.counters + (size_t)env * 8;
    cnt[0] += 1; cnt[2] = e.iter_sum; cnt[3] = e.ncon;
    if (bad) cnt[4] += 1;
    {
      int key = e.iter_sum;
      const int mpr_w = (key_mode >> 8) & 255;           // weight of one MPR run in Newton-iteration units
      key_mode &= 255;
      if (key_mode == 1) key = (cnt[5] + e.iter_sum + 1) >> 1;
      else if (key_mode == 2) key = e.solver_iter * 8;
      else if (key_mode == 3) key = e.iter_sum + (e.nefc >> 1) + mpr_w * min(e.mpr_calls, 64);
      else if (key_mode == 4) key = (3 * cnt[5] + e.iter_sum + 2) >> 2;
      else if (key_mode == 5) key = e.iter_sum + 4 * e.solver_iter;
      else if (key_mode == 6) key = e.iter_sum + e.nefc;
      else if (key_mode == 7) key = e.iter_sum + 4 * e.solver_iter + (e.nefc >> 1);
      cnt[5] = key;
    } cnt[6] = max(cnt[6], e.ncon); cnt[7] = max(cnt[7], e.nefc);
  }

  // ---- auto-reset (reset_env is a whole-warp call: lane 0's verdict on the time limit goes to every lane first) ----
  truncated = __shfl_sync(0xffffffffu, (int)truncated, 0) != 0;
  const bool reset = (is_done || truncated) && (auto_reset || bad);
  if (reset) {
    const int key_reset = (key_mode_in >> 16) ? (key_mode_in >> 16) - 1 : -1;
    int ep = st.episode[env];
    int tr, sp;
    draw_reset(seed, env_off + env, ep, t.n_traj, t.traj_len, &tr, &sp);
    __syncwarp();
    reset_env(ms, t, e, tr, sp, t.rot[0] >= 0 ? draw_rot_angle(seed, env_off + env, ep) : 0.0f);
    if (lane == 0) {
      const int prow = draw_pool_row(seed, env_off + env, ep, st.pool_K);
      st.episode[env] = ep + 1; st.counters[(size_t)env * 8 + 1] += 1;
      if (key_reset >= 0) st.counters[(size_t)env * 8 + 5] = key_reset;   // regrouping key of a fresh episode (the finished one's says nothing)
      st.dr_row[env] = prow;
      st.cursor[env] = tr * t.traj_len + sp;
      *reinterpret_cast<int2*>(&st.ep[env]) = make_int2(0, 0);
      e.prm = st.pool + (size_t)prow * m.pool_P;      // the next episode's model (LS_OBS_PARAM entries of next_obs)
    }
    __syncwarp();
    for (int k = lane; k < t.n_goal; k += 32) st.goal[(size_t)env * 4 + k] = e.goal[k];
  }
  if (next_obs) for (int k = lane; k < D; k += 32) next_obs[(size_t)env * D + k] = obs_value(t, e, k);

  // ---- store state ----
  for (int i = lane; i < nv; i += 32) {
    st.qpos[(size_t)env * nv + i] = e.qpos[i];
    st.qvel[(size_t)env * nv + i] = e.qvel[i];
    st.ws[(size_t)env * nv + i] = e.qacc_ws[i];
  }
  return reset;
}

// ----------------------------------------------------------------------------------------------------------
// step kernel: one warp per env, EnvS in dynamic shared memory
// ----------------------------------------------------------------------------------------------------------
template <class C>
__global__ void __launch_bounds__(512, 1) step_kernel(int ms, DevTask t, SolverOpts so, EngineState st,
                                                    const float* __restrict__ action, float* __restrict__ obs,
                                                    float* __restrict__ reward, uint8_t* __restrict__ done,
                                                    float* __restrict__ next_obs, int n_envs, int auto_reset,
                                                    uint64_t seed, int64_t env_off, int sync_substeps, int key_mode_in,
                                                    const unsigned char* __restrict__ stage_src, int stage_bytes) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  stage_pair_table<C>(smem_raw, stage_src, stage_bytes);
  // warps past the last env shadow it (same barriers, no stores): the block-wide barriers inside the solver have
  // data-dependent counts, so every warp of a block has to run the physics
  const int slot_raw = blockIdx.x * (blockDim.x >> 5) + warp;
  const bool ghost = slot_raw >= n_envs;
  const int env = st.perm[ghost ? n_envs - 1 : slot_raw];
  EnvS<C>& e = reinterpret_cast<EnvS<C>*>(smem_raw)[warp];
  const DevModel& m = c_models[ms];
  const int nv = m.nv, nu = m.nu;
  if (lane == 0) {
    e.prm = st.pool + (size_t)st.dr_row[env] * m.pool_P;
    e.env = env;
    e.substep = ghost ? -1 : 0;
    if (stage_bytes > 0) {
      const unsigned char* sm = smem_raw + (size_t)(blockDim.x >> 5) * sizeof(EnvS<C>);
      e.pk_tab = reinterpret_cast<const int*>(sm);
    } else { e.pk_tab = m.pair_packed; }
  }

  // ---- load state ----
  for (int i = lane; i < nv; i += 32) {
    e.qpos[i] = st.qpos[(size_t)env * nv + i];
    e.qvel[i] = st.qvel[(size_t)env * nv + i];
    e.qacc_ws[i] = st.ws[(size_t)env * nv + i];
    e.qacc[i] = 0;
  }
  for (int i = lane; i < nu; i += 32) e.ctrl[t.act_idx[i]] = action[(size_t)env * nu + i] * t.act_delta[i] + t.act_mean[i];
  if (lane < 4) e.goal[lane] = st.goal[(size_t)env * 4 + lane];
  __syncwarp();
  init_workspace(ms, e);
  if (lane == 0) e.iter_sum = 0;
  if (lane < 3 * LS_MAX_GRF) e.grf[lane] = 0;
  float rew = prev_obs_reward(t, e);

  // ---- physics ----
  if (sync_substeps) {
    // keep the warps of a block in the same phase: they then share instruction-cache lines
    for (int k = 0; k < t.n_substeps; k++) { if (k % sync_substeps == 0) __syncthreads(); physics_substeps(ms, e, so, 1, t.grf_group, t.n_grf); }
  } else {
    physics_substeps(ms, e, so, t.n_substeps, t.grf_group, t.n_grf);
  }

  if (ghost) return;
  step_epilogue<C>(ms, t, st, e, env, rew, obs, reward, done, next_obs, auto_reset, seed, env_off, key_mode_in);
}

// ----------------------------------------------------------------------------------------------------------
// sub-step kernel body: the fused step kernel above restricted to sub-steps [k0, k1) of the control step. Staging,
// reward, carry record and epilogue are the shared helpers above.
// ----------------------------------------------------------------------------------------------------------
template <class C>
__device__ __forceinline__ void substep_body(unsigned char* smem_raw, int ms, const DevTask& t, const SolverOpts& so,
                                             const EngineState& st, const float* __restrict__ action, float* __restrict__ obs,
                                             float* __restrict__ reward, uint8_t* __restrict__ done,
                                             float* __restrict__ next_obs, int n_envs, int auto_reset, uint64_t seed,
                                             int64_t env_off, int sync_substeps, int key_mode_in,
                                             const unsigned char* __restrict__ stage_src, int stage_bytes, int k0, int k1,
                                             const SplitState& split) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  stage_pair_table<C>(smem_raw, stage_src, stage_bytes);
  // warps past the last env shadow it (same barriers, no stores): the block-wide barriers inside the solver have
  // data-dependent counts, so every warp of a block has to run the physics
  const int slot_raw = blockIdx.x * (blockDim.x >> 5) + warp;
  const bool ghost = slot_raw >= n_envs;
  const int slot = ghost ? n_envs - 1 : slot_raw;
  const int rd = split.seq[0] & 1;      // bucket buffer this launch reads; it appends to the other one
  const int env = split.regroup ? bucket_env(split.bcount + rd * LS_RANK_BUCKETS,
                                             split.benv + (size_t)rd * LS_RANK_BUCKETS * n_envs, n_envs, slot)
                                : slot;
  EnvS<C>& e = reinterpret_cast<EnvS<C>*>(smem_raw)[warp];
  const DevModel& m = c_models[ms];
  const int nv = m.nv, nu = m.nu;
  if (lane == 0) {
    e.prm = st.pool + (size_t)st.dr_row[env] * m.pool_P;
    e.env = env;
    e.substep = ghost ? -1 : k0;
    if (stage_bytes > 0) {
      const unsigned char* sm = smem_raw + (size_t)(blockDim.x >> 5) * sizeof(EnvS<C>);
      e.pk_tab = reinterpret_cast<const int*>(sm);
    } else { e.pk_tab = m.pair_packed; }
  }

  // ---- load state ----
  for (int i = lane; i < nv; i += 32) {
    e.qpos[i] = st.qpos[(size_t)env * nv + i];
    e.qvel[i] = st.qvel[(size_t)env * nv + i];
    e.qacc_ws[i] = st.ws[(size_t)env * nv + i];
    e.qacc[i] = 0;
  }
  for (int i = lane; i < nu; i += 32) e.ctrl[t.act_idx[i]] = action[(size_t)env * nu + i] * t.act_delta[i] + t.act_mean[i];
  if (lane < 4) e.goal[lane] = st.goal[(size_t)env * 4 + lane];
  __syncwarp();
  init_workspace(ms, e);
  int* carry = split.carry + (size_t)env * LS_CARRY;
  float rew;
  if (k0 > 0) {
    rew = load_carry<C, false>(carry, e);   // what the previous launches of this control step left behind
  } else {
    if (lane == 0) e.iter_sum = 0;
    if (lane < 3 * LS_MAX_GRF) e.grf[lane] = 0;
    rew = prev_obs_reward(t, e);
  }

  // ---- physics ----
  if (sync_substeps) {
    // keep the warps of a block in the same phase: they then share instruction-cache lines
    for (int k = k0; k < k1; k++) { if (k % sync_substeps == 0) __syncthreads(); physics_substeps(ms, e, so, 1, t.grf_group, t.n_grf); }
  } else {
    physics_substeps(ms, e, so, k1 - k0, t.grf_group, t.n_grf);
  }
  // the regrouping key counts this launch's sub-steps: the counts at its start are those of the carry record, which the
  // warp rewrites only below (0 in the first launch; reading them here rather than keeping them live across the physics
  // keeps this kernel's stack within the fused kernel's)
  int key = launch_key(t, e, k0, k1, k0 > 0 ? carry[0] : 0, k0 > 0 ? carry[1] : 0, key_mode_in);

  if (k1 < t.n_substeps) {
    // ---- not the last launch of the control step: state and carried fields to HBM, env into its bucket ----
    if (!ghost) {
      for (int i = lane; i < nv; i += 32) {
        st.qpos[(size_t)env * nv + i] = e.qpos[i];
        st.qvel[(size_t)env * nv + i] = e.qvel[i];
        st.ws[(size_t)env * nv + i] = e.qacc_ws[i];
      }
      save_carry<C>(carry, e, rew);
      if (lane == 0 && split.regroup) append_env(split, rd ^ 1, env, n_envs, key);
    }
    return;
  }
  if (ghost) return;
  const bool reset = step_epilogue<C>(ms, t, st, e, env, rew, obs, reward, done, next_obs, auto_reset, seed, env_off,
                                      key_mode_in);
  if (lane == 0 && split.regroup) {
    if (reset && (key_mode_in >> 16)) key = (key_mode_in >> 16) - 1;
    append_env(split, rd ^ 1, env, n_envs, key);
  }
}

template <class C>
__global__ void __launch_bounds__(512, 1) substep_kernel(int ms, DevTask t, SolverOpts so, EngineState st,
                                                       const float* __restrict__ action, float* __restrict__ obs,
                                                       float* __restrict__ reward, uint8_t* __restrict__ done,
                                                       float* __restrict__ next_obs, int n_envs, int auto_reset,
                                                       uint64_t seed, int64_t env_off, int sync_substeps, int key_mode_in,
                                                       const unsigned char* __restrict__ stage_src, int stage_bytes, int k0,
                                                       int k1, SplitState split) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  substep_body<C>(smem_raw, ms, t, so, st, action, obs, reward, done, next_obs, n_envs, auto_reset, seed, env_off,
                     sync_substeps, key_mode_in, stage_src, stage_bytes, k0, k1, split);
  // The block that finishes last (every other block has read its envs from the buckets by then) empties the buckets this
  // launch read and hands the ones it filled to the next launch: no host-side launch counter, so CUDA graphs replay it.
  __syncthreads();
  int last = 0;
  if (threadIdx.x == 0) {
    __threadfence();
    last = atomicAdd(&split.seq[1], 1) == (int)gridDim.x - 1;
  }
  if (__syncthreads_or(last)) {
    const int rd = split.seq[0] & 1;
    for (int i = threadIdx.x; i < LS_RANK_BUCKETS; i += blockDim.x) split.bcount[rd * LS_RANK_BUCKETS + i] = 0;
    if (threadIdx.x == 0) { split.seq[0] = rd ^ 1; split.seq[1] = 0; }
  }
}

// ----------------------------------------------------------------------------------------------------------
// Persistent sub-step kernel (LOCOSIM_PERSIST, default where sub-step launches are): the whole control step in ONE launch
// of min(SMs, blocks) blocks. The step is cut into chunks of LOCOSIM_RESORT sub-steps; the work unit is a group of up to
// wpb envs running one chunk together. A warp that finishes a chunk of its env stores state and carry record and publishes
// the env into the key bucket of the next chunk; a block pops its next group from the lowest chunk that has enough envs
// ready, hardest keys first. So the envs are regrouped by the effort of their last chunk as in substep_kernel, but the
// block prologue (TMA staging) is paid once per step and an SM that finishes early takes the next group instead of
// idling in the wave tail of every launch.
//
// Memory ordering: an SM may hold a stale L1 line of an env it ran earlier in the same launch that another SM has since
// advanced, so everything another block of this launch may have written (state, carry, env ids, counts) is read past L1
// (ld.global.cg / ld.relaxed.gpu); publishing is a release: stores, __threadfence(), then the env id and the counts.
// No grid barrier and no co-residency assumption: a block only waits for envs that running blocks hold, so the kernel
// makes progress with any number of resident blocks.
//
// The per-env body shares the staging, reward, carry record and epilogue of the other step kernels (helpers above).
// ----------------------------------------------------------------------------------------------------------
#define LS_TL_WORDS 8     // timeline record: smid, chunk, envs, pop start, group start, group end (ns), iterations sum, max
struct PersistQueue {
  int* carry;             // [N, LS_CARRY] as SplitState::carry
  int* cnt;               // [nch + 1, 3, LS_RANK_BUCKETS] per key bucket: slots reserved, envs published, envs taken
  int* tot;               // [nch + 1, 2] per chunk: envs published, envs taken
  int* benv;              // [nch + 1, LS_RANK_BUCKETS, N] env ids of the bucket slots, -1 = empty
  int* seq;               // [2] parity of the step (which of the two chunk-0 sets it reads), blocks that have finished
  long long* tl;          // optional timeline: [1 + tl_cap, LS_TL_WORDS], tl[0] = records written (NULL in the product path)
  int tl_cap;
  int nch, chunk, pool, regroup, key_shift;
};
// bucket set of chunk c: chunk 0 of this step and chunk 0 of the next (published by the last chunk) alternate between sets 0
// and 1; chunks 1 .. nch-1 use sets 2 .. nch
__device__ __forceinline__ int persist_set(int c, int nch, int par) { return c == 0 ? par : (c == nch ? par ^ 1 : c + 1); }
__device__ __forceinline__ int ld_relaxed(const int* p) {
  int v;
  asm volatile("ld.relaxed.gpu.global.b32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_relaxed(int* p, int v) {
  asm volatile("st.relaxed.gpu.global.b32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ long long global_ns() {
  long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// publish `env` (lane 0; the warp's stores are fenced) into bucket `key` of chunk c
__device__ __forceinline__ void persist_publish(const PersistQueue& q, int par, int c, int env, int n_envs, int key) {
  const int s = persist_set(c, q.nch, par);
  key = q.regroup ? key >> q.key_shift : 0;
  const int b = key < 0 ? 0 : (key < LS_RANK_BUCKETS - 1 ? key : LS_RANK_BUCKETS - 1);
  int* cnt = q.cnt + (size_t)s * 3 * LS_RANK_BUCKETS;
  const int pos = atomicAdd(&cnt[b], 1);
  st_relaxed(&q.benv[((size_t)s * LS_RANK_BUCKETS + b) * n_envs + pos], env);
  __threadfence();
  atomicAdd(&cnt[LS_RANK_BUCKETS + b], 1);
  atomicAdd(&q.tot[2 * s], 1);
}

// next group (called by one whole warp): up to `want` envs of the lowest chunk whose ready envs reach the pool threshold
// (pool x want, or all that remain of the chunk), hardest keys first; returns the number of envs (0: the step is done)
__device__ __forceinline__ int persist_pop(const PersistQueue& q, int par, int n_envs, int want, int* s_env, int* chunk) {
  const int lane = threadIdx.x & 31;
  for (;;) {
    if (ld_relaxed(&q.tot[2 * persist_set(q.nch - 1, q.nch, par) + 1]) >= n_envs) return 0;   // every env ran the last chunk
    int c = -1, s = 0;
    for (int k = 0; k < q.nch && c < 0; k++) {
      s = persist_set(k, q.nch, par);
      const int taken = ld_relaxed(&q.tot[2 * s + 1]);
      if (taken >= n_envs) continue;
      const int avail = ld_relaxed(&q.tot[2 * s]) - taken;
      if (avail > 0 && avail >= min(q.pool * want, n_envs - taken)) c = k;
    }
    if (c < 0) { __nanosleep(256); continue; }
    int* cnt = q.cnt + (size_t)s * 3 * LS_RANK_BUCKETS;
    int* benv = q.benv + (size_t)s * LS_RANK_BUCKETS * n_envs;
    int got = 0;
    while (got < want) {
      // lane l holds buckets 127 - 4 l .. 124 - 4 l: lane order is descending key order
      int tk[4], a[4], sum = 0;
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const int b = LS_RANK_BUCKETS - 1 - 4 * lane - j;
        tk[j] = ld_relaxed(&cnt[2 * LS_RANK_BUCKETS + b]);
        a[j] = max(ld_relaxed(&cnt[LS_RANK_BUCKETS + b]) - tk[j], 0);
        sum += a[j];
      }
      int incl = sum;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
      if (__shfl_sync(0xffffffffu, incl, 31) == 0) break;
      int above = incl - sum, mine = 0, g[4];
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const int b = LS_RANK_BUCKETS - 1 - 4 * lane - j;
        g[j] = min(max(want - got - above, 0), a[j]);
        above += a[j];
        if (g[j] > 0 && atomicCAS(&cnt[2 * LS_RANK_BUCKETS + b], tk[j], tk[j] + g[j]) != tk[j]) g[j] = 0;   // raced: retry
        mine += g[j];
      }
      int off = mine;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, off, o); if (lane >= o) off += v; }
      const int total = __shfl_sync(0xffffffffu, off, 31);
      off += got - mine;
      // the claimed slots, one per lane (a bucket often gives all of them): first their indices into s_env ...
#pragma unroll
      for (int j = 0; j < 4; j++) {
        const int b = LS_RANK_BUCKETS - 1 - 4 * lane - j;
        for (int i = 0; i < g[j]; i++) s_env[off++] = b * n_envs + tk[j] + i;
      }
      __syncwarp();
      if (lane < total) {
        // ... then the env ids. A slot is reserved before its env id is stored: wait for the (running) publisher
        int* slot = benv + s_env[got + lane];
        int v;
        while ((v = ld_relaxed(slot)) < 0) __nanosleep(32);
        st_relaxed(slot, -1);
        s_env[got + lane] = v;
      }
      __syncwarp();
      if (lane == 0 && total > 0) atomicAdd(&q.tot[2 * s + 1], total);
      got += total;
    }
    if (got > 0) {
      __threadfence();            // (acquire: the envs' state is read after their ids)
      *chunk = c;
      return got;
    }
  }
}

// one chunk [k0, k1) of one env: substep_body with the env given, L1-bypassing loads, and the env published into the next
// chunk's buckets; returns the warp's Newton iterations in the chunk
template <class C>
__device__ __forceinline__ int persist_body(unsigned char* smem_raw, int ms, const DevTask& t, const SolverOpts& so,
                                            const EngineState& st, const float* __restrict__ action,
                                            float* __restrict__ obs, float* __restrict__ reward,
                                            uint8_t* __restrict__ done, float* __restrict__ next_obs, int n_envs,
                                            int auto_reset, uint64_t seed, int64_t env_off, int sync_substeps,
                                            int key_mode_in, int stage_bytes, int env, bool ghost, int c,
                                            const PersistQueue& q, int par) {
  PH_T0(t_ph);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int k0 = c * q.chunk, k1 = min(k0 + q.chunk, t.n_substeps);
  EnvS<C>& e = reinterpret_cast<EnvS<C>*>(smem_raw)[warp];
  const DevModel& m = c_models[ms];
  const int nv = m.nv, nu = m.nu;
  e.env = env;     // (every lane: a predicated store costs the persistent kernel a spill)
  e.substep = ghost ? -1 : k0;
  if (lane == 0) {
    e.prm = st.pool + (size_t)__ldcg(&st.dr_row[env]) * m.pool_P;
    if (stage_bytes > 0) {
      const unsigned char* sm = smem_raw + (size_t)(blockDim.x >> 5) * sizeof(EnvS<C>);
      e.pk_tab = reinterpret_cast<const int*>(sm);
    } else { e.pk_tab = m.pair_packed; }
  }

  // ---- load state ----
  for (int i = lane; i < nv; i += 32) {
    e.qpos[i] = __ldcg(&st.qpos[(size_t)env * nv + i]);
    e.qvel[i] = __ldcg(&st.qvel[(size_t)env * nv + i]);
    e.qacc_ws[i] = __ldcg(&st.ws[(size_t)env * nv + i]);
    e.qacc[i] = 0;
  }
  for (int i = lane; i < nu; i += 32) e.ctrl[t.act_idx[i]] = action[(size_t)env * nu + i] * t.act_delta[i] + t.act_mean[i];
  if (lane < 4) e.goal[lane] = __ldcg(&st.goal[(size_t)env * 4 + lane]);
  __syncwarp();
  init_workspace(ms, e);
  float rew;
  if (k0 > 0) {
    // what the previous chunks of this control step left behind
    rew = load_carry<C, true>(q.carry + (size_t)env * LS_CARRY, e);
  } else {
    if (lane == 0) e.iter_sum = 0;
    if (lane < 3 * LS_MAX_GRF) e.grf[lane] = 0;
    rew = prev_obs_reward(t, e);
  }
  PH_LAP(PH_PROLOGUE, t_ph);
  PH_CNT(PH_GROUPS, 1);

  // ---- physics ----
  if (sync_substeps) {
    // keep the warps of a block in the same phase: they then share instruction-cache lines
    for (int k = k0; k < k1; k++) { if (k % sync_substeps == 0) __syncthreads(); physics_substeps(ms, e, so, 1, t.grf_group, t.n_grf); }
  } else {
    physics_substeps(ms, e, so, k1 - k0, t.grf_group, t.n_grf);
  }
  // the counts at the chunk's start, read from the carry record as in substep_body (past L1, like every read of a record
  // another SM may have written)
  const int* rec = q.carry + (size_t)env * LS_CARRY;
  const int iter0 = k0 > 0 ? ld_relaxed(&rec[0]) : 0, mpr0 = k0 > 0 ? ld_relaxed(&rec[1]) : 0;
  const int iters = e.iter_sum - iter0;
  int key = launch_key(t, e, k0, k1, iter0, mpr0, key_mode_in);
  PH_T0(t_epi);

  if (k1 < t.n_substeps) {
    // ---- not the last chunk of the control step: state and carried fields to HBM, env into the next chunk's bucket ----
    if (!ghost) {
      for (int i = lane; i < nv; i += 32) {
        st.qpos[(size_t)env * nv + i] = e.qpos[i];
        st.qvel[(size_t)env * nv + i] = e.qvel[i];
        st.ws[(size_t)env * nv + i] = e.qacc_ws[i];
      }
      save_carry<C>(q.carry + (size_t)env * LS_CARRY, e, rew);
      __threadfence();
      __syncwarp();
      if (lane == 0) persist_publish(q, par, c + 1, env, n_envs, key);
    }
    PH_LAP(PH_EPILOGUE, t_epi);
    return iters;
  }
  if (ghost) return iters;
  const bool reset = step_epilogue<C>(ms, t, st, e, env, rew, obs, reward, done, next_obs, auto_reset, seed, env_off,
                                      key_mode_in);
  __threadfence();
  __syncwarp();
  if (lane == 0) {
    // into chunk 0 of the next step
    if (reset && (key_mode_in >> 16)) key = (key_mode_in >> 16) - 1;
    persist_publish(q, par, q.nch, env, n_envs, key);
  }
  PH_LAP(PH_EPILOGUE, t_epi);
  return iters;
}

template <class C>
__global__ void __launch_bounds__(512, 1) persist_kernel(int ms, DevTask t, SolverOpts so, EngineState st,
                                                       const float* __restrict__ action, float* __restrict__ obs,
                                                       float* __restrict__ reward, uint8_t* __restrict__ done,
                                                       float* __restrict__ next_obs, int n_envs, int auto_reset,
                                                       uint64_t seed, int64_t env_off, int sync_substeps, int key_mode_in,
                                                       const unsigned char* __restrict__ stage_src, int stage_bytes,
                                                       PersistQueue q) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ int s_env[16], s_n, s_c, s_par, s_it[2];
  __shared__ long long s_t[2];   // timeline: pop start, group start (in shared memory: nothing extra live across the body)
  const int warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  stage_pair_table<C>(smem_raw, stage_src, stage_bytes);   // once per block for the whole step
  if (threadIdx.x == 0) s_par = __ldcg(&q.seq[0]) & 1;
  __syncthreads();
  for (;;) {
    if (q.tl && threadIdx.x == 0) { s_t[0] = global_ns(); s_it[0] = 0; s_it[1] = 0; }
    if (warp == 0) {
      int c = 0;
      const int n = persist_pop(q, s_par, n_envs, wpb, s_env, &c);
      if (threadIdx.x == 0) { s_n = n; s_c = c; }
    }
    __syncthreads();
    const int n = s_n;
    if (n == 0) break;
    if (q.tl && threadIdx.x == 0) s_t[1] = global_ns();
    // warps past the group's last env shadow it (same barriers, no stores)
    const bool ghost = warp >= n;
    const int it = persist_body<C>(smem_raw, ms, t, so, st, action, obs, reward, done, next_obs, n_envs, auto_reset, seed,
                                   env_off, sync_substeps, key_mode_in, stage_bytes, s_env[ghost ? n - 1 : warp], ghost, s_c,
                                   q, s_par);
    if (q.tl && (threadIdx.x & 31) == 0) { if (!ghost) atomicAdd(&s_it[0], it); atomicMax(&s_it[1], it); }
    __syncthreads();
    if (q.tl && threadIdx.x == 0) {
      const long long r = (long long)atomicAdd((unsigned long long*)q.tl, 1ULL);
      if (r < q.tl_cap) {
        unsigned smid;
        asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
        long long* rec = q.tl + (r + 1) * LS_TL_WORDS;
        rec[0] = smid; rec[1] = s_c; rec[2] = n; rec[3] = s_t[0]; rec[4] = s_t[1]; rec[5] = global_ns(); rec[6] = s_it[0]; rec[7] = s_it[1];
      }
    }
  }
  // The block that finishes last (every env has run every chunk by then) empties the bucket sets of this step's chunks; the
  // set the last chunk filled becomes chunk 0 of the next step. No host-side counter, so CUDA graphs replay it.
  int last = 0;
  if (threadIdx.x == 0) {
    __threadfence();
    last = atomicAdd(&q.seq[1], 1) == (int)gridDim.x - 1;
  }
  if (__syncthreads_or(last)) {
    __threadfence();
    const int par = s_par;
    for (int c = 0; c < q.nch; c++) {
      const int s = persist_set(c, q.nch, par);
      for (int i = threadIdx.x; i < 3 * LS_RANK_BUCKETS; i += blockDim.x) q.cnt[(size_t)s * 3 * LS_RANK_BUCKETS + i] = 0;
      if (threadIdx.x < 2) q.tot[2 * s + threadIdx.x] = 0;
    }
    if (threadIdx.x == 0) { q.seq[0] = par ^ 1; q.seq[1] = 0; }
  }
}

// ----------------------------------------------------------------------------------------------------------
// Body-output kernel (locosim_set_body_outputs, locosim_set_reference_outputs), one warp and one EnvS per block, from the
// engine's state (the env's parameter-pool row as in the step kernels: masses and inertial frames differ per env under
// domain randomisation and carry tasks). `parts`: 1 = body rows, 2 = reference keys, 4 = reference rows (with 2).
// Body rows. After a step (done = that step's done bytes, every env): d_next_body, and d_body of the envs the step did not
// reset (the same state). The envs the step reset are those with a done byte under auto_reset, and those reset_env marked
// (a non-finite env) without it; reset_env has written their d_body rows from the terminal state, which the stored state no
// longer holds. After locosim_reset* (the envs of `mask`) and locosim_set_state (all, done = NULL): d_next_body.
// Why the rows are not all written by the step kernels: their terminal rows must be (nothing else sees the terminal state),
// and reset_env is a call those kernels already make; a body-output call of their own, in every epilogue, changes their
// register allocation and stack frames, which the off path must not pay for. This kernel is enqueued only while buffers
// are registered.
// Reference rows: the body outputs of the reset state of the table row at the env's cursor (reference_outputs), with the
// rotation angle of its episode and its parameter-pool row. The step kernels keep nothing for them: the terminal rows of an
// env the step reset come from the key this kernel stored after the env's previous step or reset (DevRefOut::key), with
// the cursor moved as the step moved it; whether the step found the env non-finite, from its non-finite count.
// ----------------------------------------------------------------------------------------------------------
template <class C>
__global__ void __launch_bounds__(32) body_kernel(int ms, DevTask t, EngineState st, const uint8_t* __restrict__ mask,
                                                  const uint8_t* __restrict__ done, int auto_reset, int parts, uint64_t seed,
                                                  int64_t env_off, const int2* __restrict__ rot_pin) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int env = blockIdx.x, lane = threadIdx.x & 31;
  if (mask && !mask[env]) return;
  EnvS<C>& e = *reinterpret_cast<EnvS<C>*>(smem_raw);
  const DevModel& m = c_models[ms];
  const int nv = m.nv;
  const size_t off = (size_t)env * m.nb * LS_BODY_DIM;
  if (parts & 1) {
    const DevBodyOut bo = c_bodyout[ms];
    float* body = nullptr;
    if (done && bo.body) {
      // (under auto_reset the done byte alone decides: a mark left by a step that was not followed by this kernel cannot
      // hide a row; every mark is cleared here)
      const int mark = bo.reset_mark[env];
      const bool was_reset = done[env] != 0 && (auto_reset || mark != 0);
      __syncwarp();
      if (!was_reset) body = bo.body + off;
      if (lane == 0 && mark) bo.reset_mark[env] = 0;
    }
    float* next = bo.next_body ? bo.next_body + off : nullptr;
    if (body || next) {
      if (lane == 0) e.prm = st.pool + (size_t)st.dr_row[env] * m.pool_P;
      for (int i = lane; i < nv; i += 32) {
        e.qpos[i] = st.qpos[(size_t)env * nv + i];
        e.qvel[i] = st.qvel[(size_t)env * nv + i];
      }
      __syncwarp();
      body_outputs(ms, e, body, next);
    }
  }
  const DevRefOut ro = c_refout[ms];
  if (!(parts & 2) || !ro.key) return;
  const int ncol = 2 * nv + t.n_goal;
  const int4 key = ro.key[env];
  const int cur = st.cursor[env], prow = st.dr_row[env], nbad = st.counters[(size_t)env * 8 + 4];
  const float angle = episode_angle(t, rot_pin, seed, env_off + env, env, st.episode[env]);
  float* ref = (parts & 4) && done && ro.ref ? ro.ref + off : nullptr;
  float* next = (parts & 4) && ro.next_ref ? ro.next_ref + off : nullptr;
  if (ref && done[env] != 0 && (auto_reset || nbad != key.w)) {
    // the step reset the env: d_ref describes the state it ended in, i.e. the key it started from with the cursor moved
    // once (clamped) under LS_REWARD_TRACKING or end_of_trajectory, as step_epilogue moves it; zeros where it found the
    // env non-finite
    if (nbad != key.w) {
      for (int k = lane; k < m.nb * LS_BODY_DIM; k += 32) ref[k] = 0.0f;
    } else {
      int c = key.x;
      if ((t.reward_type == LS_REWARD_TRACKING || st.end_of_trajectory) && c % t.traj_len + 1 < t.traj_len) c += 1;
      if (lane == 0) e.prm = st.pool + (size_t)key.z * m.pool_P;
      reference_outputs(ms, t, e, t.table + (size_t)c * ncol, __int_as_float(key.y), ref, (float*)nullptr);
    }
    ref = nullptr;
  }
  if (ref || next) {
    __syncwarp();
    if (lane == 0) e.prm = st.pool + (size_t)prow * m.pool_P;
    reference_outputs(ms, t, e, t.table + (size_t)cur * ncol, angle, ref, next);
  }
  if (lane == 0) ro.key[env] = make_int4(cur, __float_as_int(angle), prow, nbad);
}

// Reference rows of the dataset (locosim_create_dataset_bodies), one warp and one EnvS per block and dataset row: row r of
// locosim_create_dataset is (traj, sample) -> (traj, sample + 1); angle 0, parameters `prm` (the compiled model's own).
template <class C>
__global__ void __launch_bounds__(32) dataset_body_kernel(int ms, DevTask t, const float* __restrict__ prm,
                                                          float* __restrict__ body, float* __restrict__ next_body) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  EnvS<C>& e = *reinterpret_cast<EnvS<C>*>(smem_raw);
  const DevModel& m = c_models[ms];
  const int r = blockIdx.x, per = t.traj_len - 1, tj = r / per, sp = r - tj * per, ncol = 2 * m.nv + t.n_goal;
  const float* row = t.table + ((size_t)tj * t.traj_len + sp) * ncol;
  const size_t off = (size_t)r * m.nb * LS_BODY_DIM;
  if ((threadIdx.x & 31) == 0) e.prm = prm;
  reference_outputs(ms, t, e, row, 0.0f, body + off, (float*)nullptr);
  reference_outputs(ms, t, e, row + ncol, 0.0f, next_body + off, (float*)nullptr);
}

// ----------------------------------------------------------------------------------------------------------
// Inverse dynamics (locosim_inverse, locosim_create_dataset_inverse), one warp and one EnvS per block, the pair table read
// from global memory. EnvS::substep = -1: no output hook of the stages stores anything. The engine's state, counters and
// outputs are only read.
// ----------------------------------------------------------------------------------------------------------
// pk: the handle's staged pair table in global memory (the source of the step kernels' TMA copy, whose layout DevModel::pk_n
// then describes), or NULL: the model's table
// EnvS::env of dataset row r in inverse_kernel: the row itself, which no per-env buffer is indexed with on that path; the
// terrain unit (locosim_terrain.cu) marks it as no env (-1 - r), so that the terrain pass takes the zero origin there
#ifndef LS_DATASET_ENV
#define LS_DATASET_ENV(r) (r)
#endif
template <class C>
LS_DEV void inverse_setup(const int ms, EnvS<C>& e, const float* prm, const int env, const int* pk) {
  if ((threadIdx.x & 31) == 0) {
    e.prm = prm;
    e.pk_tab = pk ? pk : c_models[ms].pair_packed;
    e.env = env;
    e.substep = -1;
  }
  __syncwarp();
  init_workspace(ms, e);
}

// reset_value's qvel at rotation angle 0, with sin 0 = 0 and cos 0 = 1 spelled out: the same bits without sincosf
__device__ __forceinline__ float reset_qvel0(const DevTask& t, const float* row, int nv, int idx) {
  if (t.rot[0] >= 0 && (idx == t.rot[1] || idx == t.rot[2])) {
    const float vx = row[nv + t.rot[1]], vy = row[nv + t.rot[2]];
    return idx == t.rot[1] ? 1.0f * vx - 0.0f * vy : 0.0f * vx + 1.0f * vy;
  }
  return row[nv + idx];
}

// One kernel for both calls, one warp and one EnvS per block, the pair table read from global memory (no TMA staging).
//   inv_dt == 0 (locosim_inverse): block = env, at its stored state and parameter-pool row: qacc / qfrc [n_envs, nv]
//   inv_dt > 0 (locosim_create_dataset_inverse): block = row r of locosim_create_dataset, (traj, sample) -> (traj,
//     sample + 1): the reset state of (traj, sample) (angle 0, parameters `prm`, the compiled model's own) at
//     qacc = (qvel[sample + 1] - qvel[sample]) * inv_dt; qfrc [rows, nv]
template <class C>
__global__ void __launch_bounds__(32) inverse_kernel(int ms, EngineState st, DevTask t, const int* __restrict__ pk,
                                                     const float* __restrict__ qacc, const float* __restrict__ prm, float inv_dt,
                                                     float* __restrict__ qfrc) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  EnvS<C>& e = *reinterpret_cast<EnvS<C>*>(smem_raw);
  const DevModel& m = c_models[ms];
  const int r = blockIdx.x, lane = threadIdx.x & 31, nv = m.nv;
  if (inv_dt > 0.0f) {
    const int per = t.traj_len - 1, tj = r / per, sp = r - tj * per, ncol = 2 * nv + t.n_goal;
    const float* row = t.table + ((size_t)tj * t.traj_len + sp) * ncol;
    inverse_setup(ms, e, prm, LS_DATASET_ENV(r), pk);
    for (int i = lane; i < nv; i += 32) {
      e.qpos[i] = reset_value(t, row, nv, LS_OBS_QPOS, i, 0.0f);
      e.qvel[i] = reset_qvel0(t, row, nv, i);
      e.qacc[i] = (reset_qvel0(t, row + ncol, nv, i) - e.qvel[i]) * inv_dt;
    }
  } else {
    inverse_setup(ms, e, st.pool + (size_t)st.dr_row[r] * m.pool_P, r, pk);
    for (int i = lane; i < nv; i += 32) {
      e.qpos[i] = st.qpos[(size_t)r * nv + i];
      e.qvel[i] = st.qvel[(size_t)r * nv + i];
      e.qacc[i] = qacc[(size_t)r * nv + i];
    }
  }
  __syncwarp();
  inverse_dynamics(ms, e, qfrc + (size_t)r * nv);
}

// ----------------------------------------------------------------------------------------------------------
// Dynamics terms (locosim_dynamics_terms), inverse_kernel's layout: one warp and one EnvS per block (block = env), at the
// env's stored state and parameter-pool row. No collision runs, so no pair table is read. EnvS::substep = -1; the engine's
// state, counters and outputs are only read. `o` holds the whole buffers (or NULL); each env writes its own rows.
// ----------------------------------------------------------------------------------------------------------
template <class C>
__global__ void __launch_bounds__(32) dynamics_kernel(int ms, EngineState st, DynOut o) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  EnvS<C>& e = *reinterpret_cast<EnvS<C>*>(smem_raw);
  const DevModel& m = c_models[ms];
  const int r = blockIdx.x, lane = threadIdx.x & 31, nv = m.nv;
  inverse_setup(ms, e, st.pool + (size_t)st.dr_row[r] * m.pool_P, r, (const int*)nullptr);
  for (int i = lane; i < nv; i += 32) {
    e.qpos[i] = st.qpos[(size_t)r * nv + i];
    e.qvel[i] = st.qvel[(size_t)r * nv + i];
  }
  __syncwarp();
  const size_t rv = (size_t)r * nv;
  DynOut row;
  row.M = o.M ? o.M + rv * nv : nullptr;
  row.bias = o.bias ? o.bias + rv : nullptr;
  row.passive = o.passive ? o.passive + rv : nullptr;
  row.com = o.com ? o.com + (size_t)r * LS_COM_DIM : nullptr;
  row.jac = o.jac ? o.jac + rv * m.nb * 6 : nullptr;
  row.jac_com = o.jac_com ? o.jac_com + rv * 3 : nullptr;
  dynamics_terms(ms, e, row);
}

// ----------------------------------------------------------------------------------------------------------
// Forward dynamics (locosim_forward), inverse_kernel's layout: one warp and one EnvS per block (block = env), at the env's
// stored state, warm start and parameter-pool row, ctrl from `action` as the step kernels map it, the pair table read as
// inverse_kernel reads it. EnvS::substep = -1: no output hook of the stages stores anything (smooth_forces leaves the dof
// outputs' actuator scratch alone). `so` has no block barriers (one warp per block). The engine's state is only read.
// ----------------------------------------------------------------------------------------------------------
template <class C>
__global__ void __launch_bounds__(32) forward_kernel(int ms, EngineState st, DevTask t, const int* __restrict__ pk,
                                                     SolverOpts so, const float* __restrict__ action, FwdOut o) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  EnvS<C>& e = *reinterpret_cast<EnvS<C>*>(smem_raw);
  const DevModel& m = c_models[ms];
  const int r = blockIdx.x, lane = threadIdx.x & 31, nv = m.nv, nu = m.nu, nb = m.nb;
  inverse_setup(ms, e, st.pool + (size_t)st.dr_row[r] * m.pool_P, r, pk);
  for (int i = lane; i < nv; i += 32) {
    e.qpos[i] = st.qpos[(size_t)r * nv + i];
    e.qvel[i] = st.qvel[(size_t)r * nv + i];
    e.qacc_ws[i] = st.ws[(size_t)r * nv + i];
    e.qacc[i] = 0;
  }
  for (int i = lane; i < nu; i += 32) e.ctrl[t.act_idx[i]] = action[(size_t)r * nu + i] * t.act_delta[i] + t.act_mean[i];
  if (lane == 0) e.iter_sum = 0;
  __syncwarp();
  FwdOut row;
  row.dof = o.dof ? o.dof + (size_t)r * nv * LS_DOF_DIM : nullptr;
  row.body_acc = o.body_acc ? o.body_acc + (size_t)r * nb * LS_BODY_ACC_DIM : nullptr;
  row.cfrc_int = o.cfrc_int ? o.cfrc_int + (size_t)r * nb * LS_CONTACT_DIM : nullptr;
  row.cfrc_ext = o.cfrc_ext ? o.cfrc_ext + (size_t)r * nb * LS_CONTACT_DIM : nullptr;
  forward_dynamics(ms, e, so, row);
}

// ----------------------------------------------------------------------------------------------------------
// Ray casting (locosim_ray). Block (env, chunk) casts rays [chunk * LS_RAY_BLOCK, +LS_RAY_BLOCK) of env `env`: warp 0 runs
// kinematics() on the block's EnvS at the env's stored state and pool row, the block stages every geom's world frame into
// a RayGeom table behind the EnvS, then each thread casts one ray against the whole table (ray_geoms). The engine's state
// is only read. Instantiated in locosim_ray.cu only: the step kernels' translation units compile none of this code.
// ----------------------------------------------------------------------------------------------------------
#define LS_RAY_BLOCK 128
struct RayArgs {
  const float *pnt, *vec;          // [n_rays, 3] or, with LS_RAY_PER_ENV, [n_envs, n_rays, 3]
  float* dist;                     // [n_envs, n_rays]
  int* geom;                       // [n_envs, n_rays]
  float* normal;                   // [n_envs, n_rays, 3] or NULL
  int n_rays, frame, frame_body, exclude, flags;
};
template <class C>
__global__ void __launch_bounds__(LS_RAY_BLOCK) ray_kernel(int ms, EngineState st, RayArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  EnvS<C>& e = *reinterpret_cast<EnvS<C>*>(smem_raw);
  RayGeom* G = reinterpret_cast<RayGeom*>(smem_raw + sizeof(EnvS<C>));
  __shared__ int bad;
  const DevModel& m = c_models[ms];
  const int r = blockIdx.x, nv = m.nv, ng = m.ng;
  if (threadIdx.x < 32) {
    if (threadIdx.x == 0) e.prm = st.pool + (size_t)st.dr_row[r] * m.pool_P;
    for (int i = threadIdx.x; i < nv; i += 32) {
      e.qpos[i] = st.qpos[(size_t)r * nv + i];
      e.qvel[i] = st.qvel[(size_t)r * nv + i];
    }
    __syncwarp();
    const bool nf = nonfinite_state(e, nv);
    if (!nf) kinematics(ms, e);
    if (threadIdx.x == 0) bad = nf;
  }
  __syncthreads();
  if (!bad)
    for (int g = threadIdx.x; g < ng; g += blockDim.x) ray_stage_geom(ms, e, g, G[g]);
  __syncthreads();
  const int k = blockIdx.y * blockDim.x + threadIdx.x;
  if (k >= a.n_rays) return;
  const size_t o = (size_t)r * a.n_rays + k, src = 3 * ((a.flags & LS_RAY_PER_ENV) ? o : (size_t)k);
  float dist = -1, nrm[3] = {0, 0, 0};
  int geom = -1;
  if (!bad) {
    const float pnt[3] = {__ldg(a.pnt + src), __ldg(a.pnt + src + 1), __ldg(a.pnt + src + 2)};
    const float vec[3] = {__ldg(a.vec + src), __ldg(a.vec + src + 1), __ldg(a.vec + src + 2)};
    float p[3], v[3];
    ray_to_world(e, a.frame, a.frame_body, pnt, vec, p, v);
    dist = ray_geoms(G, ng, p, v, a.exclude, a.flags, &geom, nrm);
#ifdef LOCOSIM_TERRAIN
    if constexpr (C::TERRAIN) ray_terrain(ms, r, p, v, a.exclude, a.flags, &dist, &geom, nrm);
#endif
  }
  a.dist[o] = dist;
  a.geom[o] = geom;
  if (a.normal) for (int c = 0; c < 3; c++) a.normal[3 * o + c] = nrm[c];
}

// ----------------------------------------------------------------------------------------------------------
// Regrouping: the warps of a block run the solver in lock-step, so a block is as slow as its hardest env. Solver effort
// is strongly correlated from one control step to the next (lag-1 correlation of the per-step Newton iteration count
// ~0.6), so before every step the envs are bucketed by the iteration count of their previous step (counting sort,
// one block) and envs of similar effort share a block. Pure scheduling: results do not depend on the mapping.
// ----------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) rank_kernel(const int* __restrict__ counters, int* __restrict__ perm, int n_envs,
                                                    int key_shift) {
  __shared__ int hist[LS_RANK_BUCKETS];
  __shared__ int base[LS_RANK_BUCKETS];
  for (int i = threadIdx.x; i < LS_RANK_BUCKETS; i += blockDim.x) hist[i] = 0;
  __syncthreads();
  for (int i = threadIdx.x; i < n_envs; i += blockDim.x) {
    int k = counters[(size_t)i * 8 + 5] >> key_shift;
    atomicAdd(&hist[k < LS_RANK_BUCKETS - 1 ? k : LS_RANK_BUCKETS - 1], 1);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int i = 0; i < LS_RANK_BUCKETS; i++) { base[i] = acc; acc += hist[i]; }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < n_envs; i += blockDim.x) {
    int k = counters[(size_t)i * 8 + 5] >> key_shift;
    int pos = atomicAdd(&base[k < LS_RANK_BUCKETS - 1 ? k : LS_RANK_BUCKETS - 1], 1);
    perm[n_envs - 1 - pos] = i;     // hardest first: the long blocks start early, the short ones fill the tail
  }
}

// ----------------------------------------------------------------------------------------------------------
// handle
// ----------------------------------------------------------------------------------------------------------
struct locosim_handle {
  int device = 0, n_envs = 0, cfg = -1, wpb = 4, smem = 0, slot = -1, sync_substeps = 0, regroup = 1, key_shift = 0, key_mode = 3;
  int n_sm = 1;
  int resort = 0;                   // sub-steps per launch of the step kernel (>= n_substeps: one fused launch per step)
  SplitState split = {};
  int persist = 0, persist_grid = 0;   // resort < n_substeps: one persist_kernel launch of persist_grid blocks per step
  int persist_static = 0;              // static shared memory of persist_kernel<C> (bytes)
  PersistQueue pq = {};
  uint64_t seed = 0;
  int64_t env_off = 0;
  HostModel hm;
  HostTask ht;
  DevModel dm;
  DevApplied applied = {nullptr, nullptr};
  DevBodyOut bodyout = {nullptr, nullptr, nullptr};
  DevRefOut refout = {nullptr, nullptr, nullptr};
  int4* ref_key = nullptr;           // the reference keys [n_envs] (DevRefOut::key) once reference outputs were registered
  int2* rot_pin = nullptr;           // [n_envs] episode number and angle of the last rotation reset_kernel was given (episode_angle)
  uint8_t* load_mask = nullptr;      // [n_envs] the envs the last locosim_load_state loaded (load_state_kernel -> body_kernel)
  int state_fp = 0;                  // layout fingerprint of the saved-state rows (LS_STATE_TAG)
  float* d_model_row = nullptr;      // the compiled model's own parameter row (locosim_create_dataset_bodies), on first use
  DevContact contact = {nullptr, 1};
  DevDof dof = {nullptr, 1};
  float* dof_act = nullptr;          // the dof outputs' actuator-force scratch [n_envs, nu] (c_dof_act)
  DevConList conlist = {nullptr, 1};
  DevConRows conrows = {nullptr, nullptr};
  DevTask dt;
  SolverOpts so;
  EngineState st;
  int* d_mints = nullptr; float* d_mreals = nullptr; int* d_tints = nullptr; float* d_treals = nullptr;
  float* d_pool = nullptr;
  unsigned char* d_stage = nullptr; int stage_bytes = 0;
  float* terrain_origin = nullptr;   // caller-owned [n_envs, 2] terrain origin per env (locosim_set_terrain_origin), or NULL
  std::string err;
};
#ifndef LOCOSIM_EXTRA_CONFIGS_TU
static std::string g_create_error;
static bool g_slot_used[LS_MAX_SLOTS] = {false};
#endif

#define CK(call)                                                                      \
  do {                                                                                \
    cudaError_t _e = (call);                                                          \
    if (_e != cudaSuccess) {                                                          \
      h->err = std::string(#call) + ": " + cudaGetErrorString(_e);                    \
      return 1;                                                                       \
    }                                                                                 \
  } while (0)

template <class C>
static int cfg_smem() { return (int)sizeof(EnvS<C>); }
// sizeof(EnvS) decides the envs resident per SM (227 KB of dynamic shared memory per block on sm_90): a field added without
// looking costs a whole env per SM (on the 132 SMs of an H100 and 4096 envs, a few percent more blocks in the last wave).
// Guard the layout.
static_assert(sizeof(EnvS<CfgEllEuler>) * 15 <= 232448, "UnitreeA1: 15 envs per SM");
static_assert(sizeof(EnvS<CfgPyrEuler>) * 15 <= 232448, "Talos / UnitreeH1: 15 envs per SM");
static_assert(sizeof(EnvS<CfgPyrRK4>) * 14 <= 232448, "HumanoidTorque / Atlas: 14 envs per SM (293 blocks = 2.22 waves at 4096 envs on 132 SMs)");
static_assert(sizeof(EnvS<CfgPyrEuler29>) * 9 <= 232448, "UnitreeG1: 9 envs per SM");

template <class C>
static int launch_body(locosim_handle* h, const uint8_t* mask, const uint8_t* done, int auto_reset, int parts, cudaStream_t s) {
  static_assert(sizeof(EnvS<C>) <= 48 * 1024, "body_kernel: one EnvS per block within the default shared-memory limit");
  body_kernel<C><<<h->n_envs, 32, sizeof(EnvS<C>), s>>>(h->slot, h->dt, h->st, mask, done, auto_reset, parts, h->seed,
                                                        h->env_off, h->rot_pin);
  CK(cudaGetLastError());
  return 0;
}
template <class C>
static int launch_dataset_bodies(locosim_handle* h, float* body, float* next_body, cudaStream_t s) {
  const int rows = h->ht.n_traj * (h->ht.traj_len - 1);
  if (rows > 0)
    dataset_body_kernel<C><<<rows, 32, sizeof(EnvS<C>), s>>>(h->slot, h->dt, h->d_model_row, body, next_body);
  CK(cudaGetLastError());
  return 0;
}
// C with the primitive pairs filtered by collision()'s round loop (PRIMLEAN = 0: the same contact list as the lean pass, and
// the same EnvS layout). inverse_kernel is instantiated with it in every configuration, so that it compiles to the same
// registers and stack whichever pass UnitreeA1's step kernels use (LOCOSIM_PRIMLEAN), and its stages are copies of their
// own that leave the step kernels' untouched.
template <class C>
struct RoundLoop : C { enum { PRIMLEAN = 0 }; };
template <class C>
static int launch_inverse(locosim_handle* h, const float* qacc, float* qfrc, cudaStream_t s) {
  static_assert(sizeof(EnvS<C>) <= 48 * 1024, "inverse_kernel: one EnvS per block within the default shared-memory limit");
  inverse_kernel<RoundLoop<C>><<<h->n_envs, 32, sizeof(EnvS<C>), s>>>(h->slot, h->st, h->dt, (const int*)h->d_stage,
                                                                       qacc, nullptr, 0.0f, qfrc);
  CK(cudaGetLastError());
  return 0;
}
// 1 / (timestep * n_substeps), the dataset's control rate, in double from the model's fp32 timestep (the device code divides
// with -prec-div=false; a caller rebuilds the dataset's qacc bit for bit from this value)
static float dataset_inv_dt(const locosim_handle* h) {
  return (float)(1.0 / ((double)h->hm.timestep * (double)h->dt.n_substeps));
}
template <class C>
static int launch_dataset_inverse(locosim_handle* h, float* qfrc, cudaStream_t s) {
  static_assert(sizeof(EnvS<C>) <= 48 * 1024, "inverse_kernel: one EnvS per block within the default shared-memory limit");
  const int rows = h->ht.n_traj * (h->ht.traj_len - 1);
  if (rows > 0)
    inverse_kernel<RoundLoop<C>><<<rows, 32, sizeof(EnvS<C>), s>>>(h->slot, h->st, h->dt, (const int*)h->d_stage,
                                                                   nullptr, h->d_model_row, dataset_inv_dt(h), qfrc);
  CK(cudaGetLastError());
  return 0;
}
// dynamics_kernel with inverse_kernel's configuration type: the stages both call (kinematics, com_pos, crb_factor,
// passive_bias) are then the same functions
template <class C>
static int launch_dynamics(locosim_handle* h, const DynOut& o, cudaStream_t s) {
  static_assert(sizeof(EnvS<C>) <= 48 * 1024, "dynamics_kernel: one EnvS per block within the default shared-memory limit");
  dynamics_kernel<RoundLoop<C>><<<h->n_envs, 32, sizeof(EnvS<C>), s>>>(h->slot, h->st, o);
  CK(cudaGetLastError());
  return 0;
}
// forward_kernel with inverse_kernel's configuration type and pair table (the same contact list as the step kernels' first
// evaluation of a control step) and the handle's solver settings without block barriers
template <class C>
static int launch_forward(locosim_handle* h, const float* action, const FwdOut& o, cudaStream_t s) {
  static_assert(sizeof(EnvS<C>) <= 48 * 1024, "forward_kernel: one EnvS per block within the default shared-memory limit");
  SolverOpts so = h->so;
  so.sync_iters = 0;
  so.sync_phases = 0;
  forward_kernel<RoundLoop<C>><<<h->n_envs, 32, sizeof(EnvS<C>), s>>>(h->slot, h->st, h->dt, (const int*)h->d_stage, so,
                                                                       action, o);
  CK(cudaGetLastError());
  return 0;
}
// ray_kernel with inverse_kernel's configuration type (locosim_ray.cu); the caller has checked the grid's y extent
template <class C>
static int launch_ray(locosim_handle* h, const RayArgs& a, cudaStream_t s) {
  constexpr size_t smem = sizeof(EnvS<C>) + sizeof(RayGeom) * C::NG;
  static_assert(smem <= 48 * 1024, "ray_kernel: one EnvS and the geom table per block within the default shared-memory limit");
  const dim3 grid((unsigned)h->n_envs, (unsigned)((a.n_rays + LS_RAY_BLOCK - 1) / LS_RAY_BLOCK));
  ray_kernel<RoundLoop<C>><<<grid, LS_RAY_BLOCK, smem, s>>>(h->slot, h->st, a);
  CK(cudaGetLastError());
  return 0;
}
template <class C>
static int launch_step(locosim_handle* h, const float* a, float* o, float* r, uint8_t* d, float* no, int auto_reset,
                       cudaStream_t s) {
  int blocks = (h->n_envs + h->wpb - 1) / h->wpb;
  const int smem = h->smem + (h->stage_bytes ? h->stage_bytes + 16 : 0), nsub = h->dt.n_substeps;
  if (h->resort >= nsub) {
    if (h->regroup) rank_kernel<<<1, 1024, 0, s>>>(h->st.counters, h->st.perm, h->n_envs, h->key_shift);
    step_kernel<C><<<blocks, h->wpb * 32, smem, s>>>(h->slot, h->dt, h->so, h->st, a, o, r, d, no, h->n_envs, auto_reset,
                                                      h->seed, h->env_off, h->sync_substeps, h->key_mode, h->d_stage,
                                                      h->stage_bytes);
  } else if (h->persist) {
    persist_kernel<C><<<h->persist_grid, h->wpb * 32, smem, s>>>(h->slot, h->dt, h->so, h->st, a, o, r, d, no, h->n_envs,
                                                                 auto_reset, h->seed, h->env_off, h->sync_substeps,
                                                                 h->key_mode, h->d_stage, h->stage_bytes, h->pq);
  } else {
    for (int k0 = 0; k0 < nsub; k0 += h->resort)
      substep_kernel<C><<<blocks, h->wpb * 32, smem, s>>>(h->slot, h->dt, h->so, h->st, a, o, r, d, no, h->n_envs, auto_reset,
                                                         h->seed, h->env_off, h->sync_substeps, h->key_mode, h->d_stage,
                                                         h->stage_bytes, k0, k0 + h->resort < nsub ? k0 + h->resort : nsub,
                                                         h->split);
  }
  CK(cudaGetLastError());
  // body and reference outputs (only while registered): the rows the step kernel did not write
  if (h->bodyout.body || h->bodyout.next_body || h->refout.key) return launch_body<C>(h, nullptr, d, auto_reset, 7, s);
  return 0;
}
template <class C>
static int setup_cfg(locosim_handle* h) {
  int per_env = cfg_smem<C>();
  int dev_max = 0;
  CK(cudaDeviceGetAttribute(&dev_max, cudaDevAttrMaxSharedMemoryPerBlockOptin, h->device));
  int sm_total = 0;
  CK(cudaDeviceGetAttribute(&sm_total, cudaDevAttrMaxSharedMemoryPerMultiprocessor, h->device));
  // envs resident per SM for w warps per block (1 KB per block is reserved by the driver)
  auto envs_per_sm = [&](int w) {
    int sm = w * per_env;
    if (sm > dev_max) return 0;
    int b = sm_total / (sm + 1024);
    return (b > 32 ? 32 : b) * w;
  };
  int best = 1, best_env = 0;
  for (int w = 1; w <= 16; w++) { int ev = envs_per_sm(w); if (ev > best_env) { best_env = ev; best = w; } }
  // Warps of one block are kept in lock-step with block barriers (every sub-step and every Newton iteration) so that
  // they execute the same code at the same time and share instruction-cache lines; of the block sizes that keep the same
  // number of envs resident, the largest block is the fastest (H100, A1 4096 envs: 1 x 15 warps 1.24 M, 3 x 5 warps
  // 0.99 M env-steps/s) -> take it.
  h->sync_substeps = 1;
  for (int w = 16; w >= 1; w--) {
    if (envs_per_sm(w) == best_env) { best = w; break; }
  }
  {
    // A batch that does not even give every SM one full block is spread over all SMs with smaller blocks: one block per SM
    // beats half of the SMs running 14-15 warps (BASELINE config 4: Atlas.walk 1024 envs as 128 blocks of 8 on an H100's
    // 132 SMs instead of 74 of 14, next to Talos.walk 1024).
    int n_sm = 0;
    CK(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, h->device));
    // LOCOSIM_WPB=-1 keeps the largest block (MixedBatch: the lighter members of a mixed batch; small blocks of two different
    // kernels on every SM were slower after an L2 flush than one member spread and the other in full blocks).
    const bool keep = getenv("LOCOSIM_WPB") && atoi(getenv("LOCOSIM_WPB")) == -1;
    if (!keep && n_sm > 0 && (h->n_envs + best - 1) / best < n_sm) { int w = (h->n_envs + n_sm - 1) / n_sm; best = w < 1 ? 1 : (w < best ? w : best); }
  }
  if (getenv("LOCOSIM_WPB")) { int w = atoi(getenv("LOCOSIM_WPB")); if (w >= 1 && w <= 16 && w * per_env <= dev_max) best = w; }
  if (getenv("LOCOSIM_SYNC")) h->sync_substeps = atoi(getenv("LOCOSIM_SYNC"));
  h->regroup = 1;
  if (getenv("LOCOSIM_REGROUP")) h->regroup = atoi(getenv("LOCOSIM_REGROUP"));
  h->key_shift = C::RK4 ? 2 : 0;   // RK4: four solves per sub-step
  if (getenv("LOCOSIM_KEY_SHIFT")) h->key_shift = atoi(getenv("LOCOSIM_KEY_SHIFT"));
  if (getenv("LOCOSIM_KEY_MODE")) h->key_mode = atoi(getenv("LOCOSIM_KEY_MODE"));
  {
    // an MPR run holds its lock-step block about as long as `w` Newton iterations; key of a freshly reset env (+1; 0 = keep)
    int w = C::CONE == 1 ? 4 : 32, kr = C::CONE == 1 ? 1 : 0;       // (chosen by knob sweeps: tools/knob_sweep*.sh)
    if (getenv("LOCOSIM_MPR_WEIGHT")) w = atoi(getenv("LOCOSIM_MPR_WEIGHT"));
    if (getenv("LOCOSIM_KEY_RESET")) kr = atoi(getenv("LOCOSIM_KEY_RESET")) + 1;
    h->key_mode = (h->key_mode & 255) | ((w & 255) << 8) | (kr << 16);
  }
  {
    // sub-steps per launch (regrouping between launches), default by H100 A/B (bench.py, 4096 envs; fused = 10):
    // UnitreeA1.simple 1.24 M env-steps/s fused, 1.31 M at 5, 1.33 M at 2, 1.28 M at 1 -> 2 for CfgEllEuler;
    // HumanoidTorque.run (CfgPyrRK4) 0.437 M fused, 0.395 M at 5, 0.373 M at 2 -> fused. The configurations not measured
    // (Talos / H1, G1) and batches that leave SMs without a full block (the spread geometry, MixedBatch members: config 4
    // 0.76 M fused, 0.68 M at 2) keep the fused kernel.
    const int nsub = h->dt.n_substeps;
    const bool full = (h->n_envs + best - 1) / best >= h->n_sm;
    h->resort = full && C::CONE == 1 && !C::RK4 ? 2 : nsub;
    // ... and all of them in one persistent launch (persist_kernel) where the sub-step split is the default; LOCOSIM_RESORT
    // alone selects the separate launches, LOCOSIM_PERSIST=1 the persistent kernel with LOCOSIM_RESORT sub-steps per chunk
    h->persist = h->resort < nsub && !getenv("LOCOSIM_RESORT");
    if (getenv("LOCOSIM_RESORT")) h->resort = atoi(getenv("LOCOSIM_RESORT"));
    if (h->resort < 1 || h->resort > nsub) h->resort = nsub;
    if (getenv("LOCOSIM_PERSIST")) h->persist = atoi(getenv("LOCOSIM_PERSIST")) > 0;
    if (h->resort >= nsub) h->persist = 0;
    if (h->persist) {
      // bucket sets: chunk 0 of this step and of the next alternate between sets 0 and 1, chunks 1 .. nch-1 use 2 .. nch
      const size_t N = (size_t)h->n_envs;
      PersistQueue& q = h->pq;
      q.chunk = h->resort;
      q.nch = (nsub + h->resort - 1) / h->resort;
      const size_t sets = (size_t)q.nch + 1;
      q.pool = 2;                  // ready envs before a block takes a group of a chunk: pool x wpb (or all the chunk has left)
      if (getenv("LOCOSIM_PERSIST_POOL")) q.pool = atoi(getenv("LOCOSIM_PERSIST_POOL"));
      if (q.pool < 0) q.pool = 0;
      q.regroup = h->regroup;
      q.key_shift = h->key_shift;
      CK(cudaMalloc((void**)&q.carry, N * LS_CARRY * 4));
      CK(cudaMalloc((void**)&q.cnt, sets * 3 * LS_RANK_BUCKETS * 4));
      CK(cudaMalloc((void**)&q.tot, sets * 2 * 4));
      CK(cudaMalloc((void**)&q.benv, sets * LS_RANK_BUCKETS * N * 4));
      CK(cudaMalloc((void**)&q.seq, 2 * 4));
      CK(cudaMemset(q.carry, 0, N * LS_CARRY * 4));
      CK(cudaMemset(q.cnt, 0, sets * 3 * LS_RANK_BUCKETS * 4));
      CK(cudaMemset(q.tot, 0, sets * 2 * 4));
      CK(cudaMemset(q.benv, 0xff, sets * LS_RANK_BUCKETS * N * 4));
      CK(cudaMemset(q.seq, 0, 2 * 4));
      // the first step reads set 0: every env published in bucket 0, in env order
      const int n = h->n_envs, cnt0[2] = {n, n};
      CK(cudaMemcpy(q.cnt, &cnt0[0], 4, cudaMemcpyHostToDevice));
      CK(cudaMemcpy(q.cnt + LS_RANK_BUCKETS, &cnt0[1], 4, cudaMemcpyHostToDevice));
      CK(cudaMemcpy(q.tot, &n, 4, cudaMemcpyHostToDevice));
      CK(cudaMemcpy(q.benv, h->st.perm, N * 4, cudaMemcpyDeviceToDevice));
      // one resident block per SM; LOCOSIM_PERSIST_GRID caps the grid (any number of blocks makes progress)
      const int blocks = (h->n_envs + best - 1) / best;
      h->persist_grid = blocks < h->n_sm ? blocks : h->n_sm;
      if (getenv("LOCOSIM_PERSIST_GRID")) { int g = atoi(getenv("LOCOSIM_PERSIST_GRID")); if (g >= 1 && g < h->persist_grid) h->persist_grid = g; }
      // (its few static shared variables come out of the same 227 KB: the TMA staging below leaves room for them)
      cudaFuncAttributes fa;
      CK(cudaFuncGetAttributes(&fa, persist_kernel<C>));
      h->persist_static = (int)fa.sharedSizeBytes;
      CK(cudaFuncSetAttribute(persist_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize, dev_max - h->persist_static));
    } else if (h->resort < nsub) {
      const size_t N = (size_t)h->n_envs;
      CK(cudaMalloc((void**)&h->split.carry, N * LS_CARRY * 4));
      CK(cudaMalloc((void**)&h->split.bcount, 2 * LS_RANK_BUCKETS * 4));
      CK(cudaMalloc((void**)&h->split.benv, 2 * LS_RANK_BUCKETS * N * 4));
      CK(cudaMalloc((void**)&h->split.seq, 2 * 4));
      CK(cudaMemset(h->split.carry, 0, N * LS_CARRY * 4));
      CK(cudaMemset(h->split.bcount, 0, 2 * LS_RANK_BUCKETS * 4));
      CK(cudaMemset(h->split.seq, 0, 2 * 4));
      // the first launch reads buffer 0: every env in bucket 0, in env order (the identity mapping)
      const int n = h->n_envs;
      CK(cudaMemcpy(h->split.bcount, &n, 4, cudaMemcpyHostToDevice));
      CK(cudaMemcpy(h->split.benv, h->st.perm, N * 4, cudaMemcpyDeviceToDevice));
      h->split.regroup = h->regroup;
      h->split.key_shift = h->key_shift;
      CK(cudaFuncSetAttribute(substep_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize, dev_max));
    }
  }
  h->so.sync_iters = 16;    // lock-step group = the whole block
  if (getenv("LOCOSIM_SYNC_ITERS")) { int v = atoi(getenv("LOCOSIM_SYNC_ITERS")); h->so.sync_iters = v == 1 ? 16 : v; }
  if (getenv("LOCOSIM_GROUP")) h->so.sync_iters = atoi(getenv("LOCOSIM_GROUP"));
  if (h->so.sync_iters > 0 && (best + h->so.sync_iters - 1) / h->so.sync_iters > 15) h->so.sync_iters = 16;   // 15 named barriers
  h->so.sync_phases = 32;   // one more barrier where the warps enter the solver
  if (getenv("LOCOSIM_SYNC_PHASES")) h->so.sync_phases = atoi(getenv("LOCOSIM_SYNC_PHASES"));
  if (h->so.sync_iters < best) h->so.sync_phases &= 63;   // block barriers inside the Newton loop need whole-block lock-step
  h->wpb = best;
  h->smem = best * per_env;
  { int dbg = getenv("LOCOSIM_DEBUG") ? atoi(getenv("LOCOSIM_DEBUG")) : 0; CK(cudaMemcpyToSymbol(c_debug, &dbg, sizeof(int))); }
  // ---- TMA staging of the mid-phase pair table (Hopper bulk copy + mbarrier) ----
  // Default on wherever the table fits next to the per-env working sets (A1, Talos; not the RK4 configurations); on an H100
  // the A1 step time is within run-to-run noise of the unstaged one. LOCOSIM_STAGE=0 turns it off.
  if (!getenv("LOCOSIM_STAGE") || atoi(getenv("LOCOSIM_STAGE")) > 0) {
    // the PRIMITIVE part of the table (the lean loop over the convex part streams the model's table from L2)
    const int np = h->hm.np_prim;
    const int bytes = (2 * np * 4 + 15) & ~15;                   // np packed pairs directly followed by np bounds
    if (np > 0 && h->smem + bytes + 16 <= dev_max - h->persist_static) {
      CK(cudaMalloc((void**)&h->d_stage, bytes));
      CK(cudaMemset(h->d_stage, 0, bytes));
      CK(cudaMemcpy(h->d_stage, h->dm.pair_packed, 4 * np, cudaMemcpyDeviceToDevice));
      CK(cudaMemcpy(h->d_stage + 4 * np, h->dm.pair_bound, 4 * np, cudaMemcpyDeviceToDevice));
      h->dm.pk_n = np;
      CK(cudaMemcpyToSymbol(c_models, &h->dm, sizeof(DevModel), sizeof(DevModel) * h->slot));
      h->stage_bytes = bytes;
    }
  }
  // (a property of the FUNCTION, shared by every handle of this instantiation whatever its block size: always the device maximum)
  CK(cudaFuncSetAttribute(step_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize, dev_max));
  return 0;
}

#ifndef LOCOSIM_EXTRA_CONFIGS_TU
// The 31-dof configurations (CfgPyrRK4_31, CfgPyrEuler31) are compiled in their own translation unit,
// locosim_configs31.cu, linked into the same library (two nvcc processes build the library in parallel). Their entry points
// are weak: a library built from this file alone reports those models as not compiled in.
extern "C" int locosim_configs31_setup(locosim_handle* h) __attribute__((weak));
extern "C" int locosim_configs31_step(locosim_handle* h, const float* a, float* o, float* r, uint8_t* d, float* no,
                                      int auto_reset, cudaStream_t s) __attribute__((weak));
extern "C" int locosim_configs31_sync_model(locosim_handle* h) __attribute__((weak));
extern "C" int locosim_configs31_body(locosim_handle* h, const uint8_t* mask, int parts, cudaStream_t s) __attribute__((weak));
extern "C" int locosim_configs31_dataset_bodies(locosim_handle* h, float* body, float* next_body, cudaStream_t s)
    __attribute__((weak));
extern "C" int locosim_configs31_inverse(locosim_handle* h, const float* qacc, float* qfrc, cudaStream_t s)
    __attribute__((weak));
extern "C" int locosim_configs31_dataset_inverse(locosim_handle* h, float* qfrc, cudaStream_t s) __attribute__((weak));
extern "C" int locosim_configs31_dynamics(locosim_handle* h, const DynOut* o, cudaStream_t s) __attribute__((weak));
extern "C" int locosim_configs31_forward(locosim_handle* h, const float* action, const FwdOut* o, cudaStream_t s)
    __attribute__((weak));
// The ray kernels of all six configurations are compiled in a third translation unit, locosim_ray.cu, with its own
// __constant__ model slots (written at create and after a parameter-pool upload). Weak like the 31-dof entry points.
extern "C" int locosim_ray_sync_model(locosim_handle* h) __attribute__((weak));
extern "C" int locosim_ray_launch(locosim_handle* h, const RayArgs* a, cudaStream_t s) __attribute__((weak));
// The terrain configuration (CfgEllEulerTerrain, index 6) is compiled in a fourth translation unit, locosim_terrain.cu, with
// its own __constant__ slots (model, registered buffers, terrain), written by locosim_terrain_sync_model. Weak as well.
extern "C" int locosim_terrain_setup(locosim_handle* h) __attribute__((weak));
extern "C" int locosim_terrain_sync_model(locosim_handle* h) __attribute__((weak));
extern "C" int locosim_terrain_step(locosim_handle* h, const float* a, float* o, float* r, uint8_t* d, float* no,
                                    int auto_reset, cudaStream_t s) __attribute__((weak));
extern "C" int locosim_terrain_body(locosim_handle* h, const uint8_t* mask, int parts, cudaStream_t s) __attribute__((weak));
extern "C" int locosim_terrain_dataset_bodies(locosim_handle* h, float* body, float* next_body, cudaStream_t s)
    __attribute__((weak));
extern "C" int locosim_terrain_inverse(locosim_handle* h, const float* qacc, float* qfrc, cudaStream_t s)
    __attribute__((weak));
extern "C" int locosim_terrain_dataset_inverse(locosim_handle* h, float* qfrc, cudaStream_t s) __attribute__((weak));
extern "C" int locosim_terrain_dynamics(locosim_handle* h, const DynOut* o, cudaStream_t s) __attribute__((weak));
extern "C" int locosim_terrain_ray(locosim_handle* h, const RayArgs* a, cudaStream_t s) __attribute__((weak));
extern "C" int locosim_terrain_forward(locosim_handle* h, const float* action, const FwdOut* o, cudaStream_t s)
    __attribute__((weak));
// the other translation units' copies of the handle's __constant__ slots (after a registration or a pool upload)
static int sync_other_units(locosim_handle* h) {
  if ((h->cfg == 4 || h->cfg == 5) && locosim_configs31_sync_model(h)) return 1;
  if (h->cfg == 6 && locosim_terrain_sync_model(h)) return 1;
  return 0;
}

// body_kernel outside a step, for the envs of `mask` (NULL = all), the parts (see body_kernel) that are registered:
// d_next_body (1) after locosim_reset* and locosim_set_state; the reference keys (2) and d_next_ref (4) after locosim_reset*,
// the keys alone after a registration and a new parameter pool
static int next_body_rows(locosim_handle* h, const uint8_t* mask, int parts, cudaStream_t s) {
  if (!h->bodyout.next_body) parts &= ~1;
  if (!h->refout.key) parts &= ~6;
  if (!parts) return 0;
  switch (h->cfg) {
    case 0: return launch_body<CfgEllEuler>(h, mask, nullptr, 0, parts, s);
    case 1: return launch_body<CfgPyrEuler>(h, mask, nullptr, 0, parts, s);
    case 3: return launch_body<CfgPyrEuler29>(h, mask, nullptr, 0, parts, s);
    case 4:
    case 5: return locosim_configs31_body(h, mask, parts, s);
    case 6: return locosim_terrain_body(h, mask, parts, s);
    default: return launch_body<CfgPyrRK4>(h, mask, nullptr, 0, parts, s);
  }
}


extern "C" {

const char* locosim_last_error(const locosim_t* h) { return h ? h->err.c_str() : g_create_error.c_str(); }

int locosim_create(const int32_t* mi, int nmi, const double* mr, int nmr, const int32_t* ti, int nti, const double* tr,
                   int ntr, int n_envs, int device, uint64_t seed, int64_t env_off, locosim_t** out) {
  locosim_handle* h = new locosim_handle();
  *out = nullptr;
  auto fail = [&](const std::string& msg) { g_create_error = msg; delete h; return 1; };
  if (n_envs <= 0) return fail("n_envs must be positive");
  std::string err = parse_model(h->hm, mi, nmi, mr, nmr);
  if (!err.empty()) return fail(err);
  err = parse_task(h->ht, h->hm.nu, h->hm.nv, h->hm.ng, ti, nti, tr, ntr);
  if (!err.empty()) return fail(err);
  if (h->hm.nu > h->hm.nv) return fail("nu > nv");
  h->device = device; h->n_envs = n_envs; h->seed = seed; h->env_off = env_off;
  int ndev = 0;
  cudaError_t ce = cudaGetDeviceCount(&ndev);
  if (ce != cudaSuccess || ndev == 0) return fail(std::string("no CUDA device: ") + cudaGetErrorString(ce));
  if (device < 0 || device >= ndev) return fail("bad device index");
  ce = cudaSetDevice(device);
  if (ce != cudaSuccess) return fail(cudaGetErrorString(ce));
  ce = cudaDeviceGetAttribute(&h->n_sm, cudaDevAttrMultiProcessorCount, device);
  if (ce != cudaSuccess) return fail(cudaGetErrorString(ce));
  h->cfg = select_cfg(h->hm, h->ht.obs_dim);
  if (h->cfg < 0) return fail("no compiled configuration fits this model (cone / integrator / sizes: see locosim_config.h)");
  h->so.tolerance = 1e-5f; h->so.ls_tolerance = 0.1f; h->so.ls_iter = 16;
  h->so.max_iter = h->hm.iterations < 20 ? h->hm.iterations : 20;
  auto up = [&](void** dst, const void* src, size_t bytes) -> bool {
    if (cudaMalloc(dst, bytes ? bytes : 4) != cudaSuccess) return false;
    if (bytes && cudaMemcpy(*dst, src, bytes, cudaMemcpyHostToDevice) != cudaSuccess) return false;
    return true;
  };
  bool ok = up((void**)&h->d_mints, h->hm.ints.data(), h->hm.ints.size() * 4) &&
            up((void**)&h->d_mreals, h->hm.reals.data(), h->hm.reals.size() * 4) &&
            up((void**)&h->d_tints, h->ht.ints.data(), h->ht.ints.size() * 4) &&
            up((void**)&h->d_treals, h->ht.reals.data(), h->ht.reals.size() * 4);
  size_t N = (size_t)n_envs, nv = (size_t)h->hm.nv;
  ok = ok && cudaMalloc((void**)&h->st.qpos, N * nv * 4) == cudaSuccess && cudaMalloc((void**)&h->st.qvel, N * nv * 4) == cudaSuccess &&
       cudaMalloc((void**)&h->st.ws, N * nv * 4) == cudaSuccess && cudaMalloc((void**)&h->st.goal, N * 4 * 4) == cudaSuccess &&
       cudaMalloc((void**)&h->st.episode, N * 4) == cudaSuccess && cudaMalloc((void**)&h->st.counters, N * 32) == cudaSuccess &&
       cudaMalloc((void**)&h->st.dr_row, N * 4) == cudaSuccess && cudaMalloc((void**)&h->st.perm, N * 4) == cudaSuccess &&
       cudaMalloc((void**)&h->st.cursor, N * 4) == cudaSuccess &&
       cudaMalloc((void**)&h->st.ep, N * 16) == cudaSuccess && cudaMalloc((void**)&h->rot_pin, N * 8) == cudaSuccess &&
       cudaMalloc((void**)&h->load_mask, N) == cudaSuccess &&
       up((void**)&h->d_pool, h->hm.default_row.data(), h->hm.default_row.size() * 4);
  if (!ok) { std::string m = std::string("device allocation failed: ") + cudaGetErrorString(cudaGetLastError()); locosim_destroy(h); g_create_error = m; return 1; }
  cudaMemset(h->st.qpos, 0, N * nv * 4); cudaMemset(h->st.qvel, 0, N * nv * 4); cudaMemset(h->st.ws, 0, N * nv * 4);
  cudaMemset(h->st.goal, 0, N * 16); cudaMemset(h->st.episode, 0, N * 4); cudaMemset(h->st.counters, 0, N * 32);
  cudaMemset(h->st.dr_row, 0, N * 4); cudaMemset(h->st.cursor, 0, N * 4);
  cudaMemset(h->st.ep, 0, N * 16); cudaMemset(h->rot_pin, 0, N * 8); cudaMemset(h->load_mask, 0, N);
  {
    // FNV-1a over what the row layout and its indices depend on
    const int dims[7] = {LS_STATE_VERSION, h->hm.nv, h->hm.nb, h->ht.obs_dim, h->ht.n_goal, h->ht.n_traj, h->ht.traj_len};
    uint32_t f = 2166136261u;
    for (int d : dims) for (int b = 0; b < 4; b++) { f ^= ((uint32_t)d >> (8 * b)) & 255u; f *= 16777619u; }
    h->state_fp = (int)f;
  }
  h->st.max_episode_steps = 0; h->st.end_of_trajectory = 0;
  h->st.rot_angle = nullptr;
  { std::vector<int> id(N); for (size_t i = 0; i < N; i++) id[i] = (int)i; cudaMemcpy(h->st.perm, id.data(), N * 4, cudaMemcpyHostToDevice); }
  h->st.pool = h->d_pool; h->st.pool_K = 1;
  bind_model(h->dm, h->hm, h->d_mints, h->d_mreals);
  for (int k = 0; k < LS_MAX_SLOTS && h->slot < 0; k++) if (!g_slot_used[k]) { h->slot = k; g_slot_used[k] = true; }
  if (h->slot < 0) { locosim_destroy(h); g_create_error = "too many live locosim handles (max 16 per process)"; return 1; }
  if (cudaMemcpyToSymbol(c_models, &h->dm, sizeof(DevModel), sizeof(DevModel) * h->slot) != cudaSuccess ||
      cudaMemcpyToSymbol(c_applied, &h->applied, sizeof(DevApplied), sizeof(DevApplied) * h->slot) != cudaSuccess ||
      cudaMemcpyToSymbol(c_bodyout, &h->bodyout, sizeof(DevBodyOut), sizeof(DevBodyOut) * h->slot) != cudaSuccess ||
      cudaMemcpyToSymbol(c_refout, &h->refout, sizeof(DevRefOut), sizeof(DevRefOut) * h->slot) != cudaSuccess ||
      cudaMemcpyToSymbol(c_contact, &h->contact, sizeof(DevContact), sizeof(DevContact) * h->slot) != cudaSuccess ||
      cudaMemcpyToSymbol(c_dof, &h->dof, sizeof(DevDof), sizeof(DevDof) * h->slot) != cudaSuccess ||
      cudaMemcpyToSymbol(c_dof_act, &h->dof_act, sizeof(float*), sizeof(float*) * h->slot) != cudaSuccess ||
      cudaMemcpyToSymbol(c_conlist, &h->conlist, sizeof(DevConList), sizeof(DevConList) * h->slot) != cudaSuccess ||
      cudaMemcpyToSymbol(c_conrows, &h->conrows, sizeof(DevConRows), sizeof(DevConRows) * h->slot) != cudaSuccess) {
    g_create_error = std::string("cudaMemcpyToSymbol: ") + cudaGetErrorString(cudaGetLastError()); locosim_destroy(h); return 1;
  }
  bind_task(h->dt, h->ht, h->hm.nu, h->d_tints, h->d_treals);
  h->dt.po_user = h->hm.po[12];
  int rc = 0;
  switch (h->cfg) {
    case 0: rc = setup_cfg<CfgEllEuler>(h); break;
    case 1: rc = setup_cfg<CfgPyrEuler>(h); break;
    case 3: rc = setup_cfg<CfgPyrEuler29>(h); break;
    case 4:
    case 5:
      if (!locosim_configs31_setup) { h->err = "the 31-dof configurations are not compiled into this library"; rc = 1; break; }
      rc = locosim_configs31_setup(h);
      // (this unit's reset / dataset kernels read the model from its own __constant__ slots: same descriptor, staging included)
      if (!rc && cudaMemcpyToSymbol(c_models, &h->dm, sizeof(DevModel), sizeof(DevModel) * h->slot) != cudaSuccess) {
        h->err = std::string("cudaMemcpyToSymbol: ") + cudaGetErrorString(cudaGetLastError()); rc = 1;
      }
      break;
    case 6:
      if (!locosim_terrain_setup) { h->err = "the terrain configuration is not compiled into this library"; rc = 1; break; }
      rc = locosim_terrain_setup(h);
      if (!rc && cudaMemcpyToSymbol(c_models, &h->dm, sizeof(DevModel), sizeof(DevModel) * h->slot) != cudaSuccess) {
        h->err = std::string("cudaMemcpyToSymbol: ") + cudaGetErrorString(cudaGetLastError()); rc = 1;
      }
      break;
    default: rc = setup_cfg<CfgPyrRK4>(h); break;
  }
  if (!rc && locosim_ray_sync_model) rc = locosim_ray_sync_model(h);
  if (rc) { g_create_error = h->err; locosim_destroy(h); return 1; }
  *out = h;
  return 0;
}

void locosim_destroy(locosim_t* h) {
  if (!h) return;
  if (h->slot >= 0) g_slot_used[h->slot] = false;
  cudaFree(h->d_mints); cudaFree(h->d_mreals); cudaFree(h->d_tints); cudaFree(h->d_treals);
  cudaFree(h->st.qpos); cudaFree(h->st.qvel); cudaFree(h->st.ws); cudaFree(h->st.goal); cudaFree(h->st.episode);
  cudaFree(h->st.counters); cudaFree(h->st.dr_row); cudaFree(h->st.perm); cudaFree(h->st.cursor); cudaFree(h->d_pool);
  cudaFree(h->st.ep);
  cudaFree(h->d_stage);
  cudaFree(h->split.carry); cudaFree(h->split.bcount); cudaFree(h->split.benv); cudaFree(h->split.seq);
  cudaFree(h->pq.carry); cudaFree(h->pq.cnt); cudaFree(h->pq.tot); cudaFree(h->pq.benv); cudaFree(h->pq.seq);
  cudaFree(h->bodyout.reset_mark);
  cudaFree(h->ref_key); cudaFree(h->rot_pin); cudaFree(h->load_mask); cudaFree(h->d_model_row);
  cudaFree(h->dof_act);
  delete h;
}

int locosim_num_envs(const locosim_t* h) { return h->n_envs; }
int locosim_obs_dim(const locosim_t* h) { return h->ht.obs_dim; }
int locosim_action_dim(const locosim_t* h) { return h->hm.nu; }
int locosim_nq(const locosim_t* h) { return h->hm.nv; }

int locosim_set_solver(locosim_t* h, float tol, float ls_tol, int max_iter, int ls_iter) {
  if (tol <= 0 || ls_tol <= 0 || max_iter < 1 || ls_iter < 1) { h->err = "bad solver options"; return 1; }
  h->so.tolerance = tol; h->so.ls_tolerance = ls_tol; h->so.max_iter = max_iter; h->so.ls_iter = ls_iter;
  return 0;
}

int locosim_reset_rows(locosim_t* h, const uint8_t* d_mask, const int32_t* d_traj, const int32_t* d_step,
                       const int32_t* d_pool_row, float* d_obs, void* stream) {
  CK(cudaSetDevice(h->device));
  int threads = 128, blocks = (h->n_envs * 32 + threads - 1) / threads;
  reset_kernel<<<blocks, threads, 0, (cudaStream_t)stream>>>(h->slot, h->dt, h->st, d_mask, d_traj, d_step, d_pool_row, d_obs,
                                                             h->n_envs, h->seed, h->env_off, h->rot_pin);
  h->st.rot_angle = nullptr;        // pinned rotation angles apply to one reset call
  CK(cudaGetLastError());
  return next_body_rows(h, d_mask, 7, (cudaStream_t)stream);
}
int locosim_set_reset_rotation(locosim_t* h, const float* d_angle) { h->st.rot_angle = d_angle; return 0; }
int locosim_get_cursor(locosim_t* h, int32_t* d_out, void* stream) {
  CK(cudaMemcpyAsync(d_out, h->st.cursor, (size_t)h->n_envs * 4, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return 0;
}
int locosim_set_time_limit(locosim_t* h, int max_episode_steps, int end_of_trajectory) {
  if (max_episode_steps < 0 || end_of_trajectory < 0) { h->err = "bad time limit (negative)"; return 1; }
  h->st.max_episode_steps = max_episode_steps; h->st.end_of_trajectory = end_of_trajectory ? 1 : 0;
  return 0;
}
int locosim_nbody(const locosim_t* h) { return h->hm.nb; }
int locosim_set_applied_forces(locosim_t* h, float* d_xfrc, float* d_qfrc) {
  CK(cudaSetDevice(h->device));
  h->applied.xfrc = d_xfrc; h->applied.qfrc = d_qfrc;
  // (the kernels read the pointers from the handle's __constant__ slot, in both translation units)
  CK(cudaMemcpyToSymbol(c_applied, &h->applied, sizeof(DevApplied), sizeof(DevApplied) * h->slot));
  if (sync_other_units(h)) return 1;
  return 0;
}
int locosim_set_terrain_origin(locosim_t* h, float* d_origin) {
  if (h->cfg != 6) { h->err = "this model has no terrain"; return 1; }
  CK(cudaSetDevice(h->device));
  h->terrain_origin = d_origin;
  return locosim_terrain_sync_model(h);
}
int locosim_set_body_outputs(locosim_t* h, float* d_body, float* d_next_body) {
  CK(cudaSetDevice(h->device));
  if (d_body && !h->bodyout.reset_mark) CK(cudaMalloc((void**)&h->bodyout.reset_mark, (size_t)h->n_envs * 4));
  // one flag per env: set by the step kernel's reset_env where it wrote d_body, cleared by the body_kernel after the step;
  // cleared on every registration, so that no mark from earlier steps survives into the new buffers
  if (h->bodyout.reset_mark) CK(cudaMemset(h->bodyout.reset_mark, 0, (size_t)h->n_envs * 4));
  h->bodyout.body = d_body; h->bodyout.next_body = d_next_body;
  // (a __constant__ table of its own in both translation units, like the applied forces)
  CK(cudaMemcpyToSymbol(c_bodyout, &h->bodyout, sizeof(DevBodyOut), sizeof(DevBodyOut) * h->slot));
  if (sync_other_units(h)) return 1;
  return 0;
}
int locosim_set_reference_outputs(locosim_t* h, float* d_ref, float* d_next_ref) {
  CK(cudaSetDevice(h->device));
  const bool on = d_ref || d_next_ref;
  if (on && !h->ref_key) CK(cudaMalloc((void**)&h->ref_key, (size_t)h->n_envs * sizeof(int4)));
  h->refout.ref = d_ref; h->refout.next_ref = d_next_ref; h->refout.key = on ? h->ref_key : nullptr;
  // (a __constant__ table of its own in both translation units, read by body_kernel when it runs)
  CK(cudaMemcpyToSymbol(c_refout, &h->refout, sizeof(DevRefOut), sizeof(DevRefOut) * h->slot));
  if (sync_other_units(h)) return 1;
  if (!on) return 0;
  // every env's key from its current state (steps and resets keep them from here on); nothing else is written
  CK(cudaDeviceSynchronize());
  if (next_body_rows(h, nullptr, 2, 0)) return 1;
  CK(cudaDeviceSynchronize());
  return 0;
}
// the compiled model's own parameter row on the device (h->d_model_row), uploaded on first use
static int model_row(locosim_handle* h) {
  if (!h->d_model_row) {
    CK(cudaMalloc((void**)&h->d_model_row, h->hm.default_row.size() * 4));
    CK(cudaMemcpy(h->d_model_row, h->hm.default_row.data(), h->hm.default_row.size() * 4, cudaMemcpyHostToDevice));
  }
  return 0;
}
int locosim_create_dataset_bodies(locosim_t* h, float* d_body, float* d_next_body, void* stream) {
  if (!d_body || !d_next_body) { h->err = "null buffer"; return 1; }
  CK(cudaSetDevice(h->device));
  if (model_row(h)) return 1;
  cudaStream_t s = (cudaStream_t)stream;
  switch (h->cfg) {
    case 0: return launch_dataset_bodies<CfgEllEuler>(h, d_body, d_next_body, s);
    case 1: return launch_dataset_bodies<CfgPyrEuler>(h, d_body, d_next_body, s);
    case 3: return launch_dataset_bodies<CfgPyrEuler29>(h, d_body, d_next_body, s);
    case 4:
    case 5: return locosim_configs31_dataset_bodies(h, d_body, d_next_body, s);
    case 6: return locosim_terrain_dataset_bodies(h, d_body, d_next_body, s);
    default: return launch_dataset_bodies<CfgPyrRK4>(h, d_body, d_next_body, s);
  }
}
// whether any two of the caller's `n` buffers (NULL: skipped) share a byte; bytes[i] is buffer i's size
static bool buffers_overlap(const void* const* buf, const size_t* bytes, int n) {
  for (int i = 0; i < n; i++) {
    if (!buf[i]) continue;
    for (int j = 0; j < i; j++) {
      if (!buf[j]) continue;
      const char *a = (const char*)buf[i], *b = (const char*)buf[j];
      if (a < b + bytes[j] && b < a + bytes[i]) return true;
    }
  }
  return false;
}
int locosim_inverse(locosim_t* h, const float* d_qacc, float* d_qfrc_inverse, void* stream) {
  if (!d_qacc || !d_qfrc_inverse) { h->err = "null buffer"; return 1; }
  const size_t bytes = (size_t)h->n_envs * h->hm.nv * 4;
  const void* const buf[2] = {d_qacc, d_qfrc_inverse};
  const size_t sizes[2] = {bytes, bytes};
  if (buffers_overlap(buf, sizes, 2)) { h->err = "qacc and qfrc_inverse overlap"; return 1; }
  CK(cudaSetDevice(h->device));
  cudaStream_t s = (cudaStream_t)stream;
  switch (h->cfg) {
    case 0: return launch_inverse<CfgEllEuler>(h, d_qacc, d_qfrc_inverse, s);
    case 1: return launch_inverse<CfgPyrEuler>(h, d_qacc, d_qfrc_inverse, s);
    case 3: return launch_inverse<CfgPyrEuler29>(h, d_qacc, d_qfrc_inverse, s);
    case 4:
    case 5: return locosim_configs31_inverse(h, d_qacc, d_qfrc_inverse, s);
    case 6: return locosim_terrain_inverse(h, d_qacc, d_qfrc_inverse, s);
    default: return launch_inverse<CfgPyrRK4>(h, d_qacc, d_qfrc_inverse, s);
  }
}
int locosim_create_dataset_inverse(locosim_t* h, float* d_qfrc, void* stream) {
  if (!d_qfrc) { h->err = "null buffer"; return 1; }
  CK(cudaSetDevice(h->device));
  if (model_row(h)) return 1;
  cudaStream_t s = (cudaStream_t)stream;
  switch (h->cfg) {
    case 0: return launch_dataset_inverse<CfgEllEuler>(h, d_qfrc, s);
    case 1: return launch_dataset_inverse<CfgPyrEuler>(h, d_qfrc, s);
    case 3: return launch_dataset_inverse<CfgPyrEuler29>(h, d_qfrc, s);
    case 4:
    case 5: return locosim_configs31_dataset_inverse(h, d_qfrc, s);
    case 6: return locosim_terrain_dataset_inverse(h, d_qfrc, s);
    default: return launch_dataset_inverse<CfgPyrRK4>(h, d_qfrc, s);
  }
}
int locosim_dynamics_terms(locosim_t* h, float* d_M, float* d_bias, float* d_passive, float* d_com, float* d_jac,
                           float* d_jac_com, void* stream) {
  const size_t n = (size_t)h->n_envs, nv = (size_t)h->hm.nv;
  const void* const buf[6] = {d_M, d_bias, d_passive, d_com, d_jac, d_jac_com};
  const size_t bytes[6] = {n * nv * nv * 4, n * nv * 4, n * nv * 4, n * LS_COM_DIM * 4, n * h->hm.nb * 6 * nv * 4,
                           n * 3 * nv * 4};
  if (buffers_overlap(buf, bytes, 6)) { h->err = "dynamics_terms outputs overlap"; return 1; }
  if (!(d_M || d_bias || d_passive || d_com || d_jac || d_jac_com) || n == 0) return 0;
  CK(cudaSetDevice(h->device));
  const DynOut o = {d_M, d_bias, d_passive, d_com, d_jac, d_jac_com};
  cudaStream_t s = (cudaStream_t)stream;
  switch (h->cfg) {
    case 0: return launch_dynamics<CfgEllEuler>(h, o, s);
    case 1: return launch_dynamics<CfgPyrEuler>(h, o, s);
    case 3: return launch_dynamics<CfgPyrEuler29>(h, o, s);
    case 4:
    case 5: return locosim_configs31_dynamics(h, &o, s);
    case 6: return locosim_terrain_dynamics(h, &o, s);
    default: return launch_dynamics<CfgPyrRK4>(h, o, s);
  }
}
int locosim_forward(locosim_t* h, const float* d_action, float* d_dof, float* d_body_acc, float* d_cfrc_int,
                    float* d_cfrc_ext, void* stream) {
  if (!d_action) { h->err = "null action buffer"; return 1; }
  const size_t n = (size_t)h->n_envs, nv = (size_t)h->hm.nv, nb = (size_t)h->hm.nb;
  // the action is buffer 0: every output is checked against it and against the other outputs
  const void* const buf[5] = {d_action, d_dof, d_body_acc, d_cfrc_int, d_cfrc_ext};
  const size_t bytes[5] = {n * h->hm.nu * 4, n * nv * LS_DOF_DIM * 4, n * nb * LS_BODY_ACC_DIM * 4,
                           n * nb * LS_CONTACT_DIM * 4, n * nb * LS_CONTACT_DIM * 4};
  if (buffers_overlap(buf, bytes, 5)) { h->err = "forward outputs overlap"; return 1; }
  if (!(d_dof || d_body_acc || d_cfrc_int || d_cfrc_ext) || n == 0) return 0;
  CK(cudaSetDevice(h->device));
  const FwdOut o = {d_dof, d_body_acc, d_cfrc_int, d_cfrc_ext};
  cudaStream_t s = (cudaStream_t)stream;
  switch (h->cfg) {
    case 0: return launch_forward<CfgEllEuler>(h, d_action, o, s);
    case 1: return launch_forward<CfgPyrEuler>(h, d_action, o, s);
    case 3: return launch_forward<CfgPyrEuler29>(h, d_action, o, s);
    case 4:
    case 5: return locosim_configs31_forward(h, d_action, &o, s);
    case 6: return locosim_terrain_forward(h, d_action, &o, s);
    default: return launch_forward<CfgPyrRK4>(h, d_action, o, s);
  }
}
int locosim_ray(locosim_t* h, const float* d_pnt, const float* d_vec, int n_rays, int frame, int frame_body,
                int exclude_body, int flags, float* d_dist, int32_t* d_geom, float* d_normal, void* stream) {
  if (!d_pnt || !d_vec || !d_dist || !d_geom) { h->err = "null buffer"; return 1; }
  if (n_rays < 1) { h->err = "n_rays must be at least 1"; return 1; }
  if (frame < LS_RAY_WORLD || frame > LS_RAY_TRACK) { h->err = "unknown ray frame"; return 1; }
  if (flags & ~(LS_RAY_STATIC | LS_RAY_DYNAMIC | LS_RAY_PER_ENV)) { h->err = "unknown ray flag bits"; return 1; }
  if (frame_body < 0 || frame_body >= h->hm.nb) { h->err = "frame_body out of range"; return 1; }
  if (exclude_body < -1 || exclude_body >= h->hm.nb) { h->err = "exclude_body out of range"; return 1; }
  if ((n_rays + LS_RAY_BLOCK - 1) / LS_RAY_BLOCK > 65535) { h->err = "too many rays per env for one launch grid"; return 1; }
  const size_t n = (size_t)h->n_envs, nr = (size_t)n_rays, in = ((flags & LS_RAY_PER_ENV) ? n : 1) * nr * 12;
  // the outputs are buffers 0-2; each is checked against the other outputs and against both inputs
  const void* const buf_p[4] = {d_dist, d_geom, d_normal, d_pnt};
  const void* const buf_v[4] = {d_dist, d_geom, d_normal, d_vec};
  const size_t bytes[4] = {n * nr * 4, n * nr * 4, n * nr * 12, in};
  if (buffers_overlap(buf_p, bytes, 4) || buffers_overlap(buf_v, bytes, 4)) {
    h->err = "ray outputs overlap each other or the inputs"; return 1;
  }
  if (!locosim_ray_launch) { h->err = "the ray kernels are not compiled into this library"; return 1; }
  if (n == 0) return 0;
  CK(cudaSetDevice(h->device));
  const RayArgs a = {d_pnt, d_vec, d_dist, d_geom, d_normal, n_rays, frame, frame_body, exclude_body, flags};
  if (h->cfg == 6) return locosim_terrain_ray(h, &a, (cudaStream_t)stream);
  return locosim_ray_launch(h, &a, (cudaStream_t)stream);
}
int locosim_set_contact_outputs(locosim_t* h, float* d_contact) {
  CK(cudaSetDevice(h->device));
  h->contact.wrench = d_contact;
  h->contact.n_substeps = h->dt.n_substeps;
  // (a __constant__ table of its own in both translation units; the step kernels read it when they run, so a step captured
  // in a CUDA graph before this call writes the buffer at its next replay)
  CK(cudaMemcpyToSymbol(c_contact, &h->contact, sizeof(DevContact), sizeof(DevContact) * h->slot));
  if (sync_other_units(h)) return 1;
  return 0;
}
int locosim_set_dof_outputs(locosim_t* h, float* d_dof) {
  CK(cudaSetDevice(h->device));
  // the actuator-force scratch [n_envs, nu] lives as long as the handle once the outputs were first registered
  if (d_dof && !h->dof_act) {
    CK(cudaMalloc(&h->dof_act, sizeof(float) * (size_t)h->n_envs * (h->hm.nu > 0 ? h->hm.nu : 1)));
    CK(cudaMemcpyToSymbol(c_dof_act, &h->dof_act, sizeof(float*), sizeof(float*) * h->slot));
  }
  h->dof.out = d_dof;
  h->dof.n_substeps = h->dt.n_substeps;
  // (__constant__ tables of their own in both translation units, read when the kernels run, as for the contact outputs)
  CK(cudaMemcpyToSymbol(c_dof, &h->dof, sizeof(DevDof), sizeof(DevDof) * h->slot));
  if (sync_other_units(h)) return 1;
  return 0;
}
int locosim_max_contacts(const locosim_t* h) {
  switch (h->cfg) {
    case 0: return CfgEllEuler::MAXCON;
    case 1: return CfgPyrEuler::MAXCON;
    case 3: return CfgPyrEuler29::MAXCON;
    case 4: return CfgPyrRK4_31::MAXCON;
    case 5: return CfgPyrEuler31::MAXCON;
    case 6: return CfgEllEulerTerrain::MAXCON;
    default: return CfgPyrRK4::MAXCON;
  }
}
int locosim_set_contact_list_outputs(locosim_t* h, int32_t* d_ncon, float* d_con, int32_t* d_con_id) {
  const int on = (d_ncon != nullptr) + (d_con != nullptr) + (d_con_id != nullptr);
  if (on != 0 && on != 3) { h->err = "contact list: pass all three buffers or none"; return 1; }
  const size_t n = (size_t)h->n_envs, C = (size_t)locosim_max_contacts(h);
  const void* const buf[3] = {d_ncon, d_con, d_con_id};
  const size_t bytes[3] = {n * 4, n * C * LS_CONLIST_DIM * 4, n * C * LS_CONLIST_ID_DIM * 4};
  if (buffers_overlap(buf, bytes, 3)) { h->err = "contact list buffers overlap"; return 1; }
  CK(cudaSetDevice(h->device));
  h->conlist.ncon = d_ncon; h->conrows.con = d_con; h->conrows.id = d_con_id;
  h->conlist.n_substeps = h->dt.n_substeps;
  // (__constant__ tables of their own in both translation units, read when the kernels run, as for the contact outputs; the
  // rows first, so that a kernel never sees the count pointer without them)
  CK(cudaMemcpyToSymbol(c_conrows, &h->conrows, sizeof(DevConRows), sizeof(DevConRows) * h->slot));
  CK(cudaMemcpyToSymbol(c_conlist, &h->conlist, sizeof(DevConList), sizeof(DevConList) * h->slot));
  if (sync_other_units(h)) return 1;
  return 0;
}
int locosim_get_episode_stats(locosim_t* h, int32_t* d_len, float* d_ret, int32_t* d_last_len, float* d_last_ret, void* stream) {
  // (one 16-byte record per env on the device: four strided copies)
  void* dst[4] = {d_len, d_ret, d_last_len, d_last_ret};
  for (int k = 0; k < 4; k++)
    if (dst[k]) CK(cudaMemcpy2DAsync(dst[k], 4, (const char*)h->st.ep + 4 * k, 16, 4, (size_t)h->n_envs, cudaMemcpyDeviceToDevice,
                                     (cudaStream_t)stream));
  return 0;
}

// create_dataset() on the device (base.py:278-312 -> Trajectory.create_dataset utils/trajectory.py:104-151): states /
// next_states = the observation layout of consecutive samples of every trajectory of the reset table (already in HBM),
// last = 1 on the final transition of each trajectory; absorbing is all zero in the reference and is not materialised.
__global__ void dataset_kernel(int ms, DevTask t, float* __restrict__ states, float* __restrict__ next_states,
                               float* __restrict__ last) {
  const DevModel& m = c_models[ms];
  const int nv = m.nv, ncol = 2 * nv + t.n_goal, D = t.obs_dim, per = t.traj_len - 1;
  const long n_rows = (long)t.n_traj * per;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n_rows * D; i += (long)gridDim.x * blockDim.x) {
    const long r = i / D;
    const int k = (int)(i - r * D), tj = (int)(r / per), sp = (int)(r - (long)tj * per);
    const float* row = t.table + ((size_t)tj * t.traj_len + sp) * ncol;
    const int ty = t.obs_src_type[k], idx = t.obs_src_idx[k];
    float a, b;
    if (ty == LS_OBS_QPOS) { a = row[idx]; b = row[ncol + idx]; }
    else if (ty == LS_OBS_QVEL) { a = row[nv + idx]; b = row[ncol + nv + idx]; }
    else if (ty == LS_OBS_GOAL) { a = row[2 * nv + idx]; b = row[ncol + 2 * nv + idx]; }
    else { a = 0.0f; b = 0.0f; }                      // foot forces / per-model features are not trajectory data
    states[i] = a; next_states[i] = b;
    if (k == 0 && last) last[r] = sp == per - 1 ? 1.0f : 0.0f;
  }
}
int locosim_dataset_rows(const locosim_t* h) { return h->ht.n_traj * (h->ht.traj_len - 1); }
int locosim_create_dataset(locosim_t* h, float* d_states, float* d_next_states, float* d_last, void* stream) {
  if (!d_states || !d_next_states) { h->err = "null buffer"; return 1; }
  CK(cudaSetDevice(h->device));
  dataset_kernel<<<2 * h->n_sm, 256, 0, (cudaStream_t)stream>>>(h->slot, h->dt, d_states, d_next_states, d_last);
  CK(cudaGetLastError());
  return 0;
}
int locosim_reset(locosim_t* h, const uint8_t* d_mask, const int32_t* d_traj, const int32_t* d_step, float* d_obs,
                  void* stream) {
  return locosim_reset_rows(h, d_mask, d_traj, d_step, nullptr, d_obs, stream);
}

int locosim_step(locosim_t* h, const float* a, float* o, float* r, uint8_t* d, float* no, int auto_reset, void* stream) {
  if (!a || !o || !r || !d) { h->err = "null buffer"; return 1; }
  CK(cudaSetDevice(h->device));
  cudaStream_t s = (cudaStream_t)stream;
  switch (h->cfg) {
    case 0: return launch_step<CfgEllEuler>(h, a, o, r, d, no, auto_reset, s);
    case 1: return launch_step<CfgPyrEuler>(h, a, o, r, d, no, auto_reset, s);
    case 3: return launch_step<CfgPyrEuler29>(h, a, o, r, d, no, auto_reset, s);
    case 4:
    case 5: return locosim_configs31_step(h, a, o, r, d, no, auto_reset, s);
    case 6: return locosim_terrain_step(h, a, o, r, d, no, auto_reset, s);
    default: return launch_step<CfgPyrRK4>(h, a, o, r, d, no, auto_reset, s);
  }
}

int locosim_get_state(locosim_t* h, float* q, float* v, float* w, void* stream) {
  size_t bytes = (size_t)h->n_envs * h->hm.nv * 4;
  cudaStream_t s = (cudaStream_t)stream;
  if (q) CK(cudaMemcpyAsync(q, h->st.qpos, bytes, cudaMemcpyDeviceToDevice, s));
  if (v) CK(cudaMemcpyAsync(v, h->st.qvel, bytes, cudaMemcpyDeviceToDevice, s));
  if (w) CK(cudaMemcpyAsync(w, h->st.ws, bytes, cudaMemcpyDeviceToDevice, s));
  return 0;
}
int locosim_set_state(locosim_t* h, const float* q, const float* v, const float* w, void* stream) {
  size_t bytes = (size_t)h->n_envs * h->hm.nv * 4;
  cudaStream_t s = (cudaStream_t)stream;
  if (q) CK(cudaMemcpyAsync(h->st.qpos, q, bytes, cudaMemcpyDeviceToDevice, s));
  if (v) CK(cudaMemcpyAsync(h->st.qvel, v, bytes, cudaMemcpyDeviceToDevice, s));
  if (w) CK(cudaMemcpyAsync(h->st.ws, w, bytes, cudaMemcpyDeviceToDevice, s));
  else CK(cudaMemsetAsync(h->st.ws, 0, bytes, s));
  return next_body_rows(h, nullptr, 1, s);
}
int locosim_state_words(const locosim_t* h) { return LS_STATE_WORDS(h->hm.nv, h->ht.obs_dim); }
int locosim_save_state(locosim_t* h, const float* d_obs, int32_t* d_state, void* stream) {
  if (!d_obs || !d_state) { h->err = "null buffer (save_state needs the observation the envs act on next)"; return 1; }
  const size_t n = (size_t)h->n_envs;
  const void* const buf[2] = {d_obs, d_state};
  const size_t bytes[2] = {n * h->ht.obs_dim * 4, n * locosim_state_words(h) * 4};
  if (buffers_overlap(buf, bytes, 2)) { h->err = "observation and state rows overlap"; return 1; }
  if ((uintptr_t)d_state % 16) { h->err = "state rows must be 16-byte aligned"; return 1; }
  CK(cudaSetDevice(h->device));
  const int threads = 128, blocks = (h->n_envs * 32 + threads - 1) / threads;
  save_state_kernel<<<blocks, threads, 0, (cudaStream_t)stream>>>(h->dt, h->st, d_obs, reinterpret_cast<int4*>(d_state),
                                                                  h->n_envs, h->hm.nv, locosim_state_words(h), h->state_fp,
                                                                  h->seed, h->env_off, h->rot_pin);
  CK(cudaGetLastError());
  return 0;
}
int locosim_load_state(locosim_t* h, const int32_t* d_state, int n_rows, const int32_t* d_row, float* d_obs, void* stream) {
  if (!d_state || n_rows < 1) { h->err = "no state rows"; return 1; }
  if (!d_row && n_rows != h->n_envs) { h->err = "load_state without row indices needs one row per env"; return 1; }
  const size_t n = (size_t)h->n_envs;
  const void* const buf[3] = {d_state, d_row, d_obs};
  const size_t bytes[3] = {(size_t)n_rows * locosim_state_words(h) * 4, n * 4, n * h->ht.obs_dim * 4};
  if (buffers_overlap(buf, bytes, 3)) { h->err = "state rows, row indices and observation overlap"; return 1; }
  if ((uintptr_t)d_state % 16) { h->err = "state rows must be 16-byte aligned"; return 1; }
  CK(cudaSetDevice(h->device));
  cudaStream_t s = (cudaStream_t)stream;
  const int threads = 128, blocks = (h->n_envs * 32 + threads - 1) / threads;
  load_state_kernel<<<blocks, threads, 0, s>>>(h->dt, h->st, reinterpret_cast<const int4*>(d_state), n_rows, d_row, d_obs,
                                               h->n_envs, h->hm.nv, locosim_state_words(h), h->state_fp, h->rot_pin,
                                               h->bodyout.reset_mark, h->load_mask);
  CK(cudaGetLastError());
  return next_body_rows(h, h->load_mask, 7, s);
}
int locosim_set_goal(locosim_t* h, const float* g, void* stream) {
  if (!g) { h->err = "null buffer"; return 1; }
  CK(cudaMemcpyAsync(h->st.goal, g, (size_t)h->n_envs * 16, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return 0;
}
int locosim_get_counters(locosim_t* h, int32_t* d_out, void* stream) {
  CK(cudaMemcpyAsync(d_out, h->st.counters, (size_t)h->n_envs * 32, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return 0;
}
int locosim_param_pool_row_len(const locosim_t* h) { return h->hm.pool_P; }

int locosim_get_param_rows(locosim_t* h, int32_t* d_out, void* stream) {
  CK(cudaMemcpyAsync(d_out, h->st.dr_row, (size_t)h->n_envs * 4, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return 0;
}

int locosim_set_param_pool(locosim_t* h, const double* pool, int n_rows, int row_len) {
  if (!pool || n_rows < 1 || row_len != h->hm.pool_P) { h->err = "bad parameter pool (row_len must equal locosim_param_pool_row_len)"; return 1; }
  CK(cudaSetDevice(h->device));
  std::vector<float> f((size_t)n_rows * row_len);
  bool damp = false;
  for (size_t i = 0; i < f.size(); i++) {
    f[i] = (float)pool[i];
    if (!(f[i] == f[i]) || f[i] > 1e30f || f[i] < -1e30f) { h->err = "non-finite value in parameter pool"; return 1; }
  }
  for (int r = 0; r < n_rows; r++)
    for (int d = 0; d < h->hm.nv; d++) if (f[(size_t)r * row_len + h->hm.po[0] + d] > 0) damp = true;
  float* d_new = nullptr;
  CK(cudaMalloc((void**)&d_new, f.size() * 4));
  CK(cudaMemcpy(d_new, f.data(), f.size() * 4, cudaMemcpyHostToDevice));
  CK(cudaDeviceSynchronize());
  cudaFree(h->d_pool);
  h->d_pool = d_new; h->st.pool = d_new; h->st.pool_K = n_rows;
  // a dof gets a (static) frictionloss row as soon as ANY pool row gives it a positive frictionloss; in rows where
  // its value is 0 the constraint row is inert (force interval [-0, 0])
  std::vector<int> frow(h->hm.nv, -1);
  int nfric = 0;
  for (int d = 0; d < h->hm.nv; d++) {
    bool any = h->hm.default_row[h->hm.po[1] + d] > 0;
    for (int r = 0; r < n_rows && !any; r++) any = f[(size_t)r * row_len + h->hm.po[1] + d] > 0;
    if (any) frow[d] = nfric++;
  }
  CK(cudaMemcpy((void*)h->dm.dof_frow, frow.data(), frow.size() * 4, cudaMemcpyHostToDevice));
  h->dm.nfric = nfric;
  if (damp) h->dm.has_damping = 1;
  CK(cudaMemcpyToSymbol(c_models, &h->dm, sizeof(DevModel), sizeof(DevModel) * h->slot));
  if (sync_other_units(h)) return 1;
  if (locosim_ray_sync_model && locosim_ray_sync_model(h)) return 1;
  CK(cudaMemset(h->st.dr_row, 0, (size_t)h->n_envs * 4));
  if (h->refout.key) {
    // (the reference keys name the envs' pool rows: every env is on row 0 of the new pool now)
    if (next_body_rows(h, nullptr, 2, 0)) return 1;
    CK(cudaDeviceSynchronize());
  }
  return 0;
}

int locosim_kernels_per_step(const locosim_t* h) {
  const int nsub = h->dt.n_substeps;
  // (body_kernel, while body or reference outputs are registered)
  const int body = h->bodyout.body || h->bodyout.next_body || h->refout.key ? 1 : 0;
  if (h->persist) return 1 + body;
  if (h->resort < nsub) return (nsub + h->resort - 1) / h->resort + body;
  return (h->regroup ? 2 : 1) + body;
}
int locosim_set_timeline(locosim_t* h, long long* d_records, int capacity) {
  if (!h->persist) { h->err = "the timeline is recorded by the persistent sub-step kernel only"; return 1; }
  h->pq.tl = capacity > 0 ? d_records : nullptr;
  h->pq.tl_cap = capacity;
  return 0;
}
int locosim_debug_counters(unsigned long long* out8) {
  return cudaMemcpyFromSymbol(out8, g_dbg, 64) == cudaSuccess ? 0 : 1;
}
#ifdef LOCOSIM_PHASE_CLOCK
// (diagnostic build only) the phase clock summed over all slots into out[PH_N], then cleared; returns PH_N, or -1
int locosim_phase_clock(unsigned long long* out) {
  static unsigned long long buf[LS_PH_SLOTS][PH_N];
  if (cudaDeviceSynchronize() != cudaSuccess || cudaMemcpyFromSymbol(buf, g_phase, sizeof(buf)) != cudaSuccess) return -1;
  for (int p = 0; p < PH_N; p++) {
    out[p] = 0;
    for (int s = 0; s < LS_PH_SLOTS; s++) out[p] += buf[s][p];
  }
  memset(buf, 0, sizeof(buf));
  return cudaMemcpyToSymbol(g_phase, buf, sizeof(buf)) == cudaSuccess ? PH_N : -1;
}
#endif

// Measured non-tensor FP32 peak (the denominator of the FP32 utilisation bench.py reports next to the HBM roofline):
// 8 independent FMA chains per thread, 2 x 256 threads per SM slot, all SMs, best of 5 launches.
__global__ void __launch_bounds__(256) fp32_peak_kernel(float* out, int iters) {
  float a[8];
#pragma unroll
  for (int k = 0; k < 8; k++) a[k] = 1.0f + 1e-3f * (float)(threadIdx.x + k);
  const float b = 0.9999f, c = 1e-4f;
  for (int i = 0; i < iters; i++) {
#pragma unroll
    for (int u = 0; u < 8; u++) {
#pragma unroll
      for (int k = 0; k < 8; k++) a[k] = fmaf(a[k], b, c);
    }
  }
  float s = 0;
#pragma unroll
  for (int k = 0; k < 8; k++) s += a[k];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
int locosim_measure_fp32_peak(int device, double* tflops_out) {
  if (!tflops_out) return 1;
  if (cudaSetDevice(device) != cudaSuccess) return 1;
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
  const int blocks = sms * 8, threads = 256, iters = 4096;
  float* out = nullptr;
  if (cudaMalloc((void**)&out, (size_t)blocks * threads * 4) != cudaSuccess) return 1;
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  double best = 0;
  for (int rep = 0; rep < 6; rep++) {
    cudaEventRecord(e0);
    fp32_peak_kernel<<<blocks, threads>>>(out, iters);
    cudaEventRecord(e1);
    if (cudaEventSynchronize(e1) != cudaSuccess) { cudaFree(out); return 1; }
    float ms = 0;
    cudaEventElapsedTime(&ms, e0, e1);
    const double flops = 2.0 * 64.0 * (double)iters * (double)blocks * threads;
    if (rep > 0 && ms > 0) best = flops / (ms * 1e-3) / 1e12 > best ? flops / (ms * 1e-3) / 1e12 : best;
  }
  cudaEventDestroy(e0); cudaEventDestroy(e1); cudaFree(out);
  *tflops_out = best;
  return 0;
}

int locosim_launch_info(const locosim_t* h, int* wpb, int* smem, int* blocks) {
  if (wpb) *wpb = h->wpb;
  if (smem) *smem = h->smem;
  if (blocks) *blocks = (h->n_envs + h->wpb - 1) / h->wpb;
  return 0;
}

}  // extern "C"
#endif  // LOCOSIM_EXTRA_CONFIGS_TU
