// t2d_agents.cuh - the reward chain, the env epilogue t2d_env_epilogue_kernel, K10 t2d_agents_epilogue_kernel
// (status, reward and retirement of every agent row) and K11 t2d_agent_action_kernel (agent actions to their slots).
#pragma once

#include "t2d_route.cuh"
#include "t2d_world.cuh"

namespace t2d {

// ---------------------------------------------------------------------------- env epilogue
// What ParkingEnv.step does after check_status (envs/parking.py:240-256, _get_reward :148-190), for all N scenarios in
// one launch: TrafficStatus per participant from the event byte (status.py:52-61), terminated / truncated
// (parking.py:243-248), the reward chain in the reference's order, the two running extrema it keeps per episode
// (_max_iou, _min_dist_to_target) and the done mask that drives the masked reset.  One thread per participant slot;
// the thread of slot 0 also does the per-scenario part.  Reads the ego's flags through the same array, so the launch
// has no other input than the tick's outputs.
struct EnvArgs : WorldArgs {   // (the state after the tick: the ego's position for the distance shaping)
  const uint8_t* flags;        // [N][M] event byte of the tick
  const uint8_t* status;       // [N] ScenarioStatus of the tick
  const float* iou;            // [N] IoU(ego pose, target) of the tick, or nullptr (no goal)
  const float* target;         // [N][5] or nullptr
  float* max_iou;              // [N] in/out, or nullptr
  float* min_dist;             // [N] in/out, or nullptr
  float* reward;               // [N]
  uint8_t *terminated, *truncated, *done;   // [N]
  uint8_t* traffic_status;     // [N][M]
  RouteArgs route;
  double* s_best;              // [N] best arc length of the episode, or nullptr: no progress term
  int max_step, reset_trackers;
};

// The reward chain of _get_reward (parking.py:148-190) for one scored participant: st its ScenarioStatus, ts its
// TrafficStatus as check_status leaves it (only the collision and OffRoute detectors set it), step_count its scenario's
// tick count.  max_iou == nullptr skips the IoU term, min_dist == nullptr the progress term (target = the goal centre,
// (x, y) the participant's position), s_best == nullptr the route progress term (s the arc length on the route, weight
// its factor; an extension).  Out of line: the env epilogue and K10 run this one compiled copy, so that their rewards
// agree bit for bit whatever the compiler would contract in an inlined copy.
__device__ __noinline__ float reward_chain(int st, int ts, int step_count, int max_step, float iou, float* max_iou,
                                           const float* target, float* min_dist, float x, float y, float off_reward,
                                           double weight, double s, double* s_best) {
  float r;
  if (ts == 3 || ts == 4) r = -5.0f;                                             // :151-152 (+ dynamic collision, an extension)
  else if (ts == T2D_TRAFFIC_OFF_ROUTE) r = off_reward;                          // (an extension)
  else if (st == T2D_STATUS_TIME_EXCEEDED || st == T2D_STATUS_NO_ACTION) r = -1.0f;   // :153-157
  else if (st == T2D_STATUS_OUT_BOUND) r = -5.0f;                                // :158-159
  else if (st == T2D_STATUS_COMPLETED) r = 5.0f;                                 // :160-161
  else {
    r = max_step > 0 ? -tanhf((float)step_count / (float)max_step) * 0.001f : 0.0f;   // :163
    if (max_iou != nullptr) {
      const float best = *max_iou;
      r += (best == -INFINITY) ? iou : iou - best;                                 // :164-169
      *max_iou = fmaxf(best, iou);                                                 // :170
    }
    if (min_dist != nullptr) {
      const float dx = x - target[0], dy = y - target[1];
      const float d = sqrtf(dx * dx + dy * dy), best = *min_dist;                  // :172-185
      if (d < best) {                                                              // :186-188 (inf on the first step: the
        if (best != INFINITY) r += (best - d) * 0.1f;                              //  reference adds inf there; we add nothing)
        *min_dist = d;
      }
    }
    if (s_best != nullptr) {                                                       // route progress: weight (s - s_best)
      const double best = *s_best;                                                 // in fp64, one rounding to fp32; the
      if (s > best) {                                                              // first step only records s
        if (best != -INFINITY) r += __double2float_rn(__dmul_rn(weight, __dsub_rn(s, best)));
        *s_best = s;
      }
    }
  }
  return r;
}

__global__ void __launch_bounds__(256) t2d_env_epilogue_kernel(const __grid_constant__ EnvArgs A) {
  const long long total = (long long)A.N * A.M;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const unsigned f = A.flags[i];
    const uint8_t ts = (f & T2D_F_STATIC) ? 3 : ((f & T2D_F_DYNAMIC) ? 4 : 1);   // COLLISION_STATIC / COLLISION_DYNAMIC / NORMAL
    if (A.traffic_status) A.traffic_status[i] = ts;
    const int n = (int)(i / A.M);
    if (i - (long long)n * A.M != 0) continue;
    const int st = A.status[n];
    // check_status returns at the first detector that fires (parking.py:366-385): the ego's traffic status is only set
    // by the collision detector, i.e. when the scenario status says FAILED, and by OffRoute, which ranks below collision
    // and above completion
    int ego_ts = st == T2D_STATUS_FAILED ? ts : 1;
    RouteHit rh{0.0, ROUTE_NONE};
    if (A.route.route_id != nullptr && (st == T2D_STATUS_NORMAL || st == T2D_STATUS_COMPLETED)) {
      rh = route_probe(A.route, i, A.x[i], A.y[i]);
      if (rh.state == ROUTE_OFF) {
        ego_ts = T2D_TRAFFIC_OFF_ROUTE;
        if (A.traffic_status) A.traffic_status[i] = T2D_TRAFFIC_OFF_ROUTE;
      }
    }
    const bool term = st == T2D_STATUS_COMPLETED && ego_ts == 1;                   // :243-244
    const bool trunc = !term && (st != T2D_STATUS_NORMAL || ego_ts != 1);          // :245-248
    const bool scored_iou = A.iou != nullptr && A.max_iou != nullptr;
    const float r = reward_chain(st, ego_ts, A.step_count[n], A.max_step, scored_iou ? A.iou[n] : 0.0f,
                                 scored_iou ? A.max_iou + n : nullptr, A.target ? A.target + 5 * (long long)n : nullptr,
                                 (A.target && A.min_dist) ? A.min_dist + n : nullptr, A.x[i], A.y[i], A.route.off_reward,
                                 A.route.weight, rh.s, (rh.state == ROUTE_ON && A.s_best) ? A.s_best + n : nullptr);
    A.reward[n] = r;
    if (A.terminated) A.terminated[n] = term;
    if (A.truncated) A.truncated[n] = trunc;
    if (A.done) A.done[n] = term || trunc;
    if (A.reset_trackers && (term || trunc)) {   // the next episode starts fresh (ParkingEnv.reset, parking.py:276-277)
      if (A.max_iou) A.max_iou[n] = -INFINITY;
      if (A.min_dist) A.min_dist[n] = INFINITY;
      if (A.s_best) A.s_best[n] = -INFINITY;
    }
  }
}

// ---------------------------------------------------------------------------- K10 per-agent epilogue
// DESIGN.md section 1 "Per-agent status and reward": the status chain, terminated / truncated and the reward chain of the
// env epilogue for every row (n, q) of an observer list, retirement of the slots whose rows settle, and the done mask
// "no row of the scenario is NORMAL".  One warp per scenario; lane l takes rows l, l + 32, l + 64, l + 96.
// The state is the tick's result; a settled row's slot becomes 255 in type_id, the caller's writable array ...
struct AgentArgs : WorldArgs {
  GoalArgs goal;                // the rows' detectors, indexed by the row n·Q + q (target [N][Q][5] or nullptr)
  const uint8_t* flags;         // [N][M] event byte of the tick
  const int16_t* observers;     // [N][Q] or nullptr: row q is slot q
  uint8_t* retired;             // [N][M]: ... and keeps its type here (255: not retired)
  float *max_iou, *min_dist;    // [N][Q] per-episode extrema
  float* reward;                // [N][Q]
  uint8_t *terminated, *truncated, *status;   // [N][Q]
  uint8_t* done;                // [N]
  uint8_t* traffic_status;      // [N][M] or nullptr
  RouteArgs route;
  double* s_best;               // [N][Q] best arc length of the episode, or nullptr: no progress term
  int Q, max_step, reset_trackers;
};

constexpr int K10_WARPS = 8;
constexpr int K10_ROWS_PER_LANE = T2D_OBS_MAX_OBSERVERS / 32;   // Q <= 128

__global__ void __launch_bounds__(K10_WARPS * 32) t2d_agents_epilogue_kernel(const __grid_constant__ AgentArgs A) {
  const int lane = threadIdx.x & 31;
  const long long n = (long long)blockIdx.x * K10_WARPS + (threadIdx.x >> 5);
  if (n >= A.N) return;   // whole warps
  const long long s0 = n * A.M, r0 = n * A.Q;
  if (A.traffic_status) {
    for (int m = lane; m < A.M; m += 32) {
      const unsigned f = A.flags[s0 + m];
      A.traffic_status[s0 + m] = (f & T2D_F_STATIC) ? 3 : ((f & T2D_F_DYNAMIC) ? 4 : 1);
    }
    if (A.route.route_id != nullptr) __syncwarp();   // before an off-route row overwrites its slot's code
  }
  const int cnt = A.step_count[n];
  const bool time_up = A.max_step > 0 && cnt > A.max_step;                     // parking.py:366-369
  bool any_normal = false;
  unsigned settle = 0;                                                          // bit k: row lane + 32 k retires its slot
#pragma unroll 1
  for (int k = 0; k < K10_ROWS_PER_LANE; ++k) {
    const int q = lane + 32 * k;
    if (q >= A.Q) break;
    const long long r = r0 + q;
    const int j = A.observers ? A.observers[r] : q;
    const int t = (j >= 0 && j < A.M) ? A.type_id[s0 + j] : 0xff;
    if (t >= A.n_types) {   // absent row
      A.status[r] = 0; A.reward[r] = 0.0f; A.terminated[r] = 0; A.truncated[r] = 0; A.goal.iou[r] = 0.0f;
      continue;
    }
    const long long i = s0 + j;
    const float x = A.x[i], y = A.y[i];
    const float* goal = A.goal.target ? A.goal.target + 5 * r : nullptr;
    const bool has_goal = goal != nullptr && goal[0] == goal[0];
    unsigned ev = 0;
    float iou = 0.0f;
    const Vec4 g2 = params_group(A.table + t, 2);   // (pose_l, pose_w, rbound, model | shape << 8)
    // K1's condition for the ego: a solid box (pose tile: x not NaN, pose_w >= 0)
    if (has_goal && x == x && (__float_as_int(g2.w) >> 8) != SHAPE_NONE && g2.y >= 0.0f) {
      ev = ego_goal_events(A, r, x, y, A.h[i], g2.x, g2.y);   // writes goal.iou[r]
      iou = A.goal.iou[r];
    } else {
      A.goal.iou[r] = 0.0f;
    }
    const unsigned f = A.flags[i];
    int st = T2D_STATUS_NORMAL;                                                 // parking.py:366-390, lowest priority first
    if (ev & 1u) st = T2D_STATUS_COMPLETED;
    if (f & T2D_F_DYNAMIC) st = T2D_STATUS_FAILED;
    if (f & T2D_F_STATIC) st = T2D_STATUS_FAILED;
    if (f & T2D_F_OUTBOUND) st = T2D_STATUS_OUT_BOUND;
    if (ev & 2u) st = T2D_STATUS_NO_ACTION;
    if (time_up) st = T2D_STATUS_TIME_EXCEEDED;
    RouteHit rh{0.0, ROUTE_NONE};
    if (A.route.route_id != nullptr && (st == T2D_STATUS_NORMAL || st == T2D_STATUS_COMPLETED)) {   // OffRoute: below
      rh = route_probe(A.route, i, x, y);                                                            // collision, above
      if (rh.state == ROUTE_OFF) {                                                                   // completion
        st = T2D_STATUS_FAILED;
        if (A.traffic_status) A.traffic_status[i] = T2D_TRAFFIC_OFF_ROUTE;
      }
    }
    const int ts = st == T2D_STATUS_FAILED ? ((f & T2D_F_STATIC) ? 3 : ((f & T2D_F_DYNAMIC) ? 4 : T2D_TRAFFIC_OFF_ROUTE)) : 1;
    const bool term = st == T2D_STATUS_COMPLETED;
    const bool trunc = !term && st != T2D_STATUS_NORMAL;
    A.reward[r] = reward_chain(st, ts, cnt, A.max_step, iou, has_goal ? A.max_iou + r : nullptr, goal,
                               has_goal ? A.min_dist + r : nullptr, x, y, A.route.off_reward, A.route.weight, rh.s,
                               (rh.state == ROUTE_ON && A.s_best) ? A.s_best + r : nullptr);
    A.status[r] = (uint8_t)st; A.terminated[r] = term; A.truncated[r] = trunc;
    any_normal = any_normal || st == T2D_STATUS_NORMAL;
    if (st != T2D_STATUS_NORMAL) {   // retire the slot (duplicate rows store the same type)
      settle |= 1u << k;
      A.retired[i] = (uint8_t)t;
    }
  }
  // every row has read its slot's type before any slot leaves type_id
  const bool done = !__any_sync(0xffffffffu, any_normal);
  if (lane == 0) A.done[n] = done;
  __syncwarp();
#pragma unroll 1
  for (int k = 0; k < K10_ROWS_PER_LANE; ++k) {
    const int q = lane + 32 * k;
    if (q >= A.Q) break;
    if (A.reset_trackers && done) {
      A.max_iou[r0 + q] = -INFINITY; A.min_dist[r0 + q] = INFINITY;
      if (A.s_best) A.s_best[r0 + q] = -INFINITY;
    }
    if ((settle >> k) & 1u) const_cast<uint8_t*>(A.type_id)[s0 + (A.observers ? A.observers[r0 + q] : q)] = 0xff;
  }
}

// ---------------------------------------------------------------------------- K11 per-agent action
// DESIGN.md section 1 "Per-agent action": slot m of scenario n takes row q* of agent_action, the lowest q with
// observers[n][q] == m, when its type is active; nothing else is written.  One warp per scenario; lane l takes rows l,
// l + 32, l + 64, l + 96 and claims their slots with atomicMin on a per-slot owner in shared memory, so the first row
// wins whatever the order of the atomics.  Then one float2 copy per owned active slot (the fp32 bits as they are).
struct ActionArgs : WorldArgs {
  const int16_t* observers;     // [N][Q] or nullptr: row q is slot q
  const float* agent_action;    // [N][Q][2]
  float* action;                // [N][M][2]
  int Q;
};

constexpr int K11_WARPS = 8;

__global__ void __launch_bounds__(K11_WARPS * 32) t2d_agent_action_kernel(const __grid_constant__ ActionArgs A) {
  __shared__ int s_owner[K11_WARPS][T2D_MAX_PARTICIPANTS];
  const int lane = threadIdx.x & 31;
  const long long n = (long long)blockIdx.x * K11_WARPS + (threadIdx.x >> 5);
  if (n >= A.N) return;   // whole warps
  const long long s0 = n * A.M, r0 = n * A.Q;
  constexpr int K = T2D_MAX_PARTICIPANTS / 32;   // = T2D_OBS_MAX_OBSERVERS / 32: rows and slots per lane
  // every independent load first: the observer and type loads of a lane are in flight together
  int slot[K];
  unsigned type[K];
#pragma unroll
  for (int k = 0; k < K; ++k) {
    const int q = lane + 32 * k, m = q;
    slot[k] = q < A.Q ? (A.observers ? (int)A.observers[r0 + q] : q) : -1;
    type[k] = m < A.M ? A.type_id[s0 + m] : 0xffu;
  }
  int* owner = s_owner[threadIdx.x >> 5];
#pragma unroll
  for (int k = 0; k < K; ++k)
    if (lane + 32 * k < A.M) owner[lane + 32 * k] = A.Q;   // Q: no row names the slot
  __syncwarp();
#pragma unroll
  for (int k = 0; k < K; ++k)
    if (slot[k] >= 0 && slot[k] < A.M) atomicMin(&owner[slot[k]], lane + 32 * k);
  __syncwarp();
  const float2* src = reinterpret_cast<const float2*>(A.agent_action) + r0;
  float2* dst = reinterpret_cast<float2*>(A.action) + s0;
  float2 val[K];
  bool put[K];
#pragma unroll
  for (int k = 0; k < K; ++k) {   // all loads, then all stores (the two arrays may alias as far as the compiler knows)
    const int m = lane + 32 * k;
    const int q = m < A.M ? owner[m] : A.Q;
    put[k] = q < A.Q && type[k] < (unsigned)A.n_types;
    if (put[k]) val[k] = src[q];
  }
#pragma unroll
  for (int k = 0; k < K; ++k)
    if (put[k]) dst[lane + 32 * k] = val[k];
}

}  // namespace t2d
