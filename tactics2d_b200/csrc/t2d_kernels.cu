// t2d_kernels.cu - the C ABI (include/t2d_b200.h) of the batched tick, and the one translation unit that compiles every
// sm_90a kernel.  Each kernel family lives in a header of its own that compiles alone; what more than one family reads
// (the launch-shape constants, the map tile header, WorldArgs / MapArgs / GoalArgs, the PTX and vector helpers, the
// collision primitives and the goal detectors) is in t2d_world.cuh, the per-participant arithmetic in t2d_math.cuh.
//
// K1  t2d_step_kernel      fused physics -> pose -> dynamic collision (broadphase + filtered
//                          narrowphase) -> static collision against the map tile in shared
//                          memory (uniform-grid broadphase) -> out-of-bound -> status chain (t2d_tick.cuh).
//                          (+ t2d_drift_kernel: pre-pass for SingleTrackDrift participants.)
// K2  t2d_reset_kernel     masked re-initialisation from a pool of initial states (t2d_reset.cuh).
// K3  t2d_physics_kernel   flat batch through one physics model (PhysicsModelBase.step) (t2d_tick.cuh).
// K4  t2d_lidar_kernel     single-line lidar of every scenario's ego (per-edge beam windows) (t2d_lidar.cuh).
// K5  t2d_control_kernel   NPC controllers: IDM, cruise / adaptive cruise, pure pursuit, PID (t2d_control.cuh);
//                         t2d_reactive_control_kernel adds the reactive slots' own IDM desired speeds.
// K6  t2d_bev_kernel       the bird's-eye-view observation of every scenario's ego, or of every observer row (t2d_bev.cuh).
// K7  t2d_replay_kernel    log replay: recorded tracks pose the replayed slots before K1 / after K2 (t2d_replay.cuh);
//                         t2d_reactive_replay_kernel hands reactive tracks over to K5 while a reactive replay is bound.
// K8  t2d_obs_kernel       the ego-frame vector observation (t2d_obs.cuh).
// K9  t2d_obs_agents_kernel the same observation from a list of observer slots per scenario (t2d_obs.cuh).
//     t2d_env_epilogue_kernel    status, reward and done mask of every scenario's ego (t2d_agents.cuh).
// K10 t2d_agents_epilogue_kernel status, reward and retirement of every agent row of an observer list (t2d_agents.cuh).
// K11 t2d_agent_action_kernel    the action of every agent row of an observer list, scattered to its slot (t2d_agents.cuh).
// K12 t2d_route_obs_kernel       the route of every observer row in its frame, with look-ahead points (t2d_route.cuh).
// K13 t2d_episode_draw_kernel    sampled resets: the seeded pool-row draw and the row-owned columns (t2d_reset.cuh).
// K14 t2d_episode_place_kernel   sampled resets: collision-checked jitter of the start states, one warp per scenario
//                                (t2d_reset.cuh).
// K15 t2d_history_append_kernel  trajectory history: append the state after a tick, restart it after a reset (t2d_history.cuh).
// K16 t2d_history_obs_kernel     trajectory history: past poses of an observer and its agents in its current frame
//                                (t2d_history.cuh).
// K17 t2d_leader_kernel          the leader of every slot in its corridor, which K5 follows while a search is bound
//                                (t2d_leader.cuh).
// K18 t2d_lane_change_kernel     MOBIL lane changes of the IDM rows with a lateral channel, in front of K17 and K5 while
//                                a lane change is bound; t2d_lane_reset_kernel restarts the reset scenarios' lanes
//                                (t2d_lane.cuh).
// K19 t2d_yield_kernel           whom every path-following IDM car yields to at the conflict zones of its path, and where it
//                                stops, in front of K5's t2d_yield_control_kernel while yielding is bound (t2d_yield.cuh).
//     t2d_exchange_allgather_kernel   all-gather of the done masks over NVLink peer memory (t2d_exchange.cuh).
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/t2d_b200.h"
#include "t2d_math.cuh"
#include "t2d_world.cuh"
#include "t2d_tick.cuh"
#include "t2d_reset.cuh"
#include "t2d_route.cuh"
#include "t2d_agents.cuh"
#include "t2d_replay.cuh"
#include "t2d_lidar.cuh"
#include "t2d_exchange.cuh"
#include "t2d_control.cuh"
#include "t2d_bev.cuh"
#include "t2d_obs.cuh"
#include "t2d_history.cuh"
#include "t2d_leader.cuh"
#include "t2d_lane.cuh"
#include "t2d_yield.cuh"

// =============================================================================================
// C ABI
// =============================================================================================
using namespace t2d;

static thread_local std::string g_err;
static std::atomic<long long> g_launches{0};
// K1 launches per instance (launch_step's `variant`), then the one-tile launches that read the map from global memory
static std::atomic<long long> g_tick_instances[7] = {};
static std::atomic<int> g_exchanges_alive{0};   // peer-memory done exchanges in this process (see StepArgs::prefetch)
static std::mutex g_smem_mutex;
// [device]: the fallback counters of K1's FIXED instance (ORDER_COUNTERS x ORDER_COUNTER_STRIDE, zeroed), allocated by
// the first t2d_create on the device and kept for the life of the process, as a __device__ variable would be
static unsigned long long* g_order_fallbacks[64] = {};
static std::mutex g_order_mutex;
static int g_smem_configured[64][6];   // [device][kernel variant]: dynamic shared memory opted in so far (process-wide)

static int fail(int code, const std::string& msg) {
  g_err = msg;
  return code;
}
#define CUDA_TRY(expr)                                                                           \
  do {                                                                                           \
    cudaError_t _e = (expr);                                                                     \
    if (_e != cudaSuccess) return fail(T2D_E_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e)); \
  } while (0)

// Owners of the context's device and pinned host buffers.  Dropping one frees its buffer, so whatever replaces or drops
// one runs with the context's device current.
struct CudaFree {
  void operator()(void* p) const { cudaFree(p); }
};
struct CudaFreeHost {
  void operator()(void* p) const { cudaFreeHost(p); }
};
template <class T> using dev_ptr = std::unique_ptr<T, CudaFree>;
template <class T> using host_ptr = std::unique_ptr<T, CudaFreeHost>;

template <class T> static int dev_alloc(dev_ptr<T>& out, size_t n) {
  T* p = nullptr;
  CUDA_TRY(cudaMalloc(&p, n * sizeof(T)));
  out.reset(p);
  return T2D_OK;
}

template <class T> static int host_alloc(host_ptr<T>& out, size_t n, unsigned flags = cudaHostAllocDefault) {
  T* p = nullptr;
  CUDA_TRY(cudaHostAlloc(&p, n * sizeof(T), flags));
  out.reset(p);
  return T2D_OK;
}

// n host elements copied to a fresh device buffer; `out` changes only on success
template <class T> static int upload(dev_ptr<T>& out, const T* src, size_t n) {
  dev_ptr<T> d;
  if (int r = dev_alloc(d, n)) return r;
  CUDA_TRY(cudaMemcpy(d.get(), src, n * sizeof(T), cudaMemcpyHostToDevice));
  out = std::move(d);
  return T2D_OK;
}

struct t2d_exchange {
  int device = 0, world = 0, rank = 0, n_local = 0, slots = 0;
  size_t bytes = 0;
  int n_real = 0;
  int threads = 256;                             // CTA size of the exchange kernel (T2D_EXCHANGE_THREADS, read once at create)
  long long timeout_cycles = 4000000000LL;       // how long a wait may spin (~2 s of SM clocks; T2D_EXCHANGE_TIMEOUT_MS)
  unsigned char* base = nullptr;                 // slots x world x n_local done bytes | MAX_RANKS flag words | step, -, -, error
  unsigned char* peer[T2D_MAX_RANKS] = {};       // every rank's base (own included), valid after t2d_exchange_connect
  bool connected = false;
  size_t flag_off() const { return (size_t)slots * world * n_local; }
  unsigned* word(int i) const { return reinterpret_cast<unsigned*>(base + flag_off()) + T2D_MAX_RANKS + i; }   // 0 steps done, 3 error
};

// The bound map (t2d_set_map_table), replaced as a whole: a new map also drops the per-segment BEV styles of the old one
struct DeviceMap {
  dev_ptr<unsigned char> blob;         // the tiles back to back, each 128-byte aligned
  dev_ptr<uint32_t> tile_off;          // [n_tiles] byte offsets of the tiles inside blob
  const uint16_t* tile_id = nullptr;   // caller-owned DEVICE [N]; nullptr unless there is more than one tile
  int n_tiles = 0;
  bool has_segments = false;
  bool has_bounds = false;             // any tile has a boundary box
  MapHeader mh{};                      // tile 0's header
  int smem_bytes = 0;                  // what a single tile stages into shared memory
  std::vector<int> tile_nseg;          // segments of every tile, in tile order
  dev_ptr<uint8_t> seg_style;          // BEV style per segment, tiles back to back; nullptr: the default ring / open styles
  dev_ptr<uint32_t> seg_base;          // [n_tiles] first entry of every tile in seg_style
};

// The bound log (t2d_set_log / K7), replaced as a whole
struct DeviceLog {
  dev_ptr<ReplayTrack> tracks;
  dev_ptr<uint8_t> track_type;
  dev_ptr<float> rec;
  dev_ptr<int32_t> t0;
  dev_ptr<int32_t> slot_off;           // [n_rows * M + 1] schedule offsets
  dev_ptr<ReplayEntry> entries;
  dev_ptr<int32_t> slot_track1;        // [n_rows * M] instead of the two above when no schedule has two entries
  int n_tracks = 0, n_rows = 0;
  int32_t* row = nullptr;              // caller-owned DEVICE [N]
  int32_t* track_out = nullptr;        // caller-owned DEVICE [N][M] or nullptr
  uint8_t* type_id = nullptr;          // writable alias of type_id, checked against the bound one before every launch
  std::vector<uint8_t> track_type_host;   // host copy: t2d_set_type_table keeps these rows static
};

// The bound reset sampler (t2d_set_reset_sampler), replaced as a whole: the caller's struct with the jitter table moved
// into the library's own device copy
struct DeviceSampler {
  t2d_reset_sampler s{};               // s.jitter: jitter.get() or nullptr
  dev_ptr<float> jitter;               // [M][8]
};

// The trajectory history ring (t2d_set_history), replaced as a whole; the track ring exists exactly while a log schedule
// with a track output is bound (history_tracks)
struct DeviceHistory {
  int H = 0;
  dev_ptr<float> f;                    // [6][N][H][M]: x, y, heading, speed, vx, vy
  dev_ptr<uint8_t> type;               // [N][H][M]
  dev_ptr<int32_t> track;              // [N][H][M] or nullptr
  dev_ptr<long long> count;            // [N]
};

// Staging of the host steps (t2d_step_host, t2d_step_host_ego, t2d_step_host_agents); every piece is created whole the
// first time a step needs it.
static constexpr int MAX_HOST_CHUNKS = 8;

struct ChunkedUpload {   // t2d_step_host: device copy of the actions, the copy stream and its events
  dev_ptr<float> action;               // [N][M][2]
  cudaStream_t copy = nullptr;
  cudaEvent_t begin = nullptr, chunk[MAX_HOST_CHUNKS] = {};
  ~ChunkedUpload() {
    if (begin) cudaEventDestroy(begin);
    for (cudaEvent_t e : chunk)
      if (e) cudaEventDestroy(e);
    if (copy) cudaStreamDestroy(copy);
  }
};

struct Mirror {   // a packed block of device outputs and its pinned host mirror
  dev_ptr<uint8_t> dev;
  host_ptr<uint8_t> host;
};

struct MappedEgo {   // t2d_step_host_ego: [N][2] pinned + mapped host staging of the ego actions ...
  host_ptr<float> host;
  const float* dev = nullptr;          // ... and its device-side address: the kernels read it over PCIe, no copy engine involved
};

struct AgentStaging {   // t2d_step_host_agents, sized for q rows per scenario
  int q = 0;
  dev_ptr<float> action;               // [N][Q][2]
  Mirror out;                          // device: [N][Q] fp32 reward, [3][N][Q] uint8, [N] uint8 done, then [N][Q] fp32 iou;
                                       // host: the part up to done
};

// A bound lane change: the parameters, the neighbour table on the device and the caller's per-slot arrays
struct LaneChange {
  t2d_lane_change_params p;
  dev_ptr<int16_t> left, right;
  int16_t* lane_path;
  int16_t* cooldown;
  int8_t* change;
};

// A bound reactive replay: the per-track tables on the device and the caller's per-slot arrays
struct ReactiveReplay {
  dev_ptr<int16_t> track_path;
  dev_ptr<uint8_t> drive_row;
  dev_ptr<float> desired_speed;
  int16_t* drive_path;
  float* slot_desired_speed;
};

// A bound yielding (t2d_set_yielding / K19): the parameters, the zone table and priorities on the device, the stop points
// K19 writes for K5, and the caller's per-slot outputs
struct Yielding {
  t2d_yield_params p;
  dev_ptr<yield::Zone> zones;
  dev_ptr<int> zone_off;
  dev_ptr<int16_t> priority;
  dev_ptr<double2> stop_xy;            // [N][M]
  int16_t* yield_to;
  float* stop_gap;
};

struct t2d_ctx {
  int device = 0, N = 0, M = 0, G = 0;
  t2d_config cfg{};
  int n_types = 0;
  bool has_pointmass = false;
  bool has_drift = false;
  bool kin_only = false;
  float *wheel_f = nullptr, *wheel_r = nullptr;
  const float *reset_pool_wf = nullptr, *reset_pool_wr = nullptr;   // t2d_bind_reset_wheel_pool
  dev_ptr<Params> d_table;
  DeviceMap map;
  float *x = nullptr, *y = nullptr, *h = nullptr, *v = nullptr, *vx = nullptr, *vy = nullptr;
  const uint8_t* type_id = nullptr;
  int32_t* step_count = nullptr;
  int sm_count = 0;                // set by t2d_create from the device
  int max_smem_optin = 0;
  float rb_max = 0.0f;
  const float* ego_action = nullptr;   // t2d_set_ego_action
  GoalArgs goal{};                     // t2d_set_goal
  // per-agent status and reward (t2d_set_agents / K10); agent_q == 0: not bound
  int agent_q = 0;
  const int16_t* agent_observers = nullptr;
  GoalArgs agent{};                    // iou: the t2d_agents_epilogue argument
  uint8_t* agent_retired = nullptr;
  bool use_pdl = true;            // T2D_PDL=0 disables programmatic dependent launch
  int prefetch_override = -1;      // T2D_PREFETCH=0 / 1 (experiments; -1 = on unless a done exchange is alive)
  int wpc_override = 0;            // T2D_WPC=w: warps per CTA of the tick (experiments; 0 = pick from the batch size)
  int grid_limit = 0;              // T2D_GRID_LIMIT=k: at most k CTAs of the persistent tick grid per SM (experiments; 0 = occupancy)
  bool tick_generic = false;       // T2D_TICK_GENERIC=1: never launch K1's FIXED instance (tests compare the two)
  int occ_smem[9] = {-1, -1, -1, -1, -1, -1, -1, -1, -1};   // per warps-per-CTA: smem the cached occupancy was computed for
  int occ_val[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  int occ_variant[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  // NPC controllers (t2d_set_controllers / t2d_set_paths / t2d_control)
  dev_ptr<t2d_controller_params> d_ctab;
  int n_ctrl = 0;
  const uint8_t* ctrl_id = nullptr;
  const int16_t* ctrl_lead = nullptr;
  const int16_t* ctrl_path = nullptr;
  float* ctrl_last_accel = nullptr;
  bool ctrl_has_pid = false;          // the table holds a T2D_CTRL_PID row: K5 runs its PID instance
  bool ctrl_pid_reads_target = false; // ... and one of them reads the target array
  const float* pid_target = nullptr;  // t2d_set_pid: [N][M][2]
  double* pid_state = nullptr;        // t2d_set_pid: [N][M][6]
  dev_ptr<PathVertex> d_path_v;
  dev_ptr<int> d_path_off;
  int n_paths = 0;
  std::vector<PathVertex> path_host;   // host copy of the table and its offsets (t2d_set_yielding's stop points)
  std::vector<int> path_off_host;
  // leader search (t2d_set_leader_search / K17); leader_lead == nullptr: none bound, K5 reads ctrl_lead
  int16_t* leader_lead = nullptr;
  float* leader_gap = nullptr;
  double leader_half_width = 0.0, leader_max_range = 0.0;
  // lane change (t2d_set_lane_change / K18); lane == nullptr: none bound, K17 and K5 read ctrl_path
  std::unique_ptr<LaneChange> lane;
  // reactive replay (t2d_set_log_reactive); nullptr: none bound, K7 and K5 run their plain instances
  std::unique_ptr<ReactiveReplay> reactive;
  // yielding (t2d_set_yielding / K19); nullptr: none bound, K5 runs its other instances
  std::unique_ptr<Yielding> yield;
  // routes (t2d_set_routes / t2d_bind_route_trackers); route_id == nullptr: none bound
  const int16_t* route_id = nullptr;
  double route_threshold = 0.0, route_weight = 0.0;
  float route_off_reward = 0.0f;
  double* route_s_best = nullptr;        // [N] or nullptr
  double* route_agent_s_best = nullptr;  // [N][route_agent_rows] or nullptr
  int route_agent_rows = 0;
  // host steps
  std::unique_ptr<ChunkedUpload> hs_upload;
  Mirror hs_out;                       // [2][N] status, done (t2d_step_host and t2d_step_host_ego)
  MappedEgo hs_ego;
  AgentStaging ha;
  dev_ptr<uint8_t> ha_flags;           // [N][M]: the flags K10 needs when the caller keeps none
  int host_chunks = 0;                 // 0 = pick from the batch size
  // BEV observation (t2d_set_bev_styles / t2d_bev_render)
  int n_bev_styles = 0;                // 0: styles not set
  t2d_bev_style bev_style[bev::MAX_STYLES] = {};
  uint8_t bev_type_style[T2D_MAX_TYPES] = {};
  int bev_target_style = bev::NO_STYLE;
  std::unique_ptr<DeviceLog> log;      // nullptr: no log bound
  std::vector<int> type_model;         // host copy of the current type table's model ids
  std::vector<t2d_type_params> type_rows;   // ... and of its rows (t2d_set_log_reactive compares shapes)
  dev_ptr<uint8_t> order;              // [N][64] x-order hint of K1's FIXED instance (t2d_create: the identity)
  std::unique_ptr<DeviceSampler> sampler;   // t2d_set_reset_sampler; nullptr: none bound
  std::unique_ptr<DeviceHistory> hist;      // t2d_set_history; nullptr: none bound
};

enum : unsigned { NEED_STATE = 1, NEED_TABLE = 2, NEED_TICK = 4,
                  NEED_LOG = 8, NEED_CTRL = 16, NEED_PATHS = 32, NEED_PID = 64, NEED_SEARCH = 128 };

// The call-order preconditions, checked in this order: the bound state, the type table, what a tick with physics needs
// besides (a caller that launches other kernels first checks them up front), then the bindings the traffic stages read:
// the log, the controllers, the paths, the PID state and the leader search.  fn, when given, prefixes the message.
static int require(const t2d_ctx* c, unsigned need, const char* fn = nullptr) {
  const auto missing = [fn](const char* msg) { return fail(T2D_E_STATE, fn ? std::string(fn) + ": " + msg : msg); };
  if ((need & NEED_STATE) && !c->x) return missing("state not bound: call t2d_bind_state first");
  if ((need & NEED_TABLE) && (!c->d_table || c->n_types == 0))
    return missing("type table not set: call t2d_set_type_table first");
  if (need & NEED_TICK) {
    if (c->has_drift && !(c->wheel_f && c->wheel_r))
      return missing("the type table holds a SingleTrackDrift row: call t2d_bind_wheel_state first");
    if (c->log && c->log->type_id != c->type_id) return missing("state rebound after t2d_set_log: call t2d_set_log again");
  }
  if ((need & NEED_LOG) && !c->log) return missing("no log bound: call t2d_set_log or t2d_set_log_schedule first");
  if ((need & NEED_CTRL) && !c->d_ctab) return missing("controllers not set: call t2d_set_controllers first");
  if ((need & NEED_PATHS) && c->n_paths == 0) return missing("no paths bound: call t2d_set_paths first");
  if ((need & NEED_PID) && !c->pid_state) return missing("no PID state bound: call t2d_set_pid first");
  if ((need & NEED_SEARCH) && !c->leader_lead) return missing("no leader search bound: call t2d_set_leader_search first");
  return T2D_OK;
}

// The traffic bindings name what other setters bind.  A lane change and yielding read the controllers' rows and paths,
// the path table and the search's corridor; a reactive replay reads those too, and the type table's rows and the log's
// tracks.  A setter that replaces or unbinds one of these (changed: its NEED_ bit) drops every binding that reads it.
static void drop_traffic(t2d_ctx* c, unsigned changed) {
  if (changed & (NEED_CTRL | NEED_PATHS | NEED_SEARCH)) {
    c->lane.reset();
    c->yield.reset();
  }
  if (changed & (NEED_TABLE | NEED_LOG | NEED_CTRL | NEED_PATHS | NEED_SEARCH)) c->reactive.reset();
}

static WorldArgs world_args(const t2d_ctx* c) {
  return {c->x, c->y, c->h, c->v, c->vx, c->vy, c->type_id, c->step_count, c->d_table.get(), c->n_types, c->N, c->M};
}

static PathTable path_table(const t2d_ctx* c) {
  return {c->d_path_v.get(), c->d_path_off.get(), c->n_paths};
}

static RouteArgs route_args(const t2d_ctx* c) {
  return {c->route_id, path_table(c), c->route_off_reward, c->route_threshold, c->route_weight};
}

// K10 reads its progress tracker by the bound agents' rows: a tracker bound for another Q is a call-order error
static int check_route_trackers(const t2d_ctx* c, const char* fn) {
  if (c->route_id && c->route_agent_s_best && c->route_agent_rows != c->agent_q)
    return fail(T2D_E_STATE, std::string(fn) + ": the agents' route tracker has another row count than the bound agents: "
                                               "call t2d_bind_route_trackers again");
  return T2D_OK;
}

// The observer rows of the multi-agent entry `fn`: n_observers in min_rows..128, and without an observer list row q is
// slot q, so there are at most M rows
static int check_rows(const t2d_ctx* c, const char* fn, const int16_t* observers, int n_observers, int min_rows) {
  if (n_observers < min_rows || n_observers > T2D_OBS_MAX_OBSERVERS)
    return fail(T2D_E_INVALID, std::string(fn) + ": n_observers must be in " + std::to_string(min_rows) + ".." +
                                   std::to_string(T2D_OBS_MAX_OBSERVERS));
  if (!observers && n_observers > c->M)
    return fail(T2D_E_INVALID, std::string(fn) + ": without an observer list n_observers must not exceed the slots per scenario");
  return T2D_OK;
}

// Pointer alignment (nullptr counts as aligned)
static bool aligned2(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 1) == 0; }
static bool aligned4(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 3) == 0; }
static bool aligned8(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 7) == 0; }
static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// ---- trajectory history (t2d_set_history; K15 / K16)
static hist::Ring history_ring(const t2d_ctx* c) {
  const DeviceHistory& g = *c->hist;
  const size_t plane = (size_t)c->N * g.H * c->M;
  float* f = g.f.get();
  return {f, f + plane, f + 2 * plane, f + 3 * plane, f + 4 * plane, f + 5 * plane, g.type.get(), g.track.get(), g.count.get(), g.H};
}

// the track every slot shows now, when the ring records tracks
static const int32_t* history_track_now(const t2d_ctx* c) { return c->hist->track ? c->log->track_out : nullptr; }

// Gives `g` a fresh track ring filled with -1 (an entry recorded before the schedule counts as showing no track) when
// `track_out`, the bound schedule's track output, is set, and drops it otherwise
static int history_tracks(const t2d_ctx* c, DeviceHistory& g, const int32_t* track_out) {
  if (!track_out) {
    g.track.reset();
    return T2D_OK;
  }
  const size_t n = (size_t)c->N * g.H * c->M;
  dev_ptr<int32_t> t;
  if (int r = dev_alloc(t, n)) return r;
  CUDA_TRY(cudaMemset(t.get(), 0xff, n * sizeof(int32_t)));
  g.track = std::move(t);
  return T2D_OK;
}

// from scenario `first` on (t2d_set_map_table keeps tile_id only with more than one tile)
static MapArgs map_args(const DeviceMap& map, int first = 0) {
  return {map.blob.get(), map.tile_off.get(), map.tile_id ? map.tile_id + first : nullptr};
}

// after every launch: count it and report a launch error
static int launched() {
  g_launches.fetch_add(1);
  CUDA_TRY(cudaGetLastError());
  return T2D_OK;
}

// grid of a grid-stride kernel: one CTA per `per_cta` items, at most `per_sm` CTAs per SM
static int capped_grid(long long items, int per_cta, int sm_count, int per_sm) {
  return (int)std::max(1LL, std::min((items + per_cta - 1) / per_cta, (long long)sm_count * per_sm));
}

// K15 after a tick (mask == nullptr: every scenario appends) or a reset (the masked scenarios restart); no ring, no launch
static int launch_history(t2d_ctx* c, const uint8_t* mask, void* stream) {
  if (!c->hist) return T2D_OK;
  hist::AppendArgs A{world_args(c)};
  A.ring = history_ring(c); A.track_now = history_track_now(c); A.mask = mask;
  hist::t2d_history_append_kernel<<<(c->N + hist::K15_WARPS - 1) / hist::K15_WARPS, hist::K15_WARPS * 32, 0, (cudaStream_t)stream>>>(A);
  return launched();
}

// the integration steps of one interval, for the tick and t2d_physics_step
template <class Args> static void set_time_step(Args& A, int interval_ms, int delta_t_ms) {
  const int delta_t = std::min(delta_t_ms, interval_ms);
  A.n_steps = interval_ms / delta_t;                            // single_track_kinematics.py:129
  A.dt = (float)((double)delta_t / 1000.0);                     // :128
  A.dt_rem = (float)((double)(interval_ms % delta_t) / 1000.0);   // :130,152
  A.dt_d = (double)delta_t / 1000.0;
  A.dt_rem_d = (double)(interval_ms % delta_t) / 1000.0;
  A.interval_d = (double)interval_ms / 1000.0;                  // point_mass.py:86
}

extern "C" {

int t2d_version(void) { return T2D_VERSION; }
const char* t2d_last_error(void) { return g_err.c_str(); }
int64_t t2d_launch_count(void) { return (int64_t)g_launches.load(); }
int64_t t2d_tick_fixed_count(void) { return (int64_t)(g_tick_instances[4].load() + g_tick_instances[5].load()); }
int64_t t2d_tick_order_fallback_count(void) {
  std::lock_guard<std::mutex> lock(g_order_mutex);
  int64_t sum = 0;
  for (unsigned long long* d : g_order_fallbacks) {
    if (!d) continue;
    unsigned long long n[ORDER_COUNTERS * ORDER_COUNTER_STRIDE];
    if (cudaMemcpy(n, d, sizeof(n), cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
    for (int i = 0; i < ORDER_COUNTERS; ++i) sum += (int64_t)n[i * ORDER_COUNTER_STRIDE];
  }
  return sum;
}
int64_t t2d_tick_instance_count(int k) { return k >= 0 && k < 7 ? (int64_t)g_tick_instances[k].load() : -1; }

#ifdef T2D_TICK_TIMELINE
// The phase timeline of the last tick (measurement build only): [TL_MAX_WARPS][TL_POINTS][globaltimer, clock64],
// zeroed after the copy when `clear` is set.
int t2d_tick_timeline(void* dst, int64_t bytes, int clear) {
  if (!dst || bytes != (int64_t)sizeof(t2d_timeline)) return fail(T2D_E_INVALID, "timeline buffer size");
  CUDA_TRY(cudaMemcpyFromSymbol(dst, t2d_timeline, sizeof(t2d_timeline)));
  if (clear) {
    void* p = nullptr;
    CUDA_TRY(cudaGetSymbolAddress(&p, t2d_timeline));
    CUDA_TRY(cudaMemset(p, 0, sizeof(t2d_timeline)));
  }
  return T2D_OK;
}
#endif

static int check_cfg(const t2d_config* cfg) {
  if (!cfg) return fail(T2D_E_INVALID, "cfg is NULL");
  if (cfg->interval_ms <= 0) return fail(T2D_E_INVALID, "interval_ms must be > 0");
  if (cfg->delta_t_ms <= 0) return fail(T2D_E_INVALID, "delta_t_ms must be > 0");
  return T2D_OK;
}

int t2d_create(t2d_ctx** out, int device, int n_scenarios, int m_participants, const t2d_config* cfg) {
  if (!out) return fail(T2D_E_INVALID, "out is NULL");
  *out = nullptr;
  if (int r = check_cfg(cfg)) return r;
  if (n_scenarios <= 0 || m_participants <= 0) return fail(T2D_E_INVALID, "n_scenarios and m_participants must be > 0");
  if (m_participants > T2D_MAX_PARTICIPANTS)
    return fail(T2D_E_UNSUPPORTED, "m_participants > 128: a scenario must fit one warp (4 participants per lane)");
  int count = 0;
  CUDA_TRY(cudaGetDeviceCount(&count));
  if (device < 0 || device >= count) return fail(T2D_E_INVALID, "no such CUDA device");
  CUDA_TRY(cudaSetDevice(device));
  t2d_ctx* c = new t2d_ctx();
  c->device = device;
  c->N = n_scenarios;
  c->M = m_participants;
  if (const char* e = getenv("T2D_PDL")) c->use_pdl = atoi(e) != 0;
  if (const char* e = getenv("T2D_GRID_LIMIT")) c->grid_limit = std::max(0, atoi(e));
  if (const char* e = getenv("T2D_TICK_GENERIC")) c->tick_generic = atoi(e) != 0;
  if (const char* e = getenv("T2D_PREFETCH")) c->prefetch_override = atoi(e) != 0 ? 1 : 0;
  if (const char* e = getenv("T2D_WPC")) {
    const int v = atoi(e);
    if (v >= 1 && v <= MAX_WARPS_PER_CTA) c->wpc_override = v;
  }
  if (const char* e = getenv("T2D_HOST_CHUNKS")) c->host_chunks = std::max(0, std::min(atoi(e), MAX_HOST_CHUNKS));
  int g = 1;
  while (g * PPL < m_participants) g <<= 1;
  c->G = g;
  c->cfg = *cfg;
  cudaDeviceProp prop;
  CUDA_TRY(cudaGetDeviceProperties(&prop, device));
  c->sm_count = prop.multiProcessorCount;
  c->max_smem_optin = (int)prop.sharedMemPerBlockOptin;
  {
    std::lock_guard<std::mutex> lock(g_order_mutex);
    unsigned long long*& counters = g_order_fallbacks[device % 64];
    const size_t bytes = ORDER_COUNTERS * ORDER_COUNTER_STRIDE * sizeof(unsigned long long);
    if (!counters && (cudaMalloc(&counters, bytes) != cudaSuccess || cudaMemset(counters, 0, bytes) != cudaSuccess)) {
      cudaFree(counters);
      counters = nullptr;
      delete c;
      return fail(T2D_E_CUDA, "t2d_create: cannot allocate the order fallback counters");
    }
  }
  {
    std::vector<uint8_t> identity((size_t)n_scenarios * FIX_M);
    for (size_t i = 0; i < identity.size(); ++i) identity[i] = (uint8_t)(i % FIX_M);
    if (int r = upload(c->order, identity.data(), identity.size())) {
      delete c;
      return r;
    }
  }
  *out = c;
  return T2D_OK;
}

int t2d_order_hint(t2d_ctx* c, void* read_to, const void* write_from) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  CUDA_TRY(cudaSetDevice(c->device));
  const size_t bytes = (size_t)c->N * FIX_M;
  if (read_to) CUDA_TRY(cudaMemcpy(read_to, c->order.get(), bytes, cudaMemcpyDeviceToHost));
  if (write_from) CUDA_TRY(cudaMemcpy(c->order.get(), write_from, bytes, cudaMemcpyHostToDevice));
  return T2D_OK;
}

int t2d_destroy(t2d_ctx* c) {
  if (!c) return T2D_OK;
  cudaSetDevice(c->device);   // the owners free on the current device
  delete c;
  return T2D_OK;
}

int t2d_set_config(t2d_ctx* c, const t2d_config* cfg) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (int r = check_cfg(cfg)) return r;
  c->cfg = *cfg;
  return T2D_OK;
}

int t2d_set_type_table(t2d_ctx* c, const t2d_type_params* table, int n_types) {
  if (!c || !table) return fail(T2D_E_INVALID, "ctx/table is NULL");
  if (n_types <= 0 || n_types > T2D_MAX_TYPES) return fail(T2D_E_INVALID, "n_types must be in 1..64");
  static_assert(sizeof(t2d_type_params) == sizeof(AbiParams), "type table layout");
  if (c->log)
    for (uint8_t row : c->log->track_type_host)   // a bound log's tracks must stay static rows (K1 would integrate on the log)
      if (row >= n_types || table[row].model != T2D_MODEL_STATIC)
        return fail(T2D_E_INVALID, "type table: row " + std::to_string(row) + " of a replayed track must exist and be T2D_MODEL_STATIC");
  bool has_pointmass = false, has_drift = false, kin_only = true;
  float rb_max = 0.0f;
  for (int i = 0; i < n_types; ++i) {
    const t2d_type_params& p = table[i];
    if (p.shape == T2D_SHAPE_OBB) rb_max = std::max(rb_max, sqrtf(p.half_len * p.half_len + p.half_wid * p.half_wid) * 1.000002f);
    if (p.shape == T2D_SHAPE_CIRCLE) rb_max = std::max(rb_max, p.radius);
    if (p.model < 0 || p.model > T2D_MODEL_DRIFT) return fail(T2D_E_INVALID, "type table: unknown model id");
    if (p.shape < 0 || p.shape > T2D_SHAPE_NONE) return fail(T2D_E_INVALID, "type table: unknown shape id");
    const bool bicycle = p.model <= T2D_MODEL_DYNAMICS || p.model == T2D_MODEL_DRIFT;
    if (bicycle && !(p.lf + p.lr > 0.0f)) return fail(T2D_E_INVALID, "type table: lf + lr must be > 0");
    if (p.model == T2D_MODEL_DYNAMICS && !(p.lf > 0.0f && p.I_z > 0.0f))
      return fail(T2D_E_INVALID, "type table: dynamics needs lf > 0 and I_z > 0");
    if (p.model == T2D_MODEL_DRIFT && !(p.lf > 0.0f && p.I_z > 0.0f && p.mass > 0.0f && p.wheel_radius > 0.0f && p.I_yw > 0.0f))
      return fail(T2D_E_INVALID, "type table: drift needs lf, I_z, mass, wheel_radius and I_yw > 0");
    if (p.model == T2D_MODEL_DRIFT) has_drift = true;
    if (p.shape == T2D_SHAPE_OBB && !(p.half_len >= 0.0f && p.half_wid >= 0.0f))
      return fail(T2D_E_INVALID, "type table: negative OBB half extent");
    if (p.shape == T2D_SHAPE_CIRCLE && !(p.radius >= 0.0f)) return fail(T2D_E_INVALID, "type table: negative radius");
    if (p.model == T2D_MODEL_POINTMASS_NEWTON || p.model == T2D_MODEL_POINTMASS_EULER) has_pointmass = true;
    if (p.model != T2D_MODEL_KINEMATICS && p.model != T2D_MODEL_STATIC) kin_only = false;
  }
  std::vector<Params> rows(n_types + 1);
  for (int i = 0; i < n_types; ++i) {
    AbiParams a;
    memcpy(&a, &table[i], sizeof(AbiParams));
    rows[i] = derive_params(a);
  }
  {
    // row n_types: the neutral kinematic row that K1's 4-chain loop gives to slots holding another model or nothing
    // (zero speed and action in, unbounded ranges: every product stays finite and the result is discarded)
    AbiParams a{};
    a.lf = 1.0f; a.lr = 1.0f;
    a.steer_lo = a.speed_lo = a.accel_lo = -INFINITY;
    a.steer_hi = a.speed_hi = a.accel_hi = INFINITY;
    a.model = MODEL_KINEMATICS; a.shape = SHAPE_NONE;
    rows[n_types] = derive_params(a);
  }
  CUDA_TRY(cudaSetDevice(c->device));
  if (int r = upload(c->d_table, rows.data(), rows.size())) return r;
  c->n_types = n_types;
  c->type_model.resize(n_types);
  for (int i = 0; i < n_types; ++i) c->type_model[i] = table[i].model;
  c->type_rows.assign(table, table + n_types);
  drop_traffic(c, NEED_TABLE);
  c->has_pointmass = has_pointmass;
  c->has_drift = has_drift;
  c->rb_max = rb_max;
  c->kin_only = kin_only;
  for (int w = 0; w < 9; ++w) c->occ_smem[w] = -1;
  return T2D_OK;
}
// Host-side build of one static-geometry tile: the segments in list order (+ which of them close up to polygons), a
// uniform grid over their bounding box grown by one cell, per cell the ascending list of the segments that touch it and
// the "dilated" list of those within one cell of it, the clearance fields, the tile's boundary box.
struct TileIn {
  const float* segments; int n_seg;
  const int32_t* poly_start; int n_poly;
  const float* bounds;
};

static bool point_in_ring(const float* seg, int s0, int s1, double px, double py) {   // even-odd over the ring's edges
  bool in = false;
  for (int i = s0; i < s1; ++i) {
    const double x1 = seg[4 * i], y1 = seg[4 * i + 1], x2 = seg[4 * i + 2], y2 = seg[4 * i + 3];
    if ((y1 > py) != (y2 > py) && px < (x2 - x1) * (py - y1) / (y2 - y1) + x1) in = !in;
  }
  return in;
}

static int build_tile(const TileIn& t, float cell_size, float reach, std::vector<unsigned char>& blob) {
  const float* segments = t.segments;
  const int n_seg = t.n_seg;
  if (n_seg < 0 || n_seg > T2D_MAX_SEGMENTS) return fail(T2D_E_INVALID, "n_seg must be in 0..32767");
  if (n_seg > 0 && !segments) return fail(T2D_E_INVALID, "segments is NULL");
  if (t.n_poly < 0 || (t.n_poly > 0 && !t.poly_start)) return fail(T2D_E_INVALID, "poly_start is NULL");
  if (t.bounds && !(t.bounds[0] <= t.bounds[1] && t.bounds[2] <= t.bounds[3])) return fail(T2D_E_INVALID, "bounds must be (xmin<=xmax, ymin<=ymax)");
  for (int p = 0; p < t.n_poly; ++p) {
    const int s0 = t.poly_start[p], s1 = t.poly_start[p + 1];
    if (s0 < 0 || s1 > n_seg || s1 - s0 < 3 || (p > 0 && s0 < t.poly_start[p])) return fail(T2D_E_INVALID, "poly_start: rings must be ascending, inside the segment list and have >= 3 edges");
    // one object = one or more closed rings back to back (an Area's exterior, then its holes): every edge ends where the
    // next one starts, except the edge that returns to its ring's first vertex - the next edge starts the next ring
    int r0 = s0;
    for (int i = s0; i < s1; ++i) {
      if (segments[4 * i + 2] == segments[4 * r0] && segments[4 * i + 3] == segments[4 * r0 + 1]) { r0 = i + 1; continue; }
      if (i + 1 == s1 || segments[4 * i + 2] != segments[4 * (i + 1)] || segments[4 * i + 3] != segments[4 * (i + 1) + 1])
        return fail(T2D_E_INVALID, "poly_start: a ring's edges must chain and close");
    }
  }
  MapHeader mh{};
  mh.n_seg = n_seg; mh.n_poly = t.n_poly;
  mh.has_bounds = t.bounds ? 1 : 0;
  if (t.bounds) { mh.bxmin = t.bounds[0]; mh.bxmax = t.bounds[1]; mh.bymin = t.bounds[2]; mh.bymax = t.bounds[3]; }
  if (n_seg == 0) {   // bounds only
    mh.gx = mh.gy = 0; mh.total_bytes = mh.smem_bytes = mh.off_fine = sizeof(MapHeader);
    blob.assign(sizeof(MapHeader), 0);
    memcpy(blob.data(), &mh, sizeof(mh));
    return T2D_OK;
  }
  float xmin = INFINITY, xmax = -INFINITY, ymin = INFINITY, ymax = -INFINITY;
  for (int i = 0; i < n_seg * 4; ++i)
    if (!std::isfinite(segments[i])) return fail(T2D_E_INVALID, "segments must be finite");
  for (int i = 0; i < n_seg; ++i) {
    const float* s = segments + 4 * i;
    xmin = std::min(xmin, std::min(s[0], s[2])); xmax = std::max(xmax, std::max(s[0], s[2]));
    ymin = std::min(ymin, std::min(s[1], s[3])); ymax = std::max(ymax, std::max(s[1], s[3]));
  }
  const float span = std::max(xmax - xmin, ymax - ymin);
  float cell = cell_size > 0.0f ? cell_size : 8.0f;
  // keep the grid small enough for shared memory: at most 64 x 64 cells over the box grown by one cell (the dilation)
  while (span / cell > 62.0f) cell *= 2.0f;
  // reach of the dilated lists: the largest bounding radius of the type table (as the kernel inflates it) when a table is
  // set - shorter lists in dense maps - else one cell; a participant that reaches further takes the out-of-line walk
  const float dil = reach > 0.0f ? std::min(cell, reach * 1.0002f + 2e-3f) : cell;
  const float margin = 1e-3f * std::max(1.0f, std::max(std::fabs(xmin) + std::fabs(xmax), std::fabs(ymin) + std::fabs(ymax)) * 1e-3f);
  const float x0 = xmin - dil - margin, y0 = ymin - dil - margin;
  const int gx = std::max(1, (int)std::floor((xmax + dil + margin - x0) / cell) + 1);
  const int gy = std::max(1, (int)std::floor((ymax + dil + margin - y0) / cell) + 1);
  const float inv = 1.0f / cell;
  // cells[c] lists (ascending) the segments that pass within `grow` of cell c's box (conservatively: the segment's line
  // against the box grown by `grow` on every side)
  auto bin_segments = [&](float grow) {
    std::vector<std::vector<uint16_t>> cells((size_t)gx * gy);
    for (int i = 0; i < n_seg; ++i) {
      const float* s = segments + 4 * i;
      const float g = grow + margin;
      const float sx0 = std::min(s[0], s[2]) - g, sx1 = std::max(s[0], s[2]) + g;
      const float sy0 = std::min(s[1], s[3]) - g, sy1 = std::max(s[1], s[3]) + g;
      int cx0 = std::max(0, (int)std::floor((sx0 - x0) * inv)), cx1 = std::min(gx - 1, (int)std::floor((sx1 - x0) * inv));
      int cy0 = std::max(0, (int)std::floor((sy0 - y0) * inv)), cy1 = std::min(gy - 1, (int)std::floor((sy1 - y0) * inv));
      for (int cy = cy0; cy <= cy1; ++cy)
        for (int cx = cx0; cx <= cx1; ++cx) {
          // exact-enough cull: does the segment's line pass within the grown cell box?
          const float bx0 = x0 + cx * cell - g, bx1 = x0 + (cx + 1) * cell + g;
          const float by0 = y0 + cy * cell - g, by1 = y0 + (cy + 1) * cell + g;
          const double dx = (double)s[2] - s[0], dy = (double)s[3] - s[1];
          const double hx = 0.5 * ((double)bx1 - bx0), hy = 0.5 * ((double)by1 - by0);
          const double mx = 0.5 * ((double)bx1 + bx0), my = 0.5 * ((double)by1 + by0);
          const double cr = std::fabs(((double)s[0] - mx) * dy - ((double)s[1] - my) * dx);
          if (cr > hx * std::fabs(dy) + hy * std::fabs(dx) + 1e-6 * (std::fabs(dx) + std::fabs(dy) + 1.0)) continue;
          cells[(size_t)cy * gx + cx].push_back((uint16_t)i);
        }
    }
    return cells;
  };
  const std::vector<std::vector<uint16_t>> cells = bin_segments(0.0f);
  // the dilated lists serve participants with reach r <= dil from the cell under their centre: every segment within r
  // of the centre is within dil of that cell's box (+ a 0.1 % + 1 mm guard for the fp32 cell index)
  const std::vector<std::vector<uint16_t>> dcells = bin_segments(dil * 1.001f + 1e-3f);
  size_t n_items = 0, n_ditems = 0;
  for (auto& v : cells) n_items += v.size();
  for (auto& v : dcells) n_ditems += v.size();
  int fine = 4;   // bounded host work: cells x segments <= ~1e8 distance evaluations
  while (fine > 1 && (double)gx * gy * fine * fine * n_seg > 1e8) fine >>= 1;
  mh.gx = gx; mh.gy = gy; mh.n_items = (int)n_items; mh.n_ditems = (int)n_ditems; mh.fine = fine;
  mh.x0 = x0; mh.y0 = y0; mh.inv_cell = inv; mh.cell = cell; mh.dil = dil;
  auto up16 = [](size_t v) { return (v + 15) / 16 * 16; };
  mh.off_seg = (uint32_t)up16(sizeof(MapHeader));
  mh.off_cell = (uint32_t)up16(mh.off_seg + (size_t)n_seg * 16);
  mh.off_items = (uint32_t)up16(mh.off_cell + ((size_t)gx * gy + 1) * 4);
  mh.off_dcell = (uint32_t)up16(mh.off_items + n_items * 2);
  mh.off_ditems = (uint32_t)up16(mh.off_dcell + ((size_t)gx * gy + 1) * 4);
  mh.off_objfirst = (uint32_t)up16(mh.off_ditems + n_ditems * 2);
  mh.off_poly = (uint32_t)up16(mh.off_objfirst + (size_t)n_seg * 2);
  mh.off_pbox = (uint32_t)up16(mh.off_poly + ((size_t)t.n_poly + 1) * 4);
  mh.off_clear = (uint32_t)up16(mh.off_pbox + (size_t)t.n_poly * 16);
  mh.off_fine = (uint32_t)up16(mh.off_clear + (size_t)gx * gy * 4);
  mh.smem_bytes = mh.off_fine;   // the fine field is read through L1 / L2, everything in front of it may be staged
  mh.total_bytes = (uint32_t)up16(mh.off_fine + (size_t)gx * fine * gy * fine);
  blob.assign(mh.total_bytes, 0);
  memcpy(blob.data(), &mh, sizeof(mh));
  memcpy(blob.data() + mh.off_seg, segments, (size_t)n_seg * 16);
  auto write_lists = [&](const std::vector<std::vector<uint16_t>>& lists, uint32_t off_start, uint32_t off_items) {
    uint32_t* cs = reinterpret_cast<uint32_t*>(blob.data() + off_start);
    uint16_t* it = reinterpret_cast<uint16_t*>(blob.data() + off_items);
    uint32_t acc = 0;
    for (size_t ci = 0; ci < lists.size(); ++ci) {
      cs[ci] = acc;
      for (uint16_t sg : lists[ci]) it[acc++] = sg;
    }
    cs[lists.size()] = acc;
  };
  write_lists(cells, mh.off_cell, mh.off_items);
  write_lists(dcells, mh.off_dcell, mh.off_ditems);
  // the object a segment belongs to, named by the object's first segment: an open polyline piece is its own object, the
  // edges of a polygon share the polygon's first edge (StaticCollision.update reports the first OBJECT hit, collision.py:37-43)
  uint16_t* objfirst = reinterpret_cast<uint16_t*>(blob.data() + mh.off_objfirst);
  for (int i = 0; i < n_seg; ++i) objfirst[i] = (uint16_t)i;
  int32_t* pstart = reinterpret_cast<int32_t*>(blob.data() + mh.off_poly);
  float* pbox = reinterpret_cast<float*>(blob.data() + mh.off_pbox);
  for (int p = 0; p < t.n_poly; ++p) {
    const int s0 = t.poly_start[p], s1 = t.poly_start[p + 1];
    pstart[p] = s0;
    float bx0 = INFINITY, bx1 = -INFINITY, by0 = INFINITY, by1 = -INFINITY;
    for (int i = s0; i < s1; ++i) {
      objfirst[i] = (uint16_t)s0;
      bx0 = std::min(bx0, segments[4 * i]); bx1 = std::max(bx1, segments[4 * i]);
      by0 = std::min(by0, segments[4 * i + 1]); by1 = std::max(by1, segments[4 * i + 1]);
    }
    pbox[4 * p] = bx0; pbox[4 * p + 1] = bx1; pbox[4 * p + 2] = by0; pbox[4 * p + 3] = by1;
  }
  pstart[t.n_poly] = t.n_poly > 0 ? t.poly_start[t.n_poly] : 0;
  // clearance fields: lower bound of the distance from any point of a cell to the nearest segment
  // (distance from the cell centre minus the half diagonal); ZERO inside a polygon - a pose deep inside an obstacle
  // touches no edge but intersects the Area all the same.  Coarse (float per cell) and fine (bytes of CLEAR_QUANT metres,
  // fine x fine per coarse cell, read through L1 / L2).
  auto centre_dist = [&](double px, double py) {
    for (int p = 0; p < t.n_poly; ++p)
      if (px >= pbox[4 * p] && px <= pbox[4 * p + 1] && py >= pbox[4 * p + 2] && py <= pbox[4 * p + 3] &&
          point_in_ring(segments, t.poly_start[p], t.poly_start[p + 1], px, py))
        return 0.0;
    double best = INFINITY;
    for (int i = 0; i < n_seg; ++i) {
      const float* sg = segments + 4 * i;
      const double dx = (double)sg[2] - sg[0], dy = (double)sg[3] - sg[1], ux = px - sg[0], uy = py - sg[1];
      const double dd = dx * dx + dy * dy;
      double tt = dd > 0.0 ? (ux * dx + uy * dy) / dd : 0.0;
      tt = std::min(1.0, std::max(0.0, tt));
      const double ex = ux - tt * dx, ey = uy - tt * dy;
      best = std::min(best, ex * ex + ey * ey);
    }
    return std::sqrt(best);
  };
  float* clr = reinterpret_cast<float*>(blob.data() + mh.off_clear);
  {
    const double half_diag = 0.5 * std::sqrt(2.0) * (double)cell * 1.0001 + 2.0 * margin;
    for (int cy = 0; cy < gy; ++cy)
      for (int cx = 0; cx < gx; ++cx) {
        const double d = centre_dist((double)x0 + (cx + 0.5) * (double)cell, (double)y0 + (cy + 0.5) * (double)cell) - half_diag;
        clr[(size_t)cy * gx + cx] = d > 0.0 ? (float)(d * 0.9999) : 0.0f;
      }
  }
  uint8_t* fine_field = blob.data() + mh.off_fine;
  {
    const double fc = (double)cell / fine;
    const double half_diag = 0.5 * std::sqrt(2.0) * fc * 1.001 + 2.0 * margin + 1e-3 * fc;
    for (int iy = 0; iy < gy * fine; ++iy)
      for (int ix = 0; ix < gx * fine; ++ix) {
        const double d = centre_dist((double)x0 + (ix + 0.5) * fc, (double)y0 + (iy + 0.5) * fc) - half_diag;
        const double q = std::floor(std::max(0.0, d) / CLEAR_QUANT);
        fine_field[(size_t)iy * gx * fine + ix] = (uint8_t)std::min(255.0, q);
      }
  }
  return T2D_OK;
}

int t2d_set_map_table(t2d_ctx* c, const t2d_map_tile* tiles, int n_tiles, const uint16_t* tile_id, float cell_size) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (n_tiles < 0 || n_tiles > T2D_MAX_TILES) return fail(T2D_E_INVALID, "n_tiles must be in 0..T2D_MAX_TILES");
  if (n_tiles > 0 && !tiles) return fail(T2D_E_INVALID, "tiles is NULL");
  if (n_tiles > 1 && !tile_id) return fail(T2D_E_INVALID, "tile_id is NULL (needed with more than one tile)");
  DeviceMap m;
  std::vector<unsigned char> all;
  std::vector<uint32_t> offs((size_t)n_tiles);
  for (int i = 0; i < n_tiles; ++i) {
    TileIn t{tiles[i].segments, tiles[i].n_seg, tiles[i].poly_start, tiles[i].n_poly, tiles[i].bounds};
    std::vector<unsigned char> blob;
    if (int r = build_tile(t, cell_size, c->rb_max, blob)) return r;
    offs[i] = (uint32_t)all.size();
    all.insert(all.end(), blob.begin(), blob.end());
    all.resize((all.size() + 127) / 128 * 128, 0);   // every tile starts 128-byte aligned
    m.has_bounds = m.has_bounds || tiles[i].bounds != nullptr;
    m.has_segments = m.has_segments || tiles[i].n_seg > 0;
    m.tile_nseg.push_back(tiles[i].n_seg);
    if (i == 0) memcpy(&m.mh, blob.data(), sizeof(MapHeader));
  }
  CUDA_TRY(cudaSetDevice(c->device));
  if (n_tiles > 0) {
    if (int r = upload(m.blob, all.data(), all.size())) return r;
    if (int r = upload(m.tile_off, offs.data(), offs.size())) return r;
  }
  m.n_tiles = n_tiles;
  m.tile_id = n_tiles > 1 ? tile_id : nullptr;
  m.smem_bytes = (int)m.mh.smem_bytes;   // what a single tile stages into shared memory
  c->map = std::move(m);
  return T2D_OK;
}

int t2d_set_map_polygons(t2d_ctx* c, const float* segments, int n_seg, const int32_t* poly_start, int n_poly, const float* bounds,
                         float cell_size) {
  if (n_seg == 0 && !bounds) return t2d_set_map_table(c, nullptr, 0, nullptr, cell_size);
  t2d_map_tile t{};
  t.segments = segments; t.n_seg = n_seg; t.poly_start = poly_start; t.n_poly = n_poly; t.bounds = bounds;
  return t2d_set_map_table(c, &t, 1, nullptr, cell_size);
}

int t2d_set_map(t2d_ctx* c, const float* segments, int n_seg, const float* bounds, float cell_size) {
  return t2d_set_map_polygons(c, segments, n_seg, nullptr, 0, bounds, cell_size);
}

int t2d_bind_state(t2d_ctx* c, float* x, float* y, float* heading, float* speed, float* vx, float* vy,
                   const uint8_t* type_id, int32_t* step_count) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (!x || !y || !heading || !speed || !vx || !vy || !type_id || !step_count)
    return fail(T2D_E_INVALID, "t2d_bind_state: NULL array");
  c->x = x; c->y = y; c->h = heading; c->v = speed; c->vx = vx; c->vy = vy;
  c->type_id = type_id; c->step_count = step_count;
  return T2D_OK;
}

int t2d_bind_wheel_state(t2d_ctx* c, float* omega_front, float* omega_rear) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if ((omega_front == nullptr) != (omega_rear == nullptr)) return fail(T2D_E_INVALID, "t2d_bind_wheel_state: one array is NULL");
  c->wheel_f = omega_front; c->wheel_r = omega_rear;
  return T2D_OK;
}

int t2d_bind_reset_wheel_pool(t2d_ctx* c, const float* pool_omega_front, const float* pool_omega_rear) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if ((pool_omega_front == nullptr) != (pool_omega_rear == nullptr)) return fail(T2D_E_INVALID, "t2d_bind_reset_wheel_pool: one array is NULL");
  c->reset_pool_wf = pool_omega_front; c->reset_pool_wr = pool_omega_rear;
  return T2D_OK;
}

// t2d_set_log (row_track, slot_off == nullptr) and t2d_set_log_schedule: validate everything, then replace the bound log.
// A row_track binding becomes a schedule of at most one entry per slot.
static int set_log(t2d_ctx* c, const t2d_log* L, const char* who, const int32_t* slot_off, const int32_t* slot_track,
                   int n_entries, int32_t* track_out) {
  const std::string fn = who;
  if (int r = require(c, NEED_STATE | NEED_TABLE)) return r;
  if (L->n_tracks <= 0 || L->n_rows <= 0) return fail(T2D_E_INVALID, fn + ": n_tracks and n_rows must be >= 1");
  if (!L->first_ms || !L->n_frames || !L->period_ms || !L->type_row || !L->records || !L->t0_ms || !L->log_row || !L->type_id)
    return fail(T2D_E_INVALID, fn + ": NULL array");
  if (slot_off == nullptr && !L->row_track) return fail(T2D_E_INVALID, fn + ": NULL array");
  if (slot_off != nullptr && L->row_track) return fail(T2D_E_INVALID, fn + ": row_track must be NULL (the schedule binds the slots)");
  if (L->type_id != c->type_id)
    return fail(T2D_E_INVALID, fn + ": type_id is not the array bound with t2d_bind_state");
  const int K = L->n_tracks, M = c->M;
  const long long PM = (long long)L->n_rows * M;
  std::vector<ReplayTrack> tracks((size_t)K);
  std::vector<long long> last((size_t)K);
  long long n_rec = 0;
  for (int k = 0; k < K; ++k) {
    if (L->period_ms[k] <= 0) return fail(T2D_E_INVALID, fn + ": track " + std::to_string(k) + ": period_ms must be > 0");
    if (L->n_frames[k] < 1) return fail(T2D_E_INVALID, fn + ": track " + std::to_string(k) + ": no frames");
    const int row = L->type_row[k];
    if (row >= c->n_types) return fail(T2D_E_INVALID, fn + ": track " + std::to_string(k) + ": type_row outside the type table");
    if (c->type_model[row] != T2D_MODEL_STATIC)
      return fail(T2D_E_INVALID, fn + ": track " + std::to_string(k) + ": type_row is not a T2D_MODEL_STATIC row");
    tracks[k] = ReplayTrack{L->first_ms[k], L->period_ms[k], L->n_frames[k], (int32_t)n_rec};
    last[k] = (long long)L->first_ms[k] + (long long)(L->n_frames[k] - 1) * L->period_ms[k];
    n_rec += L->n_frames[k];
    if (n_rec > INT32_MAX / 5) return fail(T2D_E_UNSUPPORTED, fn + ": too many records");
  }
  for (long long i = 0; i < 5 * n_rec; ++i)
    if (!std::isfinite(L->records[i])) return fail(T2D_E_INVALID, fn + ": record " + std::to_string(i / 5) + " is not finite");
  std::vector<int32_t> off((size_t)PM + 1, 0);
  std::vector<ReplayEntry> entries;
  std::vector<int> seen((size_t)K, -1);
  if (slot_off == nullptr) {
    for (int p = 0; p < L->n_rows; ++p)
      for (int m = 0; m < M; ++m) {
        const long long s = (long long)p * M + m;
        const int k = L->row_track[s];
        if (k < -1 || k >= K) return fail(T2D_E_INVALID, fn + ": row_track entry outside [-1, n_tracks)");
        if (k >= 0) {
          if (seen[k] == p) return fail(T2D_E_INVALID, fn + ": track " + std::to_string(k) + " bound twice in row " + std::to_string(p));
          seen[k] = p;
          // a slot's final entry is never probed: its last stamp only has to be an int32, not exact
          entries.push_back(ReplayEntry{(int32_t)std::min<long long>(last[k], INT32_MAX), k});
        }
        off[s + 1] = (int32_t)entries.size();
      }
  } else {
    if (!slot_track && n_entries > 0) return fail(T2D_E_INVALID, fn + ": NULL array");
    if (n_entries < 0) return fail(T2D_E_INVALID, fn + ": n_entries must be >= 0");
    if (slot_off[0] != 0 || slot_off[PM] != n_entries)
      return fail(T2D_E_INVALID, fn + ": slot_off must run from 0 to n_entries");
    for (long long s = 0; s < PM; ++s)
      if (slot_off[s + 1] < slot_off[s]) return fail(T2D_E_INVALID, fn + ": slot_off is not monotone at slot " + std::to_string(s));
    entries.resize((size_t)n_entries);
    for (int p = 0; p < L->n_rows; ++p)
      for (int m = 0; m < M; ++m) {
        const long long s = (long long)p * M + m;
        for (int e = slot_off[s]; e < slot_off[s + 1]; ++e) {
          const int k = slot_track[e];
          const std::string at = fn + ": row " + std::to_string(p) + " slot " + std::to_string(m) + ": ";
          if (k < 0 || k >= K) return fail(T2D_E_INVALID, at + "slot_track entry outside [0, n_tracks)");
          if (seen[k] == p) return fail(T2D_E_INVALID, at + "track " + std::to_string(k) + " scheduled twice in the row");
          seen[k] = p;
          if (e > slot_off[s] && (long long)L->first_ms[k] <= last[slot_track[e - 1]])
            return fail(T2D_E_INVALID, at + "track " + std::to_string(k) + " does not start after the previous entry ends");
          if (last[k] > INT32_MAX) return fail(T2D_E_UNSUPPORTED, at + "track " + std::to_string(k) + ": last stamp exceeds int32 ms");
          entries[e] = ReplayEntry{(int32_t)last[k], k};
        }
      }
    std::copy(slot_off, slot_off + PM + 1, off.begin());
  }
  // at most one entry per slot (every row_track binding): the slots' tracks as one array, no search
  bool single = true;
  for (long long s = 0; s < PM && single; ++s) single = off[s + 1] - off[s] <= 1;
  CUDA_TRY(cudaSetDevice(c->device));
  auto g = std::make_unique<DeviceLog>();
  if (single) {
    std::vector<int32_t> one((size_t)PM, -1);
    for (long long s = 0; s < PM; ++s)
      if (off[s + 1] > off[s]) one[s] = entries[off[s]].track;
    if (int r = upload(g->slot_track1, one.data(), one.size())) return r;
  } else {
    if (int r = upload(g->slot_off, off.data(), off.size())) return r;
    if (int r = upload(g->entries, entries.data(), entries.size())) return r;
  }
  if (int r = upload(g->tracks, tracks.data(), tracks.size())) return r;
  if (int r = upload(g->track_type, L->type_row, (size_t)K)) return r;
  if (int r = upload(g->rec, L->records, 5 * (size_t)n_rec)) return r;
  if (int r = upload(g->t0, L->t0_ms, (size_t)L->n_rows)) return r;
  g->track_type_host.assign(L->type_row, L->type_row + K);
  g->n_tracks = K; g->n_rows = L->n_rows;
  g->row = L->log_row; g->type_id = L->type_id; g->track_out = track_out;
  if (c->hist) {   // the ring's tracks restart with the log (a rejected call keeps both as they were)
    DeviceHistory tracks;
    tracks.H = c->hist->H;
    if (int r = history_tracks(c, tracks, track_out)) return r;
    c->hist->track = std::move(tracks.track);
  }
  c->log = std::move(g);
  drop_traffic(c, NEED_LOG);
  return T2D_OK;
}

int t2d_set_log(t2d_ctx* c, const t2d_log* L) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (!L) {
    CUDA_TRY(cudaSetDevice(c->device));
    c->log.reset();
    drop_traffic(c, NEED_LOG);
    if (c->hist) c->hist->track.reset();
    return T2D_OK;
  }
  return set_log(c, L, "t2d_set_log", nullptr, nullptr, 0, nullptr);
}

int t2d_set_log_schedule(t2d_ctx* c, const t2d_log* L, const int32_t* slot_off, const int32_t* slot_track, int32_t n_entries,
                         int32_t* track_out) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (!L || !slot_off) return fail(T2D_E_INVALID, "t2d_set_log_schedule: log / slot_off is NULL (t2d_set_log(ctx, NULL) unbinds)");
  return set_log(c, L, "t2d_set_log_schedule", slot_off, slot_track, n_entries, track_out);
}

// K7 over the scenarios [first, first + count): tick mode (mask == nullptr, offset 1) or reset mode (the masked scenarios
// take row pool_index[n] / n, offset 0).
static int launch_replay(t2d_ctx* c, void* stream, int first, int count, int offset, const uint8_t* mask, const int32_t* pool_index) {
  const DeviceLog& g = *c->log;
  if (g.type_id != c->type_id) return fail(T2D_E_STATE, "state rebound after t2d_set_log: call t2d_set_log again");
  const size_t p0 = (size_t)first * c->M;
  ReplayArgs R{};
  R.x = c->x + p0; R.y = c->y + p0; R.h = c->h + p0; R.v = c->v + p0; R.vx = c->vx + p0; R.vy = c->vy + p0;
  R.type_id = g.type_id + p0;
  R.step_count = c->step_count + first;
  R.log_row = g.row + first;
  R.mask = mask ? mask + first : nullptr;
  R.pool_index = pool_index ? pool_index + first : nullptr;
  R.log_row_out = mask ? g.row + first : nullptr;
  R.tracks = g.tracks.get(); R.track_type = g.track_type.get(); R.rec = g.rec.get();
  R.t0 = g.t0.get(); R.slot_off = g.slot_off.get(); R.entries = g.entries.get(); R.slot_track1 = g.slot_track1.get();
  R.track_out = g.track_out ? g.track_out + p0 : nullptr;
  R.N = count; R.M = c->M; R.n_rows = g.n_rows; R.offset = offset; R.interval_ms = c->cfg.interval_ms;
  const int grid = capped_grid((long long)count * c->M, 256, c->sm_count, 8);
  if (c->reactive) {   // the reactive instance: handovers to K5, and the driving rows after them
    const ReactiveReplay& rr = *c->reactive;
    ReactiveReplayArgs X{};
    static_cast<ReplayArgs&>(X) = R;
    X.track_path = rr.track_path.get(); X.drive_row = rr.drive_row.get(); X.desired_speed = rr.desired_speed.get();
    X.drive_path = rr.drive_path + p0; X.slot_desired_speed = rr.slot_desired_speed + p0;
    X.pid_state = c->pid_state ? c->pid_state + 6 * p0 : nullptr;
    X.last_accel = c->ctrl_last_accel ? c->ctrl_last_accel + p0 : nullptr;
    t2d_reactive_replay_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(X);
    return launched();
  }
  t2d_replay_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(R);
  return launched();
}

// Warps per CTA of the tick.  One wave (the usual case: every warp tile is resident at once and the kernel's duration is
// one tile's lifetime): the SM with the most warps sets the pace, and every CTA costs a launch + prologue (barrier
// init, TMA staging), weighed below as 0.42 of a warp on the fullest SM (1-warp CTAs are not considered: the prologue
// is paid per warp there).  Several waves: persistent CTAs of the largest size.  On an H100 (132 SMs) 4096 x 64 is 2048 warp
// tiles, more than the conservative 132 x 14, so it takes 8-warp CTAs; at the launch bounds' 2 CTAs per SM all 256 of them are
// resident at once anyway (one wave).  On an H100 80GB HBM3 SXM at a 400 W power limit (T2D_WPC, 40000 timed steps) 8 and 4 warps
// per CTA measured within 2 % of each other and 2 warps per CTA about 45 % slower.
static int pick_wpc(long long tiles, int sm_count) {
  const int resident_warps = 14;   // per SM at the kernel's register budget, rounded down to what every variant reaches
  if (tiles > (long long)sm_count * resident_warps) return MAX_WARPS_PER_CTA;
  int best = 2;
  double best_cost = 1e30;
  for (int w = 2; w <= MAX_WARPS_PER_CTA; ++w) {
    const long long ctas = (tiles + w - 1) / w;
    const long long per_sm = (ctas + sm_count - 1) / sm_count;
    const double cost = (double)(per_sm * w) + 0.42 * (double)per_sm;
    if (cost < best_cost - 1e-9 || (cost < best_cost + 1e-9 && w > best)) { best_cost = cost; best = w; }
  }
  return best;
}

// Launches K1 over the scenarios [first, first + count) of the bound state with the ego action `ego` (nullptr: row 0 of
// `action`); the per-participant / per-scenario pointers passed in (action, flags, ..., done) address scenario `first`
// already, `ego` scenario 0.
static int launch_step(t2d_ctx* c, const float* action, const float* ego, uint8_t* flags, int16_t* hit_index, int16_t* hit_segment,
                       uint8_t* scn_status, uint8_t* done, void* stream, int do_physics, int first = 0, int count = -1) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (int r = require(c, NEED_STATE | NEED_TABLE)) return r;
  if (do_physics && !action) return fail(T2D_E_INVALID, "action is NULL");
  if (do_physics)
    if (int r = require(c, NEED_TICK)) return r;
  CUDA_TRY(cudaSetDevice(c->device));
  if (count < 0) count = c->N - first;
  if (first < 0 || count <= 0 || first + count > c->N) return fail(T2D_E_INVALID, "scenario range out of bounds");
  const DeviceMap& map = c->map;
  const size_t p0 = (size_t)first * c->M;
  StepArgs A{};
  A.x = c->x + p0; A.y = c->y + p0; A.h = c->h + p0; A.v = c->v + p0; A.vx = c->vx + p0; A.vy = c->vy + p0;
  A.type_id = c->type_id + p0; A.step_count = c->step_count + first;
  A.wheel_f = c->wheel_f ? c->wheel_f + p0 : nullptr; A.wheel_r = c->wheel_r ? c->wheel_r + p0 : nullptr;
  A.action = action; A.ego_action = ego ? ego + 2 * (size_t)first : nullptr; A.flags = flags; A.hit_index = hit_index; A.hit_segment = hit_segment;
  A.scn_status = scn_status; A.done = done;
  A.order = c->order.get() + (size_t)first * FIX_M;
  A.order_fallbacks = g_order_fallbacks[c->device % 64];
  const bool map_table = map.n_tiles > 1;
  const MapArgs mp = map_args(map, first);
  A.map_blob = mp.map_blob; A.tile_off = mp.tile_off; A.tile_id = mp.tile_id; A.map_bytes = map.smem_bytes; A.mh = map.mh;
  A.map_in_smem = (!map_table && map.blob && map.mh.n_seg > 0 && map.smem_bytes <= MAP_SMEM_LIMIT) ? 1 : 0;
  A.table = c->d_table.get(); A.n_types = c->n_types;
  A.N = count; A.M = c->M; A.G = c->G;
  set_time_step(A, c->cfg.interval_ms, c->cfg.delta_t_ms);
  A.max_step = c->cfg.max_step; A.cfg_flags = c->cfg.flags;
  // the boundary box: tile 0's (with a map table every lane reads its own tile's)
  A.do_physics = do_physics; A.has_bounds = map.has_bounds ? 1 : 0;
  A.bxmin = map.mh.bxmin; A.bxmax = map.mh.bxmax; A.bymin = map.mh.bymin; A.bymax = map.mh.bymax;
  A.prefetch = c->prefetch_override >= 0 ? c->prefetch_override : (g_exchanges_alive.load() == 0 ? 1 : 0);
  // (drift / replay: K1 passes the pre-pass's vx, vy through)
  A.needs_vel_in = (c->has_pointmass || c->has_drift || (do_physics && c->log)) ? 1 : 0;
  bool vec = (c->M % PPL == 0) && aligned16(A.x) && aligned16(A.y) && aligned16(A.h) && aligned16(A.v) && aligned16(A.vx) &&
             aligned16(A.vy) && aligned4(A.type_id) && aligned16(action) && aligned4(flags) && aligned8(hit_index) &&
             aligned8(hit_segment);
  A.vec_ok = vec ? 1 : 0;

  A.rb_max = c->rb_max;
  A.goal = c->goal;
  if (A.goal.target) {   // the rows from `first` on (t2d_set_goal binds the three outputs with every target)
    A.goal.target += 5 * (size_t)first; A.goal.iou += first; A.goal.last_pose += 4 * (size_t)first; A.goal.noact_count += first;
  }
  const int table_bytes = (((c->n_types + 1) * (int)sizeof(Params) + 15) / 16) * 16;   // + the neutral row
  const int spw = 32 / c->G;
  const long long tiles = ((long long)count + spw - 1) / spw;
  int wpc = pick_wpc(tiles, c->sm_count);
  if (c->wpc_override > 0) wpc = c->wpc_override;   // T2D_WPC (experiments), read once at t2d_create
  {
    int off = (A.map_in_smem ? A.map_bytes : 0) + table_bytes;
    A.off_poseA = off; off += wpc * POSE_PER_WARP * (int)sizeof(float4);
    A.off_poseB = off; off += wpc * POSE_PER_WARP * (int)sizeof(float4);
    A.off_hit = off; off += wpc * POSE_PER_WARP * (int)sizeof(int);
    A.off_queue = off; off += wpc * QCAP * 4;
    A.off_sorted = off; off += wpc * POSE_PER_WARP * (int)sizeof(float4);
    A.off_qcount = off; off += ((wpc + 3) & ~3) * 4;
    A.off_bar = off; off += 16;
    A.wpc = wpc;
    A.table_bytes = table_bytes;
    A.n_tiles = (int)tiles;
    A.g_shift = 0;
    while ((1 << A.g_shift) < c->G) ++A.g_shift;
    const int MP = c->G * PPL;
    A.mp_shift = 0;
    while ((1 << A.mp_shift) < MP) ++A.mp_shift;
  }
  const int smem = A.off_bar + 16;
  if (smem > c->max_smem_optin) return fail(T2D_E_UNSUPPORTED, "shared memory budget exceeded");
  using kernel_t = void (*)(StepArgs);
  kernel_t kern;
  // the C2-shaped instance exactly when this tick has the shape it is compiled for (FIX_M ...)
  const bool fixed = c->kin_only && !c->tick_generic && c->M == FIX_M && c->G == FIX_G && do_physics && A.vec_ok &&
                     !A.needs_vel_in && A.ego_action == nullptr && A.goal.target == nullptr;
  if (fixed) kern = map_table ? (kernel_t)t2d_step_kernel<true, true, true> : (kernel_t)t2d_step_kernel<true, false, true>;
  else if (c->kin_only) kern = map_table ? (kernel_t)t2d_step_kernel<true, true, false> : (kernel_t)t2d_step_kernel<true, false, false>;
  else kern = map_table ? (kernel_t)t2d_step_kernel<false, true, false> : (kernel_t)t2d_step_kernel<false, false, false>;
  const int variant = (fixed ? 4 : c->kin_only ? 2 : 0) + (map_table ? 1 : 0);
  {
    // cudaFuncSetAttribute applies to the kernel function for the whole process and SETS the value: worlds of
    // different sizes share it, so the opt-in is tracked per (device, kernel variant) and only ever raised.
    std::lock_guard<std::mutex> lock(g_smem_mutex);
    int& configured = g_smem_configured[c->device % 64][variant];
    if (smem > configured) {
      CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
      configured = smem;
    }
  }
  if (do_physics && c->log)
    if (int r = launch_replay(c, stream, first, count, 1, nullptr, nullptr)) return r;
  if (do_physics && c->has_drift) {
    t2d_drift_kernel<<<capped_grid((long long)count * c->M, 128, c->sm_count, 16), 128, 0, (cudaStream_t)stream>>>(A);
    if (int r = launched()) return r;
  }
  const long long ctas_needed = (tiles + wpc - 1) / wpc;
  if (c->occ_smem[wpc] != smem || c->occ_variant[wpc] != variant) {
    int per_sm = 1;
    CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, wpc * 32, smem));
    c->occ_val[wpc] = per_sm < 1 ? 1 : per_sm;
    c->occ_smem[wpc] = smem;
    c->occ_variant[wpc] = variant;
  }
  int per_sm_ctas = c->occ_val[wpc];
  if (c->grid_limit > 0) per_sm_ctas = std::min(per_sm_ctas, c->grid_limit);   // T2D_GRID_LIMIT: leave CTA slots to other streams
  const long long resident = (long long)c->sm_count * per_sm_ctas;
  const int grid = (int)std::max(1LL, std::min(ctas_needed, resident));
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((unsigned)grid);
  cfg.blockDim = dim3((unsigned)(wpc * 32));
  cfg.dynamicSmemBytes = (size_t)smem;
  cfg.stream = (cudaStream_t)stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = c->use_pdl ? 1 : 0;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  CUDA_TRY(cudaLaunchKernelEx(&cfg, kern, A));
  if (int r = launched()) return r;
  g_tick_instances[variant].fetch_add(1);
  if (!map_table && map.blob && map.mh.n_seg > 0 && !A.map_in_smem) g_tick_instances[6].fetch_add(1);
  return T2D_OK;
}

// K5 with the ego action `ego` (nullptr: row 0 of `action`)
// A call K5 could not complete is refused before anything is launched: PID rows without their state or target.
static int check_pid_binding(const t2d_ctx* c) {
  if (!c->ctrl_has_pid) return T2D_OK;
  if (!c->pid_state) return fail(T2D_E_INVALID, "a PID controller row is bound without its state: call t2d_set_pid first");
  if (c->ctrl_pid_reads_target && !c->pid_target)
    return fail(T2D_E_INVALID, "a PID controller row reads the target, and none is bound: call t2d_set_pid with one");
  return T2D_OK;
}

// ---- leader search (t2d_set_leader_search / t2d_find_leaders; K17)
static int check_leader_args(const char* fn, double half_width, double max_range, const int16_t* lead, const float* gap) {
  if (!(std::isfinite(half_width) && half_width > 0.0 && half_width <= 100.0))
    return fail(T2D_E_INVALID, std::string(fn) + ": half_width must be finite and in (0, 100] m");
  if (!(std::isfinite(max_range) && max_range > 0.0 && max_range <= 1.0e5))
    return fail(T2D_E_INVALID, std::string(fn) + ": max_range must be finite and in (0, 1e5] m");
  if (!aligned2(lead) || !aligned4(gap))
    return fail(T2D_E_INVALID, std::string(fn) + ": lead must be 2-byte and gap 4-byte aligned");
  return T2D_OK;
}

// The slots' current paths: a bound reactive replay's drive_path, a bound lane change's lane_path (never both), else the
// controllers' path_id
static const int16_t* current_path(const t2d_ctx* c) {
  return c->reactive ? c->reactive->drive_path : c->lane ? c->lane->lane_path : c->ctrl_path;
}

// K17 on the bound state and the controllers' paths; the caller has checked the arguments and the bindings
static int launch_leaders(t2d_ctx* c, double half_width, double max_range, int16_t* lead, float* gap, void* stream) {
  CUDA_TRY(cudaSetDevice(c->device));
  leader::Args A{world_args(c)};
  A.path_id = current_path(c); A.paths = path_table(c);
  A.half_width = half_width; A.max_range = max_range; A.lead = lead; A.gap = gap;
  leader::t2d_leader_kernel<<<(c->N + leader::WARPS - 1) / leader::WARPS, leader::WARPS * 32, 0, (cudaStream_t)stream>>>(A);
  return launched();
}

// K18 on the bound state with the bound lane change and search; the caller has checked the bindings
static int launch_lane_change(t2d_ctx* c, void* stream) {
  const LaneChange& L = *c->lane;
  lane::Args A{world_args(c)};
  A.ctab = c->d_ctab.get(); A.n_ctrl = c->n_ctrl; A.ctrl_id = c->ctrl_id; A.paths = path_table(c);
  A.left = L.left.get(); A.right = L.right.get();
  A.half_width = c->leader_half_width; A.max_range = c->leader_max_range;
  A.politeness = L.p.politeness; A.threshold = L.p.threshold; A.b_safe = L.p.b_safe; A.min_gap = L.p.min_gap;
  A.cooldown = L.p.cooldown;
  A.lane_path = L.lane_path; A.cool = L.cooldown; A.change = L.change;
  lane::t2d_lane_change_kernel<<<(c->N + lane::WARPS - 1) / lane::WARPS, lane::WARPS * 32, 0, (cudaStream_t)stream>>>(A);
  return launched();
}

// K19 on the bound state with the bound yielding and search; the caller has checked the bindings
static int launch_yields(t2d_ctx* c, int16_t* yield_to, float* stop_gap, void* stream) {
  const Yielding& Y = *c->yield;
  CUDA_TRY(cudaSetDevice(c->device));
  yield::Args A{world_args(c)};
  A.path_id = current_path(c); A.route_id = c->route_id;
  A.ctrl_id = c->ctrl_id; A.ctab = c->d_ctab.get(); A.n_ctrl = c->n_ctrl; A.paths = path_table(c);
  A.zones = Y.zones.get(); A.zone_off = Y.zone_off.get(); A.priority = Y.priority.get();
  A.half_width = c->leader_half_width; A.max_range = c->leader_max_range;
  A.critical_gap = Y.p.critical_gap; A.two_commit_decel = 2.0 * Y.p.commit_decel; A.v_min = Y.p.v_min;
  A.yield_to = yield_to; A.stop_gap = stop_gap; A.stop_xy = Y.stop_xy.get();
  yield::t2d_yield_kernel<<<(c->N + yield::WARPS - 1) / yield::WARPS, yield::WARPS * 32, 0, (cudaStream_t)stream>>>(A);
  return launched();
}

static int launch_control(t2d_ctx* c, float* action, const float* ego, void* stream) {
  if (int r = require(c, NEED_STATE | NEED_TABLE | NEED_CTRL)) return r;
  if (int r = check_pid_binding(c)) return r;
  if (!action) return fail(T2D_E_INVALID, "action is NULL");
  if (!aligned8(action)) return fail(T2D_E_INVALID, "action must be 8-byte aligned");
  CUDA_TRY(cudaSetDevice(c->device));
  // a bound lane change decides first (it is only bound with a search), on the state K17 and K5 read next
  if (c->lane)
    if (int r = launch_lane_change(c, stream)) return r;
  // a bound search finds the leaders on the state K5 reads next, and K5 follows them instead of the controllers' lead_index
  if (c->leader_lead)
    if (int r = launch_leaders(c, c->leader_half_width, c->leader_max_range, c->leader_lead, c->leader_gap, stream)) return r;
  // bound yielding (only with a search) finds the stops on the same state, and K5 brakes for them
  if (c->yield)
    if (int r = launch_yields(c, c->yield->yield_to, c->yield->stop_gap, stream)) return r;
  CtrlArgs A{world_args(c)};
  A.ctab = c->d_ctab.get(); A.n_ctrl = c->n_ctrl; A.ctrl_id = c->ctrl_id; A.path_id = current_path(c);
  A.lead = c->leader_lead ? c->leader_lead : c->ctrl_lead; A.paths = path_table(c);
  A.last_accel = c->ctrl_last_accel; A.action = action; A.ego_action = ego;
  A.steer_first = (c->cfg.flags & T2D_CFG_STEER_FIRST) ? 1 : 0;
  A.pid_target = c->pid_target; A.pid_state = c->pid_state;
  const int warps_per_cta = 4;
  auto kern = c->ctrl_has_pid ? t2d_control_kernel<true> : t2d_control_kernel<false>;
  if (c->reactive) {   // the reactive slots' own desired speeds (only bound with a PID state)
    A.slot_desired_speed = c->reactive->slot_desired_speed;
    kern = t2d_reactive_control_kernel;
  }
  if (c->yield) {   // the stops K19 has just written (slot_desired_speed stays nullptr without a reactive replay)
    A.stop_gap = c->yield->stop_gap; A.stop_xy = c->yield->stop_xy.get();
    kern = t2d_yield_control_kernel;
  }
  kern<<<capped_grid(c->N, warps_per_cta, c->sm_count, 16), warps_per_cta * 32, 0, (cudaStream_t)stream>>>(A);
  return launched();
}

struct HostPart {   // a part of a packed read-back that goes to a caller's array (dst == nullptr: not wanted)
  void* dst;
  size_t off, bytes;
};

// Copies the first `bytes` of a packed device block to its pinned mirror, waits for the stream, and copies the parts out
static int read_back(const Mirror& m, size_t bytes, cudaStream_t s, std::initializer_list<HostPart> parts) {
  CUDA_TRY(cudaMemcpyAsync(m.host.get(), m.dev.get(), bytes, cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaStreamSynchronize(s));
  for (const HostPart& p : parts)
    if (p.dst) memcpy(p.dst, m.host.get() + p.off, p.bytes);
  return T2D_OK;
}

static int make_mirror(Mirror& out, size_t dev_bytes, size_t host_bytes) {
  Mirror m;
  if (int r = dev_alloc(m.dev, dev_bytes)) return r;
  if (int r = host_alloc(m.host, host_bytes)) return r;
  out = std::move(m);
  return T2D_OK;
}

// the [2][N] status / done block of t2d_step_host and t2d_step_host_ego
static int status_done_staging(t2d_ctx* c) {
  return c->hs_out.dev ? T2D_OK : make_mirror(c->hs_out, 2 * (size_t)c->N, 2 * (size_t)c->N);
}

int t2d_set_goal(t2d_ctx* c, const float* target, float arrival_threshold, int no_action_max_step, float* iou_out, float* last_pose,
                 int32_t* no_action_count) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (target && (!iou_out || !last_pose || !no_action_count)) return fail(T2D_E_INVALID, "t2d_set_goal: NULL output array");
  if (target && !(arrival_threshold > 0.0f && arrival_threshold <= 1.0f)) return fail(T2D_E_INVALID, "arrival_threshold must be in (0, 1]");
  c->goal = {target, iou_out, last_pose, no_action_count, arrival_threshold, no_action_max_step};
  return T2D_OK;
}

int t2d_step(t2d_ctx* c, const float* action, uint8_t* flags, int16_t* hit_index, int16_t* hit_segment, uint8_t* scn_status,
             uint8_t* done, void* stream) {
  if (int r = launch_step(c, action, c ? c->ego_action : nullptr, flags, hit_index, hit_segment, scn_status, done, stream, 1))
    return r;
  return launch_history(c, nullptr, stream);
}

int t2d_step_host(t2d_ctx* c, const float* action_host, uint8_t* flags, int16_t* hit_index, int16_t* hit_segment,
                  uint8_t* scn_status_host, uint8_t* done_host, void* stream) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (!action_host) return fail(T2D_E_INVALID, "action is NULL");
  CUDA_TRY(cudaSetDevice(c->device));
  const int N = c->N, M = c->M;
  if (!c->hs_upload) {
    auto u = std::make_unique<ChunkedUpload>();
    if (int r = dev_alloc(u->action, (size_t)N * M * 2)) return r;
    CUDA_TRY(cudaStreamCreateWithFlags(&u->copy, cudaStreamNonBlocking));
    CUDA_TRY(cudaEventCreateWithFlags(&u->begin, cudaEventDisableTiming));
    for (cudaEvent_t& e : u->chunk) CUDA_TRY(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    c->hs_upload = std::move(u);
  }
  if (int r = status_done_staging(c)) return r;
  ChunkedUpload& u = *c->hs_upload;
  uint8_t* out = c->hs_out.dev.get();
  // Chunks of whole scenarios: the copy of chunk k + 1 (copy engine, own stream) runs under the kernel of chunk k.
  // A kernel that does not fill the GPU lasts one tile's lifetime whatever the batch, so splitting a small upload only
  // adds a fixed cost per chunk; it pays once a chunk alone fills the GPU, i.e. from ~1 M participants (8 MiB of
  // actions) per chunk upwards.
  int chunks = c->host_chunks;
  if (chunks <= 0) chunks = (int)std::min<long long>(MAX_HOST_CHUNKS, std::max<long long>(1, (long long)N * M / (1 << 20)));
  int per = (N + chunks - 1) / chunks;
  per = (per + 31) & ~31;   // whole warp tiles (<= 32 scenarios per warp): a chunked tick groups lanes exactly as t2d_step does
  cudaStream_t s = (cudaStream_t)stream;
  const bool split = per < N;   // a single chunk needs no second stream
  if (split) {
    CUDA_TRY(cudaEventRecord(u.begin, s));            // the copies follow whatever the caller queued on `stream`
    CUDA_TRY(cudaStreamWaitEvent(u.copy, u.begin, 0));
  }
  int k = 0;
  for (int first = 0; first < N; first += per, ++k) {
    const int count = std::min(per, N - first);
    const size_t a0 = (size_t)first * M * 2;
    CUDA_TRY(cudaMemcpyAsync(u.action.get() + a0, action_host + a0, (size_t)count * M * 2 * sizeof(float), cudaMemcpyHostToDevice,
                             split ? u.copy : s));
    if (split) {
      CUDA_TRY(cudaEventRecord(u.chunk[k], u.copy));
      CUDA_TRY(cudaStreamWaitEvent(s, u.chunk[k], 0));
    }
    const size_t p0 = (size_t)first * M;
    if (int r = launch_step(c, u.action.get() + a0, c->ego_action, flags ? flags + p0 : nullptr, hit_index ? hit_index + p0 : nullptr,
                            hit_segment ? hit_segment + p0 : nullptr, out + first, out + N + first, stream, 1, first, count))
      return r;
  }
  if (int r = launch_history(c, nullptr, stream)) return r;   // after the last chunk
  return read_back(c->hs_out, 2 * (size_t)N, s, {{scn_status_host, 0, (size_t)N}, {done_host, (size_t)N, (size_t)N}});
}

int t2d_set_prefetch(t2d_ctx* c, int mode) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (mode < -1 || mode > 1) return fail(T2D_E_INVALID, "prefetch mode must be -1 (policy), 0 (off) or 1 (on)");
  c->prefetch_override = mode;
  return T2D_OK;
}

int t2d_set_ego_action(t2d_ctx* c, const float* ego_action) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (!aligned8(ego_action)) return fail(T2D_E_INVALID, "ego_action must be 8-byte aligned");
  c->ego_action = ego_action;
  return T2D_OK;
}

int t2d_step_host_ego(t2d_ctx* c, const float* ego_action_host, float* action, uint8_t* flags, int16_t* hit_index, int16_t* hit_segment,
                      uint8_t* scn_status_host, uint8_t* done_host, void* stream) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (!ego_action_host || !action) return fail(T2D_E_INVALID, "ego_action / action is NULL");
  CUDA_TRY(cudaSetDevice(c->device));
  const int N = c->N;
  if (!c->hs_ego.host) {
    // pinned AND mapped: the first kernel of the step reads the 8 N bytes straight from host memory (one PCIe round trip
    // inside the kernel) instead of waiting for a copy-engine transfer and the stream dependency behind it
    MappedEgo e;
    if (int r = host_alloc(e.host, (size_t)N * 2, cudaHostAllocMapped)) return r;
    float* dev = nullptr;
    CUDA_TRY(cudaHostGetDevicePointer(&dev, e.host.get(), 0));
    e.dev = dev;
    c->hs_ego = std::move(e);
  }
  if (int r = status_done_staging(c)) return r;
  if (c->d_ctab)
    if (int r = check_pid_binding(c)) return r;
  memcpy(c->hs_ego.host.get(), ego_action_host, (size_t)N * 2 * sizeof(float));
  const float* ego = c->hs_ego.dev;
  if (c->d_ctab) {
    // the controllers' launch fetches the ego actions and writes them into row 0 of `action`; the other participants'
    // actions never leave the device; the tick then reads everything from `action`
    if (int r = launch_control(c, action, ego, stream)) return r;
    ego = nullptr;
  }
  uint8_t* out = c->hs_out.dev.get();
  if (int r = launch_step(c, action, ego, flags, hit_index, hit_segment, out, out + N, stream, 1)) return r;
  if (int r = launch_history(c, nullptr, stream)) return r;
  return read_back(c->hs_out, 2 * (size_t)N, (cudaStream_t)stream,
                   {{scn_status_host, 0, (size_t)N}, {done_host, (size_t)N, (size_t)N}});
}

int t2d_env_epilogue(t2d_ctx* c, const uint8_t* flags, const uint8_t* scn_status, float* reward, uint8_t* terminated,
                     uint8_t* truncated, uint8_t* traffic_status, uint8_t* done, float* max_iou, float* min_dist,
                     int reset_trackers_on_done, void* stream) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (int r = require(c, NEED_STATE)) return r;
  if (!flags || !scn_status || !reward) return fail(T2D_E_INVALID, "t2d_env_epilogue: flags / scn_status / reward is NULL");
  CUDA_TRY(cudaSetDevice(c->device));
  EnvArgs A{world_args(c)};
  A.flags = flags; A.status = scn_status;
  A.iou = c->goal.target ? c->goal.iou : nullptr; A.target = c->goal.target;
  A.max_iou = max_iou; A.min_dist = min_dist;
  A.reward = reward; A.terminated = terminated; A.truncated = truncated; A.done = done; A.traffic_status = traffic_status;
  A.max_step = c->cfg.max_step; A.reset_trackers = reset_trackers_on_done ? 1 : 0;
  A.route = route_args(c); A.s_best = c->route_id ? c->route_s_best : nullptr;
  t2d_env_epilogue_kernel<<<capped_grid((long long)c->N * c->M, 256, c->sm_count, 8), 256, 0, (cudaStream_t)stream>>>(A);
  return launched();
}

int t2d_set_agents(t2d_ctx* c, const int16_t* observers, int32_t n_observers, const float* goals, float arrival_threshold,
                   int no_action_max_step, float* last_pose, int32_t* noact_count, uint8_t* retired_type) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (!observers && n_observers == 0) {   // unbind
    c->agent_q = 0; c->agent_observers = nullptr; c->agent = {}; c->agent_retired = nullptr;
    return T2D_OK;
  }
  if (int r = check_rows(c, "t2d_set_agents", observers, n_observers, 1)) return r;
  if (!last_pose || !noact_count || !retired_type) return fail(T2D_E_INVALID, "t2d_set_agents: NULL state array");
  if (goals && !(arrival_threshold > 0.0f && arrival_threshold <= 1.0f)) return fail(T2D_E_INVALID, "arrival_threshold must be in (0, 1]");
  c->agent_q = n_observers; c->agent_observers = observers; c->agent_retired = retired_type;
  c->agent = {goals, nullptr, last_pose, noact_count, arrival_threshold, no_action_max_step};
  return T2D_OK;
}

int t2d_agents_epilogue(t2d_ctx* c, const uint8_t* flags, float* reward, uint8_t* terminated, uint8_t* truncated,
                        uint8_t* agent_status, float* iou, uint8_t* done, float* max_iou, float* min_dist, uint8_t* traffic_status,
                        int reset_trackers_on_done, void* stream) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (int r = require(c, NEED_STATE | NEED_TABLE)) return r;
  if (c->agent_q == 0) return fail(T2D_E_STATE, "t2d_agents_epilogue: no agents bound: call t2d_set_agents first");
  if (!flags || !reward || !terminated || !truncated || !agent_status || !iou || !done || !max_iou || !min_dist)
    return fail(T2D_E_INVALID, "t2d_agents_epilogue: NULL array");
  if (int r = check_route_trackers(c, "t2d_agents_epilogue")) return r;
  CUDA_TRY(cudaSetDevice(c->device));
  AgentArgs A{world_args(c)};
  A.route = route_args(c); A.s_best = c->route_id ? c->route_agent_s_best : nullptr;
  A.goal = c->agent; A.goal.iou = iou;
  A.flags = flags; A.observers = c->agent_observers; A.retired = c->agent_retired;
  A.max_iou = max_iou; A.min_dist = min_dist; A.reward = reward; A.terminated = terminated; A.truncated = truncated;
  A.status = agent_status; A.done = done; A.traffic_status = traffic_status;
  A.Q = c->agent_q; A.max_step = c->cfg.max_step;
  A.reset_trackers = reset_trackers_on_done ? 1 : 0;
  t2d_agents_epilogue_kernel<<<(c->N + K10_WARPS - 1) / K10_WARPS, K10_WARPS * 32, 0, (cudaStream_t)stream>>>(A);
  return launched();
}

// K11 over the bound state's type ids; the caller has checked the arguments
static int launch_agent_action(t2d_ctx* c, const int16_t* observers, int Q, const float* agent_action, float* action,
                               void* stream) {
  CUDA_TRY(cudaSetDevice(c->device));
  ActionArgs A{world_args(c)};
  A.observers = observers; A.agent_action = agent_action; A.action = action; A.Q = Q;
  t2d_agent_action_kernel<<<(c->N + K11_WARPS - 1) / K11_WARPS, K11_WARPS * 32, 0, (cudaStream_t)stream>>>(A);
  return launched();
}

int t2d_scatter_agent_action(t2d_ctx* c, const int16_t* observers, int32_t n_observers, const float* agent_action,
                             float* action, void* stream) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (int r = check_rows(c, "t2d_scatter_agent_action", observers, n_observers, 1)) return r;
  if (!agent_action || !action) return fail(T2D_E_INVALID, "t2d_scatter_agent_action: agent_action / action is NULL");
  if (!aligned8(agent_action) || !aligned8(action))
    return fail(T2D_E_INVALID, "t2d_scatter_agent_action: agent_action and action must be 8-byte aligned");
  if (int r = require(c, NEED_STATE | NEED_TABLE)) return r;
  return launch_agent_action(c, observers, n_observers, agent_action, action, stream);
}

int t2d_step_host_agents(t2d_ctx* c, const float* agent_action_host, float* action, uint8_t* flags, int16_t* hit_index,
                         int16_t* hit_segment, float* max_iou, float* min_dist, int reset_trackers_on_done, float* reward_host,
                         uint8_t* terminated_host, uint8_t* truncated_host, uint8_t* agent_status_host, uint8_t* done_host,
                         void* stream) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (!agent_action_host || !action || !max_iou || !min_dist || !done_host)
    return fail(T2D_E_INVALID, "t2d_step_host_agents: agent_action / action / max_iou / min_dist / done is NULL");
  if (!aligned8(action)) return fail(T2D_E_INVALID, "t2d_step_host_agents: action must be 8-byte aligned");
  if (int r = require(c, NEED_STATE | NEED_TABLE | NEED_TICK)) return r;
  if (c->agent_q == 0) return fail(T2D_E_STATE, "t2d_step_host_agents: no agents bound: call t2d_set_agents first");
  if (int r = check_route_trackers(c, "t2d_step_host_agents")) return r;
  if (c->d_ctab)
    if (int r = check_pid_binding(c)) return r;
  CUDA_TRY(cudaSetDevice(c->device));
  const int N = c->N, M = c->M, Q = c->agent_q;
  const size_t nq = (size_t)N * Q;
  const size_t out_bytes = 7 * nq + N;                   // reward, terminated, truncated, status, done
  const size_t iou_off = (out_bytes + 15) & ~(size_t)15;
  if (c->ha.q != Q) {   // staging for the bound Q
    AgentStaging a;
    if (int r = dev_alloc(a.action, nq * 2)) return r;
    if (int r = make_mirror(a.out, iou_off + nq * sizeof(float), out_bytes)) return r;
    a.q = Q;
    c->ha = std::move(a);
  }
  if (!flags && !c->ha_flags)
    if (int r = dev_alloc(c->ha_flags, (size_t)N * M)) return r;
  uint8_t* fl = flags ? flags : c->ha_flags.get();
  uint8_t* o = c->ha.out.dev.get();
  float* d_reward = reinterpret_cast<float*>(o);
  uint8_t* d_term = o + 4 * nq;
  uint8_t* d_trunc = d_term + nq;
  uint8_t* d_status = d_trunc + nq;
  uint8_t* d_done = d_status + nq;
  float* d_iou = reinterpret_cast<float*>(o + iou_off);
  // One copy-engine transfer of the actions, as t2d_step_host (from pinned caller memory it is a DMA; pageable memory
  // goes through the driver's staging).  Staging them in mapped host memory for K11 to read over PCIe, as
  // t2d_step_host_ego does with its 8 N bytes, made the whole call about 1.5x slower at 2 MiB (DESIGN.md section 7).
  cudaStream_t s = (cudaStream_t)stream;
  CUDA_TRY(cudaMemcpyAsync(c->ha.action.get(), agent_action_host, nq * 2 * sizeof(float), cudaMemcpyHostToDevice, s));
  if (int r = launch_agent_action(c, c->agent_observers, Q, c->ha.action.get(), action, stream)) return r;
  if (c->d_ctab)
    if (int r = launch_control(c, action, c->ego_action, stream)) return r;
  if (int r = launch_step(c, action, c->ego_action, fl, hit_index, hit_segment, nullptr, nullptr, stream, 1)) return r;
  if (int r = launch_history(c, nullptr, stream)) return r;   // the post-tick state, before K10 retires slots
  if (int r = t2d_agents_epilogue(c, fl, d_reward, d_term, d_trunc, d_status, d_iou, d_done, max_iou, min_dist, nullptr,
                                  reset_trackers_on_done, stream))
    return r;
  return read_back(c->ha.out, out_bytes, s,
                   {{reward_host, 0, 4 * nq}, {terminated_host, 4 * nq, nq}, {truncated_host, 5 * nq, nq},
                    {agent_status_host, 6 * nq, nq}, {done_host, 7 * nq, (size_t)N}});
}

int t2d_check_events(t2d_ctx* c, uint8_t* flags, int16_t* hit_index, int16_t* hit_segment, void* stream) {
  return launch_step(c, nullptr, c ? c->ego_action : nullptr, flags, hit_index, hit_segment, nullptr, nullptr, stream, 0);
}

// The arguments t2d_reset and t2d_reset_sampled share
static int check_reset(t2d_ctx* c, const uint8_t* mask, int n_pool, const float* pool_x, const float* pool_y,
                       const float* pool_heading, const float* pool_speed) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (int r = require(c, NEED_STATE)) return r;
  if (!mask || !pool_x || !pool_y || !pool_heading || !pool_speed) return fail(T2D_E_INVALID, "t2d_reset: NULL array");
  if (n_pool <= 0) return fail(T2D_E_INVALID, "n_pool must be > 0");
  if (c->log && n_pool != c->log->n_rows) return fail(T2D_E_INVALID, "t2d_reset: with a log bound, pool row p is episode row p (n_pool == n_rows)");
  if (c->log && c->log->type_id != c->type_id) return fail(T2D_E_STATE, "state rebound after t2d_set_log: call t2d_set_log again");
  return T2D_OK;
}

// K2 (and K7) of t2d_reset, after check_reset; t2d_reset_sampled runs it between K13 and K14
static int launch_reset(t2d_ctx* c, const uint8_t* mask, const int32_t* pool_index, int n_pool, const float* pool_x,
                        const float* pool_y, const float* pool_heading, const float* pool_speed, const float* pool_vx,
                        const float* pool_vy, void* stream) {
  CUDA_TRY(cudaSetDevice(c->device));
  ResetArgs A{world_args(c)};
  A.mask = mask; A.pool_index = pool_index;
  A.px = pool_x; A.py = pool_y; A.ph = pool_heading; A.pv = pool_speed; A.pvx = pool_vx; A.pvy = pool_vy;
  A.goal = c->goal;
  A.wheel_f = c->wheel_f; A.wheel_r = c->wheel_r; A.pool_wf = c->reset_pool_wf; A.pool_wr = c->reset_pool_wr;
  A.last_accel = c->ctrl_last_accel; A.pid_state = c->pid_state; A.n_pool = n_pool;
  if (c->agent_q > 0) {   // the bound type_id is the caller's writable device array (K10 retires slots in it)
    A.agent_type_id = const_cast<uint8_t*>(c->type_id); A.agent_retired = c->agent_retired;
    A.agent = c->agent; A.agent_q = c->agent_q;
  }
  t2d_reset_kernel<<<capped_grid((long long)c->N * c->M, 256, c->sm_count, 8), 256, 0, (cudaStream_t)stream>>>(A);
  if (int r = launched()) return r;
  if (c->lane) {   // the new episodes start from their starting lanes
    lane::ResetArgs R{mask, c->ctrl_path, c->lane->lane_path, c->lane->cooldown, c->lane->change, (long long)c->N, c->M};
    lane::t2d_lane_reset_kernel<<<capped_grid((long long)c->N * c->M, 256, c->sm_count, 8), 256, 0, (cudaStream_t)stream>>>(R);
    if (int r = launched()) return r;
  }
  if (c->log) return launch_replay(c, stream, 0, c->N, 0, mask, pool_index);   // the new episode's traffic at t0
  return T2D_OK;
}

int t2d_reset(t2d_ctx* c, const uint8_t* mask, const int32_t* pool_index, int n_pool, const float* pool_x, const float* pool_y,
              const float* pool_heading, const float* pool_speed, const float* pool_vx, const float* pool_vy, void* stream) {
  if (int r = check_reset(c, mask, n_pool, pool_x, pool_y, pool_heading, pool_speed)) return r;
  if (int r = launch_reset(c, mask, pool_index, n_pool, pool_x, pool_y, pool_heading, pool_speed, pool_vx, pool_vy, stream))
    return r;
  return launch_history(c, mask, stream);   // entry 0 of the new episode: the state after the whole reset
}

// A row-owned pool needs what it writes into: checked when the sampler is bound and before every sampled reset (the
// goal, the map table or the routes may have been unbound since)
static int check_sampler_targets(const t2d_ctx* c, const t2d_reset_sampler& s) {
  if (s.pool_target && !c->goal.target) return fail(T2D_E_STATE, "reset sampler: a target pool needs a t2d_set_goal target");
  if (s.pool_tile_id && !c->map.tile_id) return fail(T2D_E_STATE, "reset sampler: a tile pool needs a map table of more than one tile");
  if (s.pool_route_id && !c->route_id) return fail(T2D_E_STATE, "reset sampler: a route pool needs t2d_set_routes");
  return T2D_OK;
}

int t2d_set_reset_sampler(t2d_ctx* c, const t2d_reset_sampler* s) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (!s) {
    c->sampler.reset();
    return T2D_OK;
  }
  if (int r = require(c, NEED_STATE | NEED_TABLE)) return r;
  if (s->tries < 1 || s->tries > 32) return fail(T2D_E_INVALID, "reset sampler: tries must be in 1..32");
  if (!s->episode || !s->pool_row || !s->reset_try) return fail(T2D_E_INVALID, "reset sampler: NULL episode / pool_row / reset_try");
  const bool pools = s->pool_type_id || s->pool_target || s->pool_tile_id || s->pool_route_id;
  if (pools && s->n_rows <= 0) return fail(T2D_E_INVALID, "reset sampler: row pools need n_rows > 0");
  if (s->jitter)
    for (int k = 0; k < c->M * 4; ++k) {
      const float lo = s->jitter[2 * k], hi = s->jitter[2 * k + 1];
      if (!(std::isfinite(lo) && std::isfinite(hi) && lo <= hi))
        return fail(T2D_E_INVALID, "reset sampler: every jitter range must be finite with lo <= hi");
    }
  if (int r = check_sampler_targets(c, *s)) return r;
  CUDA_TRY(cudaSetDevice(c->device));
  auto d = std::make_unique<DeviceSampler>();
  d->s = *s;
  if (s->jitter) {
    if (int r = upload(d->jitter, s->jitter, (size_t)c->M * 8)) return r;
    d->s.jitter = d->jitter.get();
  }
  CUDA_TRY(cudaMemset(s->episode, 0, sizeof(uint32_t) * c->N));
  c->sampler = std::move(d);
  return T2D_OK;
}

int t2d_reset_sampled(t2d_ctx* c, const uint8_t* mask, int n_pool, const float* pool_x, const float* pool_y,
                      const float* pool_heading, const float* pool_speed, const float* pool_vx, const float* pool_vy,
                      void* stream) {
  if (int r = check_reset(c, mask, n_pool, pool_x, pool_y, pool_heading, pool_speed)) return r;
  if (!c->sampler) return fail(T2D_E_STATE, "t2d_reset_sampled: no reset sampler bound");
  if (int r = require(c, NEED_TABLE)) return r;
  const t2d_reset_sampler& s = c->sampler->s;
  if (int r = check_sampler_targets(c, s)) return r;
  if ((s.pool_type_id || s.pool_target || s.pool_tile_id || s.pool_route_id) && n_pool != s.n_rows)
    return fail(T2D_E_INVALID, "t2d_reset_sampled: the pool must have the sampler's n_rows rows");
  if (!s.sample_rows && n_pool < c->N) return fail(T2D_E_INVALID, "t2d_reset_sampled: without row draws the pool needs one row per scenario");
  CUDA_TRY(cudaSetDevice(c->device));
  DrawArgs D{};
  D.mask = mask; D.episode = s.episode; D.pool_row = s.pool_row; D.seed = s.seed; D.sample_rows = s.sample_rows;
  D.N = c->N; D.M = c->M; D.P = n_pool;
  // the row-owned columns are written into the caller's bound arrays (type_id, the goal target, the map table's tile_id,
  // the route ids), which the library documents as rewritable between ticks
  D.pool_type = s.pool_type_id; D.type_id = const_cast<uint8_t*>(c->type_id);
  D.retired = c->agent_q > 0 ? c->agent_retired : nullptr;
  D.pool_target = s.pool_target; D.target = const_cast<float*>(c->goal.target);
  D.pool_tile = s.pool_tile_id; D.tile_id = const_cast<uint16_t*>(c->map.tile_id);
  D.pool_route = s.pool_route_id; D.route_id = const_cast<int16_t*>(c->route_id);
  t2d_episode_draw_kernel<<<capped_grid((long long)c->N * c->M, 256, c->sm_count, 8), 256, 0, (cudaStream_t)stream>>>(D);
  if (int r = launched()) return r;
  if (int r = launch_reset(c, mask, s.pool_row, n_pool, pool_x, pool_y, pool_heading, pool_speed, pool_vx, pool_vy, stream))
    return r;
  PlaceArgs P{world_args(c)};
  P.mask = mask; P.episode = s.episode; P.reset_try = s.reset_try; P.seed = s.seed;
  P.jitter = s.jitter; P.tries = s.tries; P.avoid_target = s.avoid_target; P.target = c->goal.target;
  P.map = map_args(c->map); P.mh = c->map.mh; P.has_bounds = c->map.has_bounds ? 1 : 0;
  P.wheel_f = c->wheel_f; P.wheel_r = c->wheel_r; P.pool_wheels = c->reset_pool_wf != nullptr;
  t2d_episode_place_kernel<<<(unsigned)((c->N + K14_WARPS - 1) / K14_WARPS), K14_WARPS * 32, 0, (cudaStream_t)stream>>>(P);
  if (int r = launched()) return r;
  return launch_history(c, mask, stream);   // entry 0 of the new episode: the placed state
}

// K4 over the rows of an observer list (observers == nullptr: row q is slot q); the callers have checked their arguments
static int launch_lidar(t2d_ctx* c, const int16_t* observers, int Q, int n_beams, float max_range, const double* beam_cos_sin,
                        float* scan, void* stream) {
  CUDA_TRY(cudaSetDevice(c->device));
  LidarArgs A{world_args(c)};
  A.map = map_args(c->map);
  A.beam_cs = beam_cos_sin; A.observers = observers; A.scan = scan;
  A.Q = Q; A.n_beams = n_beams; A.range = (double)max_range;
  const long long grid = ((long long)c->N * Q + LIDAR_WARPS - 1) / LIDAR_WARPS;
  if (grid > INT32_MAX) return fail(T2D_E_UNSUPPORTED, "lidar: more than 2^33 rows (one warp per row)");
  t2d_lidar_kernel<<<(unsigned)grid, LIDAR_WARPS * 32, 0, (cudaStream_t)stream>>>(A);
  return launched();
}

int t2d_lidar_scan(t2d_ctx* c, int n_beams, float max_range, const double* beam_cos_sin, float* scan, void* stream) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (int r = require(c, NEED_STATE | NEED_TABLE)) return r;
  if (n_beams <= 0 || !(max_range > 0.0f) || !beam_cos_sin || !scan) return fail(T2D_E_INVALID, "t2d_lidar_scan: bad argument");
  return launch_lidar(c, nullptr, 1, n_beams, max_range, beam_cos_sin, scan, stream);
}

int t2d_lidar_scan_agents(t2d_ctx* c, const int16_t* observers, int32_t n_observers, int n_beams, float max_range,
                          const double* beam_cos_sin, float* scan, void* stream) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (int r = check_rows(c, "t2d_lidar_scan_agents", observers, n_observers, 1)) return r;
  if (n_beams <= 0 || !(max_range > 0.0f) || !beam_cos_sin || !scan)
    return fail(T2D_E_INVALID, "t2d_lidar_scan_agents: n_beams must be > 0, max_range > 0, beam_cos_sin and scan not NULL");
  if (int r = require(c, NEED_STATE | NEED_TABLE)) return r;
  return launch_lidar(c, observers, n_observers, n_beams, max_range, beam_cos_sin, scan, stream);
}

int t2d_set_bev_styles(t2d_ctx* c, const t2d_bev_style* table, int n_styles, const uint8_t* type_style, const uint8_t* seg_style,
                       int n_seg_total, int target_style) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (int r = require(c, NEED_TABLE)) return r;
  if (!table || n_styles < 4 || n_styles > T2D_MAX_BEV_STYLES) return fail(T2D_E_INVALID, "n_styles must be in 4..64");
  if (!type_style) return fail(T2D_E_INVALID, "type_style is NULL");
  for (int i = 0; i < n_styles; ++i)
    if (!(table[i].line_width_pt >= 0.0f && table[i].line_width_pt <= 100.0f))
      return fail(T2D_E_INVALID, "style line width must be in [0, 100] pt");
  auto ok = [&](int s) { return s == bev::NO_STYLE || (s >= 0 && s < n_styles); };
  for (int t = 0; t < c->n_types; ++t)
    if (!ok(type_style[t])) return fail(T2D_E_INVALID, "type_style: no such style");
  if (!ok(target_style)) return fail(T2D_E_INVALID, "target_style: no such style");
  const std::vector<int>& nseg = c->map.tile_nseg;
  long long total = 0;
  for (int k : nseg) total += k;
  if (seg_style) {
    if (n_seg_total != total) return fail(T2D_E_INVALID, "n_seg_total differs from the segments of the map's tiles");
    for (long long s = 0; s < total; ++s)
      if (!ok(seg_style[s])) return fail(T2D_E_INVALID, "seg_style: no such style");
  }
  CUDA_TRY(cudaSetDevice(c->device));
  dev_ptr<uint8_t> d_style;
  dev_ptr<uint32_t> d_base;
  if (seg_style && total > 0) {
    std::vector<uint32_t> base(nseg.size());
    uint32_t acc = 0;
    for (size_t i = 0; i < base.size(); ++i) { base[i] = acc; acc += (uint32_t)nseg[i]; }
    if (int r = upload(d_style, seg_style, (size_t)total)) return r;
    if (int r = upload(d_base, base.data(), base.size())) return r;
  }
  // opt in to the kernel's shared memory here: t2d_bev_render must stay free of anything a graph capture rejects
  CUDA_TRY(cudaFuncSetAttribute(bev::t2d_bev_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(bev::Smem)));
  CUDA_TRY(cudaFuncSetAttribute(bev::t2d_bev_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(bev::Smem)));
  c->map.seg_style = std::move(d_style);
  c->map.seg_base = std::move(d_base);
  memcpy(c->bev_style, table, sizeof(t2d_bev_style) * (size_t)n_styles);
  memset(c->bev_type_style, bev::NO_STYLE, sizeof(c->bev_type_style));
  memcpy(c->bev_type_style, type_style, (size_t)c->n_types);
  c->bev_target_style = target_style;
  c->n_bev_styles = n_styles;
  return T2D_OK;
}

// K6 over the rows of an observer list (rows: t2d_bev_render_agents) or over the egos (t2d_bev_render); the arguments
// both entries take are checked here, with messages prefixed by fn
static int launch_bev(t2d_ctx* c, const std::string& fn, bool rows, const int16_t* observers, int Q, const float* goals,
                      int width, int height, const float* range, int rgb, uint8_t* out, void* stream) {
  if (int r = require(c, NEED_STATE)) return r;
  if (c->n_bev_styles == 0) return fail(T2D_E_STATE, "BEV styles not set: call t2d_set_bev_styles first");
  if (!range || !out) return fail(T2D_E_INVALID, fn + ": range / out is NULL");
  if (width < 1 || height < 1 || width > bev::MAX_SIDE || height > bev::MAX_SIDE)
    return fail(T2D_E_INVALID, fn + ": width and height must be in 1..1024");
  for (int k = 0; k < 4; ++k)
    if (!(range[k] > 0.0f && range[k] <= 1.0e5f)) return fail(T2D_E_INVALID, fn + ": every range must be in (0, 1e5] m");
  const long long grid = (long long)c->N * Q;   // one CTA per row
  if (grid > INT32_MAX) return fail(T2D_E_UNSUPPORTED, fn + ": more than 2^31 - 1 rows (one CTA per row)");
  // the window (matplotlib_renderer.py:152-164, auto_scale :200-224), in the float64 oracle's operation order
  const double L = range[0], R = range[1], F = range[2], B = range[3];
  const double x_min = -L, x_max = R, y_min = -B, y_max = F;
  const double ww = x_max - x_min, wh = y_max - y_min;
  const double cx = (x_min + x_max) / 2, cy = (y_min + y_max) / 2;
  const double aspect = (double)height / (double)width;
  double nw, nh;
  if (wh / ww > aspect) { nw = wh / aspect; nh = wh; }
  else { nw = ww; nh = ww * aspect; }
  const double nx0 = cx - nw / 2, nx1 = cx + nw / 2, ny0 = cy - nh / 2, ny1 = cy + nh / 2;
  bev::Args A{world_args(c)};
  A.win.xmin = nx0; A.win.ymax = ny1;
  A.win.px = (nx1 - nx0) / width; A.win.py = (ny1 - ny0) / height;
  for (int s = 0; s < c->n_bev_styles; ++s) {
    const t2d_bev_style& st = c->bev_style[s];
    const double hw = (double)st.line_width_pt * 200.0 / 72.0 / 2.0 * A.win.px;   // points at the renderer's 200 dpi
    A.hw2[s] = hw * hw;
    A.style_rgb[s][0] = st.r; A.style_rgb[s][1] = st.g; A.style_rgb[s][2] = st.b;
    A.style_z[s] = st.z;
  }
  memcpy(A.type_style, c->bev_type_style, sizeof(A.type_style));
  A.map = map_args(c->map); A.seg_style = c->map.seg_style.get(); A.seg_base = c->map.seg_base.get();
  A.target = c->goal.target; A.target_style = c->bev_target_style;
  A.ring_style = T2D_BEV_STYLE_RING; A.open_style = T2D_BEV_STYLE_OPEN;
  A.observers = observers; A.goals = goals; A.Q = Q;
  A.W = width; A.H = height; A.rgb = rgb ? 1 : 0; A.out = out;
  CUDA_TRY(cudaSetDevice(c->device));
  if (rows) bev::t2d_bev_kernel<true><<<(unsigned)grid, bev::CTA, sizeof(bev::Smem), (cudaStream_t)stream>>>(A);
  else bev::t2d_bev_kernel<false><<<(unsigned)grid, bev::CTA, sizeof(bev::Smem), (cudaStream_t)stream>>>(A);
  return launched();
}

int t2d_bev_render(t2d_ctx* c, int width, int height, const float* range, int rgb, uint8_t* out, void* stream) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  return launch_bev(c, "t2d_bev_render", false, nullptr, 1, nullptr, width, height, range, rgb, out, stream);
}

int t2d_bev_render_agents(t2d_ctx* c, const int16_t* observers, int32_t n_observers, const float* goals, int width, int height,
                          const float* range, int rgb, uint8_t* out, void* stream) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (int r = check_rows(c, "t2d_bev_render_agents", observers, n_observers, 1)) return r;
  return launch_bev(c, "t2d_bev_render_agents", true, observers, n_observers, goals, width, height, range, rgb, out, stream);
}

// What t2d_observe and t2d_observe_agents share: the checks of cfg and out (messages prefixed with fn) and K8's arguments
static int obs_args(const t2d_ctx* c, const std::string& fn, const t2d_obs_config* cfg, float* out, int16_t* agent_index,
                    int16_t* segment_index, obs::Args& A) {
  if (!cfg) return fail(T2D_E_INVALID, fn + ": cfg is NULL");
  if (cfg->k_agents < 0 || cfg->k_agents > T2D_OBS_MAX_AGENTS) return fail(T2D_E_INVALID, fn + ": k_agents must be in 0..127");
  if (cfg->k_segments < 0 || cfg->k_segments > T2D_OBS_MAX_SEGMENTS)
    return fail(T2D_E_INVALID, fn + ": k_segments must be in 0..256");
  if (!(cfg->agent_range > 0.0f && cfg->agent_range <= 1.0e5f) || !(cfg->segment_range > 0.0f && cfg->segment_range <= 1.0e5f))
    return fail(T2D_E_INVALID, fn + ": agent_range and segment_range must be in (0, 1e5] m");
  if (!out) return fail(T2D_E_INVALID, fn + ": out is NULL");
  static_assert(T2D_OBS_MAX_AGENTS == obs::MAX_K && T2D_OBS_MAX_SEGMENTS == obs::MAX_S, "K8's shared lists hold the ABI's limits");
  static_cast<WorldArgs&>(A) = world_args(c);
  A.max_step = c->cfg.max_step; A.map = map_args(c->map); A.target = c->goal.target;
  A.K = cfg->k_agents; A.S = cfg->k_segments;
  A.F = obs::EGO_F + obs::GOAL_F + obs::AGENT_F * A.K + obs::SEG_F * A.S;
  const double ra = cfg->agent_range, rs = cfg->segment_range;
  A.ra2 = ra * ra; A.rs2 = rs * rs;
  A.out = out; A.agent_index = agent_index; A.segment_index = segment_index;
  return T2D_OK;
}

int t2d_observe(t2d_ctx* c, const t2d_obs_config* cfg, float* out, int16_t* agent_index, int16_t* segment_index, void* stream) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  obs::Args A{};
  if (int r = obs_args(c, "t2d_observe", cfg, out, agent_index, segment_index, A)) return r;
  if (int r = require(c, NEED_STATE | NEED_TABLE)) return r;
  CUDA_TRY(cudaSetDevice(c->device));
  const int grid = (c->N + obs::WARPS - 1) / obs::WARPS;
  obs::t2d_obs_kernel<<<grid, obs::WARPS * 32, 0, (cudaStream_t)stream>>>(A);
  return launched();
}

int t2d_observe_agents(t2d_ctx* c, const t2d_obs_config* cfg, const int16_t* observers, int32_t n_observers,
                       const float* goals, float* out, int16_t* agent_index, int16_t* segment_index, void* stream) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  obs::AgentArgs G{};
  if (int r = obs_args(c, "t2d_observe_agents", cfg, out, agent_index, segment_index, G.a)) return r;
  if (int r = check_rows(c, "t2d_observe_agents", observers, n_observers, 1)) return r;
  if (int r = require(c, NEED_STATE | NEED_TABLE)) return r;
  G.observers = observers; G.goals = goals; G.Q = n_observers;
  CUDA_TRY(cudaSetDevice(c->device));
  const long long rows = (long long)c->N * n_observers;
  const int grid = (int)std::min<long long>((rows + obs::WARPS - 1) / obs::WARPS, 1ll << 30);   // the kernel strides past 2^32 rows
  obs::t2d_obs_agents_kernel<<<grid, obs::WARPS * 32, 0, (cudaStream_t)stream>>>(G);
  return launched();
}

int t2d_set_history(t2d_ctx* c, int32_t length) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (length < 0 || length > T2D_HISTORY_MAX) return fail(T2D_E_INVALID, "t2d_set_history: length must be in 0..64");
  CUDA_TRY(cudaSetDevice(c->device));
  if (length == 0) {
    c->hist.reset();
    return T2D_OK;
  }
  static_assert(T2D_HISTORY_MAX == hist::MAX_H && T2D_HISTORY_FIELDS == hist::HIST_F, "K16's stage holds the ABI's limits");
  auto g = std::make_unique<DeviceHistory>();
  g->H = length;
  const size_t plane = (size_t)c->N * length * c->M;
  if (int r = dev_alloc(g->f, 6 * plane)) return r;
  if (int r = dev_alloc(g->type, plane)) return r;
  if (int r = dev_alloc(g->count, (size_t)c->N)) return r;
  CUDA_TRY(cudaMemset(g->f.get(), 0, 6 * plane * sizeof(float)));
  CUDA_TRY(cudaMemset(g->type.get(), 0xff, plane));
  CUDA_TRY(cudaMemset(g->count.get(), 0, (size_t)c->N * sizeof(long long)));
  if (int r = history_tracks(c, *g, c->log ? c->log->track_out : nullptr)) return r;
  c->hist = std::move(g);
  return T2D_OK;
}

int t2d_history_view(t2d_ctx* c, t2d_history_ring* out) {
  if (!c || !out) return fail(T2D_E_INVALID, "t2d_history_view: ctx / out is NULL");
  *out = t2d_history_ring{};
  if (!c->hist) return T2D_OK;
  const hist::Ring R = history_ring(c);
  out->length = R.H;
  out->x = R.x; out->y = R.y; out->heading = R.h; out->speed = R.v; out->vx = R.vx; out->vy = R.vy;
  out->type_id = R.type; out->track = R.track; out->count = reinterpret_cast<int64_t*>(R.count);
  return T2D_OK;
}

int t2d_observe_history(t2d_ctx* c, const int16_t* observers, int32_t n_observers, const int16_t* agent_index, int32_t k_agents,
                        float* out, void* stream) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (int r = check_rows(c, "t2d_observe_history", observers, n_observers, 0)) return r;
  if (n_observers == 0 && observers) return fail(T2D_E_INVALID, "t2d_observe_history: an observer list needs n_observers >= 1");
  if (k_agents < 0 || k_agents > T2D_OBS_MAX_AGENTS) return fail(T2D_E_INVALID, "t2d_observe_history: k_agents must be in 0..127");
  if (k_agents > 0 && !agent_index) return fail(T2D_E_INVALID, "t2d_observe_history: agent_index is NULL");
  if (!out) return fail(T2D_E_INVALID, "t2d_observe_history: out is NULL");
  if (int r = require(c, NEED_STATE | NEED_TABLE)) return r;
  if (!c->hist) return fail(T2D_E_STATE, "t2d_observe_history: no history bound: call t2d_set_history first");
  CUDA_TRY(cudaSetDevice(c->device));
  hist::ObsArgs A{world_args(c)};
  A.ring = history_ring(c); A.track_now = history_track_now(c);
  A.observers = observers; A.Q = n_observers; A.agent_index = agent_index; A.K = k_agents; A.out = out;
  const long long rows = (long long)c->N * std::max(1, n_observers);
  const int grid = (int)std::min<long long>((rows + hist::K16_WARPS - 1) / hist::K16_WARPS, 1ll << 30);   // the kernel strides
  hist::t2d_history_obs_kernel<<<grid, hist::K16_WARPS * 32, 0, (cudaStream_t)stream>>>(A);
  return launched();
}

int t2d_set_controllers(t2d_ctx* c, const t2d_controller_params* table, int n_rows, const uint8_t* ctrl_id,
                        const int16_t* lead_index, const int16_t* path_id, float* last_accel) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  CUDA_TRY(cudaSetDevice(c->device));
  if (!table) {
    c->d_ctab.reset();
    c->n_ctrl = 0; c->ctrl_id = nullptr; c->ctrl_lead = nullptr; c->ctrl_path = nullptr;
    c->ctrl_last_accel = nullptr;
    c->ctrl_has_pid = c->ctrl_pid_reads_target = false;
    drop_traffic(c, NEED_CTRL);
    return T2D_OK;
  }
  if (n_rows <= 0 || n_rows > T2D_MAX_CONTROLLERS) return fail(T2D_E_INVALID, "n_rows must be in 1..T2D_MAX_CONTROLLERS");
  if (!ctrl_id || !last_accel) return fail(T2D_E_INVALID, "t2d_set_controllers: ctrl_id / last_accel is NULL");
  bool has_pid = false, reads_target = false;
  for (int i = 0; i < n_rows; ++i) {
    const t2d_controller_params& p = table[i];
    if (p.kind < T2D_CTRL_EXTERNAL || p.kind > T2D_CTRL_PID) return fail(T2D_E_INVALID, "unknown controller kind");
    if (p.kind == T2D_CTRL_PID) {   // PIDController.__init__'s checks, pid_controller.py:81-102
      if (!(p.dt > 0.0)) return fail(T2D_E_INVALID, "PID row: dt must be positive");
      if (!(p.max_steering > 0.0)) return fail(T2D_E_INVALID, "PID row: max_steering must be positive");
      if (!(p.max_accel > 0.0f)) return fail(T2D_E_INVALID, "PID row: max_accel must be positive");
      if (!(p.min_accel < 0.0f)) return fail(T2D_E_INVALID, "PID row: min_accel must be negative (deceleration)");
      if (!(p.max_accel > p.min_accel)) return fail(T2D_E_INVALID, "PID row: max_accel must be greater than min_accel");
      if (!(p.derivative_filter_alpha > 0.0 && p.derivative_filter_alpha <= 1.0))
        return fail(T2D_E_INVALID, "PID row: derivative_filter_alpha must be in range (0, 1]");
      if (p.pid_lateral < T2D_PID_LAT_NONE || p.pid_lateral > T2D_PID_LAT_PATH_CROSS_TRACK)
        return fail(T2D_E_INVALID, "PID row: unknown lateral source");
      if (p.pid_longitudinal != T2D_PID_LON_NONE && p.pid_longitudinal != T2D_PID_LON_TARGET)
        return fail(T2D_E_INVALID, "PID row: unknown longitudinal source");
      if ((p.pid_lateral == T2D_PID_LAT_CROSS_TRACK || p.pid_lateral == T2D_PID_LAT_PATH_CROSS_TRACK) && !(p.wheel_base > 0.0f))
        return fail(T2D_E_INVALID, "PID row: wheel_base must be positive");   // pid_controller.py:357-358
      has_pid = true;
      reads_target = reads_target || p.pid_longitudinal == T2D_PID_LON_TARGET || p.pid_lateral == T2D_PID_LAT_HEADING ||
                     p.pid_lateral == T2D_PID_LAT_CROSS_TRACK;
    }
    if (p.kind == T2D_CTRL_IDM && p.pid_lateral != T2D_PID_LAT_NONE) {   // lane keeping: the PID row's lateral checks
      if (p.pid_lateral != T2D_PID_LAT_PATH_HEADING && p.pid_lateral != T2D_PID_LAT_PATH_CROSS_TRACK)
        return fail(T2D_E_INVALID, "IDM row: the lateral channel must be a PATH source");
      if (!(p.dt > 0.0)) return fail(T2D_E_INVALID, "IDM row with a lateral channel: dt must be positive");
      if (!(p.max_steering > 0.0)) return fail(T2D_E_INVALID, "IDM row with a lateral channel: max_steering must be positive");
      if (!(p.derivative_filter_alpha > 0.0 && p.derivative_filter_alpha <= 1.0))
        return fail(T2D_E_INVALID, "IDM row with a lateral channel: derivative_filter_alpha must be in range (0, 1]");
      if (p.pid_lateral == T2D_PID_LAT_PATH_CROSS_TRACK && !(p.wheel_base > 0.0f))
        return fail(T2D_E_INVALID, "IDM row with a lateral channel: wheel_base must be positive");
      has_pid = true;   // K5's PID instance runs the channel, on t2d_set_pid's state
    }
    if (p.kind == T2D_CTRL_PURE_PURSUIT && !(p.min_pre_aiming_distance > 0.0f))
      return fail(T2D_E_INVALID, "min_pre_aiming_distance must be positive");   // pure_pursuit_controller.py:30-31
    if (p.kind >= T2D_CTRL_CRUISE && p.target_speed < 0.0f)
      return fail(T2D_E_INVALID, "target_speed must be non-negative");          // acceleration_controller.py:48-49
  }
  if (int r = upload(c->d_ctab, table, (size_t)n_rows)) return r;
  c->n_ctrl = n_rows; c->ctrl_id = ctrl_id; c->ctrl_lead = lead_index; c->ctrl_path = path_id; c->ctrl_last_accel = last_accel;
  c->ctrl_has_pid = has_pid; c->ctrl_pid_reads_target = reads_target;
  drop_traffic(c, NEED_CTRL);
  return T2D_OK;
}

int t2d_set_pid(t2d_ctx* c, const float* target, double* state) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (!state) {
    if (target) return fail(T2D_E_INVALID, "t2d_set_pid: a target needs a state");
    c->pid_target = nullptr; c->pid_state = nullptr;
    return T2D_OK;
  }
  if (!aligned8(target) || !aligned8(state))
    return fail(T2D_E_INVALID, "t2d_set_pid: target / state must be 8-byte aligned");
  c->pid_target = target; c->pid_state = state;
  return T2D_OK;
}

int t2d_set_paths(t2d_ctx* c, const float* xy, const int32_t* offsets, int n_paths) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  CUDA_TRY(cudaSetDevice(c->device));
  if (n_paths == 0 || !xy) {   // unbind
    c->d_path_v.reset(); c->d_path_off.reset(); c->n_paths = 0; c->path_host.clear(); c->path_off_host.clear();
    drop_traffic(c, NEED_PATHS);
    return T2D_OK;
  }
  if (n_paths < 0 || !offsets) return fail(T2D_E_INVALID, "t2d_set_paths: bad argument");
  if (offsets[0] != 0) return fail(T2D_E_INVALID, "offsets[0] must be 0");
  for (int p = 0; p < n_paths; ++p)
    if (offsets[p + 1] - offsets[p] < 2) return fail(T2D_E_INVALID, "a path needs at least 2 vertices");
  const int V = offsets[n_paths];
  std::vector<PathVertex> pv((size_t)V);
  for (int p = 0; p < n_paths; ++p) {
    double acc = 0.0;   // the running arc length of LineString.interpolate's walk, in float64
    for (int i = offsets[p]; i < offsets[p + 1]; ++i) {
      pv[i].x = xy[2 * i]; pv[i].y = xy[2 * i + 1];
      pv[i].cum = acc;
      pv[i].len = 0.0;
      if (i + 1 < offsets[p + 1]) {
        pv[i].len = hypot((double)xy[2 * i + 2] - (double)xy[2 * i], (double)xy[2 * i + 3] - (double)xy[2 * i + 1]);
        acc += pv[i].len;
      }
    }
  }
  dev_ptr<PathVertex> d_v;
  dev_ptr<int> d_off;
  if (int r = upload(d_v, pv.data(), pv.size())) return r;
  if (int r = upload(d_off, offsets, (size_t)n_paths + 1)) return r;
  c->d_path_v = std::move(d_v); c->d_path_off = std::move(d_off); c->n_paths = n_paths;
  c->path_host = std::move(pv);
  c->path_off_host.assign(offsets, offsets + n_paths + 1);
  drop_traffic(c, NEED_PATHS);
  return T2D_OK;
}

int t2d_set_routes(t2d_ctx* c, const int16_t* route_id, double threshold, double progress_weight, float off_route_reward) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (route_id) {
    if (!(std::isfinite(threshold) && threshold >= 0.0))
      return fail(T2D_E_INVALID, "t2d_set_routes: threshold must be finite and >= 0");
    if (!std::isfinite(progress_weight) || !std::isfinite(off_route_reward))
      return fail(T2D_E_INVALID, "t2d_set_routes: progress_weight and off_route_reward must be finite");
  }
  c->route_id = route_id;
  c->route_threshold = route_id ? threshold : 0.0;
  c->route_weight = route_id ? progress_weight : 0.0;
  c->route_off_reward = route_id ? off_route_reward : 0.0f;
  return T2D_OK;
}

int t2d_bind_route_trackers(t2d_ctx* c, double* s_best, double* agent_s_best, int32_t n_agent_rows) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (agent_s_best && (n_agent_rows < 1 || n_agent_rows > T2D_OBS_MAX_OBSERVERS))
    return fail(T2D_E_INVALID, "t2d_bind_route_trackers: n_agent_rows must be in 1..128");
  if (!aligned8(s_best) || !aligned8(agent_s_best))
    return fail(T2D_E_INVALID, "t2d_bind_route_trackers: the trackers must be 8-byte aligned");
  c->route_s_best = s_best;
  c->route_agent_s_best = agent_s_best;
  c->route_agent_rows = agent_s_best ? n_agent_rows : 0;
  return T2D_OK;
}

int t2d_route_observe(t2d_ctx* c, const int16_t* observers, int32_t n_observers, int n_points, float spacing, float* out,
                      void* stream) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (int r = check_rows(c, "t2d_route_observe", observers, n_observers, 1)) return r;
  if (n_points < 0 || n_points > T2D_ROUTE_MAX_POINTS) return fail(T2D_E_INVALID, "t2d_route_observe: n_points must be in 0..256");
  if (!(spacing > 0.0f) || !std::isfinite(spacing)) return fail(T2D_E_INVALID, "t2d_route_observe: spacing must be finite and > 0");
  if (!out) return fail(T2D_E_INVALID, "t2d_route_observe: out is NULL");
  if (int r = require(c, NEED_STATE | NEED_TABLE)) return r;
  CUDA_TRY(cudaSetDevice(c->device));
  RouteObsArgs A{world_args(c)};
  A.route = route_args(c); A.observers = observers; A.out = out; A.Q = n_observers; A.P = n_points;
  A.spacing = (double)spacing;
  t2d_route_obs_kernel<<<(c->N + K12_WARPS - 1) / K12_WARPS, K12_WARPS * 32, 0, (cudaStream_t)stream>>>(A);
  return launched();
}

int t2d_control(t2d_ctx* c, float* action, void* stream) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  return launch_control(c, action, c->ego_action, stream);
}

int t2d_set_leader_search(t2d_ctx* c, double half_width, double max_range, int16_t* lead, float* gap) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (!lead) {   // unbind
    c->leader_lead = nullptr; c->leader_gap = nullptr; c->leader_half_width = c->leader_max_range = 0.0;
    drop_traffic(c, NEED_SEARCH);
    return T2D_OK;
  }
  if (int r = check_leader_args("t2d_set_leader_search", half_width, max_range, lead, gap)) return r;
  if (int r = require(c, NEED_STATE | NEED_TABLE)) return r;
  c->leader_lead = lead; c->leader_gap = gap; c->leader_half_width = half_width; c->leader_max_range = max_range;
  return T2D_OK;
}

int t2d_find_leaders(t2d_ctx* c, double half_width, double max_range, int16_t* lead, float* gap, void* stream) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (!lead) return fail(T2D_E_INVALID, "t2d_find_leaders: lead is NULL");
  if (int r = check_leader_args("t2d_find_leaders", half_width, max_range, lead, gap)) return r;
  if (int r = require(c, NEED_STATE | NEED_TABLE)) return r;
  return launch_leaders(c, half_width, max_range, lead, gap, stream);
}

int t2d_set_lane_change(t2d_ctx* c, const t2d_lane_change_params* p, const int16_t* left, const int16_t* right,
                        int16_t* lane_path, int16_t* cooldown, int8_t* change) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (!p) {   // unbind
    c->lane.reset();
    return T2D_OK;
  }
  if (!(std::isfinite(p->politeness) && p->politeness >= 0.0))
    return fail(T2D_E_INVALID, "t2d_set_lane_change: politeness must be finite and >= 0");
  if (!std::isfinite(p->threshold)) return fail(T2D_E_INVALID, "t2d_set_lane_change: threshold must be finite");
  if (!(std::isfinite(p->b_safe) && p->b_safe > 0.0))
    return fail(T2D_E_INVALID, "t2d_set_lane_change: b_safe must be finite and > 0");
  if (!(std::isfinite(p->min_gap) && p->min_gap > 0.0))
    return fail(T2D_E_INVALID, "t2d_set_lane_change: min_gap must be finite and > 0");
  if (p->cooldown < 0 || p->cooldown > 32767) return fail(T2D_E_INVALID, "t2d_set_lane_change: cooldown must be in 0..32767");
  if (!left || !right || !lane_path || !cooldown)
    return fail(T2D_E_INVALID, "t2d_set_lane_change: left / right / lane_path / cooldown is NULL");
  if (!aligned2(lane_path) || !aligned2(cooldown))
    return fail(T2D_E_INVALID, "t2d_set_lane_change: lane_path and cooldown must be 2-byte aligned");
  if (int r = require(c, NEED_STATE | NEED_TABLE | NEED_CTRL | NEED_PATHS | NEED_SEARCH, "t2d_set_lane_change")) return r;
  if (!c->ctrl_path) return fail(T2D_E_STATE, "t2d_set_lane_change: the controllers have no path_id");
  if (c->reactive) return fail(T2D_E_STATE, "t2d_set_lane_change: a reactive replay is bound (lane changes on track paths are not supported)");
  if (p->min_gap > c->leader_max_range)
    return fail(T2D_E_INVALID, "t2d_set_lane_change: min_gap must not exceed the search's max_range");
  for (int q = 0; q < c->n_paths; ++q) {
    if (left[q] < -1 || left[q] >= c->n_paths || right[q] < -1 || right[q] >= c->n_paths)
      return fail(T2D_E_INVALID, "t2d_set_lane_change: a neighbour must be -1 or a path of the table");
    if (left[q] == q || right[q] == q) return fail(T2D_E_INVALID, "t2d_set_lane_change: a path cannot be its own neighbour");
  }
  CUDA_TRY(cudaSetDevice(c->device));
  auto L = std::make_unique<LaneChange>();
  L->p = *p;
  if (int r = upload(L->left, left, (size_t)c->n_paths)) return r;
  if (int r = upload(L->right, right, (size_t)c->n_paths)) return r;
  L->lane_path = lane_path; L->cooldown = cooldown; L->change = change;
  const size_t nm = (size_t)c->N * c->M;
  CUDA_TRY(cudaMemcpy(lane_path, c->ctrl_path, nm * sizeof(int16_t), cudaMemcpyDeviceToDevice));
  CUDA_TRY(cudaMemset(cooldown, 0, nm * sizeof(int16_t)));
  if (change) CUDA_TRY(cudaMemset(change, 0, nm));
  c->lane = std::move(L);
  return T2D_OK;
}

// ---- yielding (t2d_set_yielding / t2d_find_yields; K19)
// p's point at arc length clamp(s, 0, L): on the first segment of non-zero length that reaches s (the last one past L),
// x0 + t dx with t = (s - acc) / len and len = sqrt(dx dx + dy dy), the arc lengths of closest_on_path
static void point_at(const PathVertex* pv, int n_vert, double s, double& x, double& y) {
  double acc = 0.0;
  s = std::max(s, 0.0);
  x = pv[0].x; y = pv[0].y;
  for (int i = 0; i + 1 < n_vert; ++i) {
    const double dx = pv[i + 1].x - pv[i].x, dy = pv[i + 1].y - pv[i].y;
    const double l2 = dx * dx + dy * dy;
    if (!(l2 > 0.0)) continue;
    const double len = std::sqrt(l2);
    const double t = std::min((s - acc) / len, 1.0);
    x = pv[i].x + t * dx; y = pv[i].y + t * dy;
    if (s <= acc + len) return;
    acc = acc + len;
  }
}

int t2d_set_yielding(t2d_ctx* c, const t2d_yield_params* p, const t2d_conflict_zone* zones, const int32_t* zone_off,
                     const int16_t* priority, int16_t* yield_to, float* stop_gap) {
  const std::string fn = "t2d_set_yielding";
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (!p) {   // unbind
    c->yield.reset();
    return T2D_OK;
  }
  if (!(std::isfinite(p->critical_gap) && p->critical_gap > 0.0))
    return fail(T2D_E_INVALID, fn + ": critical_gap must be finite and > 0");
  if (!(std::isfinite(p->commit_decel) && p->commit_decel > 0.0))
    return fail(T2D_E_INVALID, fn + ": commit_decel must be finite and > 0");
  if (!(std::isfinite(p->v_min) && p->v_min > 0.0)) return fail(T2D_E_INVALID, fn + ": v_min must be finite and > 0");
  if (!zone_off || !yield_to || !stop_gap) return fail(T2D_E_INVALID, fn + ": zone_off / yield_to / stop_gap is NULL");
  if (!aligned2(yield_to) || !aligned4(stop_gap) || !aligned8(zones) || !aligned4(zone_off) || !aligned2(priority))
    return fail(T2D_E_INVALID, fn + ": yield_to, priority must be 2-byte, stop_gap, zone_off 4-byte and zones 8-byte aligned");
  if (int r = require(c, NEED_STATE | NEED_TABLE | NEED_CTRL | NEED_PATHS | NEED_SEARCH, fn.c_str())) return r;
  const int P = c->n_paths;
  if (zone_off[0] != 0) return fail(T2D_E_INVALID, fn + ": zone_off[0] must be 0");
  for (int k = 0; k < P; ++k)
    if (zone_off[k + 1] < zone_off[k]) return fail(T2D_E_INVALID, fn + ": zone_off must not decrease");
  const int Z = zone_off[P];
  if (Z > 0 && !zones) return fail(T2D_E_INVALID, fn + ": zones is NULL");
  for (int k = 0; k < P; ++k) {
    for (int z = zone_off[k]; z < zone_off[k + 1]; ++z) {
      const t2d_conflict_zone& r = zones[z];
      const std::string at = fn + ": zone " + std::to_string(z) + ": ";
      if (r.q < 0 || r.q >= P) return fail(T2D_E_INVALID, at + "q outside [0, n_paths)");
      if (r.q == k) return fail(T2D_E_INVALID, at + "q is the zone's own path");
      if (!(std::isfinite(r.s_in_p) && std::isfinite(r.s_out_p) && std::isfinite(r.s_in_q) && std::isfinite(r.s_out_q)))
        return fail(T2D_E_INVALID, at + "an arc length is not finite");
      if (!(r.s_in_p <= r.s_out_p && r.s_in_q <= r.s_out_q)) return fail(T2D_E_INVALID, at + "s_in > s_out");
      if (z > zone_off[k] && !(zones[z - 1].s_in_p <= r.s_in_p))
        return fail(T2D_E_INVALID, at + "the zones of a path must be sorted by s_in_p");
    }
  }
  std::vector<yield::Zone> dz((size_t)std::max(Z, 1));   // with the stop points, on the host copy of the table
  const std::vector<int>& off = c->path_off_host;
  for (int k = 0; k < P; ++k)
    for (int z = zone_off[k]; z < zone_off[k + 1]; ++z) {
      const t2d_conflict_zone& r = zones[z];
      yield::Zone& d = dz[z];
      d.s_in_p = r.s_in_p; d.s_in_q = r.s_in_q; d.s_out_q = r.s_out_q; d.q = r.q; d.reserved = 0;
      point_at(c->path_host.data() + off[k], off[k + 1] - off[k], r.s_in_p, d.stop_x, d.stop_y);
    }
  std::vector<int16_t> prio((size_t)P, 0);   // priority == NULL: all 0
  if (priority) std::copy(priority, priority + P, prio.begin());
  CUDA_TRY(cudaSetDevice(c->device));
  auto Y = std::make_unique<Yielding>();
  Y->p = *p;
  if (int r = upload(Y->zones, dz.data(), dz.size())) return r;
  if (int r = upload(Y->zone_off, zone_off, (size_t)P + 1)) return r;
  if (int r = upload(Y->priority, prio.data(), prio.size())) return r;
  if (int r = dev_alloc(Y->stop_xy, (size_t)c->N * c->M)) return r;
  Y->yield_to = yield_to; Y->stop_gap = stop_gap;
  c->yield = std::move(Y);
  return T2D_OK;
}

int t2d_find_yields(t2d_ctx* c, int16_t* yield_to, float* stop_gap, void* stream) {
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (!yield_to || !stop_gap) return fail(T2D_E_INVALID, "t2d_find_yields: yield_to / stop_gap is NULL");
  if (!aligned2(yield_to) || !aligned4(stop_gap))
    return fail(T2D_E_INVALID, "t2d_find_yields: yield_to must be 2-byte and stop_gap 4-byte aligned");
  if (int r = require(c, NEED_STATE | NEED_TABLE)) return r;
  if (!c->yield) return fail(T2D_E_STATE, "t2d_find_yields: no yielding bound: call t2d_set_yielding first");
  return launch_yields(c, yield_to, stop_gap, stream);
}

int t2d_set_log_reactive(t2d_ctx* c, const t2d_reactive_replay* r) {
  const std::string fn = "t2d_set_log_reactive";
  if (!c) return fail(T2D_E_INVALID, "ctx is NULL");
  if (!r) {   // unbind
    c->reactive.reset();
    return T2D_OK;
  }
  if (!r->track_path || !r->drive_row || !r->desired_speed || !r->drive_path || !r->slot_desired_speed)
    return fail(T2D_E_INVALID, fn + ": NULL array");
  if (!aligned2(r->drive_path) || !aligned4(r->slot_desired_speed))
    return fail(T2D_E_INVALID, fn + ": drive_path must be 2-byte and slot_desired_speed 4-byte aligned");
  const unsigned need = NEED_STATE | NEED_TABLE | NEED_LOG | NEED_CTRL | NEED_PATHS | NEED_PID | NEED_SEARCH;
  if (int e = require(c, need, fn.c_str())) return e;
  if (c->lane) return fail(T2D_E_STATE, fn + ": a lane change is bound (lane changes on track paths are not supported)");
  if (r->n_tracks != c->log->n_tracks)
    return fail(T2D_E_INVALID, fn + ": n_tracks must be the bound log's (" + std::to_string(c->log->n_tracks) + ")");
  for (int k = 0; k < r->n_tracks; ++k) {
    const std::string at = fn + ": track " + std::to_string(k) + ": ";
    const int p = r->track_path[k];
    if (p < -1 || p >= c->n_paths) return fail(T2D_E_INVALID, at + "track_path outside [-1, n_paths)");
    if (p < 0) continue;   // plain replay: its drive row and desired speed are not read
    const int row = r->drive_row[k];
    if (row >= c->n_types) return fail(T2D_E_INVALID, at + "drive_row outside the type table");
    const t2d_type_params& d = c->type_rows[row];
    const t2d_type_params& s = c->type_rows[c->log->track_type_host[k]];
    if (d.model == T2D_MODEL_STATIC) return fail(T2D_E_INVALID, at + "drive_row is a T2D_MODEL_STATIC row");
    if (d.shape != s.shape || d.half_len != s.half_len || d.half_wid != s.half_wid || d.radius != s.radius)
      return fail(T2D_E_INVALID, at + "drive_row has another shape or other extents than the track's row");
    if (!(std::isfinite(r->desired_speed[k]) && r->desired_speed[k] > 0.0f))
      return fail(T2D_E_INVALID, at + "desired_speed must be finite and > 0");
  }
  CUDA_TRY(cudaSetDevice(c->device));
  auto g = std::make_unique<ReactiveReplay>();
  if (int e = upload(g->track_path, r->track_path, (size_t)r->n_tracks)) return e;
  if (int e = upload(g->drive_row, r->drive_row, (size_t)r->n_tracks)) return e;
  if (int e = upload(g->desired_speed, r->desired_speed, (size_t)r->n_tracks)) return e;
  g->drive_path = r->drive_path; g->slot_desired_speed = r->slot_desired_speed;
  const size_t nm = (size_t)c->N * c->M;
  CUDA_TRY(cudaMemset(r->drive_path, 0xff, nm * sizeof(int16_t)));   // -1: no slot is reactive before a reset
  CUDA_TRY(cudaMemset(r->slot_desired_speed, 0, nm * sizeof(float)));
  c->reactive = std::move(g);
  return T2D_OK;
}

int t2d_exchange_create(t2d_exchange** out, int device, int world, int rank, int n_local, int slots, void* ipc_handle_out) {
  if (!out || !ipc_handle_out) return fail(T2D_E_INVALID, "out / ipc_handle_out is NULL");
  *out = nullptr;
  if (world < 1 || world > T2D_MAX_RANKS || rank < 0 || rank >= world) return fail(T2D_E_INVALID, "bad world / rank");
  if (n_local <= 0 || slots < 2 || slots > 64) return fail(T2D_E_INVALID, "n_local must be > 0 and slots in 2..64");
  static_assert(sizeof(cudaIpcMemHandle_t) == T2D_IPC_HANDLE_BYTES, "IPC handle size");
  CUDA_TRY(cudaSetDevice(device));
  t2d_exchange* x = new t2d_exchange();
  x->device = device; x->world = world; x->rank = rank; x->n_real = n_local; x->n_local = (n_local + 15) & ~15; x->slots = slots;
  x->threads = std::min(256, 32 * world);                 // one warp per peer
  if (const char* e = getenv("T2D_EXCHANGE_THREADS")) {   // experiments: a smaller CTA finds a home on a busy SM sooner
    const int v = atoi(e);
    if (v >= 32 && v <= 512 && v % 32 == 0 && v >= world) x->threads = v;
  }
  if (const char* e = getenv("T2D_EXCHANGE_TIMEOUT_MS")) {
    const double ms = atof(e);
    if (ms > 0.0) x->timeout_cycles = (long long)(ms * 2.0e6);   // ~2 GHz SM clock
  }
  x->bytes = x->flag_off() + (T2D_MAX_RANKS + 4) * sizeof(unsigned);
  cudaError_t e = cudaMalloc(&x->base, x->bytes);
  if (e == cudaSuccess) e = cudaMemset(x->base, 0, x->bytes);
  cudaIpcMemHandle_t h;
  if (e == cudaSuccess) e = cudaIpcGetMemHandle(&h, x->base);
  if (e != cudaSuccess) {
    if (x->base) cudaFree(x->base);
    delete x;
    return fail(T2D_E_CUDA, std::string("t2d_exchange_create: ") + cudaGetErrorString(e));
  }
  memcpy(ipc_handle_out, &h, sizeof(h));
  CUDA_TRY(cudaDeviceSynchronize());
  g_exchanges_alive.fetch_add(1);
  *out = x;
  return T2D_OK;
}

int t2d_exchange_connect(t2d_exchange* x, const void* handles) {
  if (!x || !handles) return fail(T2D_E_INVALID, "exchange / handles is NULL");
  CUDA_TRY(cudaSetDevice(x->device));
  for (int p = 0; p < x->world; ++p) {
    if (p == x->rank) { x->peer[p] = x->base; continue; }
    cudaIpcMemHandle_t h;
    memcpy(&h, static_cast<const unsigned char*>(handles) + (size_t)p * sizeof(h), sizeof(h));
    void* ptr = nullptr;
    const cudaError_t e = cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) {   // do not leak the mappings opened so far
      for (int q = 0; q < p; ++q)
        if (q != x->rank && x->peer[q]) { cudaIpcCloseMemHandle(x->peer[q]); x->peer[q] = nullptr; }
      return fail(T2D_E_CUDA, std::string("cudaIpcOpenMemHandle: ") + cudaGetErrorString(e));
    }
    x->peer[p] = static_cast<unsigned char*>(ptr);
  }
  x->connected = true;
  return T2D_OK;
}

int t2d_exchange_allgather_lagged(t2d_exchange* x, const uint8_t* done_local, uint8_t* dst, int lag, void* stream) {
  if (!x || !done_local || !dst) return fail(T2D_E_INVALID, "exchange / done_local / dst is NULL");
  if (!x->connected) return fail(T2D_E_STATE, "exchange not connected: call t2d_exchange_connect first");
  if (lag < 0 || 2 * lag + 2 > x->slots) return fail(T2D_E_INVALID, "lag needs a ring of at least 2 * lag + 2 slots");
  CUDA_TRY(cudaSetDevice(x->device));
  AllGatherArgs A{};
  for (int p = 0; p < x->world; ++p) A.peer[p] = x->peer[p];
  A.base = x->base; A.local = done_local; A.dst = dst;
  A.world = x->world; A.rank = x->rank; A.n_local = x->n_local; A.n_real = x->n_real; A.slots = x->slots;
  A.lag = lag; A.timeout = x->timeout_cycles;
  t2d_exchange_allgather_kernel<<<1, x->threads, 0, (cudaStream_t)stream>>>(A);
  g_launches.fetch_add(1);
  CUDA_TRY(cudaGetLastError());
  return T2D_OK;
}

int t2d_exchange_allgather(t2d_exchange* x, const uint8_t* done_local, uint8_t* dst, void* stream) {
  return t2d_exchange_allgather_lagged(x, done_local, dst, 0, stream);
}

int t2d_exchange_status(t2d_exchange* x, uint32_t* steps, uint32_t* timed_out) {
  if (!x) return fail(T2D_E_INVALID, "exchange is NULL");
  CUDA_TRY(cudaSetDevice(x->device));
  unsigned w[4];
  CUDA_TRY(cudaMemcpy(w, x->word(0), sizeof(w), cudaMemcpyDeviceToHost));
  if (steps) *steps = w[0];
  if (timed_out) *timed_out = w[3];
  return T2D_OK;
}

int t2d_exchange_destroy(t2d_exchange* x) {
  if (!x) return T2D_OK;
  cudaSetDevice(x->device);
  for (int p = 0; p < x->world; ++p)
    if (x->connected && p != x->rank && x->peer[p]) cudaIpcCloseMemHandle(x->peer[p]);
  if (x->base) cudaFree(x->base);
  g_exchanges_alive.fetch_sub(1);
  delete x;
  return T2D_OK;
}

int t2d_physics_step(int device, const t2d_type_params* params, int interval_ms, int delta_t_ms, int n, float* x, float* y,
                     float* heading, float* speed, float* vx, float* vy, float* omega_front, float* omega_rear,
                     const float* action, float* applied, void* stream) {
  if (!params) return fail(T2D_E_INVALID, "params is NULL");
  if (n < 0) return fail(T2D_E_INVALID, "n must be >= 0");
  if (n == 0) return T2D_OK;
  if (!x || !y || !heading || !speed || !vx || !vy || !action) return fail(T2D_E_INVALID, "t2d_physics_step: NULL array");
  if (interval_ms <= 0 || delta_t_ms <= 0) return fail(T2D_E_INVALID, "interval_ms and delta_t_ms must be > 0");
  if (params->model < 0 || params->model > T2D_MODEL_DRIFT) return fail(T2D_E_INVALID, "unknown model id");
  if (params->model == T2D_MODEL_DRIFT && !(omega_front && omega_rear))
    return fail(T2D_E_INVALID, "t2d_physics_step: SingleTrackDrift needs the wheel-speed arrays");
  CUDA_TRY(cudaSetDevice(device));
  PhysArgs A{};
  A.wheel_f = omega_front; A.wheel_r = omega_rear;
  {
    AbiParams a;
    memcpy(&a, params, sizeof(AbiParams));
    A.p = derive_params(a);
  }
  A.x = x; A.y = y; A.h = heading; A.v = speed; A.vx = vx; A.vy = vy; A.action = action; A.applied = applied;
  A.n = n;
  set_time_step(A, interval_ms, delta_t_ms);
  int sms = 0;
  CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
  t2d_physics_kernel<<<capped_grid(n, 256, sms, 8), 256, 0, (cudaStream_t)stream>>>(A);
  return launched();
}

}  // extern "C"
