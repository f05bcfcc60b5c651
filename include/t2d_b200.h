/*
 * t2d_b200.h - C ABI of the GPU-native (H100, sm_90a) batched env.step() hot path for tactics2d.
 *
 * The reference (WoodOxen/tactics2d, pure Python) has no FFI layer: its boundary for
 * this path is five duck-typed Python interfaces.  This library is what a ctypes
 * binding behind those interfaces calls; every entry point names the reference
 * interface it replaces (paths relative to the reference root):
 *
 *   t2d_physics_step     PhysicsModelBase.step            tactics2d/physics/physics_model_base.py:27-38
 *                        SingleTrackKinematics.step       tactics2d/physics/single_track_kinematics.py:178-198
 *                        SingleTrackDynamics.step         tactics2d/physics/single_track_dynamics.py:231-251
 *                        PointMass.step                   tactics2d/physics/point_mass.py:209-232
 *   t2d_set_type_table   ParticipantBase / templates      tactics2d/participant/element/participant_template.py:42-257,
 *                                                         vehicle.py:111-118,179-221, cyclist.py:76-94, pedestrian.py:70-88
 *   t2d_set_map          StaticCollision.reset / OutBound.reset
 *                                                         tactics2d/traffic/event_detection/collision.py:45-46, out_bound.py:50-65
 *   t2d_bind_wheel_state the omega_wf / omega_wr arguments of SingleTrackDrift.step
 *                                                         tactics2d/physics/single_track_drift.py:467-499
 *   t2d_bind_state       Trajectory.add_state / current state
 *                                                         tactics2d/participant/trajectory/trajectory.py:115-149
 *   t2d_step             ScenarioManager.update + check_status
 *                                                         tactics2d/traffic/scenario_manager.py:63-73,
 *                                                         tactics2d/envs/parking.py:352-392 (tick), :243-248 (done rule)
 *                        ParticipantBase.get_pose         tactics2d/participant/element/vehicle.py:263-281
 *                        DynamicCollision.update          tactics2d/traffic/event_detection/collision.py:18-25
 *                        StaticCollision.update           tactics2d/traffic/event_detection/collision.py:37-43
 *                        OutBound.update                  tactics2d/traffic/event_detection/out_bound.py:37-48
 *                        TimeExceed.update                tactics2d/traffic/event_detection/time_exceed.py:26-33
 *   t2d_set_goal         Arrival.update / NoAction.update  tactics2d/traffic/event_detection/arrival.py:32-47, no_action.py:32-53
 *   t2d_lidar_scan       SingleLineLidar._scan_obstacles   tactics2d/sensor/lidar.py:128-221
 *   t2d_lidar_scan_agents
 *                        (no reference counterpart: the reference's SingleLineLidar bound to each row's slot)
 *   t2d_set_bev_styles   the colour / z-order tables of MatplotlibRenderer   tactics2d/renderer/matplotlib_config.py,
 *                                                         sensor/camera.py:56-87 (style key of an element)
 *   t2d_bev_render       BEVCamera.update + MatplotlibRenderer.update / save_single_frame(return_array=True)
 *                                                         tactics2d/sensor/camera.py:333-386,
 *                                                         renderer/matplotlib_renderer.py:542-768
 *   t2d_bev_render_agents
 *                        (no reference counterpart: the reference's BEVCamera bound to each row's slot)
 *   t2d_set_controllers  IDMController / AccelerationController / PurePursuitController / PIDController objects
 *                                                         tactics2d/controller/idm_controller.py:33-58,
 *                                                         acceleration_controller.py:33-80, pure_pursuit_controller.py:26-49,
 *                                                         pid_controller.py:41-157
 *   t2d_set_paths        the `waypoints` LineString of PurePursuitController.step   pure_pursuit_controller.py:76,92
 *   t2d_set_pid          the PIDController keyword targets and its per-object state, per slot   pid_controller.py:126-132
 *   t2d_control          ControllerBase.step for every controlled participant
 *                                                         idm_controller.py:59-141, acceleration_controller.py:82-145,
 *                                                         pure_pursuit_controller.py:51-98, pid_controller.py:159-406
 *   t2d_set_leader_search / t2d_find_leaders
 *                        (no reference counterpart) the leader of every slot in its corridor, for the controllers'
 *                        `leading_state` / `front_state`
 *   t2d_set_lane_change  (no reference counterpart) MOBIL lane changes (Kesting, Treiber and Helbing 2007) for the IDM
 *                        rows with a lateral channel, decided on the device before every t2d_control
 *   t2d_set_yielding / t2d_find_yields
 *                        (no reference counterpart) yielding at the conflict zones of crossing and merging paths for
 *                        path-following IDM traffic, decided on the device before every t2d_control
 *   t2d_check_events     the same detectors on caller-supplied poses (no physics)
 *   t2d_reset            ScenarioManager.reset / ParticipantBase.reset
 *                                                         tactics2d/envs/parking.py:397-441, participant_base.py:236-246
 *   t2d_set_log          Trajectory.get_state / Vehicle.get_pose of logged participants at a frame
 *                                                         participant/trajectory/trajectory.py:97-113, vehicle.py:263-281
 *   t2d_set_log_schedule the same, with several tracks replayed one after the other in a slot
 *   t2d_set_log_reactive (no reference counterpart) reactive log agents: a track handed over to path-following IDM after
 *                        its first sample
 *   t2d_observe          (no reference counterpart) the ego-frame vector observation: ego motion, goal, nearest
 *                        participants and nearest map segments of every scenario's ego
 *   t2d_observe_agents   (no reference counterpart) the same observation seen from a list of observer slots per scenario,
 *                        for multi-agent control
 *   t2d_set_agents / t2d_agents_epilogue
 *                        (no reference counterpart) status, reward and retirement of every agent row of an observer list
 *   t2d_scatter_agent_action
 *                        (no reference counterpart) one action per agent row, written into its slot of the action array
 *   t2d_step_host_agents (no reference counterpart) the multi-agent step for a caller whose buffers live in host memory
 *   t2d_set_routes / t2d_bind_route_trackers
 *                        OffRoute.reset / OffRoute.update   tactics2d/traffic/event_detection/off_route.py:24-51
 *                        (+ a route-progress reward term, an extension)
 *   t2d_route_observe    (no reference counterpart) the route of each observer row in its frame, with look-ahead points
 *   t2d_set_history      Trajectory.add_state / Trajectory.reset(state) / history_states of every participant slot
 *                                                         tactics2d/participant/trajectory/trajectory.py:115-149,170-188
 *   t2d_observe_history  (no reference counterpart) the recent past of an observer and its agents in its current frame
 *
 * Conventions
 *   - plain pointers and sizes only; no torch / C++ types cross the ABI;
 *   - every function returns 0 on success or a negative T2D_E_* code; the message of the
 *     last error on the calling thread is t2d_last_error(); no exception crosses;
 *   - all array arguments of t2d_step / t2d_check_events / t2d_reset / t2d_physics_step are
 *     DEVICE pointers owned by the caller (PyTorch tensors' data_ptr()); the library never
 *     allocates or frees them.  t2d_set_type_table / t2d_set_map take HOST pointers and copy;
 *   - work is enqueued on the cudaStream_t passed as `stream` (NULL = legacy default
 *     stream) and the call returns without a host synchronisation;
 *   - a context belongs to one device and is not thread-safe.
 *
 * Layout: structure-of-arrays, scenario-major.  Participant (n, m) of an N x M world lives
 * at index n*M + m of every [N, M] array.  fp32 state, uint8 type ids, int16 hit indices.
 */
#ifndef T2D_B200_H
#define T2D_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define T2D_VERSION 100 /* 0.1.0 */

/* error codes */
#define T2D_OK 0
#define T2D_E_INVALID (-1)     /* bad argument */
#define T2D_E_CUDA (-2)        /* a CUDA runtime call failed; see t2d_last_error() */
#define T2D_E_UNSUPPORTED (-3) /* configuration outside what the kernels cover */
#define T2D_E_STATE (-4)       /* call order: state not bound, type table not set ... */

/* physics model ids (t2d_type_params.model) */
#define T2D_MODEL_KINEMATICS 0       /* SingleTrackKinematics  */
#define T2D_MODEL_DYNAMICS 1         /* SingleTrackDynamics    */
#define T2D_MODEL_POINTMASS_NEWTON 2 /* PointMass(backend="newton") */
#define T2D_MODEL_POINTMASS_EULER 3  /* PointMass(backend="euler")  */
#define T2D_MODEL_STATIC 4           /* no motion (Obstacle, obstacle.py:14-19) */
#define T2D_MODEL_DRIFT 5            /* SingleTrackDrift (built-in tyre); needs t2d_bind_wheel_state */

/* collision shape ids (t2d_type_params.shape) */
#define T2D_SHAPE_OBB 0    /* Vehicle / Cyclist / Other bounding box, vehicle.py:132-142 */
#define T2D_SHAPE_CIRCLE 1 /* Pedestrian ((x, y), width/2), pedestrian.py:85-88 */
#define T2D_SHAPE_NONE 2   /* takes part in physics only */

#define T2D_TYPE_INACTIVE 255 /* type id of an empty participant slot */
#define T2D_MAX_TYPES 64
#define T2D_MAX_PARTICIPANTS 128 /* per scenario (one warp spans a scenario) */
#define T2D_MAX_SEGMENTS 32767   /* hit_segment is int16 */
#define T2D_MAX_RANKS 16         /* GPUs of one node sharing a done exchange */
#define T2D_IPC_HANDLE_BYTES 64  /* sizeof(cudaIpcMemHandle_t) */

/* per-participant event byte (t2d_step `flags`) */
#define T2D_F_DYNAMIC 1  /* TrafficStatus.COLLISION_DYNAMIC, status.py:55 */
#define T2D_F_STATIC 2   /* TrafficStatus.COLLISION_STATIC,  status.py:54 */
#define T2D_F_OUTBOUND 4 /* ScenarioStatus.OUT_BOUND,        status.py:26 */

/* scenario status byte = ScenarioStatus, tactics2d/traffic/status.py:23-28 */
#define T2D_STATUS_NORMAL 1
#define T2D_STATUS_COMPLETED 2
#define T2D_STATUS_TIME_EXCEEDED 3
#define T2D_STATUS_OUT_BOUND 4
#define T2D_STATUS_NO_ACTION 5
#define T2D_STATUS_FAILED 6

/* t2d_config.flags */
#define T2D_CFG_ANY_PARTICIPANT 1 /* any active participant's event ends the scenario (default: only participant 0, the ego) */
#define T2D_CFG_STEER_FIRST 2     /* action[...,0] is steering, [...,1] acceleration (env order, parking.py:239) */

typedef struct t2d_ctx t2d_ctx;

typedef struct t2d_config {
  int32_t interval_ms; /* State.frame advance per step; ScenarioManager.step_size (scenario_manager.py:50) */
  int32_t delta_t_ms;  /* Euler sub-step; PhysicsModelBase._DELTA_T = 5 (physics_model_base.py:23) */
  int32_t max_step;    /* TimeExceed.max_step; <= 0 disables the check */
  int32_t flags;       /* T2D_CFG_* */
} t2d_config;

/* One row per participant type.  Ranges are [lo, hi]; "no constraint" (the reference's
 * None) is (-INFINITY, +INFINITY). */
typedef struct t2d_type_params {
  float half_len, half_wid; /* OBB half extents (length/2, width/2) */
  float radius;             /* circle radius (width/2) */
  float lf, lr;             /* axle distances from the geometry centre */
  float steer_lo, steer_hi;
  float speed_lo, speed_hi;
  float accel_lo, accel_hi;
  float mass, mass_height, mu, I_z, cf, cr; /* SingleTrackDynamics only */
  int32_t model;                            /* T2D_MODEL_* */
  int32_t shape;                            /* T2D_SHAPE_* */
  float wheel_radius, T_sb, T_se, I_yw;     /* SingleTrackDrift only (single_track_drift.py:98-107: 0.344, 0.76, 1, 1.7);
                                               the drift model also reads lf, lr, mass, I_z and the three ranges */
} t2d_type_params;

int t2d_version(void);
const char* t2d_last_error(void);

int t2d_create(t2d_ctx** out, int device, int n_scenarios, int m_participants, const t2d_config* cfg);
int t2d_destroy(t2d_ctx* ctx);
int t2d_set_config(t2d_ctx* ctx, const t2d_config* cfg);

/* HOST pointers; copied. */
int t2d_set_type_table(t2d_ctx* ctx, const t2d_type_params* table, int n_types);
/* segments: host float[n_seg][4] = (x1, y1, x2, y2), collidable map polyline pieces in list
 * order (the order defines "first hit"); bounds: host float[4] = (xmin, xmax, ymin, ymax) as
 * Map.boundary gives it, or NULL for no out-of-bound check; cell_size: broadphase grid pitch
 * in metres (<= 0: choose automatically). */
int t2d_set_map(t2d_ctx* ctx, const float* segments, int n_seg, const float* bounds, float cell_size);

/* Static objects that are AREAS, and a different map per scenario.
 * StaticCollision.update tests `agent_pose.intersects(static_object.geometry)` against a list of static objects
 * (traffic/event_detection/collision.py:37-43); in the reference's envs those are Area polygons - the walls and obstacles
 * of a parking lot, regenerated by every reset (envs/parking.py:397-441) - and a pose wholly inside a polygon intersects
 * it without touching an edge.  poly_start (host int32 [n_poly + 1], ascending) marks the segments that close up to
 * rings: ring p = segments [poly_start[p], poly_start[p + 1]), each edge ending where the next begins and the last at the
 * first one's start (Area.geometry's exterior); segments outside every ring are open polyline pieces (RoadLine).
 * With rings present, hit_segment names the first OBJECT hit in list order by its first segment: poly_start[p] for ring p
 * (an edge of it was touched, or the pose centre lies inside it), the segment itself for an open piece. */
int t2d_set_map_polygons(t2d_ctx* ctx, const float* segments, int n_seg, const int32_t* poly_start, int n_poly,
                         const float* bounds, float cell_size);
/* One tile = the static objects + boundary of one map (host arrays, copied).  tile_id: DEVICE uint16 [N], owned by the
 * caller and read by every tick: the tile of each scenario (may be rewritten between ticks, e.g. by a reset that draws a
 * new parking lot); NULL is allowed when n_tiles == 1.  Every scenario then collides with its own tile's objects, is
 * bounded by its own tile's box, and t2d_lidar_scan sees its own tile's segments.
 * t2d_set_map / t2d_set_map_polygons / t2d_set_map_table: n_tiles == 0 (no segments and no bounds) unbinds.  Rejected
 * (the previous map, its tile_id and its per-segment BEV styles stay bound): any malformed tile. */
#define T2D_MAX_TILES 4096
typedef struct {
  const float* segments;     /* [n_seg][4] */
  int32_t n_seg;
  const int32_t* poly_start; /* [n_poly + 1] or NULL */
  int32_t n_poly;
  const float* bounds;       /* [4] xmin, xmax, ymin, ymax or NULL */
} t2d_map_tile;
int t2d_set_map_table(t2d_ctx* ctx, const t2d_map_tile* tiles, int n_tiles, const uint16_t* tile_id, float cell_size);

/* DEVICE pointers, each [N, M] (step_count: [N]); read and written in place by t2d_step. */
int t2d_bind_state(t2d_ctx* ctx, float* x, float* y, float* heading, float* speed, float* vx, float* vy,
                   const uint8_t* type_id, int32_t* step_count);

/* SingleTrackDrift carries two more state variables per participant, the front / rear wheel angular speeds that
 * SingleTrackDrift.step takes and returns (single_track_drift.py:467-499).  DEVICE pointers [N, M], read and written in
 * place by t2d_step for participants whose type has model T2D_MODEL_DRIFT; required only when the type table holds
 * such a row. */
int t2d_bind_wheel_state(t2d_ctx* ctx, float* omega_front, float* omega_rear);

/* One tick of all N scenarios.  action: [N, M, 2] fp32.  Outputs (any may be NULL):
 * flags [N, M] uint8, hit_index [N, M] int16 (lowest colliding participant or -1),
 * hit_segment [N, M] int16 (lowest colliding map segment or -1), scn_status [N] uint8,
 * done [N] uint8. */
int t2d_step(t2d_ctx* ctx, const float* action, uint8_t* flags, int16_t* hit_index, int16_t* hit_segment,
             uint8_t* scn_status, uint8_t* done, void* stream);

/* The same tick for a caller whose buffers live in HOST memory - what a ctypes / numpy binding of the reference's
 * env.step(action) -> (..., terminated, truncated, info["status"]) would hand over (envs/parking.py:444-468).
 * action_host: [N, M, 2] fp32 (pinned memory recommended), scn_status_host / done_host: [N] uint8 in host memory
 * (either may be NULL); flags / hit_index / hit_segment stay DEVICE arrays as in t2d_step (any may be NULL).
 * The library stages the actions in chunks of whole scenarios on its own copy stream so that the host->device copy of
 * one chunk runs under the kernel of the previous one, reads status + done back in one device->host copy and
 * synchronises `stream` before returning: the host arrays are valid on return. */
int t2d_step_host(t2d_ctx* ctx, const float* action_host, uint8_t* flags, int16_t* hit_index, int16_t* hit_segment,
                  uint8_t* scn_status_host, uint8_t* done_host, void* stream);

/* The detectors alone on the bound poses (x, y, heading); no physics, no step counting. */
int t2d_check_events(t2d_ctx* ctx, uint8_t* flags, int16_t* hit_index, int16_t* hit_segment, void* stream);

/* Arrival (tactics2d/traffic/event_detection/arrival.py:32-47) and NoAction (no_action.py:32-53) for the ego
 * (participant 0) of every scenario, evaluated inside t2d_step.  All pointers are DEVICE arrays owned by the caller:
 * target [N][5] = (cx, cy, heading, half_len, half_wid) of the target-area rectangle (NULL disables both detectors),
 * iou_out [N] receives IoU(ego pose, target) (Arrival.update's second return value), last_pose [N][4] and
 * no_action_count [N] are the detector state (zero them before the first step; t2d_reset clears them).
 * arrival_threshold: IoU >= threshold -> T2D_STATUS_COMPLETED (reference 0.95); no_action_max_step: more than that
 * many consecutive ticks with IoU(pose, previous pose) > 0.999 -> T2D_STATUS_NO_ACTION (reference 100; <= 0 disables).
 * Status priority (envs/parking.py:361-392): time exceeded, no action, out of bound, collision, completed. */
int t2d_set_goal(t2d_ctx* ctx, const float* target, float arrival_threshold, int no_action_max_step, float* iou_out,
                 float* last_pose, int32_t* no_action_count);

/* Masked re-initialisation (ScenarioManager.reset, envs/parking.py:397-441; ParticipantBase.reset): for every scenario n
 * with mask[n] != 0 copy row pool_index[n] (row n when pool_index is NULL) of the [n_pool, M] pool arrays into the bound
 * state and zero step_count[n]; pool_vx / pool_vy may be NULL (then speed x (cos, sin)(heading)).  Everything else the
 * world owns per participant starts fresh too: the NoAction detector state of t2d_set_goal, the controllers' last_accel
 * (0), the PID state of t2d_set_pid (0), and the SingleTrackDrift wheel speeds bound with t2d_bind_wheel_state - from the pool columns of
 * t2d_bind_reset_wheel_pool when bound, else free rolling (speed / wheel_radius).  With agents bound (t2d_set_agents)
 * the retired slots take their types back and the per-row NoAction state is cleared. */
int t2d_reset(t2d_ctx* ctx, const uint8_t* mask, const int32_t* pool_index, int n_pool, const float* pool_x,
              const float* pool_y, const float* pool_heading, const float* pool_speed, const float* pool_vx,
              const float* pool_vy, void* stream);
/* Optional initial wheel speeds for t2d_reset: DEVICE arrays [n_pool][M] indexed like the other pool columns (NULL, NULL unbinds). */
int t2d_bind_reset_wheel_pool(t2d_ctx* ctx, const float* pool_omega_front, const float* pool_omega_rear);

/* ---- sampled resets: a seeded pool-row draw and collision-checked random start states -------------------------------
 * ParkingEnv.reset draws a new start state on every reset (envs/parking.py:397-441) and keeps a draw only when the
 * vehicle's box meets no obstacle and not the target area (ParkingLotGenerator._verify_start_state,
 * map/generator/generate_parking_lot.py:231-237).  The contract is DESIGN.md section 1 "Sampled resets":
 *   draws      Philox4x32-10, key (seed low, seed high), counter (d, n, episode[n], 0);
 *   row        d = 0: row = (u0 * P) >> 32 over the P pool rows (sample_rows; else row n), written to pool_row[n];
 *   columns    the optional DEVICE pools are copied from the row into what they belong to: pool_type_id [n_rows][M] into
 *              the bound type_id (with agents bound the scenario's retired list is cleared), pool_target [n_rows][5] into
 *              the t2d_set_goal target, pool_tile_id [n_rows] into the map table's tile_id (ids < n_tiles at every
 *              sampled reset: the library does not read the device pool to check them),
 *              pool_route_id [n_rows][M] into the t2d_set_routes route_id;
 *   jitter     after K2 (and K7) slot m = 0 .. M-1 of every masked scenario, unless inactive or retired or its jitter row
 *              is all zero, tries t < tries with draw d = 1 + 32 m + t: (x + dx, y + dy, wrap(h + dh), v + dv), dx ... from
 *              the (lo, hi) ranges of jitter[m] (HOST fp32 [M][4][2], copied; NULL: none).  The lowest t whose pose is
 *              inside its tile's box, meets no collidable segment or Area of its tile and no other active slot at its
 *              current state (and, for slot 0 with avoid_target, not the goal target) wins; reset_try[n][m] = t, or -1
 *              when no try is accepted (the pool state is kept) or the slot is not jittered.  A moved slot's vx, vy are
 *              v (cos h, sin h); a moved SingleTrackDrift slot rolls freely (v / wheel_radius), or keeps the wheel speeds
 *              of a bound t2d_bind_reset_wheel_pool;
 *   episode    [N] uint32, zeroed when a sampler is bound; each sampled reset of scenario n draws with e = episode[n]
 *              and then increments it.
 * episode [N], pool_row [N] int32 and reset_try [N][M] int8 are caller-owned DEVICE buffers that must stay alive while
 * bound.  NULL unbinds.  Rejected (the previous sampler stays bound): tries outside 1..32, a NULL episode / pool_row /
 * reset_try, row pools with n_rows <= 0, a jitter range that is not finite or has lo > hi (T2D_E_INVALID); a pool whose
 * destination is not bound (T2D_E_STATE). */
typedef struct t2d_reset_sampler {
  uint64_t seed;
  int32_t sample_rows;            /* 1: draw the row; 0: scenario n runs pool row n */
  int32_t tries;                  /* 1..32 */
  int32_t avoid_target;           /* slot 0 must not meet its goal target */
  int32_t n_rows;                 /* rows of the pools below (the reset's n_pool must match) */
  const float* jitter;            /* HOST [M][4][2] or NULL */
  const uint8_t* pool_type_id;    /* DEVICE [n_rows][M] or NULL */
  const float* pool_target;       /* DEVICE [n_rows][5] or NULL */
  const uint16_t* pool_tile_id;   /* DEVICE [n_rows] or NULL */
  const int16_t* pool_route_id;   /* DEVICE [n_rows][M] or NULL */
  uint32_t* episode;              /* DEVICE [N] */
  int32_t* pool_row;              /* DEVICE [N] */
  int8_t* reset_try;              /* DEVICE [N][M] */
} t2d_reset_sampler;
int t2d_set_reset_sampler(t2d_ctx* ctx, const t2d_reset_sampler* sampler);
/* A sampled reset of the scenarios with mask[n] != 0 (envs/parking.py:397-441, generate_parking_lot.py:231-237): K13
 * (row draw, row-owned columns), t2d_reset with pool_index = pool_row (K2, then K7 with a log: the drawn row is the
 * replayed one), K14 (jitter).  Pool arguments as t2d_reset's.  Rejected without a launch: whatever t2d_reset rejects,
 * no sampler bound or a pool destination no longer bound (T2D_E_STATE), row pools with n_pool != n_rows, no row draws
 * with n_pool < N (T2D_E_INVALID). */
int t2d_reset_sampled(t2d_ctx* ctx, const uint8_t* mask, int n_pool, const float* pool_x, const float* pool_y,
                      const float* pool_heading, const float* pool_speed, const float* pool_vx, const float* pool_vy,
                      void* stream);

/* ---- log replay: recorded tracks drive participants around a simulated ego ------------------------------------------
 * Trajectory.get_state(frame) / Vehicle.get_pose(frame) (participant/trajectory/trajectory.py:97-113,
 * participant/element/vehicle.py:263-281) for every replayed slot of every scenario, on the device.  The contract
 * (sampling, interpolation between frames, absent tracks) is DESIGN.md section 1 "Log replay".
 * A track k is present on [first_ms[k], first_ms[k] + (n_frames[k] - 1) * period_ms[k]] and holds n_frames[k] records
 * (x, y, heading, vx, vy), fp32, in records starting at record sum(n_frames[0..k-1]).  Its type_row must be a
 * T2D_MODEL_STATIC row of the type table: the tick then only builds the pose of a replayed slot and checks it like any
 * other participant.  Episode row p starts at t0_ms[p] and binds slot m to track row_track[p * M + m] (-1: not
 * replayed; a track at most once per row).  Before every tick, scenario n samples its row log_row[n] at
 * t = t0_ms[row] + (step_count[n] + 1) * interval_ms, the time the tick produces: a replayed slot takes the track's
 * state at t, and type_id T2D_TYPE_INACTIVE while the track is absent.  t2d_check_events does not replay.
 * t2d_reset sets log_row[n] = pool_index[n] (n without pool_index) for the masked scenarios, needs n_pool == n_rows,
 * and samples those scenarios at t0 at once.  While a log is bound the tick keeps every static slot's vx, vy. */
typedef struct t2d_log {
  int32_t n_tracks;           /* >= 1 */
  const int32_t* first_ms;    /* HOST [n_tracks] time stamp of the first record */
  const int32_t* n_frames;    /* HOST [n_tracks] >= 1 */
  const int32_t* period_ms;   /* HOST [n_tracks] > 0 */
  const uint8_t* type_row;    /* HOST [n_tracks] type-table row, model T2D_MODEL_STATIC */
  const float* records;       /* HOST [sum n_frames][5] x, y, heading, vx, vy; finite */
  int32_t n_rows;             /* >= 1 */
  const int32_t* t0_ms;       /* HOST [n_rows] */
  const int32_t* row_track;   /* HOST [n_rows][M] in [-1, n_tracks); NULL for t2d_set_log_schedule */
  int32_t* log_row;           /* DEVICE [N], caller-owned: the row each scenario runs */
  uint8_t* type_id;           /* DEVICE [N][M]: the type_id array of t2d_bind_state - the replay writes it, so the
                                 writable pointer is passed here and must equal the bound one */
} t2d_log;
/* Host arrays are copied.  NULL unbinds.  Rejected (the previous log stays bound): malformed tables, a non-static track
 * row, a type_id other than the bound one.  A later t2d_set_type_table that makes a track's row non-static is
 * rejected too. */
int t2d_set_log(t2d_ctx* ctx, const t2d_log* log);
/* Slot schedules (DESIGN.md section 1 "Log replay", "Slot schedules"): slot m of row p replays, one after the other,
 * the tracks slot_track[slot_off[p * M + m] .. slot_off[p * M + m + 1]), whose presence intervals [first, last] must be
 * strictly increasing and disjoint (last of an entry < first of the next).  At sample time t the slot shows the entry
 * present at t, else T2D_TYPE_INACTIVE with its state untouched; t2d_set_log's row_track is the case of at most one
 * entry per slot.  log->row_track must be NULL; every other field is checked as t2d_set_log checks it.
 *   slot_off    HOST int32 [n_rows * M + 1], slot_off[0] == 0, monotone, slot_off[n_rows * M] == n_entries
 *   slot_track  HOST int32 [n_entries] in [0, n_tracks); a track at most once per row, over all the row's slots;
 *               every scheduled track's last stamp must fit int32 ms
 *   track_out   optional caller-owned DEVICE int32 [N][M]: every replay launch (ticks, t2d_step_host chunks, t2d_reset)
 *               writes the track each slot it samples shows, -1 while the slot shows none or is not replayed
 * Host arrays are copied.  Rejected (the previous log stays bound): any malformed field. */
int t2d_set_log_schedule(t2d_ctx* ctx, const t2d_log* log, const int32_t* slot_off, const int32_t* slot_track,
                         int32_t n_entries, int32_t* track_out);
/* Reactive replay (DESIGN.md section 1 "Reactive replay"): a track k with track_path[k] >= 0 is reactive.  At every
 * replay launch that samples a slot showing a reactive track k at time t (the sample time above):
 *   handover   (reset mode, or t - interval_ms < first_ms[k] <= t in tick mode): the slot is posed from the log and takes
 *              type_row[k] exactly as plain replay does, and drive_path[n][m] = track_path[k],
 *              slot_desired_speed[n][m] = desired_speed[k], the lateral PID state pid_state[n][m][0:3] (t2d_set_pid) and
 *              last_accel[n][m] (t2d_set_controllers) are zeroed.  The tick does not integrate this static row.
 *   simulated  (every later sample up to the track's last stamp): the state is left alone, type_id = drive_row[k] (the
 *              tick integrates it with K5's action), drive_path and slot_desired_speed as at the handover.
 * After the last stamp the slot is T2D_TYPE_INACTIVE as in plain replay.  Every other slot the launch samples (plain
 * tracks, absent tracks, slots without a track, the ego) gets drive_path = -1.  K17 and K5 read drive_path instead of the
 * controllers' path_id, and K5's IDM rows take slot_desired_speed instead of the row's desired_speed where drive_path >=
 * 0; the caller gives those slots an IDM row with a PATH lateral channel.
 *   track_path          HOST int16 [n_tracks] a path of t2d_set_paths, -1: plain replay
 *   drive_row           HOST uint8 [n_tracks] for a reactive track a row of the type table that is not
 *                       T2D_MODEL_STATIC, with type_row[k]'s shape, half_len, half_wid and radius (not read otherwise)
 *   desired_speed       HOST float [n_tracks] finite and > 0 on a reactive track (m/s; not read otherwise)
 *   drive_path          DEVICE int16 [N][M], caller-owned, 2-byte aligned; set to -1 by the call
 *   slot_desired_speed  DEVICE float [N][M], caller-owned, 4-byte aligned; set to 0 by the call
 * Host arrays are copied.  NULL unbinds; with nothing bound every launch is the plain one.  t2d_set_log,
 * t2d_set_log_schedule, t2d_set_paths, t2d_set_controllers, t2d_set_type_table and unbinding the leader search drop the
 * binding; t2d_set_lane_change is rejected while it is bound.  Rejected (the previous binding stays whole): n_tracks
 * other than the log's, a NULL array, a track_path entry outside [-1, n_paths), a drive_row of a reactive track outside
 * the table, static or of another shape or extents, a desired speed that is not finite and > 0, misaligned device arrays
 * (T2D_E_INVALID); state, type table, log, controllers, paths, PID state or leader search not bound, or a lane change
 * bound (T2D_E_STATE).  The history ring (t2d_set_history) does not keep a reactive slot's handover entry: its type id
 * changes on the next tick. */
typedef struct t2d_reactive_replay {
  int32_t n_tracks;               /* the bound log's n_tracks */
  const int16_t* track_path;      /* HOST [n_tracks] */
  const uint8_t* drive_row;       /* HOST [n_tracks] */
  const float* desired_speed;     /* HOST [n_tracks] */
  int16_t* drive_path;            /* DEVICE [N][M] */
  float* slot_desired_speed;      /* DEVICE [N][M] */
} t2d_reactive_replay;
int t2d_set_log_reactive(t2d_ctx* ctx, const t2d_reactive_replay* replay);

/* Single-line lidar of the ego (participant 0) of every scenario: SingleLineLidar._scan_obstacles
 * (tactics2d/sensor/lidar.py:128-221).  n_beams = point_density (lidar.py:49), max_range = perception range;
 * beam_cos_sin: DEVICE double [n_beams][2] = (cos, sin) of the beam angles linspace(0, 2 pi, n_beams, endpoint=False)
 * (lidar.py:160); scan: DEVICE float [N][n_beams], +inf where nothing is hit within the range.  Obstacles are the map
 * segments given to t2d_set_map and the pose rings of the other box-shaped participants. */
int t2d_lidar_scan(t2d_ctx* ctx, int n_beams, float max_range, const double* beam_cos_sin, float* scan, void* stream);

/* Per-agent lidar: t2d_lidar_scan with the sensor on any list of observer slots per scenario (the reference's
 * SingleLineLidar bound with bind_with(j) to each row's slot; DESIGN.md section 1 "Per-agent lidar").  Row (n, q), q < Q =
 * n_observers (1..T2D_OBS_MAX_OBSERVERS), is the scan from slot j = observers[n][q] at its fp32 (x, y, heading), whatever
 * j's shape: the beams are in j's frame, the obstacles are the scenario's map segments and the pose rings of every other
 * active box-shaped slot, slot 0 included.  observers: DEVICE int16 [N][Q], or NULL for slot q in row q of every scenario
 * (needs Q <= M).  A value outside [0, M) or an empty slot (type_id >= n_types, a retired one included) gives an absent
 * row (every beam +inf); duplicates give identical rows.  beam_cos_sin as t2d_lidar_scan; scan: DEVICE float
 * [N][Q][n_beams] (64-bit offsets: N·Q·n_beams may exceed 2^31).  With observers NULL and Q = 1 the call is
 * t2d_lidar_scan.  Rejected without a launch: n_observers outside 1..128, observers == NULL with n_observers > M,
 * n_beams <= 0, max_range not > 0 (NaN included), beam_cos_sin or scan NULL (T2D_E_INVALID), state or type table not bound
 * (T2D_E_STATE), more than 2^33 rows (T2D_E_UNSUPPORTED).  One launch, no allocation, no synchronisation: capturable in
 * a CUDA graph. */
int t2d_lidar_scan_agents(t2d_ctx* ctx, const int16_t* observers /* DEVICE [N][Q] or NULL */, int32_t n_observers /* Q */,
                          int n_beams, float max_range, const double* beam_cos_sin, float* scan /* DEVICE [N][Q][n_beams] */,
                          void* stream);

/* ---- bird's-eye-view observation of the ego of every scenario ------------------------------------------------------
 * t2d_set_bev_styles + t2d_bev_render replace BEVCamera.update (tactics2d/sensor/camera.py:333-386) followed by
 * MatplotlibRenderer.update / save_single_frame(return_array=True) (renderer/matplotlib_renderer.py:542-768): the
 * 200 x 200 x 3 uint8 observation of ParkingEnv / RacingEnv (envs/parking.py:130, racing.py:102).  The contract, and
 * where it deliberately differs from the reference's renderer, is DESIGN.md section 1 "BEV observation".
 * A style is a colour, a z order (larger is drawn on top; equal z keeps the draw order) and the stroke width in points
 * that open map segments of that style are drawn with (the renderer's 200 dpi: w = line_width_pt * 200 / 72 pixels).
 * Rows with a fixed meaning: */
#define T2D_MAX_BEV_STYLES 64
#define T2D_BEV_STYLE_BACKGROUND 0 /* pixels no primitive covers */
#define T2D_BEV_STYLE_ARROW 1      /* the heading triangle of every drawn box participant */
#define T2D_BEV_STYLE_RING 2       /* a map ring object without a per-segment style */
#define T2D_BEV_STYLE_OPEN 3       /* an open map segment without a per-segment style */
#define T2D_BEV_NOT_DRAWN 255
typedef struct t2d_bev_style {
  uint8_t r, g, b;
  int8_t z;
  float line_width_pt;
} t2d_bev_style;
/* HOST arrays, copied.  table: n_styles rows (4..T2D_MAX_BEV_STYLES); type_style [n_types]: the style of every
 * participant type (T2D_BEV_NOT_DRAWN: not drawn; box types are drawn as their pose ring plus the heading triangle, disc
 * types as their disc, SHAPE_NONE types never); seg_style [n_seg_total]: the style of every map segment of the current
 * map, tiles back to back in tile order (a ring object takes the style of its first segment), or NULL for the defaults
 * T2D_BEV_STYLE_RING / T2D_BEV_STYLE_OPEN; target_style: the style of the t2d_set_goal rectangle (T2D_BEV_NOT_DRAWN: not
 * drawn).  t2d_set_map / t2d_set_map_polygons / t2d_set_map_table drop the per-segment styles back to the defaults. */
int t2d_set_bev_styles(t2d_ctx* ctx, const t2d_bev_style* table, int n_styles, const uint8_t* type_style,
                       const uint8_t* seg_style, int n_seg_total, int target_style);
/* Renders every scenario's view into out: DEVICE uint8 [N][height][width][3] RGB when rgb != 0, else [N][height][width]
 * style indices (RGB = the style's colour).  range: HOST float [4] = (left, right, front, back) in metres, each in
 * (0, 1e5]; width, height in 1..1024.  One launch, no allocation, no synchronisation: capturable in a CUDA graph. */
int t2d_bev_render(t2d_ctx* ctx, int width, int height, const float* range, int rgb, uint8_t* out, void* stream);
/* Per-agent BEV: t2d_bev_render seen from any list of observer slots per scenario (no reference counterpart: the
 * reference's BEVCamera bound to each row's slot, sensor_base.py:89-95; DESIGN.md section 1 "Per-agent BEV").  Row (n, q),
 * q < Q = n_observers (1..T2D_OBS_MAX_OBSERVERS), is the view centred on slot j = observers[n][q] at its fp32 (x, y,
 * heading), +x along its heading, whatever j's shape; it draws what t2d_bev_render draws for the scenario, j's own body
 * included.  observers: DEVICE int16 [N][Q], or NULL for slot q in row q (needs Q <= M).  A value outside [0, M) or an
 * empty slot (type_id >= n_types, a retired one included) gives an absent row: every pixel the background (style 0); it
 * does not take t2d_bev_render's no-ego view.  goals: DEVICE float [N][Q][5] (cx, cy, heading, half_len, half_wid), the
 * goal rectangle of every row (NaN cx: none), or NULL: the rows observed by slot 0 draw the t2d_set_goal target, the
 * others none; drawn in the target style either way.  out: DEVICE uint8 [N][Q][height][width][3] RGB, or
 * [N][Q][height][width] style indices (64-bit offsets).  A row observed by slot 0 without goals equals t2d_bev_render's
 * image whenever slot 0 is present.  Rejected without a launch: what t2d_bev_render rejects, n_observers outside
 * 1..128, observers == NULL with n_observers > M (T2D_E_INVALID), N·Q above 2^31 - 1 (T2D_E_UNSUPPORTED).  One launch, no
 * allocation, no synchronisation: capturable in a CUDA graph. */
int t2d_bev_render_agents(t2d_ctx* ctx, const int16_t* observers /* DEVICE [N][Q] or NULL */, int32_t n_observers /* Q */,
                          const float* goals /* DEVICE [N][Q][5] or NULL */, int width, int height,
                          const float* range /* HOST [4] */, int rgb, uint8_t* out /* DEVICE [N][Q][H][W](3) */,
                          void* stream);

/* ---- vector observation of the ego of every scenario -----------------------------------------------------------------
 * One fp32 row of F = 16 + 11 k_agents + 9 k_segments values per scenario, everything in the frame of participant 0 (origin
 * at its centre, +x along its heading).  The contract is DESIGN.md section 1 "Vector observation".  Blocks in this order:
 *   ego      [8]  valid, speed, v_long, v_lat, half_len, half_wid, is_disc, t_frac (= step_count / max_step, 0 without one)
 *   goal     [8]  valid, ex, ey, cos dh, sin dh, half_len, half_wid, dist   (the t2d_set_goal target; zeros without one)
 *   agents   [K][11] valid, ex, ey, cos dh, sin dh, v_x, v_y, half_len, half_wid, is_disc, dist: the K nearest other
 *                 participants (slots >= 1, active, shape not NONE) whose centre lies within agent_range, by (d^2, slot)
 *   segments [S][9]  valid, ex1, ey1, ex2, ey2, ecx, ecy, dist, in_ring: the S nearest segments of the scenario's map tile
 *                 within segment_range of the ego centre, by (d^2, segment index); (ecx, ecy) is the closest point
 * Absent and padding rows are zeros with index -1; with the ego slot empty the whole row is zeros. */
#define T2D_OBS_MAX_AGENTS 127
#define T2D_OBS_MAX_SEGMENTS 256
typedef struct t2d_obs_config {
  int32_t k_agents;    /* 0..T2D_OBS_MAX_AGENTS */
  int32_t k_segments;  /* 0..T2D_OBS_MAX_SEGMENTS */
  float agent_range;   /* metres, (0, 1e5]; closed: d^2 <= r^2 in fp64 */
  float segment_range; /* metres, (0, 1e5] */
} t2d_obs_config;
/* out: DEVICE float [N][F]; agent_index: DEVICE int16 [N][k_agents] (the slot of each agent row) or NULL; segment_index:
 * DEVICE int16 [N][k_segments] (the segment's index in its tile) or NULL.  Reads the goal target when one is bound and the
 * map tile(s) when set.  Rejected without a launch: k_agents / k_segments out of bounds, a range that is not finite or not
 * in (0, 1e5], out == NULL (T2D_E_INVALID), state not bound (T2D_E_STATE).  One launch, no allocation, no
 * synchronisation: capturable in a CUDA graph. */
int t2d_observe(t2d_ctx* ctx, const t2d_obs_config* cfg, float* out, int16_t* agent_index, int16_t* segment_index,
                void* stream);

/* ---- per-agent vector observation: the same row seen from any list of observer slots ---------------------------------
 * DESIGN.md section 1 "Per-agent vector observation".  Row (n, q), q < Q = n_observers (1..T2D_OBS_MAX_OBSERVERS), is
 * t2d_observe's row with slot j = observers[n][q] in the place of participant 0: the frame and the ego block are j's, the
 * agent candidates are every other slot (slot 0 included) that is active, has a shape and lies within agent_range, by
 * (d^2, slot), and the segments are measured from j's centre.  observers: DEVICE int16 [N][Q], or NULL for slot q in row q
 * of every scenario (needs Q <= M).  A value outside [0, M) or an empty slot (type_id >= n_types) gives an absent row
 * (zeros, every index -1); duplicates are allowed; the kernel applies this to the device data, nothing is checked on the host.
 * Goal block: goals == NULL - the rows observed by slot 0 take the t2d_set_goal target, every other row zeros; else goals is
 * DEVICE float [N][Q][5] (cx, cy, heading, half_len, half_wid) per row, a row whose cx is NaN gets zeros.  t_frac is the
 * scenario's.  With observers [n] = {0} and goals == NULL a row is bit-identical to t2d_observe's.
 * out: DEVICE float [N][Q][F] (F as t2d_observe, 64-bit offsets: N·Q·F may exceed 2^31); agent_index: DEVICE int16 [N][Q][K]
 * or NULL; segment_index: DEVICE int16 [N][Q][S] or NULL.  Rejected without a launch: everything t2d_observe rejects,
 * n_observers outside 1..128, observers == NULL with n_observers > M (T2D_E_INVALID), state not bound (T2D_E_STATE).
 * One launch, no allocation, no synchronisation: capturable in a CUDA graph. */
#define T2D_OBS_MAX_OBSERVERS 128
int t2d_observe_agents(t2d_ctx* ctx, const t2d_obs_config* cfg, const int16_t* observers /* DEVICE [N][Q] or NULL */,
                       int32_t n_observers /* Q */, const float* goals /* DEVICE [N][Q][5] or NULL */,
                       float* out /* DEVICE [N][Q][F] */, int16_t* agent_index /* [N][Q][K] or NULL */,
                       int16_t* segment_index /* [N][Q][S] or NULL */, void* stream);

/* On-device NPC controllers (tactics2d/controller).  A controller row is one configured controller object; the fields
 * are the reference's attribute names.  kind selects the law:
 *   T2D_CTRL_IDM           IDMController.step               (steering 0; free flow, or car following when a leader is set;
 *                                                            with pid_lateral PATH_HEADING / PATH_CROSS_TRACK the steering
 *                                                            is a PID row's lateral channel on the slot's path, see below)
 *   T2D_CTRL_CRUISE        AccelerationController.step      (steering 0; cruise, or adaptive cruise with a leader)
 *   T2D_CTRL_PURE_PURSUIT  PurePursuitController.step       (pure-pursuit steering on a path + the cruise laws)
 *   T2D_CTRL_PID           PIDController.step               (PID steering and acceleration with per-slot state, t2d_set_pid) */
#define T2D_CTRL_EXTERNAL 0 /* the caller's action is kept */
#define T2D_CTRL_IDM 1
#define T2D_CTRL_CRUISE 2
#define T2D_CTRL_PURE_PURSUIT 3
#define T2D_CTRL_PID 4
#define T2D_MAX_CONTROLLERS 64

/* Where a PID row takes its lateral error from (pid_controller.py:249-283).  HEADING / CROSS_TRACK read column 1 of the
 * t2d_set_pid target (target_heading in rad / cross_track_error in m); the PATH_* sources derive it from the slot's
 * path_id polyline (t2d_set_paths): PATH_CROSS_TRACK is the signed offset of the closest path point, positive when the
 * path lies to the vehicle's left, PATH_HEADING the direction of the closest segment as target_heading.  NONE: steering 0
 * and the lateral half of the state untouched (control_mode "longitudinal"). */
#define T2D_PID_LAT_NONE 0
#define T2D_PID_LAT_HEADING 1
#define T2D_PID_LAT_CROSS_TRACK 2
#define T2D_PID_LAT_PATH_HEADING 3
#define T2D_PID_LAT_PATH_CROSS_TRACK 4
/* Longitudinal error: TARGET = target_speed (column 0 of the target) - speed; NONE: acceleration 0 ("lateral") */
#define T2D_PID_LON_NONE 0
#define T2D_PID_LON_TARGET 1

typedef struct t2d_controller_params {
  int32_t kind; /* T2D_CTRL_* */
  /* IDMController.__init__, idm_controller.py:33-58 */
  float desired_speed, time_headway, min_spacing, max_acceleration, comfortable_deceleration, delta;
  /* AccelerationController attributes, acceleration_controller.py:33-39 (after update_driving_style, :62-80) */
  float target_speed, kp, accel_change_rate, delta_t, max_accel, min_accel, interval;
  /* PurePursuitController: min_pre_aiming_distance, interval (pure_pursuit_controller.py:26-36), wheel_base (:76) */
  float min_pre_aiming_distance, pp_interval, wheel_base;
  /* PIDController attributes, pid_controller.py:41-134 (after update_driving_style, :136-157).  The channel's limits are
   * max_accel / min_accel above; a CROSS_TRACK / PATH_CROSS_TRACK row scales the lateral output by 2.0 / wheel_base. */
  int32_t pid_lateral;      /* T2D_PID_LAT_* */
  int32_t pid_longitudinal; /* T2D_PID_LON_* */
  double dt, kp_lat, ki_lat, kd_lat, max_steering, kp_lon, ki_lon, kd_lon, derivative_filter_alpha;
} t2d_controller_params; /* 152 bytes: 4 bytes of padding before dt */

/* table: HOST array of n_rows (<= T2D_MAX_CONTROLLERS) rows, copied.  The rest are DEVICE arrays owned by the caller:
 * ctrl_id [N, M] uint8 = row of the participant's controller (255, or a row of kind EXTERNAL: not controlled);
 * lead_index [N, M] int16 = the participant's leading vehicle inside its scenario (`leading_state` / `front_state`),
 * -1 for none (NULL: nobody has one); while a leader search is bound (t2d_set_leader_search) t2d_control ignores it and
 * takes every leader from the search, found on the same state in the same call; path_id [N, M] int16 = the pure-pursuit path, -1 for none (NULL allowed);
 * last_accel [N, M] float = |acceleration| each participant applied on the previous tick (State.accel,
 * participant/trajectory/state.py:171-185), read and rewritten by t2d_control; zero it before the first tick.
 * Lane keeping (an extension, DESIGN.md section 1 "Lane keeping for IDM rows"): an IDM row whose pid_lateral is
 * T2D_PID_LAT_PATH_HEADING or T2D_PID_LAT_PATH_CROSS_TRACK keeps its IDM acceleration and steers with the lateral half of
 * the PID law on the slot's path (kp_lat / ki_lat / kd_lat, dt, derivative_filter_alpha, max_steering, wheel_base; the
 * same code and rounding as a PID row with pid_longitudinal NONE, the same state[..., 0:3] of t2d_set_pid, never the
 * target).  Such a row needs t2d_set_pid's state like a PID row; its pid_longitudinal is not read.  An IDM row with
 * pid_lateral NONE is the reference's IDM.
 * table == NULL removes the controllers.  Every call that is not rejected drops a bound lane change
 * (t2d_set_lane_change).  Rejected (the previous binding stays whole): an unknown kind, a PID row with
 * dt <= 0, max_steering <= 0, max_accel <= 0, min_accel >= 0, max_accel <= min_accel, derivative_filter_alpha outside
 * (0, 1], an unknown source, or wheel_base <= 0 with a cross-track source, and an IDM row whose pid_lateral is neither
 * NONE nor a PATH source, or that has one with dt <= 0, max_steering <= 0, derivative_filter_alpha outside (0, 1], or
 * wheel_base <= 0 with PATH_CROSS_TRACK. */
int t2d_set_controllers(t2d_ctx* ctx, const t2d_controller_params* table, int n_rows, const uint8_t* ctrl_id,
                        const int16_t* lead_index, const int16_t* path_id, float* last_accel);

/* Pure-pursuit paths: HOST arrays, copied.  xy [V][2] vertices of all paths back to back, offsets [n_paths + 1] (path p
 * owns vertices offsets[p] .. offsets[p + 1] - 1, at least 2).  n_paths == 0 or xy == NULL unbinds.  Rejected (the
 * previous paths stay bound): malformed offsets.  Every call that is not rejected drops a bound lane change. */
int t2d_set_paths(t2d_ctx* ctx, const float* xy, const int32_t* offsets, int n_paths);

/* ---- route following: the OffRoute detector, route progress and the route observation --------------------------------
 * DESIGN.md section 1 "Route following".  A route is a polyline of the t2d_set_paths table.  route_id: DEVICE int16 [N][M]
 * owned by the caller (like tile_id; it may be rewritten between steps): the route of every slot, -1, or any id the table
 * does not hold, for none; a route whose segments all have zero length is none too.  For a slot with a route, (x, y) its
 * fp32 centre, the closest point is the first strict minimum of the squared distance over the route's segments of non-zero
 * length (the projection clamped to the segment, as K5's PATH sources), d its distance, s its arc length (the lengths of
 * the earlier segments of non-zero length summed in list order, plus t len), L the total length; fp64, one rounding per
 * operation.
 *   OffRoute (off_route.py:24-35, route.distance(centre) > threshold): a scored participant with a route whose status is
 * NORMAL or COMPLETED is off route when d > threshold (status chain: time exceeded, no action, out of bound, collision,
 * off route, completed).  t2d_env_epilogue: the ego's traffic status becomes T2D_TRAFFIC_OFF_ROUTE (the scenario status
 * stays the tick's), the step is truncated and its reward is off_route_reward.  K10 (t2d_agents_epilogue): the row's
 * status becomes FAILED, its slot's traffic status OFF_ROUTE, the row is truncated with reward off_route_reward and its
 * slot retires.  t2d_step / t2d_step_host_ego leave status and done to the tick, unchanged.
 *   Progress (an extension): a NORMAL row on its route adds fp32(progress_weight (s - s_best)) to its reward when
 * s > s_best, then s_best = s.  s_best is an fp64 tracker per scored row (initialise to -inf: the first step only records
 * s), reset where max_iou / min_dist are.
 * route_id == NULL unbinds; with no routes bound (or all -1) every output of both epilogues is what it is without this
 * call.  Rejected (the previous binding stays whole): a threshold that is negative or not finite, a progress_weight or
 * off_route_reward that is not finite (T2D_E_INVALID).  The default off_route_reward of the Python layer is -5, the
 * out-of-bound penalty. */
int t2d_set_routes(t2d_ctx* ctx, const int16_t* route_id, double threshold, double progress_weight, float off_route_reward);
/* The progress trackers, DEVICE fp64 and owned by the caller: s_best [N] for t2d_env_epilogue, agent_s_best [N][n_agent_rows]
 * for t2d_agents_epilogue (n_agent_rows must equal the bound agents' Q when it runs, else T2D_E_STATE).  Either may be
 * NULL: no progress term there.  They are read only while routes are bound.  Rejected: n_agent_rows outside 1..128 with
 * an agent tracker, a tracker that is not 8-byte aligned (T2D_E_INVALID). */
int t2d_bind_route_trackers(t2d_ctx* ctx, double* s_best, double* agent_s_best, int32_t n_agent_rows);

#define T2D_TRAFFIC_OFF_ROUTE 5  /* TrafficStatus.OFF_ROUTE, status.py */
#define T2D_ROUTE_OBS_FIELDS 5   /* has_route, lateral offset, heading error, s / L, L - s */
#define T2D_ROUTE_MAX_POINTS 256 /* look-ahead points per row of t2d_route_observe */
/* K12 (no reference counterpart): one fp32 row of T2D_ROUTE_OBS_FIELDS + 2 n_points per observer row, in the frame of the
 * observer's slot (origin its centre, +x along its heading): has_route (1), the signed lateral offset u.x (c.y - y) -
 * u.y (c.x - x) (positive when the route lies to the left), the heading error atan2(u.y, u.x) - heading wrapped to
 * (-pi, pi], s / L, L - s, then n_points points (x, y) at arc length min(s + k spacing, L), k = 1..n_points.  observers
 * DEVICE int16 [N][Q], Q = n_observers in 1..T2D_OBS_MAX_OBSERVERS, or NULL for slot q in row q (Q <= M).  Rows whose
 * observer is outside [0, M), whose slot is empty or retired, or whose slot has no route are zeros.  out: DEVICE fp32
 * [N][Q][T2D_ROUTE_OBS_FIELDS + 2 n_points].  Rejected without a launch: n_observers outside 1..128, observers == NULL
 * with n_observers > M, n_points outside 0..T2D_ROUTE_MAX_POINTS, spacing not finite or <= 0, out == NULL
 * (T2D_E_INVALID), state or type table not bound (T2D_E_STATE).  One launch, no allocation: capturable in a CUDA graph. */
int t2d_route_observe(t2d_ctx* ctx, const int16_t* observers, int32_t n_observers, int n_points, float spacing, float* out,
                      void* stream);

/* ---- trajectory history: the recent states of every participant slot, and past poses in an observer's frame ------------
 * Trajectory.add_state appends every tick's State and Trajectory.reset(state) starts the history again from that state
 * (participant/trajectory/trajectory.py:115-149,170-188).  The contract is DESIGN.md section 1 "Trajectory history".
 * t2d_set_history(ctx, H), H in 1..T2D_HISTORY_MAX, allocates the library's ring (N M H 25 bytes, plus 4 bytes per entry
 * while a log schedule with a track_out is bound) and H = 0 frees it.  A new binding is empty (every count 0).  Rejected
 * (the previous ring stays bound, entries and all): H outside 0..64 (T2D_E_INVALID), an allocation that fails (T2D_E_CUDA).
 *   append   t2d_step, t2d_step_host (after its last chunk), t2d_step_host_ego and t2d_step_host_agents (before K10)
 *            append the post-tick state of every scenario: entry e = count[n] goes to ring index e % H, count[n] + 1;
 *   restart  t2d_reset and t2d_reset_sampled restart every masked scenario: entry 0 = the state after the whole reset (the
 *            log replay and the sampled placement included), count = 1; the other scenarios keep their history;
 *   alone    t2d_set_state-style writes, t2d_check_events and every observation leave the ring untouched;
 *   valid    entry e of slot m counts for the slot's current occupant iff it is one of the last min(count, H) entries, its
 *            recorded type id is < n_types and equals the slot's current one, and - with a schedule's track_out bound - its
 *            recorded track equals the slot's current track_out value.  Binding a log drops the recorded tracks (they
 *            read -1 afterwards: not replayed).
 * With no ring bound nothing of this launches. */
#define T2D_HISTORY_MAX 64
#define T2D_HISTORY_FIELDS 7 /* valid, ex, ey, cos dh, sin dh, v_x, v_y */
int t2d_set_history(t2d_ctx* ctx, int32_t length);
/* K16: for every observer row, its own past (block 0) and the past of K agent slots (block 1 + k), lag 0 (the newest entry)
 * first, T2D_HISTORY_FIELDS values per lag in the observer's CURRENT frame, with the arithmetic of t2d_observe's agent rows
 * applied to the recorded pose and velocity.  n_observers == 0 (observers NULL): one row per scenario, observed by slot 0
 * (t2d_observe's rows); n_observers = Q in 1..T2D_OBS_MAX_OBSERVERS: the rows of observers DEVICE int16 [N][Q], or NULL for
 * slot q in row q (Q <= M), as t2d_observe_agents.  agent_index: DEVICE int16 [rows][k_agents] as t2d_observe /
 * t2d_observe_agents return it (-1: none), k_agents in 0..T2D_OBS_MAX_AGENTS, NULL when k_agents == 0.  out: DEVICE fp32
 * [rows][1 + k_agents][H][T2D_HISTORY_FIELDS] (64-bit offsets).  An observer outside [0, M) or whose slot is empty gives a
 * zero row; an agent slot outside [0, M) and an entry that is not valid give zero lags.  When the newest entry is the
 * current state, block 1 + k at lag 0, fields 1..6, equals fields 1..6 of t2d_observe's agent row k bit for bit.
 * Rejected without a launch: n_observers outside 0..128, observers with n_observers == 0, observers == NULL with
 * n_observers > M, k_agents outside 0..127, agent_index NULL with k_agents > 0, out NULL (T2D_E_INVALID), state or type table
 * not bound, no ring bound (T2D_E_STATE).  One launch, no allocation, no synchronisation: capturable in a CUDA graph. */
int t2d_observe_history(t2d_ctx* ctx, const int16_t* observers, int32_t n_observers, const int16_t* agent_index,
                        int32_t k_agents, float* out, void* stream);
/* The bound ring's DEVICE arrays, for read-back utilities and tests (length 0 and NULL pointers without a ring).  They belong
 * to the library and live until the next t2d_set_history or t2d_destroy; track is NULL unless tracks are recorded. */
typedef struct t2d_history_ring {
  int32_t length;                                 /* H */
  float *x, *y, *heading, *speed, *vx, *vy;       /* [N][H][M] */
  uint8_t* type_id;                               /* [N][H][M] */
  int32_t* track;                                 /* [N][H][M] or NULL */
  int64_t* count;                                 /* [N] entries since the scenario's episode began */
} t2d_history_ring;
int t2d_history_view(t2d_ctx* ctx, t2d_history_ring* out);

/* Overwrites action[n][m] = (accel, steer) ((steer, accel) with T2D_CFG_STEER_FIRST) of every controlled participant from
 * the bound state, then stores |applied acceleration| of the WHOLE action buffer in last_accel (bicycles: the accel clipped
 * to the type's range; point masses: |(ax, ay)|).  Call it after the external actions are in the buffer and before
 * t2d_step.  action: DEVICE [N, M, 2] fp32. */
int t2d_control(t2d_ctx* ctx, float* action, void* stream);

/* ---- leader search (K17, no reference counterpart: the reference's controllers take the leader from their caller) ------
 * DESIGN.md section 1 "Leader search".  fp64, one rounding per operation.  A follower is every slot with type_id < n_types
 * (controlled or not) at a position that is not NaN; a candidate is every other slot with type_id < n_types and a shape
 * other than T2D_SHAPE_NONE at a position that is not NaN (replayed slots and discs count, empty and retired slots do not).
 *   path frame     the follower's path_id of the bound controllers is in [0, n_paths) and that path has a segment of
 *                  non-zero length: follower and candidates are projected onto it as t2d_set_routes' closest point (arc
 *                  length s, distance d); a candidate qualifies when d <= half_width and 0 < gap = s_j - s_i <= max_range;
 *   heading frame  every other follower (all of them without controllers or paths): with (c, s) the sine and cosine of
 *                  its fp32 heading as t2d_observe computes them, ex = c dx + s dy and ey = -s dx + c dy of the candidate's
 *                  offset; it qualifies when ex > 0, |ey| <= half_width and ex <= max_range, and gap = ex (bit for bit
 *                  the ex of the t2d_observe_agents row for the same pair).
 * The leader is the qualifying candidate of smallest (gap, slot).  lead: DEVICE int16 [N][M], -1 for none; gap: DEVICE
 * fp32 [N][M], the gap rounded once, +inf for none.  half_width in (0, 100] m, max_range in (0, 1e5] m, both finite.
 *   t2d_set_leader_search binds a search: every t2d_control, t2d_step_host_ego and t2d_step_host_agents then launches K17
 * in front of the controllers, into the caller-owned lead / gap (gap may be NULL), and the controllers follow `lead`
 * instead of set_controllers' lead_index (the laws themselves, and their centre distance, are unchanged).  lead == NULL
 * unbinds; with no search bound nothing of this launches.  The search keeps no state: resets need nothing.
 *   t2d_find_leaders writes the leaders of the bound state into lead / gap once: one launch, no allocation, capturable.
 * Rejected without a launch (a rejected set keeps the previous binding whole): half_width or max_range outside its range
 * or not finite, lead NULL for find, lead not 2-byte or gap not 4-byte aligned (T2D_E_INVALID), state or type table not
 * bound (T2D_E_STATE). */
int t2d_set_leader_search(t2d_ctx* ctx, double half_width, double max_range, int16_t* lead, float* gap);
int t2d_find_leaders(t2d_ctx* ctx, double half_width, double max_range, int16_t* lead, float* gap, void* stream);
/* Unbinding the search (lead == NULL) also drops a bound lane change. */

/* ---- lane changes (K18, no reference counterpart): MOBIL (Kesting, Treiber and Helbing 2007) ---------------------------
 * DESIGN.md section 1 "Lane changes".  Evaluated on the state K5 reads next, fp64 with one rounding per operation except
 * the IDM accelerations, which are K5's own idm_law.  Candidates are the leader search's; a candidate is on path r when
 * its distance to r (t2d_set_routes' closest point) is <= the bound search's half_width, s^r is its arc length there.
 *   A lane changer is a slot whose controller row is an IDM row with a lateral channel, whose current path
 * p = lane_path[n][m] has a segment of non-zero length, whose cooldown is 0 and which is itself on p.  Its target lanes
 * are left[p] and right[p] when >= 0.  On a target q: blocked when a candidate on q has |s^q_j - s^q_c| < min_gap; the new
 * leader l' is the candidate on q of smallest gap s^q_j - s^q_c in (0, max_range] (ties: lower slot), the new follower n
 * the same behind; the old leader l and follower o are the same on p.  a(f | L) is idm_law with f's own IDM row (the
 * changer's row when f has none); a missing leader is free flow, a missing follower gives 0 to both its terms.
 *   safe       a(n | c) >= -b_safe, or no new follower;
 *   incentive  (a(c | l') - a(c | l)) + politeness ((a(n | c) - a(n | l')) + (a(o | l) - a(o | c))).
 * Among the unblocked safe sides with incentive > threshold the larger incentive wins (a tie goes left): lane_path = q,
 * cooldown = params.cooldown, change = +1 (left) / -1 (right).  Every other slot: change = 0 and a positive cooldown
 * counts down by 1.  All decisions of a scenario are made on the same state (two cars may take the same gap).
 *   t2d_set_lane_change binds it: left / right HOST int16 [n_paths] (-1: none), copied; lane_path, cooldown DEVICE int16
 * [N][M] and change DEVICE int8 [N][M] (may be NULL) owned by the caller.  The call copies the controllers' path_id into
 * lane_path and zeroes cooldown (and change).  While bound, t2d_control, t2d_step_host_ego and t2d_step_host_agents launch
 * K18, then K17, then K5; K17 (also under t2d_find_leaders) and K5's path reads take lane_path instead of path_id, which is
 * never written (it stays the episode's starting lane).  t2d_reset / t2d_reset_sampled copy path_id into lane_path and
 * zero cooldown and change for the reset scenarios.  p == NULL unbinds; with nothing bound nothing of this launches.
 * t2d_set_controllers, t2d_set_paths and unbinding the leader search drop the binding.
 * Rejected (a rejected call keeps the previous binding whole): politeness < 0 or not finite, threshold not finite,
 * b_safe <= 0 or not finite, min_gap <= 0, min_gap > max_range or not finite, cooldown outside 0..32767, NULL left / right
 * / lane_path / cooldown, a left / right entry outside [-1, n_paths) or naming its own path, lane_path or cooldown not
 * 2-byte aligned (T2D_E_INVALID); state, type table, controllers, their path_id, paths or the leader search not bound
 * (T2D_E_STATE). */
typedef struct t2d_lane_change_params {
  double politeness; /* p: weight of the followers' accelerations */
  double threshold;  /* a_th (m/s^2): the incentive must exceed it */
  double b_safe;     /* (m/s^2): the new follower's predicted deceleration limit */
  double min_gap;    /* (m): the blocking distance along the target lane, in (0, max_range] */
  int32_t cooldown;  /* ticks without a decision after a change, 0..32767 */
  int32_t reserved;  /* 0 */
} t2d_lane_change_params; /* 40 bytes */
int t2d_set_lane_change(t2d_ctx* ctx, const t2d_lane_change_params* p, const int16_t* left, const int16_t* right,
                        int16_t* lane_path, int16_t* cooldown, int8_t* change);

/* ---- yielding at conflict zones (K19, no reference counterpart) --------------------------------------------------------
 * DESIGN.md section 1 "Yielding at conflict zones".  fp64 with one rounding per operation, on the state K5 reads next.
 * The zone table is built on the host from the bound path table (tactics2d_b200.traffic.conflict_zones): for path p,
 * rows zone_off[p] .. zone_off[p + 1] - 1, sorted by s_in_p, each naming the other path q and the arc intervals
 * [s_in_p, s_out_p] on p and [s_in_q, s_out_q] on q where the two come within the zone width (widened by a margin).
 *   A slot's path is its current path (K17's: drive_path, lane_path or path_id) when that has a segment of non-zero length,
 * else its route (t2d_set_routes, read at every launch) when that has one, which makes it a partner only.  s_k is its arc
 * length on that path (t2d_set_routes' closest point), u_k = max(v_k, v_min).  A yielder is a slot with type_id < n_types,
 * a position that is not NaN, an IDM controller row and a usable current path p.  It considers the zones of p with
 * v_i^2 / (2 commit_decel) < d_i = s_in_p - s_i <= the search's max_range.  The partners of a zone are the leader search's
 * candidates whose path is q, with d_j = s_in_q - s_j and t_j = max(d_j, 0) / u_j; a partner is cleared when
 * s_j > s_out_q and excluded when its distance to p is <= the search's half_width and its arc length on p is > s_i.  i
 * must yield to a partner that is neither when d_j <= v_j^2 / (2 commit_decel), or t_j <= critical_gap and priority[q] >
 * priority[p], or t_j <= critical_gap, priority[q] == priority[p] and (d_j, j) < (d_i, i).  The yield zone is the
 * considered zone of smallest d_i (then lowest row) with a must-yield partner: yield_to = its lowest such partner slot,
 * stop_gap = d_i rounded once; -1 and +inf for every other slot.  K5 (t2d_yield_control_kernel) then gives an IDM row with
 * a finite stop_gap min(IDM on its leader, IDM on the stop point standing at speed 0), the stop point being p's point at
 * arc length clamp(s_in_p, 0, L).
 *   t2d_set_yielding binds it: zones HOST [zone_off[n_paths]], zone_off HOST int32 [n_paths + 1], priority HOST int16
 * [n_paths] or NULL (all 0), all copied; yield_to DEVICE int16 [N][M] and stop_gap DEVICE fp32 [N][M] owned by the caller.
 * While bound, t2d_control, t2d_step_host_ego and t2d_step_host_agents launch K18 (if bound), K17, K19, then K5.  K19
 * keeps no state: resets need nothing.  p == NULL unbinds; with nothing bound nothing of this launches and K5 runs its
 * other instances.  t2d_set_controllers, t2d_set_paths and unbinding the leader search drop the binding.
 *   t2d_find_yields writes the yields of the bound state into yield_to / stop_gap once (and the stop points K5 reads): one
 * launch, no allocation, capturable.
 * Rejected (a rejected call keeps the previous binding whole): critical_gap, commit_decel or v_min not finite and > 0,
 * NULL zone_off / yield_to / stop_gap (or zones with rows), zone_off[0] != 0 or decreasing, a zone with q outside
 * [0, n_paths) or q == p, an arc length that is not finite, s_in > s_out, the zones of a path not sorted by s_in_p,
 * misaligned arrays (T2D_E_INVALID); state, type table, controllers, paths or the leader search not bound, or no yielding
 * bound for find (T2D_E_STATE). */
typedef struct t2d_yield_params {
  double critical_gap; /* (s): a partner this close in time to its zone entry is a gap too small to take */
  double commit_decel; /* (m/s^2): a car that cannot stop before its zone at this deceleration is committed */
  double v_min;        /* (m/s): the speed floor of the partners' time to their zone */
} t2d_yield_params;    /* 24 bytes */
typedef struct t2d_conflict_zone {
  int32_t q;           /* the other path */
  int32_t reserved;    /* 0 */
  double s_in_p, s_out_p, s_in_q, s_out_q;   /* (m) arc lengths on p and on q */
} t2d_conflict_zone;   /* 40 bytes */
int t2d_set_yielding(t2d_ctx* ctx, const t2d_yield_params* p, const t2d_conflict_zone* zones, const int32_t* zone_off,
                     const int16_t* priority, int16_t* yield_to, float* stop_gap);
int t2d_find_yields(t2d_ctx* ctx, int16_t* yield_to, float* stop_gap, void* stream);

/* Inputs and memory of the PID rows: DEVICE arrays owned by the caller.  target [N][M][2] fp32 = (target_speed, lateral
 * target: target_heading in rad for HEADING rows, cross_track_error in m for CROSS_TRACK rows; PATH rows ignore it);
 * state [N][M][6] fp64 = (lat_integral, lat_prev_error, lat_prev_derivative, lon_integral, lon_prev_error,
 * lon_prev_derivative) of every slot, all zero for a freshly reset controller.  t2d_control reads and rewrites the state
 * row of each slot a PID row drives (only the half of an enabled channel); t2d_reset zeroes the rows of the reset
 * scenarios.  state == NULL unbinds both; a target without a state is rejected.  While a PID row is bound, t2d_control
 * refuses (T2D_E_INVALID, nothing launched) without a state, or without a target when a row reads it. */
int t2d_set_pid(t2d_ctx* ctx, const float* target, double* state);

/* ---- the env layer: ego action, host-resident ego caller, reward / terminated / truncated ------------------------------
 * ParkingEnv.step takes ONE action, the ego's (steering, accel) (envs/parking.py:219-239); the other participants of a
 * batched scenario are driven on the device (t2d_control) or by the rows of the caller's action array.
 * t2d_set_ego_action binds a DEVICE array [N][2] (or NULL to unbind): while bound, t2d_control and t2d_step take the
 * action of participant 0 of every scenario from it (t2d_control also writes it into row 0 of `action`). */
int t2d_set_ego_action(t2d_ctx* ctx, const float* ego_action /* device [N][2], 8-byte aligned */);
/* One tick for a caller whose policy lives on the host and drives only the ego: stages ego_action_host [N][2] in pinned,
 * device-mapped host memory that the first kernel reads directly (8 N bytes over PCIe instead of the 8 N M of
 * t2d_step_host, and no copy-engine transfer in front of the kernels), runs t2d_control when controllers are set (the other
 * participants' rows of `action`, a DEVICE array [N][M][2] owned by the caller, never leave the device), the tick, and
 * copies status + done back ([N] each, HOST); synchronises `stream` before returning. */
int t2d_step_host_ego(t2d_ctx* ctx, const float* ego_action_host, float* action, uint8_t* flags, int16_t* hit_index,
                      int16_t* hit_segment, uint8_t* scn_status_host, uint8_t* done_host, void* stream);
/* What ParkingEnv.step computes after check_status (envs/parking.py:240-256, _get_reward :148-190), for all scenarios in
 * one launch, from the tick's outputs `flags` [N][M] and `scn_status` [N]: traffic_status [N][M] (TrafficStatus codes,
 * status.py:52-61; may be NULL), terminated / truncated / done [N] (may be NULL), reward [N] by the reference's chain
 * (-5 collision, -1 time exceeded / no action, -5 out of bound, +5 completed, else time penalty + IoU gain + 0.1 x
 * progress towards the target).  max_iou / min_dist [N]: the per-episode extrema the reward keeps (ParkingEnv._max_iou,
 * _min_dist_to_target; initialise to -inf / +inf; NULL when no goal is set); with reset_trackers_on_done they are
 * re-initialised for the scenarios that are done, so that `done` can go straight into t2d_reset.  All arrays DEVICE. */
int t2d_env_epilogue(t2d_ctx* ctx, const uint8_t* flags, const uint8_t* scn_status, float* reward, uint8_t* terminated,
                     uint8_t* truncated, uint8_t* traffic_status, uint8_t* done, float* max_iou, float* min_dist,
                     int reset_trackers_on_done, void* stream);

/* ---- per-agent status, reward and retirement (no reference counterpart) ---------------------------------------------
 * DESIGN.md section 1 "Per-agent status and reward".  The agents are the rows of an observer list, as in
 * t2d_observe_agents: observers DEVICE int16 [N][Q], Q = n_observers in 1..T2D_OBS_MAX_OBSERVERS, or NULL for slot q in
 * row q (Q <= M).  Row (n, q) is active when observers[n][q] is in [0, M) and that slot's type_id < n_types when the
 * epilogue runs; an inactive row is absent (status 0, reward 0, terminated / truncated 0, iou 0).  Duplicates are allowed.
 * goals: DEVICE float [N][Q][5] (cx, cy, heading, half_len, half_wid) or NULL; a NaN cx means the row has no goal.  A row
 * with a goal whose slot is a box has the Arrival / NoAction detectors of t2d_set_goal (same threshold rule, same
 * arithmetic), with per-row state last_pose [N][Q][4] and noact_count [N][Q] (zero them before the first step).
 * retired_type DEVICE uint8 [N][M] (fill with 255 before the first step): a row that settles (status not NORMAL) retires
 * its slot - the type goes into retired_type and type_id becomes 255, so the bound type_id must be writable.
 * While agents are bound, t2d_reset also restores the retired types of the masked scenarios (before its log replay, which
 * rewrites replayed slots as before) and clears their per-row NoAction state.  observers == NULL with n_observers == 0
 * unbinds.  Rejected: n_observers outside 1..128, observers == NULL with n_observers > M, a NULL state array, a threshold
 * outside (0, 1] with goals (T2D_E_INVALID).  The arrays are the caller's and must stay alive while bound. */
int t2d_set_agents(t2d_ctx* ctx, const int16_t* observers, int32_t n_observers, const float* goals, float arrival_threshold,
                   int no_action_max_step, float* last_pose, int32_t* noact_count, uint8_t* retired_type);
/* K10: for every row, the status chain of t2d_step applied to its own slot (time exceeded, no action, out of bound,
 * collision, completed, normal), terminated / truncated / reward by t2d_env_epilogue's rules, iou [N][Q] (0 without
 * detectors), the per-episode extrema max_iou / min_dist [N][Q] (initialise to -inf / +inf), retirement, and
 * done[n] = 1 when no row of scenario n is NORMAL (a scenario whose rows are all absent is done at every step).  With
 * reset_trackers_on_done the extrema of the done scenarios restart.  traffic_status [N][M] may be NULL; every other array
 * is required (T2D_E_INVALID).  State not bound or no agents bound: T2D_E_STATE.  All arrays DEVICE; one launch, no
 * allocation, no synchronisation: capturable in a CUDA graph. */
int t2d_agents_epilogue(t2d_ctx* ctx, const uint8_t* flags, float* reward, uint8_t* terminated, uint8_t* truncated,
                        uint8_t* agent_status, float* iou, uint8_t* done, float* max_iou, float* min_dist,
                        uint8_t* traffic_status, int reset_trackers_on_done, void* stream);

/* ---- per-agent action (no reference counterpart) ---------------------------------------------------------------------
 * DESIGN.md section 1 "Per-agent action".  agent_action DEVICE fp32 [N][Q][2], one action per row of an observer list
 * (observers DEVICE int16 [N][Q], Q = n_observers in 1..T2D_OBS_MAX_OBSERVERS, or NULL for slot q in row q, Q <= M), in
 * the world's action order.  K11: for slot m of scenario n, let q* be the LOWEST q with observers[n][q] == m; when q*
 * exists and type_id[n][m] < n_types, action[n][m] = agent_action[n][q*] (the fp32 bits as they are).  Nothing else is
 * written: slots no row names, rows out of range, rows whose slot is empty or retired, and duplicate rows after the first
 * leave action as it was.  Call it before t2d_control: a slot with a controller then takes its controller's action, and
 * the controllers see the agents' own accelerations in last_accel.  While t2d_set_ego_action is bound, slot 0 still
 * takes the ego action in t2d_control and t2d_step.  Needs no t2d_set_agents.  Rejected without a launch: n_observers
 * outside 1..128, observers == NULL with n_observers > M, a NULL or not 8-byte aligned agent_action / action
 * (T2D_E_INVALID), state not bound (T2D_E_STATE).  One launch, no allocation, no synchronisation: capturable in a CUDA
 * graph. */
int t2d_scatter_agent_action(t2d_ctx* ctx, const int16_t* observers /* DEVICE [N][Q] or NULL */, int32_t n_observers,
                             const float* agent_action /* DEVICE [N][Q][2] */, float* action /* DEVICE [N][M][2] */,
                             void* stream);
/* One multi-agent step for a caller whose policy lives on the host: the counterpart of t2d_step_host_ego for the agents
 * bound with t2d_set_agents (their observer list and Q).  Copies agent_action_host HOST [N][Q][2] (pinned memory
 * recommended) into a device staging buffer with one host->device copy on `stream` (reallocated when Q changes, freed by
 * t2d_destroy), scatters it into the caller's DEVICE action [N][M][2] with K11, runs t2d_control when controllers are
 * set, the tick (log replay and drift as usual) and K10,
 * copies reward (fp32), terminated, truncated, agent status (uint8; [N][Q] each) and done ([N]) back in ONE device->host
 * copy and synchronises `stream`: the host arrays are valid on return.  flags [N][M], hit_index, hit_segment: DEVICE,
 * any may be NULL (K10 then reads the library's own flags).  max_iou / min_dist: DEVICE [N][Q], the per-episode extrema
 * of t2d_agents_epilogue.  Host outputs may be NULL, except done_host.  No reset inside the call.  Rejected without a
 * launch: a NULL context, agent_action_host, action, max_iou, min_dist or done_host, an action that is not 8-byte
 * aligned (T2D_E_INVALID), state not bound or no agents bound (T2D_E_STATE). */
int t2d_step_host_agents(t2d_ctx* ctx, const float* agent_action_host /* HOST [N][Q][2] */, float* action /* DEVICE [N][M][2] */,
                         uint8_t* flags, int16_t* hit_index, int16_t* hit_segment, float* max_iou, float* min_dist,
                         int reset_trackers_on_done, float* reward_host, uint8_t* terminated_host, uint8_t* truncated_host,
                         uint8_t* agent_status_host, uint8_t* done_host, void* stream);

/* ---- done-mask exchange across the GPUs of one node, over peer memory (NVLink / NVSwitch) -------------------------
 * Scenarios are sharded across ranks (one process per GPU); the one exchange of the path is "every rank learns every
 * rank's done mask of this tick" - the terminated / truncated vector a central learner or reset scheduler reads
 * (envs/parking.py:243-248 per scenario).  t2d_exchange_allgather is that all-gather as ONE small kernel per rank:
 * it stores the rank's mask into a ring slot on EVERY rank (peer stores), signals the step on every rank's flag word
 * (release, system scope), waits for all ranks' signals of the same step (acquire; bounded - a rank that never shows
 * up sets the sticky timed_out word instead of hanging the GPU) and copies the slot to the caller's array.
 *
 * Set-up: every rank calls t2d_exchange_create (fills a 64-byte CUDA IPC handle), the ranks pass the handles around
 * by any host channel (torch.distributed in this repository), every rank calls t2d_exchange_connect with all `world`
 * handles in rank order.  n_local = scenarios per rank (rows are padded to a multiple of 16); slots >= 2 = ring depth.
 * Every rank must call t2d_exchange_allgather the same number of times, in stream order on each rank. */
typedef struct t2d_exchange t2d_exchange;
int t2d_exchange_create(t2d_exchange** out, int device, int world, int rank, int n_local, int slots, void* ipc_handle_out);
int t2d_exchange_connect(t2d_exchange* x, const void* handles /* host, world x T2D_IPC_HANDLE_BYTES */);
/* done_local: DEVICE uint8 [n_local] (t2d_step's `done`); dst: DEVICE uint8 [world * ((n_local + 15) & ~15)], rank order. */
int t2d_exchange_allgather(t2d_exchange* x, const uint8_t* done_local, uint8_t* dst, void* stream);
/* The same exchange taken off the critical path: the call posts this step's mask (put + signal, nothing to wait for)
 * and delivers into dst the gathered masks of the step `lag` calls earlier, whose signals have long arrived (the first
 * `lag` calls deliver nothing and leave dst untouched).  The consumer of the gathered masks - a central learner or
 * reset scheduler - is behind the simulation anyway; the ticks of the ranks no longer meet once per step.
 * Needs slots >= 2 * lag + 2.  lag = 0 is t2d_exchange_allgather.  If a rank fails to signal within the time-out
 * (T2D_EXCHANGE_TIMEOUT_MS, default ~2 s) dst is filled with 0xFF and the sticky timed_out word is set. */
int t2d_exchange_allgather_lagged(t2d_exchange* x, const uint8_t* done_local, uint8_t* dst, int lag, void* stream);
int t2d_exchange_status(t2d_exchange* x, uint32_t* steps, uint32_t* timed_out);
int t2d_exchange_destroy(t2d_exchange* x);

/* Flat batch of `n` independent participants through ONE model (PhysicsModelBase.step):
 * state arrays are read and written in place; action [n, 2]; applied [n, 2] (may be NULL)
 * receives the clipped (accel, steer) the reference returns next to the State.  omega_front / omega_rear [n]: the wheel
 * speeds of SingleTrackDrift.step (in / out); NULL for every other model. */
int t2d_physics_step(int device, const t2d_type_params* params /*host*/, int interval_ms, int delta_t_ms, int n,
                     float* x, float* y, float* heading, float* speed, float* vx, float* vy, float* omega_front,
                     float* omega_rear, const float* action, float* applied, void* stream);

/* Tuning knob of t2d_step, no effect on results: the tick can ask L2 for its first input lines while the previous grid is
 * still draining (and for the next tile inside its persistent loop).  mode 1: on, 0: off, -1 (default): on unless a
 * peer-memory done exchange is alive in the process (on one GPU it saves ~1 us per tick at 4096 x 64; next to the
 * exchange kernel on 8 GPUs it measured slower).  A caller that can time both settings picks with this (bench.py does at
 * N > 1); the environment variable T2D_PREFETCH sets the initial mode at t2d_create. */
int t2d_set_prefetch(t2d_ctx* ctx, int mode);

/* Number of kernels this library has launched since load (bench.py's gpu_launches). */
int64_t t2d_launch_count(void);

/* Number of ticks launched through the tick kernel's instance compiled for M = 64: kinematic types only, aligned
   state, no ego action and no goal (the others run the generic instance, which computes the same bits).
   The environment variable T2D_TICK_GENERIC=1, read at t2d_create, keeps a world on the generic instance. */
int64_t t2d_tick_fixed_count(void);

/* Number of warp tiles of that instance, on the current device, whose x sort fell back to the sort network.  The
   instance starts every scenario's sort from the slot order it left after the scenario's previous tick (an [N][64] hint
   the world holds, the identity at t2d_create; set_state, reset and the other kernels leave it alone) and falls back
   when two repair passes do not sort it.  Returns -1 when the counters cannot be read. */
int64_t t2d_tick_order_fallback_count(void);

/* The order hint of t2d_tick_order_fallback_count: copies its N x 64 bytes to the HOST buffer read_to (unless NULL),
   then overwrites it with the N x 64 bytes at the HOST buffer write_from (unless NULL).  Whatever the hint holds, every
   tick computes the same results; only the time the sort takes depends on it.  For tests and diagnostics. */
int t2d_order_hint(t2d_ctx* ctx, void* read_to, const void* write_from);

/* Number of launches of the tick kernel (t2d_step and every call that ticks or checks events) since load that the CUDA
   runtime accepted (a fault while the kernel runs is not seen here), per instance:
   k = 0 / 1: fp64 models compiled in (the table holds a type that is neither kinematic nor static), one map tile / a map
   table; k = 2 / 3: kinematic and static types only, one tile / table; k = 4 / 5: the M = 64 instance of
   t2d_tick_fixed_count, one tile / table.  k = 6: launches with one map tile too large for shared memory, which read it
   from global memory.  Returns -1 for any other k. */
int64_t t2d_tick_instance_count(int k);

#ifdef __cplusplus
}
#endif
#endif /* T2D_B200_H */
