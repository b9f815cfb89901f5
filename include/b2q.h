/* b2q.h — C ABI of the H100-native batched A1 simulator + rollout engine (libb2q.so).
 *
 * This is the drop-in boundary for the ONE hot path of PaddleRobotics QuadrupedalRobots/ETGRL: everything
 * below `env.reset / env.step` (and, for the policy, below `agent.predict / agent.sample`).  Plain C types
 * only; every array argument is a DEVICE pointer owned by the caller (e.g. a torch tensor's data_ptr);
 * the library owns only the opaque handle and its internal struct-of-arrays env state.  All work is
 * stream-ordered on the caller's cudaStream_t (passed as void*); no call synchronises the host except
 * b2q_create/b2q_destroy.  Every function returns 0 on success, a negative B2Q_E* code otherwise and
 * never throws; b2q_last_error() gives the message.  There is no CPU fallback: without a CUDA device
 * b2q_create fails with B2Q_ECUDA.
 *
 * Element type of all real-valued device arrays: float when B2QConfig.precision == 0 (the product
 * path), double when == 1 (the same kernels instantiated in float64 — a validation build used by the
 * parity tests to separate algorithmic from rounding differences).
 *
 * Reference interfaces replaced (paths relative to QuadrupedalRobots/ETGRL):
 *   b2q_create      rlschool.make_env('Quadrupedal', ...)                  train.py:305-309, env_test.py:43-46
 *   b2q_obs_dim     env.observation_space.shape[0]                         train.py:311
 *   b2q_act_dim     env.action_space.shape[0]                              train.py:312
 *   b2q_reset       env.reset(ETG_w=, ETG_b=, x_noise=) / reset(dynamic_param=)   train.py:131, Dynamic_parallel_model.py:55
 *   b2q_step        env.step(action, donef=) -> obs, reward, done, info    train.py:147,195,228
 *                   = Minitaur.Step minitaur.py:248-260 + stepSimulation :244 + ETG/IK a1.py:97-110
 *                     + obs pack EnvWrapper.py:60-109 + reward/termination
 *   b2q_set_dynamics  dynamic_param dict (param2dynamic_dict)              train.py:112-126
 *   b2q_mlp_*       Actor.forward / SAC.predict / SAC.sample               model/mujoco_model.py:53-60, alg/sac.py:60-75
 *   b2q_es_fitness  fitness_list.append(episode_reward) per individual     train.py:404-413
 */
#ifndef B2Q_H
#define B2Q_H
#include <stdint.h>
#include <stddef.h>
#ifdef __cplusplus
extern "C" {
#endif

#define B2Q_OK 0
#define B2Q_EINVAL (-1)
#define B2Q_ECUDA (-2)
#define B2Q_ENOMEM (-3)

#define B2Q_ACT_DIM 12
#define B2Q_OBS_DIM 49   /* full layout: dis3 | contact4 | rpy3 drpy3 | q12 qd12 | ETG12  (EnvWrapper.py:60-109 order); b2q_obs_dim(h) <= 49 */
#define B2Q_INFO_DIM 56
#define B2Q_STATE_DIM 37 /* pos3 quat4(xyzw) vlin3 vang3 (world) q12 qd12 */
#define B2Q_DYN_DIM 48   /* kp12 kd12 mu latency_s g3 basemass baseinertia3 legmass3 leginertia12 */
#define B2Q_ETG_H 20

/* info columns (per env row of B2Q_INFO_DIM): the keys train.py consumes (velx :156, reward terms :150-155,
 * ETG_act env_test.py:54, joint_angle / obs-IMU Dynamic_parallel_model.py:63-64, real_action) */
enum {
  B2Q_INFO_VELX = 0, B2Q_INFO_TORSO = 1, B2Q_INFO_FEET = 2, B2Q_INFO_UP = 3, B2Q_INFO_TAU = 4, B2Q_INFO_STAND = 5,
  B2Q_INFO_BADFOOT = 6, B2Q_INFO_FOOTCONTACT = 7, B2Q_INFO_DONE = 8, B2Q_INFO_NAN = 9, B2Q_INFO_ENERGY = 10,
  B2Q_INFO_BASE_Z = 11, B2Q_INFO_ETG_ACT = 12 /*..23*/, B2Q_INFO_REAL_ACTION = 24 /*..35*/,
  B2Q_INFO_RPY = 36 /*..38*/, B2Q_INFO_DRPY = 39 /*..41*/, B2Q_INFO_JOINT_ANGLE = 42 /*..53*/, B2Q_INFO_FALL = 54,
  B2Q_INFO_STEP = 55
};

typedef struct B2QConfig {
  int32_t num_envs;
  int32_t device;            /* CUDA ordinal */
  int32_t precision;         /* 0 float32 (product), 1 float64 (validation) */
  int32_t threads_per_block; /* 0 = default (32: one warp = 8 robots per CTA) */
  double sim_dt;             /* 0.002 */
  int32_t action_repeat;     /* 13 */
  int32_t solver_iters;      /* int(300/action_repeat) = 23 */
  double erp, warmstart, contact_margin;
  int32_t action_interp;     /* Minitaur.ProcessAction, minitaur.py:1384-1401 */
  double torque_limit;       /* <=0 off */
  int32_t settle_steps;      /* a1.py:294-297 */
  int32_t max_episode_steps; /* >0: done also when an env's own step counter reaches it (per-env form of donef=(steps>max_step), train.py:147) */
  int32_t etg_enabled;       /* 1; 0 = make_env(ETG=0): action is the joint offset itself (Dynamic_parallel_model.py:49,59-60) */
  int32_t action_filter;     /* 2nd-order Butterworth low-pass on the joint targets (minitaur.py:250-251, action_filter.py:111-216) */
  double filter_highcut;     /* Hz; 4.0 (action_filter.py:44) */
  double etg_T, etg_T2, etg_sigma_sq, etg_amp, etg_phase0, etg_phase1; /* train.py:296-297 */
  double w_torso, w_feet, w_up, w_tau, w_stand, w_badfoot, w_footcontact, w_done, reward_p, vel_d; /* train.py:478-484 */
  double foot_radius;
  int32_t ring_depth;        /* control steps of observation history kept (control latency <= ring_depth*R-2 substeps) */
  int32_t auto_reset;        /* reset an env inside step when it reports done */
  int32_t terrain_type;      /* 0 plane, 1 height field */
  int32_t hf_nx, hf_ny;
  double hf_x0, hf_y0, hf_cell;
  const double* hf_host;     /* HOST pointer, [hf_ny][hf_nx], copied at create */
  int32_t clip_motor_commands; /* A1.ApplyAction -> _ClipMotorCommands (a1.py:428-458; enable_clip_motor_commands, default 0 as a1.py:229) */
  double max_angle_change;   /* MAX_MOTOR_ANGLE_CHANGE_PER_STEP = 0.2 rad per substep (a1.py:62) */
  /* ---- round 2 additions (all default to the round-1 behaviour) ---- */
  /* observation layout = sensor_mode of the reference (train.py:259-277; SimpleEnv.get_observation, deployment/envs/EnvWrapper.py:60-109):
   * blocks in sorted-key order  BaseDisplacement(3) | FootContactSensor(4) | IMU(6 or 3) | MotorAngle(12) / MotorAngleAcc(24) | ETG(12) */
  int32_t sensor_dis;        /* 1 */
  int32_t sensor_contact;    /* 1 */
  int32_t sensor_imu;        /* 1 = rpy+drpy (6), 2 = drpy only (3), 0 = off */
  int32_t sensor_motor;      /* 1 = angles+velocities (24), 2 = angles only (12), 0 = off */
  int32_t sensor_etg;        /* 1 */
  int32_t obs_normal;        /* 1 = normalised as EnvWrapper.py:66-106 (`normal`, train.py:306); 0 = raw sensor units */
  double noise_stdev[5];     /* Minitaur._AddSensorNoise stdevs: motor angle, motor velocity, motor torque, base rpy, base rpy rate
                              * (minitaur.py:59,635,762,785,805,880,1206-1211); all 0 = off */
  uint64_t noise_seed;       /* counter-based RNG key (Philox4x32-10 over (seed, env, step)) */
  int32_t stuck_termination; /* 1: done when the base position std over the last 10 control steps <= 2e-4 after step 10 (rlschool [EXT]) */
  int32_t body_collisions;   /* 1: `badfoot` counts non-toe leg links / trunk corners touching the terrain (not only low knees) */
  int32_t motor_mode;        /* 0 POSITION (laikago_motor.py:139-145), 1 TORQUE (laikago_motor.py:131-134: the action IS the torque),
                              * 2 HYBRID (laikago_motor.py:152-164): the action is [N][12][5] = per motor (q*, kp, qd*, kd, tau_ff), b2q_act_dim = 60,
                              * tau = -kp (q - q*) - kd (qd - qd*) + tau_ff; taken as commanded (no ETG / pose offset, interpolation or filter) */
  int32_t joint_limits;      /* 1: URDF joint limits (a1.py:186-223) as unilateral rows of the contact solve (one slot per leg) */
  int32_t external_force;    /* 1: per-env base push set with b2q_set_external_force (random_param['random_force'], train.py:254) */
  double base_damping[4];    /* Bullet btMultiBody base damping: linear k1,k2, angular k1,k2 (force = m v (k1 + k2 |v|)); 0 = off */
  double etg_foot_y_inset;   /* ETG nominal footholds pulled towards the body midline by this much (make_env(step_y=), train.py:463; balancebeam) */
  int32_t knee_contacts;     /* 1: the knee spheres (calf-joint origin, r 0.02) collide with the terrain: 3 more solver rows per leg (non-toe link contact response) */
} B2QConfig;

typedef struct B2QEnv* B2QHandle;

void b2q_default_config(B2QConfig* cfg);
int b2q_create(const B2QConfig* cfg, B2QHandle* out);
int b2q_destroy(B2QHandle h);
const char* b2q_last_error(B2QHandle h);   /* h may be NULL: last create error */
const char* b2q_version(void);
int b2q_num_envs(B2QHandle h);
int b2q_obs_dim(B2QHandle h);
int b2q_act_dim(B2QHandle h);
int b2q_info_dim(B2QHandle h);
int b2q_elem_size(B2QHandle h);            /* 4 or 8 */

/* dyn [N,48] (NULL = defaults for masked envs): repacks and re-settles the masked envs (snapshot for reset). */
int b2q_set_dynamics(B2QHandle h, const uint8_t* env_mask, const void* dyn, void* stream);
/* env_mask [N] u8 or NULL (= all). etg_w [N,3,20], etg_b [N,3] or NULL (keep). obs_out [N,49] or NULL. */
int b2q_reset(B2QHandle h, const uint8_t* env_mask, const void* etg_w, const void* etg_b, void* obs_out, void* stream);
/* b2q_reset plus a per-env initial x offset of the base [N] (env.reset(x_noise=...), train.py:131,505); x_offset may be NULL. */
int b2q_reset_ex(B2QHandle h, const uint8_t* env_mask, const void* etg_w, const void* etg_b, const void* x_offset, void* obs_out, void* stream);
/* world-frame force [N,3] applied at the base COM during every following control step (NULL = clear); needs cfg.external_force. */
int b2q_set_external_force(B2QHandle h, const void* force, void* stream);
/* action [N,12] (already scaled by act_bound, joint-space residual). obs [N,obs_dim], reward [N], done [N] u8, info [N,56]. */
int b2q_step(B2QHandle h, const void* action, int donef, void* obs, void* reward, uint8_t* done, void* info, void* stream);
/* The same step with HOST buffers (the reference-facing call: numpy in / numpy out), synchronous: on return obs / reward /
 * done (and info if non-NULL) hold this step's results.  With page-locked host memory (b2q_host_alloc, cudaHostAlloc,
 * torch pin_memory) the step kernel reads the action rows from and stores its coalesced observation block to the host
 * buffers directly over PCIe (no separate copies; the info rows are staged in shared memory and stored as one block per
 * CTA like the observations).  Pageable buffers are staged through device memory with cudaMemcpyAsync.  Environment variable B2Q_HOST_IO (read at b2q_create)
 * selects 0 = always memcpy, 1 = zero-copy actions only, 2 = zero-copy actions and outputs (default). */
int b2q_step_host(B2QHandle h, const void* action_host, int donef, void* obs_host, void* reward_host, uint8_t* done_host,
                  void* info_host, void* stream);
void* b2q_host_alloc(size_t bytes);   /* page-locked host memory, NULL on failure */
void b2q_host_free(void* p);
/* tests / checkpointing */
int b2q_get_state(B2QHandle h, void* state_out /*[N,37]*/, void* stream);
int b2q_set_state(B2QHandle h, const void* state_in /*[N,37]*/, void* stream);
int b2q_get_step_count(B2QHandle h, int32_t* out /*[N] device*/, void* stream);
/* number of kernels this handle has launched so far (bench.py's gpu_launches) */
int64_t b2q_launch_count(B2QHandle h);
/* changes cfg.max_episode_steps for every following step (BCtrain.py:313-314 lengthens the episodes during a run); >= 0, 0 = no step
 * limit.  Host-side only: a step already enqueued keeps the limit it was launched with.  A handle that never calls it keeps the
 * value of b2q_create. */
int b2q_set_max_episode_steps(B2QHandle h, int max_episode_steps);

/* Terrain atlas: env i of a height-field handle (terrain_type 1) reads tile tile_of_env[i] of `n_tiles` height fields instead of the
 * create-time one.  Every tile lies on the handle's grid (hf_nx, hf_ny, hf_x0, hf_y0, hf_cell).  tiles_host is a HOST array
 * [n_tiles][hf_ny][hf_nx], tile_of_env a HOST array [N] of indices in [0, n_tiles); both are copied.  The call waits for the stream,
 * replaces any earlier atlas, and re-settles every env's reset snapshot on its tile with the dynamics it has: call b2q_reset before the
 * next step.  From then on the handle runs the atlas kernels, in which env i computes what a plain height-field handle created on tile
 * tile_of_env[i] computes.  Returns B2Q_EINVAL for a plane handle, n_tiles < 1 or an index out of range.  An atlas handle refuses
 * b2q_snapshot_save, b2q_snapshot_load and b2q_render with B2Q_EINVAL. */
int b2q_set_terrain_tiles(B2QHandle h, const double* tiles_host, int n_tiles, const int32_t* tile_of_env, void* stream);

/* Whole-handle snapshot, for stopping a run and continuing it bit for bit.  The blob holds everything a later b2q_step / b2q_reset
 * reads: the SoA pool (state, snapshot, snap_obs, param, ETG packs, observation ring, position history, external force, step
 * counters) and the handle's mutable host fields (max_episode_steps).  It starts with a header: magic, format version, sizes,
 * precision, N, ring depth, obs_dim, the B2QConfig fields (pointers and device left out) and a hash of the height field.
 * dst / src are DEVICE pointers of b2q_snapshot_bytes(h) bytes, 16-byte aligned.  Save is stream-ordered with no host sync.  Load
 * reads the header to the host (one small copy, waited for), returns B2Q_EINVAL for a blob of another configuration, format or size
 * (b2q_last_error names the first field that differs) and otherwise enqueues the copy of the pool. */
int64_t b2q_snapshot_bytes(B2QHandle h);
int b2q_snapshot_save(B2QHandle h, void* dst, void* stream);
int b2q_snapshot_load(B2QHandle h, const void* src, void* stream);

#ifdef __cplusplus
}
#endif
#endif
