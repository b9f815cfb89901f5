"""ETG-RL training loop on the GPU engine — the batched counterpart of ETGRL/train.py:252-449 (same phases, same flag names
where they exist): SAC episodes with one learner step per control step (train.py:163-169) over N parallel envs, and every
`ES_EVERY_STEPS` env steps an ES phase of `ES_TRAIN_STEPS` generations over the ETG control points (train.py:392-437).
Everything per-step stays on the device: obs -> fused MLP (wgmma) -> step kernel -> device replay -> SAC learn (CUDA graph), and the
per-episode statistics of train.py:150-157 (b2q_train_episode_stats), which every log record reads.  Every --eval_every_steps the block of
train.py:370-390 runs: a deterministic evaluation on --train_eval_envs envs, the e_step growth of --e_step_growth, the checkpoint of --outdir.
The reference's flags are honoured or refused before any device work (check_supported); --epsilon, --gamma, --random, --timesteps and
--timeinterval are accepted and ignored, as in the reference.

    python -m paddlerobotics_b200.train --num_envs 4096 --max_steps 2000000 --ES 1
    python -m paddlerobotics_b200.train --train_eval_envs 16 --e_step_growth 50 --outdir train_log
    python -m paddlerobotics_b200.train --outdir ckpt --save_state 1; python -m paddlerobotics_b200.train --outdir ckpt --resume ckpt/exp0/state.pt --max_steps N
    torchrun --nproc_per_node 8 -m paddlerobotics_b200.train --num_envs 32768 --batch 32768 --max_steps 16000000 --outdir ckpt

Under torchrun (WORLD_SIZE > 1) --num_envs, --batch, --memory and --popsize stay global sizes, split evenly over the ranks: each rank steps
its contiguous shard of the envs, keeps its own replay ring and samples its share of the batch; the data-parallel learner (sync "exact")
all-reduces the gradients between its phases, so every rank holds the same weights.  The step counters and cadences stay global.  Rank r
seeds torch with --seed + r (warm-up actions, exploration noise, --sensor_noise) and keys the learner's noise by r; NumPy's generator, which
the ES solver draws from, gets --seed on every rank.  Only rank 0 prints, evaluates (--train_eval_envs, --eval) and writes checkpoints.
--save_state / --resume run on one GPU only.
"""
import argparse
import json
import os
import time

import numpy as np
import torch

from . import _lib, dist_run, dynamics_grid, run_state
from .agent import MujocoAgent, SACLearner, flatten_params
from .env import VecQuadrupedalEnv, apply_dynamic_param, dynamic_param_row
from .es import PopulationEvaluator, SimpleGA, TrainEpisodeStats, solutions_to_etg_device
from .etg import ETG_layer, Opt_with_points
from .replay import ReplayMemory
from .run_state import write_atomic
from .terrain import GRID_KEYS, make_terrain, make_terrain_tiles, terrain_grid

GAMMA, TAU, ALPHA, ACTOR_LR, CRITIC_LR = 0.99, 0.005, 0.2, 3e-4, 3e-4     # train.py:43-47


def parser():
    p = argparse.ArgumentParser()
    p.add_argument("--num_envs", type=int, default=4096)
    p.add_argument("--max_steps", type=int, default=400000, help="total env steps (all envs)")
    p.add_argument("--batch", type=int, default=4096)
    p.add_argument("--warmup_steps", type=int, default=40960)          # WARMUP_STEPS = 1e4 per env-step in the reference
    p.add_argument("--memory", type=int, default=1000000)              # MEMORY_SIZE, train.py:41
    p.add_argument("--e_step", type=int, default=400)                  # train.py:476
    p.add_argument("--act_bound", type=float, default=0.3)             # train.py:488
    p.add_argument("--ETG_T", type=float, default=0.5)
    p.add_argument("--footheight", type=float, default=0.1)
    p.add_argument("--steplen", type=float, default=0.05)
    p.add_argument("--ES", type=int, default=1)
    p.add_argument("--popsize", type=int, default=40)
    p.add_argument("--es_rollouts", type=int, default=4)
    p.add_argument("--es_every_steps", type=int, default=200000)       # ES_EVERY_STEPS = 5e4 per env in the reference
    p.add_argument("--es_train_steps", type=int, default=3)            # ES_TRAIN_STEPS = 10
    p.add_argument("--es_rpm", type=int, default=0, help="1: the ES phase also feeds SAC: the incumbent's episode and the first rollout of every "
                   "individual are appended to the replay memory (run_EStrain_episode, train.py:240-241; the reference's default is 1)")
    p.add_argument("--sigma", type=float, default=0.02)
    p.add_argument("--sigma_decay", type=float, default=0.99)
    p.add_argument("--seed", type=int, default=0)
    p.add_argument("--log_every", type=int, default=50)
    p.add_argument("--overlap", type=int, default=1, help="run the SAC update on a second stream beside the env step")
    p.add_argument("--graph_iter", type=int, default=1, help="capture one whole training iteration (policy forward, env step, replay append + sample, SAC update) "
                   "in ONE CUDA graph and replay it per control step (needs --overlap 1)")
    p.add_argument("--torso", type=float, default=1.5); p.add_argument("--feet", type=float, default=0.3); p.add_argument("--up", type=float, default=0.6)
    p.add_argument("--tau", type=float, default=0.07); p.add_argument("--badfoot", type=float, default=0.1); p.add_argument("--footcontact", type=float, default=0.1)
    p.add_argument("--task_mode", type=str, default="stairstair")      # train.py:462
    p.add_argument("--step_y", type=float, default=0.05)               # train.py:463
    p.add_argument("--outdir", type=str, default="", help="where itr_<steps>.pt / .npz are written (train.py:386-390); empty = no checkpoints")
    p.add_argument("--suffix", type=str, default="exp0")
    p.add_argument("--eval_every_steps", type=int, default=0, help="checkpoint cadence in env steps; 0 = EVAL_EVERY_STEPS (1e4) per env")
    p.add_argument("--load", type=str, default="", help="itr_*.pt to restore the agent from (and the .npz next to it for w, b, param)")
    p.add_argument("--eval", type=int, default=0, help="1: evaluate the --load checkpoint instead of training (run_evaluate_episodes, train.py:182-211,438-449)")
    p.add_argument("--eval_envs", type=int, default=1, help="envs of the --eval episode (one episode each, no auto-reset)")
    p.add_argument("--terrain_grid", type=int, default=0, help=TERRAIN_GRID_HELP)
    p.add_argument("--dynamics_grid", type=int, default=0, help=dynamics_grid.HELP)
    p.add_argument("--render_dir", type=str, default="", help="--eval: write env 0's camera image of every step to DIR/img{step}.png (train.py:196-199); empty = no frames")
    p.add_argument("--render_width", type=int, default=640)
    p.add_argument("--render_height", type=int, default=480)
    p.add_argument("--dynamic_param", type=str, default="", help="PATH.npy: a 48-vector in [-1, 1] (dynamic_train's dynamic_param{epoch}.npy) -> "
                   "param2dynamic_dict -> every env of training, the ES phase and --eval (train.py:302-303); empty = nominal dynamics")
    p.add_argument("--ETG_path", type=str, default="None", help="a pretrained ETG (.npz with `param`, e.g. pretrain's itr_*.npz): its 12 control-point "
                   "offsets seed the ES solver and the first gait (train.py:281-299); a missing file keeps zero offsets.  Not with --load")
    p.add_argument("--train_eval_envs", type=int, default=0, help="K > 0: every --eval_every_steps, one deterministic episode (at most 601 steps) on each of "
                   "K envs of a separate handle (run_evaluate_episodes, train.py:370-383) and one JSON record; 0 = no evaluation")
    p.add_argument("--save_state", type=int, default=0, help="1: write the whole training state to <outdir>/<suffix>/state.pt after every evaluation block "
                   "(after its iteration's ES phase) and when --max_steps is reached, replacing the previous file atomically (needs --outdir)")
    p.add_argument("--resume", type=str, default="", help="a state.pt of --save_state: continue that run with its arguments (bit for bit until the first learn, then as close as two "
                   "uninterrupted runs: the learner sums with f32 atomics); only --max_steps, "
                   "--log_every, --outdir, --suffix and --save_state may be given with other values")
    p.add_argument("--e_step_growth", type=int, default=0, help="G > 0: every --eval_every_steps, `if e_step < 600: e_step += G` (train.py:384-385; the "
                   "reference's G is 50); 0 = a fixed --e_step")
    p.add_argument("--dist_backend", type=str, default="nccl", choices=dist_run.BACKENDS, help="under torchrun: the process group's backend; gloo lets "
                   "several ranks share one GPU, and needs --graph_iter 0 (a gloo collective cannot be captured in a CUDA graph)")
    # ---- the rest of the reference's flags (train.py:452-505), with its defaults
    p.add_argument("--act_mode", type=str, default="traj", choices=("traj", "pose", "torque"), help="motor mode and act_bound (train.py:279,315-320)")
    p.add_argument("--normal", type=int, default=1)
    p.add_argument("--vel_d", type=float, default=0.5)
    p.add_argument("--reward_p", type=float, default=5)
    p.add_argument("--ETG", type=int, default=1, help="0: no ETG, the policy's action is the whole residual (needs --ES 0)")
    p.add_argument("--ETG_T2", type=float, default=0.5)
    p.add_argument("--ETG_H", type=int, default=20)
    p.add_argument("--stand", type=float, default=0)
    p.add_argument("--enable_action_filter", type=int, default=0)
    for k in ("dis", "motor", "imu", "contact", "ETG"):
        p.add_argument("--sensor_" + k, type=int, default=1)
    for k in ("ETG_obs", "footpose", "dynamic", "exforce"):
        p.add_argument("--sensor_" + k, type=int, default=0)
    p.add_argument("--sensor_noise", type=int, default=0, help="1: Gaussian sensor noise (SENSOR_NOISE_STDDEV), seeded by --seed")
    p.add_argument("--RNN_mode", type=str, default="None")
    p.add_argument("--random_dynamic", type=int, default=0)
    p.add_argument("--random_force", type=int, default=0)
    p.add_argument("--x_noise", type=int, default=0)
    p.add_argument("--render", type=int, default=0)
    for k, t, d in (("epsilon", float, 0.4), ("gamma", float, 0.95), ("random", int, 0), ("timesteps", int, 5), ("timeinterval", int, 1)):
        p.add_argument("--" + k, type=t, default=d, help="accepted and ignored, as in the reference")
    return p


def check_supported(args):
    """Options the batched engine does not provide raise before any device work (the make_env rule: honoured or raised, never ignored)."""
    if args.ETG_H != 20:
        raise NotImplementedError("--ETG_H %d: the RBF layer width is fixed at 20 in the kernel" % args.ETG_H)
    if args.ETG_T2 != args.ETG_T:
        raise NotImplementedError("--ETG_T2 %g != --ETG_T %g: the second ETG period is not provided" % (args.ETG_T2, args.ETG_T))
    if args.stand != 0:
        raise NotImplementedError("--stand %g: the stand reward term is not provided" % args.stand)
    for k in ("ETG_obs", "footpose", "dynamic", "exforce"):
        if getattr(args, "sensor_" + k):
            raise NotImplementedError("--sensor_%s 1: this rlschool-only observation block is not provided" % k)
    if args.RNN_mode not in ("None", "", None):
        raise NotImplementedError("--RNN_mode %s: recurrent observation modes are not provided" % args.RNN_mode)
    if args.random_dynamic:
        raise NotImplementedError("--random_dynamic 1: per-episode dynamics randomisation is not provided")
    if args.random_force:
        raise NotImplementedError("--random_force 1: per-episode pushes are not provided in the batched env")
    if args.x_noise:
        raise NotImplementedError("--x_noise 1: the device auto-reset starts every episode at x = 0")
    if args.render:
        raise NotImplementedError("--render 1: there is no GUI window; --eval 1 --render_dir writes the camera frames")


def obs_width(args):
    """The observation width the --sensor_* flags select (env.observation_dim of the training env)."""
    from .deploy import obs_dim_of
    return obs_dim_of(args.sensor_dis, args.sensor_motor, args.sensor_imu, args.sensor_contact, args.sensor_ETG)


def check_args(p, args):
    """The argument errors of main, raised (p.error) before any device work."""
    check_terrain_grid(p, args)
    if getattr(args, "terrain_grid", 0) and args.sensor_noise:
        p.error("--terrain_grid 1 with --sensor_noise 1: the step kernel keys its sensor noise by the env's index in the handle, so a "
                "geometry's envs would not draw the noise of the same --eval 1 episode")
    check_dynamics_grid(p, args)
    if getattr(args, "dynamics_grid", 0) and args.sensor_noise:
        p.error("--dynamics_grid 1 with --sensor_noise 1: the step kernel keys its sensor noise by the env's index in the handle, so a "
                "setting's envs would not draw the noise of the same --eval 1 episode")
    if args.ES and not args.ETG:
        p.error("--ETG 0 with --ES 1: the ES phase searches the ETG, which --ETG 0 turns off")
    if args.train_eval_envs < 0 or args.e_step_growth < 0:
        p.error("--train_eval_envs and --e_step_growth must be >= 0")
    if args.load:
        import torch
        have = int(torch.load(args.load, map_location="cpu")["actor_model.l1.weight"].shape[1])
        if have != obs_width(args):
            p.error("--load %s: the actor takes %d inputs, but the --sensor_* flags give a %d-wide observation" % (args.load, have, obs_width(args)))


RESUME_FREE = ("max_steps", "log_every", "outdir", "suffix", "save_state", "resume")     # the flags a --resume may change
RESUME_CONFLICTS = (("--load", "load"), ("--ETG_path", "ETG_path"), ("--eval 1", "eval"))


def check_world(p, args, world):
    """The refusals of a run over `world` > 1 ranks, raised before any device work."""
    if args.save_state or args.resume:
        raise NotImplementedError("--save_state / --resume with WORLD_SIZE %d: every rank's env shard, replay ring and generators would need their own "
                                  "state file; run it on one GPU" % world)
    dist_run.check_divisible(p, world, num_envs=args.num_envs, batch=args.batch, memory=args.memory, popsize=args.popsize)
    if args.dist_backend == "gloo" and args.graph_iter:
        p.error("--dist_backend gloo with --graph_iter 1: gloo collectives run on the host and cannot be captured in the iteration's CUDA graph; "
                "give --graph_iter 0, or use nccl")


def resume_args(p, argv, saved):
    """The arguments of a --resume run: the saved run's, with the RESUME_FREE flags of this command line.  Any other flag given on the
    command line with a value other than the saved one is an argument error (p.error) naming the flags, as are --load, --ETG_path and
    --eval 1, which set what the state restores."""
    return run_state.resume_args(p, parser, argv, saved, RESUME_FREE, RESUME_CONFLICTS, "the agent, the ETG and the training loop")


def grow_e_step(e_step, growth):
    """train.py:384-385 with the reference's 50 as `growth`."""
    if e_step < EVAL_MAX_STEP:
        e_step += growth
    return e_step


def block_due(total, test_flag, every):
    """train.py:370-372's test of the evaluation / e_step / checkpoint block after the control step that took the env-step count to `total`:
    (due, test_flag).  test_flag starts at 1, not at the reference's 0, so the first block (also this loop's first checkpoint) comes at the
    first multiple of `every`, not after the first iteration.  When `every` is a multiple of the number of envs (the default 1e4 per env),
    the blocks fall on the iterations where the env-step count reaches each multiple."""
    if (total + 1) // every >= test_flag:
        while (total + 1) // every >= test_flag:
            test_flag += 1
        return True, test_flag
    return False, test_flag


def etg_prior(ETG_T=0.5, footheight=0.1, steplen=0.05):
    """(layer, w0, b0, prior_points) of the default gait fit (train.py:296-299)."""
    layer = ETG_layer(ETG_T, 0.026, 20, 0.04, np.array([-np.pi / 2, 0]), 0.2, ETG_T)
    w0, b0, prior_points = Opt_with_points(ETG=layer, ETG_T=ETG_T, Footheight=footheight, Steplength=steplen)
    return layer, w0, b0, prior_points


def initial_etg(args):
    """The ES init rule of train.py:281-287 / pretrain.py:171-177: (param [12], w, b).  If --ETG_path is an existing file, param is its `param`
    (12 values, a 6x2 array is flattened; any other size raises ValueError naming the file) and (w, b) = Opt_with_points(prior_points + param)
    warm-started from (w0, b0), the fit train.py:349-352 makes of the solver's best param; otherwise (zeros, w0, b0).  Nothing is written:
    the reference's data/zero_param.npz is not created."""
    layer, w0, b0, prior_points = etg_prior(args.ETG_T, args.footheight, args.steplen)
    path = args.ETG_path
    if not path or path == "None" or not os.path.isfile(path):
        return np.zeros(12), w0, b0
    with np.load(path) as z:
        if "param" not in z.files:
            raise ValueError("%s: an ETG file needs a `param` array (12 control-point offsets)" % path)
        param = np.asarray(z["param"], dtype=np.float64)
    if param.size != 12:
        raise ValueError("%s: `param` must hold 12 control-point offsets, got shape %s" % (path, list(param.shape)))
    param = param.reshape(-1).copy()
    w, b, _ = Opt_with_points(ETG=layer, ETG_T=args.ETG_T, w0=w0, b0=b0, points=prior_points + param.reshape(-1, 2))
    return param, w, b


def env_config(args):
    """The reward weights of the command line (train.py:255-261) and the ETG period go to BOTH the training env and the ES evaluator: ES
    must optimise the reward SAC is trained on, with the gait (w, b) is fitted to."""
    return dict(w_torso=args.torso, w_feet=args.feet, w_up=args.up, w_tau=args.tau, w_badfoot=args.badfoot, w_footcontact=args.footcontact,
                heightfield=make_terrain(args.task_mode, step_y=args.step_y), stuck_termination=1, body_collisions=1,
                etg_foot_y_inset=args.step_y if args.task_mode == "balancebeam" else 0.0, etg_T=float(args.ETG_T), etg_T2=float(args.ETG_T))


def train_env_config(args, rank=0):
    """env_config plus the observation, action and reward flags of this command (the make_env keywords of train.py:305-309).  Joint limits and
    knee contacts stay off, as in every earlier version of this command (quadrupedal_config turns them on).  --sensor_noise draws from
    --seed + rank."""
    from .env import SENSOR_NOISE_STDDEV, _motor_mode
    cfg = env_config(args)
    cfg.update(vel_d=float(args.vel_d), reward_p=float(args.reward_p), obs_normal=int(bool(args.normal)), action_filter=int(bool(args.enable_action_filter)),
               etg_enabled=int(bool(args.ETG)), motor_mode=_motor_mode(args.act_mode), sensor_dis=int(bool(args.sensor_dis)),
               sensor_contact=int(bool(args.sensor_contact)), sensor_imu=int(args.sensor_imu), sensor_motor=int(args.sensor_motor), sensor_etg=int(bool(args.sensor_ETG)))
    if args.sensor_noise:
        cfg.update(noise_stdev=SENSOR_NOISE_STDDEV, noise_seed=int(args.seed) + rank)
    return cfg


def make_envs(args, env_cfg, policy=None, act_bound=None, rank=0, world=1, device=0):
    """The training env (this rank's shard of --num_envs) and the ES phase's PopulationEvaluator (this rank's shard of the population; None
    without --ES), both on the --dynamic_param dynamics."""
    env = apply_dynamic_param(VecQuadrupedalEnv(args.num_envs // world, device=device, auto_reset=True, max_episode_steps=args.e_step, **env_cfg),
                              args.dynamic_param)
    evaluator = None
    if args.ES:
        evaluator = PopulationEvaluator(args.popsize, args.es_rollouts, max_steps=args.e_step, rank=rank, world=world, device=device, policy=policy,
                                        act_bound=args.act_bound if act_bound is None else act_bound, **env_cfg)
        apply_dynamic_param(evaluator.env, args.dynamic_param)
    return env, evaluator


def make_eval_env(args, env_cfg, n, device=0):
    """An env of n envs without auto-reset on the training configuration and the --dynamic_param dynamics (--eval, --train_eval_envs)."""
    return apply_dynamic_param(VecQuadrupedalEnv(n, device=device, auto_reset=False, **env_cfg), args.dynamic_param)


def main(argv=None):
    p = parser()
    args = p.parse_args(argv)
    rank, world, local = dist_run.ranks()
    if world > 1:
        check_world(p, args, world)
    state = None
    if args.resume:
        state = run_state.load_state(p, args.resume, "train")
        args = resume_args(p, argv, state["args"])
    if args.save_state and not args.outdir:
        p.error("--save_state 1 writes <outdir>/<suffix>/state.pt: it needs --outdir")
    check_supported(args)
    torch.manual_seed(args.seed + rank); np.random.seed(args.seed)
    env_cfg = train_env_config(args, rank)
    run_args = dict(vars(args))                      # what a --save_state file records
    if state is not None:
        args = argparse.Namespace(**run_args)
        args.load, args.ETG_path = "", "None"        # the state supersedes the saved run's starting agent and ETG
    if args.load and args.ETG_path not in ("", "None"):
        p.error("--ETG_path and --load both set the ETG: --load restores (w, b, param) from the .npz next to the checkpoint")
    if args.eval and not args.load:
        p.error("--eval 1 evaluates a checkpoint: it needs --load itr_*.pt")
    check_args(p, args)
    if args.eval:
        if rank != 0:
            return []                                                                                                             # --eval runs on rank 0 alone
        world = 1
    with dist_run.process_group(world, local, getattr(args, "dist_backend", "nccl")) as dev:     # a state file may predate the flag
        from .bctrain import act_bound_of
        bound = act_bound_of(args)                                                                                                # train.py:315-320
        # a uniform bound stays a Python scalar: the same float32 products as before the per-motor bounds of --act_mode pose
        bound = float(bound[0]) if np.all(bound == bound[0]) else torch.as_tensor(bound, dtype=torch.float32, device=torch.device("cuda", dev))
        if args.eval:
            return evaluate(args, env_cfg, bound)
        return run(args, env_cfg, bound, state, run_args, rank, world, dev)


def run(args, env_cfg, bound, state, run_args, rank=0, world=1, dev=0):
    """The training loop on this rank (device `dev`) of `world` ranks; returns the records rank 0 printed, [] on the other ranks.  `state`: a
    --save_state file to continue from (one rank only)."""
    import torch.distributed as dist
    layer = ETG_layer(args.ETG_T, 0.026, 20, 0.04, np.array([-np.pi / 2, 0]), 0.2, args.ETG_T)
    w0, b0, prior_points = Opt_with_points(ETG=layer, ETG_T=args.ETG_T, Footheight=args.footheight, Steplength=args.steplen)     # train.py:298-299
    n_all = args.num_envs                       # the global env count: what `total` advances by per iteration
    n = n_all // world                          # this rank's shard
    key = rank << 40                            # the rank's offset of every counter-RNG seed: rank 0 keeps the single-GPU keys

    def say(rec, keep=True):
        if rank == 0:
            if keep:
                log.append(rec)
            print(json.dumps(rec), flush=True)

    def all_sum(t):
        if world > 1:
            dist.all_reduce(t)
        return t

    def warm():
        # train.py:141's rpm.size() >= WARMUP_STEPS over the global ring: until the first learn every rank has appended the same rows, and
        # afterwards the ring only grows, so W x this rank's fill level decides it on every rank alike without a collective
        return rpm.size() * world >= args.warmup_steps

    def check_replicas():
        if world > 1 and not dist_run.all_equal(learner.replica_state()):
            raise RuntimeError("the ranks' learners differ: the data-parallel update must leave every rank with the same weights and moments")
    # the evaluator's policy reads `learner` when it runs, so it may be built before the learner
    env, evaluator = make_envs(args, env_cfg, policy=lambda o: learner.actor.forward(o)[0][0], act_bound=bound, rank=rank, world=world, device=dev)
    eval_env = make_eval_env(args, env_cfg, args.train_eval_envs, device=dev) if args.train_eval_envs and rank == 0 else None
    od = env.observation_dim
    agent = MujocoAgent(od, 12, device=dev, seed=args.seed)
    ETG_best_param, w, b = initial_etg(args)                                                                                      # ES_solver.get_best_param(), train.py:348
    if args.load:
        agent.restore(args.load)
        z = np.load(args.load[:-3] + ".npz")                                                                                      # train.py:439-441
        w, b, ETG_best_param = z["w"], z["b"], z["param"].reshape(-1)
    outdir = os.path.join(args.outdir, args.suffix) if args.outdir and rank == 0 else ""
    if outdir:
        os.makedirs(outdir, exist_ok=True)
    ckpt_every = args.eval_every_steps or int(1e4) * n_all
    test_flag = 1
    e_step = args.e_step
    batch = args.batch // world
    learner = SACLearner(agent, batch, gamma=GAMMA, tau=TAU, alpha=ALPHA, actor_lr=ACTOR_LR, critic_lr=CRITIC_LR, world=world, seed_key=key)
    if world > 1 and not dist_run.all_equal(torch.cat(flatten_params(agent.params))):
        raise RuntimeError("the ranks built different agents from --seed %d" % args.seed)
    rpm = ReplayMemory(args.memory // world, od, 12, device=dev, device_cursor=bool(args.graph_iter and args.overlap))
    solver = SimpleGA(12, sigma_init=args.sigma, sigma_decay=args.sigma_decay, sigma_limit=0.005, elite_ratio=0.1, weight_decay=0.005,
                      popsize=args.popsize, param=ETG_best_param.copy())                                                          # train.py:288-295
    obs = env.reset(w, b).clone()
    total, it, last_es, t0 = 0, 0, 0, time.perf_counter()
    s_learn = torch.cuda.Stream(device=env.device)
    # the per-episode statistics of run_train_episode (train.py:150-157,175,359-366): one b2q_train_episode_stats launch per control step in
    # both loop modes, read and emptied by every log record
    stats = TrainEpisodeStats(_lib.load(), n, env.device, EVAL_TERMS)
    last_log = (0, 0.0)
    log = []
    # ---- one whole iteration as ONE CUDA graph (--graph_iter): everything step-dependent lives in device memory — the replay cursor, the learner's
    #      step counter (which also keys the rsample() noise), torch's graph-safe generator for the exploration noise — so the captured launches are
    #      valid for every later step.  The learner runs on its own stream inside the graph, beside the env step, exactly as in the eager loop below.
    #      The episode step limit is a kernel argument of the captured env step: a new limit (--e_step_growth) drops the graph, and the loop captures
    #      it again after one eager iteration.
    iter_graph = None
    if state is not None:
        env.load_state_dict(state["env"]); learner.load_state_dict(state["learner"]); rpm.load_state_dict(state["rpm"])
        stats.load_state_dict(state["stats"]); solver.load_state_dict(state["solver"])
        obs.copy_(state["obs"])
        L = state["loop"]
        total, it, last_es, test_flag, e_step, last_log = L["total"], L["it"], L["last_es"], L["test_flag"], L["e_step"], (L["last_log_total"], 0.0)
        ETG_best_param, w, b = state["ETG_best_param"], state["w"], state["b"]
        torch.set_rng_state(state["torch_rng"]); torch.cuda.set_rng_state(state["cuda_rng"], env.device)

    def save_state():
        torch.cuda.synchronize()
        write_atomic(os.path.join(outdir, "state.pt"), {
            "args": run_args, "env": env.state_dict(), "learner": learner.state_dict(), "rpm": rpm.state_dict(), "stats": stats.state_dict(),
            "solver": solver.state_dict(), "obs": obs.cpu(), "ETG_best_param": np.array(ETG_best_param), "w": np.array(w), "b": np.array(b),
            "loop": {"total": total, "it": it, "last_es": last_es, "test_flag": test_flag, "e_step": e_step, "last_log_total": last_log[0]},
            "graph": iter_graph is not None, "torch_rng": torch.get_rng_state(), "cuda_rng": torch.cuda.get_rng_state(env.device)})

    def graph_iteration():
        cur = torch.cuda.current_stream()
        act = learner.actor.forward(obs, mode=1, eps=torch.randn(n, 12, device=env.device))[0][0]     # agent.sample(obs)
        batch_t = rpm.sample_batch(batch, out=learner.static_batch())
        s_learn.wait_stream(cur)
        with torch.cuda.stream(s_learn):
            learner.learn(*batch_t, graph=False, pull=False)
        nobs, rew, done, info = env.step(act * bound)
        stats.step(rew, done, info, env._stream())
        rpm.append(obs, act, rew, nobs, 1.0 - done.float())
        cur.wait_stream(s_learn)
        obs.copy_(nobs)
    def capture_iteration():
        torch.cuda.synchronize()
        cap = torch.cuda.Stream(device=env.device)
        cap.wait_stream(torch.cuda.current_stream())
        g = torch.cuda.CUDAGraph()
        mirrors = (rpm._curr_pos, rpm._curr_size, rpm._samples)
        with torch.cuda.graph(g, stream=cap):
            graph_iteration()
        rpm._curr_pos, rpm._curr_size, rpm._samples = mirrors     # capture records launches, it does not run them: the ring has not moved
        torch.cuda.current_stream().wait_stream(cap)
        return g
    if state is not None and state["graph"]:
        # the saved run was replaying its captured iteration: capture it again, without the eager iteration that precedes a first capture
        # (its exploration noise would come from seed=it+1, not from torch's generator).  The captured learn() takes learner.steps + 1 as its
        # seed, and the saved run's graph holds the value learner.steps had after its capture, which replays leave unchanged.
        learner.steps -= 1
        learner.static_batch()     # allocated eagerly, as the uninterrupted run's eager iterations did: not from the graph's pool
        iter_graph = capture_iteration()
    while total < args.max_steps:
        if iter_graph is not None:
            iter_graph.replay()
            rpm.advance(n)
            rew, done = env.reward, env.done
            total += n_all; it += 1
        else:
            if not warm():
                act = torch.rand(n, 12, device=env.device) * 2 - 1                         # train.py:141-142
            else:
                act = learner.actor.forward(obs, mode=1, seed=it + 1 + key)[0][0]         # agent.sample(obs)
            learning = warm()
            if learning and args.overlap:
                # the learner step (latency-bound small kernels) runs on its own stream NEXT TO the env step (one warp per scheduler):
                # it samples transitions up to t-1 and its new weights are first used by the policy forward of step t+1, exactly as
                # in the sequential order, except that transition t itself joins the replay one update later
                batch_t = rpm.sample_batch(batch, out=learner.static_batch())
                s_learn.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(s_learn):
                    for x in batch_t:
                        x.record_stream(s_learn)
                    learner.learn(*batch_t, graph=True, pull=False)
            nobs, rew, done, info = env.step(act * bound)
            stats.step(rew, done, info, env._stream())
            rpm.append(obs, act, rew, nobs, 1.0 - done.float())                            # terminal = 1 - done, train.py:148-149,159
            if learning and args.overlap:
                torch.cuda.current_stream().wait_stream(s_learn)
            obs.copy_(nobs)
            total += n_all; it += 1
            if warm() and not (learning and args.overlap):
                learner.learn(*rpm.sample_batch(batch, out=learner.static_batch()), graph=True, pull=False)   # one update per control step, train.py:163-169
            if args.graph_iter and args.overlap and learning and it % args.log_every != 0:
                # warm-up is over and one eager learning iteration has run: capture the iteration once
                iter_graph = capture_iteration()
        if it % args.log_every == 0:
            torch.cuda.synchronize()
            el = time.perf_counter() - t0
            rate_int = (total - last_log[0]) / max(el - last_log[1], 1e-9); last_log = (total, el)
            ep = stats.take() if world == 1 else stats.take(all_sum)
            if world == 1:
                step_rew, done_frac, loss = float(rew.mean()), float(done.float().mean()), learner.losses
            else:                                   # global means: the envs of every rank, the shard losses averaged
                g = all_sum(torch.cat([torch.stack([rew.double().sum(), done.double().sum()]), learner.losses[:2].double()])).tolist()
                step_rew, done_frac, loss = g[0] / n_all, g[1] / n_all, (g[2] / world, g[3] / world)
            closed = ep["episodes"] + ep["nonfinite_episodes"] > 0
            rec = {"env_steps": total, "iters": it, "env_steps_per_s": total / el, "interval_env_steps_per_s": rate_int, "mean_step_reward": step_rew, "done_frac": done_frac,
                   "episode_return": ep["return"],
                   "critic_loss": float(loss[0]) if warm() else None, "actor_loss": float(loss[1]) if warm() else None,
                   "train_episodes": ep["episodes"] if closed else None, "train_nonfinite_episodes": ep["nonfinite_episodes"] if closed else None,
                   "train_episode_step": ep["length"]}
            for k in EVAL_TERMS:
                rec["train_episode_" + k], rec["train_mean_" + k] = ep["terms"][k], ep["mean_terms"][k]
            rec["train_success_rate"] = ep["success_rate"]
            say(rec)
        due, test_flag = block_due(total, test_flag, ckpt_every)
        if due:                                                                         # train.py:370-390, in its order
            if eval_env is not None:
                r = run_evaluate_episodes(eval_env, w, b, policy=lambda o, s: learner.actor.forward(o)[0][0], act_bound=bound, max_step=EVAL_MAX_STEP)
                say(eval_record(total, r, e_step))
            check_replicas()     # its all-gather is also where the other ranks wait for rank 0's evaluation
            if args.e_step_growth:
                grown = grow_e_step(e_step, args.e_step_growth)
                if grown != e_step:
                    e_step = grown
                    env.set_max_episode_steps(e_step)
                    iter_graph = None                                                   # the captured env step holds the old limit
            if outdir:                                                                  # agent.save + np.savez(w, b, param), train.py:386-390
                learner.pull()
                agent.save(os.path.join(outdir, "itr_%d.pt" % total))
                np.savez(os.path.join(outdir, "itr_%d.npz" % total), w=w, b=b, param=ETG_best_param)
        if evaluator is not None and total - last_es >= args.es_every_steps and warm():
            last_es = total
            # the incumbent ETG seeds best_reward (train.py:395-396): a sampled individual replaces it only if it is actually better
            es_replay = rpm if args.es_rpm else None
            # popsize copies of ONE gait: only one episode goes to the replay (train.py:395)
            inc_fit, _ = evaluator.evaluate(np.repeat(np.asarray(w)[None], args.popsize, 0), np.repeat(np.asarray(b)[None], args.popsize, 0),
                                            replay=es_replay, record=np.arange(args.popsize) == 0)
            es_rows = [int(all_sum(evaluator.rows.clone()))] if args.es_rpm else []
            inc = inc_fit.double().cpu().numpy()
            best_fit = float(np.nanmean(inc)) if np.isfinite(inc).any() else -np.inf
            best_param = ETG_best_param.copy()
            for gen in range(args.es_train_steps):                                     # train.py:397-418
                sol = solver.ask()
                ws, bs = solutions_to_etg_device(sol, prior_points, w0, b0, ETG_T=args.ETG_T, device=dev)
                fit, mlen = evaluator.evaluate(ws.cpu().numpy(), bs.cpu().numpy(), replay=es_replay)
                fit_np = fit.double().cpu().numpy()
                fit_np = np.where(np.isfinite(fit_np), fit_np, -1e9)                    # a diverged rollout must lose, not poison tell()
                solver.tell(fit_np)
                if fit_np.max() > best_fit:
                    best_fit, best_param = float(fit_np.max()), np.asarray(sol[int(fit_np.argmax())]).copy()
                rec = {"ES_gen": gen, "fitness_max": float(fit_np.max()), "fitness_mean": float(fit_np.mean()), "mean_len": float(mlen.mean())}
                if args.es_rpm:
                    es_rows.append(int(all_sum(evaluator.rows.clone())))
                    rec["rpm_rows"] = es_rows[-1]
                say(rec, keep=False)
            if args.es_rpm:
                # the masked appends advanced the ring's device cursor; one read brings the host mirrors level before the loop uses them
                rpm.sync_host()
                rpm_size = rpm.size() if world == 1 else int(all_sum(torch.tensor(rpm.size(), device=env.device)))
                say({"ES_rpm_rows": sum(es_rows), "env_steps": total, "rpm_size": rpm_size}, keep=False)
            ETG_best_param = best_param
            pts = prior_points + ETG_best_param.reshape(-1, 2)                          # train.py:433-437
            w, b, _ = Opt_with_points(ETG=layer, ETG_T=args.ETG_T, w0=w0, b0=b0, points=pts)
            solver.reset(ETG_best_param)
            obs.copy_(env.reset(w, b)); stats.restart()     # in place: the captured iteration graph reads and writes these tensors; cut episodes are dropped
        if due and args.save_state:
            save_state()
    if args.save_state:
        save_state()
    torch.cuda.synchronize()
    learner.pull()
    check_replicas()
    if eval_env is not None:
        eval_env.close()
    return log


def eval_record(total, r, e_step):
    """The eval/* scalars of train.py:376-383 for one run_evaluate_episodes result; e_step is the training episode limit in force."""
    rec = {"eval_env_steps": total, "eval_episode_reward": r["mean_return"], "eval_episode_step": r["mean_length"]}
    for k in EVAL_TERMS:
        rec["eval_episode_" + k] = r["terms"][k]
        rec["eval_mean_" + k] = r["terms"][k] / r["mean_length"]
    rec["eval_success_rate"] = r["success_rate"]
    rec["e_step"] = e_step
    return rec


EVAL_MAX_STEP = 600                                                         # run_evaluate_episodes(agent, env, 600, ...), train.py:445
EVAL_TERMS = ("torso", "feet", "up", "tau", "badfoot", "footcontact")       # the info terms summed per episode, train.py:202-207


def run_evaluate_episodes(env, w, b, policy=None, act_bound=0.3, max_step=EVAL_MAX_STEP, x_offset=None, render=None):
    """run_evaluate_episodes (train.py:182-211, BCtrain.py:147-176): one episode per env of `env` (no auto-reset) on the ETG (w, b), at most
    max_step + 1 control steps (the reference's loop breaks after step max_step + 1; donef forces the done flag of that step).
    policy(obs, steps) -> [N,12] in [-1, 1], scaled by act_bound, with steps the 1-based control step (bctrain keys the student's sensor
    noise by it); None = zero residual (the open-loop ETG).  x_offset: [N] start displacements along x for env.reset (bctrain --x_noise 1).
    Each env's return, length, EVAL_TERMS sums and velx success count freeze at its first done, all in one b2q_es_accumulate_terms launch
    per step.  render(steps): per-step hook.
    Returns {mean_return, mean_length, terms: {term: mean episode sum}, success_rate: mean over envs of count / length, per_env}, per_env
    holding the [N] device tensors these means are taken over: {return, length, terms: {term: episode sum}, success_rate}."""
    from . import _lib
    from .es import EpisodeStats
    n = env.num_envs
    stats = EpisodeStats(_lib.load(), n, env.dtype, env.device, EVAL_TERMS)
    stream = env._stream()
    zero = torch.zeros(n, 12, dtype=env.dtype, device=env.device) if policy is None else None
    obs = env.reset(w, b, x_offset=x_offset)
    for steps in range(1, max_step + 2):
        act = zero if policy is None else policy(obs, steps) * act_bound                                 # agent.predict(obs), train.py:193
        obs, rew, done, info = env.step(act, donef=steps > max_step)
        if render is not None:
            render(steps)
        stats.step(rew, done, info, stream)
        if not bool(stats.alive.any()):
            break
    return {"mean_return": float(stats.ret.double().mean()), "mean_length": float(stats.len.double().mean()),
            "terms": {k: float(stats.term_sum[j].double().mean()) for j, k in enumerate(EVAL_TERMS)},
            "success_rate": float(stats.success_rate().double().mean()),
            "per_env": {"return": stats.ret, "length": stats.len, "terms": {k: stats.term_sum[j] for j, k in enumerate(EVAL_TERMS)},
                        "success_rate": stats.success_rate()}}


TERRAIN_GRID_HELP = ("--eval 1: score on every stair / slope geometry of the task's grid (terrain.terrain_grid: train.py:48-50's step heights, "
                     "widths and slopes) in one batched rollout of --eval_envs envs per geometry; one JSON line per geometry and a summary")


def check_terrain_grid(p, args):
    """The argument errors of --terrain_grid 1 (train, pretrain, bctrain), raised (p.error) before any device work."""
    if not getattr(args, "terrain_grid", 0):
        return
    if not args.eval:
        p.error("--terrain_grid 1 scores a checkpoint or gait on every geometry of the task's grid: it needs --eval 1")
    if args.render_dir:
        p.error("--terrain_grid 1 with --render_dir: the camera ray-casts one height field, and a grid evaluation steps one per geometry")
    if args.task_mode not in GRID_KEYS:
        p.error("--terrain_grid 1 with --task_mode %s: this terrain has no step height, width or slope to vary (grids exist for %s)"
                % (args.task_mode, ", ".join(GRID_KEYS)))


def evaluate_settings(env, settings, summary, w, b, policy=None, act_bound=0.3, max_step=EVAL_MAX_STEP, x_offset=None):
    """The grid evaluations' shared core: the --eval 1 episode of n = env.num_envs / len(settings) envs for every setting, all in `env`,
    which the caller has set up so that env s * n + j runs env j of setting s.  policy(obs, steps) sees every setting's rows at once;
    x_offset: [n] start offsets, the same for every setting.  Each setting's record is its dict followed by run_evaluate_episodes' record
    over its envs, taken as run_evaluate_episodes takes it.  Prints one JSON line per setting, then summary(records); closes env;
    returns the records and the summary."""
    S = len(settings)
    n = env.num_envs // S
    r = run_evaluate_episodes(env, w, b, policy=policy, act_bound=act_bound, max_step=max_step, x_offset=None if x_offset is None else np.tile(x_offset, S))
    pe = r["per_env"]
    cols = [pe["return"], pe["length"], pe["success_rate"]] + [pe["terms"][k] for k in EVAL_TERMS]
    means = torch.stack([torch.stack([c[s * n:(s + 1) * n].double().mean() for c in cols]) for s in range(S)]).tolist()
    env.close()
    recs = []
    for setting, m in zip(settings, means):
        rec = dict(setting, mean_return=m[0], mean_length=m[1], success_rate=m[2], terms={k: m[3 + j] for j, k in enumerate(EVAL_TERMS)})
        recs.append(rec)
        print(json.dumps(rec), flush=True)
    summ = summary(recs)
    print(json.dumps(summ), flush=True)
    return recs + [summ]


def evaluate_terrain_grid(args, env_cfg, w, b, policy=None, act_bound=0.3, max_step=EVAL_MAX_STEP, x_offset=None):
    """--eval 1 --terrain_grid 1 of train, pretrain and bctrain: evaluate_settings on every geometry of terrain_grid(--task_mode), in one
    terrain-atlas env with env_cfg's configuration and the --dynamic_param dynamics.  A geometry's record leads with its grid values; the
    summary gives the number of geometries, the mean return over them, and the worst geometry and its return."""
    geoms = terrain_grid(args.task_mode)
    tiles, x0, y0, cell = make_terrain_tiles(args.task_mode, geoms, args.step_y)
    n, G = args.eval_envs, len(geoms)
    env = make_eval_env(args, dict(env_cfg, heightfield=(tiles[0], x0, y0, cell)), n * G)
    env.set_terrain_tiles(tiles, np.repeat(np.arange(G, dtype=np.int32), n))
    del tiles

    def summary(recs):
        worst = min(range(G), key=lambda g: recs[g]["mean_return"])
        return {"geometries": G, "eval_envs": n, "task_mode": args.task_mode, "mean_return": float(np.mean([rc["mean_return"] for rc in recs])),
                "worst": geoms[worst], "worst_return": recs[worst]["mean_return"]}
    return evaluate_settings(env, geoms, summary, w, b, policy=policy, act_bound=act_bound, max_step=max_step, x_offset=x_offset)


def check_dynamics_grid(p, args):
    """The argument errors of --dynamics_grid 1 (train, pretrain, bctrain), raised (p.error) before any device work."""
    if not getattr(args, "dynamics_grid", 0):
        return
    if not args.eval:
        p.error("--dynamics_grid 1 scores a checkpoint or gait on every setting of the dynamics sweep: it needs --eval 1")
    if getattr(args, "terrain_grid", 0):
        p.error("--dynamics_grid 1 with --terrain_grid 1: one grid evaluation at a time (each runs one setting per group of envs)")
    if args.render_dir:
        p.error("--dynamics_grid 1 with --render_dir: the frames show env 0, and a grid evaluation steps one setting per group of envs")


def evaluate_dynamics_grid(args, env_cfg, w, b, policy=None, act_bound=0.3, max_step=EVAL_MAX_STEP, x_offset=None):
    """--eval 1 --dynamics_grid 1 of train, pretrain and bctrain: evaluate_settings on the 82 settings of dynamics_grid.settings(), in one
    env with env_cfg's configuration (the --task_mode terrain) whose rows come from one set_dynamics call: env s * eval_envs + j has the
    run's --dynamic_param (or nominal) row with setting s's group at its level.  A setting's record leads with its group, level and the
    group's engine values; the summary gives the centre's return and, per group, the worst level, its return and the range of the
    return over the levels, most sensitive group first."""
    rows = dynamics_grid.swept_rows(dynamic_param_row(args.dynamic_param))
    n = args.eval_envs
    env = VecQuadrupedalEnv(n * len(rows), auto_reset=False, **env_cfg)
    env.set_dynamics(np.repeat(rows, n, 0))

    def summary(recs):
        return {"settings": len(recs), "eval_envs": n, "task_mode": args.task_mode, "dynamic_param": args.dynamic_param or None,
                "centre_return": recs[0]["mean_return"], "groups": dynamics_grid.group_summary(recs[1:], "mean_return")}
    return evaluate_settings(env, dynamics_grid.setting_records(), summary, w, b, policy=policy, act_bound=act_bound, max_step=max_step,
                             x_offset=x_offset)


def frame_writer(env, args):
    """--render_dir: a render hook that writes env 0's camera image of the current step to DIR/img{step}.png (train.py:196-199)."""
    from .render import write_png
    os.makedirs(args.render_dir, exist_ok=True)

    def frame(steps):
        rgba = env.get_camera_image(args.render_width, args.render_height, env_ids=[0])[0]
        write_png(os.path.join(args.render_dir, "img%d.png" % steps), rgba[0].cpu().numpy())
    return frame


def evaluate(args, env_cfg, act_bound):
    """--eval 1: one deterministic episode per env of the restored agent and ETG (w, b) on the training env's config, at most
    EVAL_MAX_STEP + 1 control steps (run_evaluate_episodes).  Prints and returns one JSON record; with --terrain_grid 1 or
    --dynamics_grid 1, the records of evaluate_terrain_grid or evaluate_dynamics_grid."""
    n = args.eval_envs
    z = np.load(args.load[:-3] + ".npz")                                                                                      # train.py:439-441
    w, b = z["w"], z["b"]
    if args.terrain_grid or getattr(args, "dynamics_grid", 0):
        agent = MujocoAgent(obs_width(args), 12, seed=args.seed)
        agent.restore(args.load)
        grid = evaluate_terrain_grid if args.terrain_grid else evaluate_dynamics_grid
        return grid(args, env_cfg, w, b, policy=lambda o, s: agent.predict_batch(o), act_bound=act_bound, max_step=EVAL_MAX_STEP)
    env = make_eval_env(args, env_cfg, n)
    agent = MujocoAgent(env.observation_dim, 12, seed=args.seed)
    agent.restore(args.load)
    r = run_evaluate_episodes(env, w, b, policy=lambda o, s: agent.predict_batch(o), act_bound=act_bound, max_step=EVAL_MAX_STEP,
                              render=frame_writer(env, args) if args.render_dir else None)
    rec = {"eval_envs": n, "mean_return": r["mean_return"], "mean_length": r["mean_length"], "terms": r["terms"]}
    print(json.dumps(rec), flush=True)
    env.close()
    return rec


if __name__ == "__main__":
    main()
