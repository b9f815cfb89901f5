"""Behaviour-cloning training on the GPU engine — the batched counterpart of ETGRL/BCtrain.py:87-199,201-327 (same flags and defaults
where they exist).  A 46-dim student that sees only the noisy obs[3:] (no base displacement: the hardware cannot measure it,
EnvWrapper.py:75-76) is cloned from a 49-dim SAC expert:

    observe (one kernel: student rows + sensor noise + ring append) -> student sample -> env step (auto-reset at e_step + 1 steps)
    every multiple of train_per_steps env steps: train_per_time shuffled passes over the ring, range(0, size - batch, batch) batches,
    replayed from CUDA graphs of (device gather, seeded BC update) steps (SACLearner.bc_sweep)
    every eval_every_steps env steps: run_random_eval (student vs expert, ref_ratio), e_step += 50 while < 600, itr_<steps>.pt

The one deviation from the reference's schedule: BCtrain trains at the end of the episode in which the multiple was crossed, the
batched loop at the control step that crosses it, over the first min(multiple, memory) rows of the ring (exactly the rows the
reference's ring held at that multiple).  The learner work per collected row is the reference's.

    python -m paddlerobotics_b200.bctrain --ref_agent expert.pt --ETG_path expert.npz --num_envs 4096
    python -m paddlerobotics_b200.bctrain --ref_agent expert.pt --ETG_path expert.npz --save_state 1; python -m paddlerobotics_b200.bctrain --resume BCtrain_log/exp0/state.pt --max_steps N
"""
import argparse
import json
import os
import time

import numpy as np
import torch

from . import bc
from .agent import MujocoAgent, SACLearner
from .env import VecQuadrupedalEnv, apply_dynamic_param, etg_of_path, quadrupedal_config
from .dynamics_grid import HELP as DYNAMICS_GRID_HELP
from .train import (TERRAIN_GRID_HELP, check_dynamics_grid, check_terrain_grid, evaluate_dynamics_grid, evaluate_terrain_grid, frame_writer,
                    run_evaluate_episodes)

ACTOR_LR, CRITIC_LR = 3e-4, 3e-4            # BCtrain.py:44-45
EVAL_STEPS, RANDOM_EVAL_STEPS = 600, 800    # run_evaluate_episodes(agent, env, 600, ...) BCtrain.py:321; run_random_eval(..., 800, ...) :302
E_STEP_GROWTH, E_STEP_MAX = 50, 600         # BCtrain.py:313-314


def parser():
    p = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    # ---- BCtrain.py:330-375
    p.add_argument("--outdir", type=str, default="BCtrain_log")
    p.add_argument("--max_steps", type=float, default=1e6, help="total env steps (all envs)")
    p.add_argument("--load", type=str, default="", help="student itr_*.pt to start from (or to evaluate with --eval 1)")
    p.add_argument("--eval", type=int, default=0, help="1: one deterministic episode of the --load student (run_evaluate_episodes, BCtrain.py:147-176)")
    p.add_argument("--suffix", type=str, default="exp0")
    p.add_argument("--task_mode", type=str, default="stairstair")
    p.add_argument("--step_y", type=float, default=0.05)
    p.add_argument("--random_dynamic", type=int, default=0)
    p.add_argument("--random_force", type=int, default=0)
    p.add_argument("--render", type=int, default=0)
    p.add_argument("--normal", type=int, default=1)
    p.add_argument("--vel_d", type=float, default=0.6)
    p.add_argument("--ETG", type=int, default=1)
    p.add_argument("--ETG_T", type=float, default=0.5)
    p.add_argument("--reward_p", type=float, default=1)
    p.add_argument("--e_step", type=int, default=400)
    p.add_argument("--act_mode", type=str, default="traj", choices=("traj", "pose", "torque"))
    p.add_argument("--ref_agent", type=str, default="data/model/StairStair_3_itr_960231.pt", help="the 49-dim SAC expert (.pt)")
    p.add_argument("--ETG_path", type=str, default="data/model/StairStair_3_itr_960231.npz", help="the expert's gait (.npz{w,b})")
    p.add_argument("--ETG_H", type=int, default=20)
    p.add_argument("--stand", type=float, default=0)
    p.add_argument("--torso", type=float, default=1)
    p.add_argument("--up", type=float, default=0.1)
    p.add_argument("--tau", type=float, default=0.1)
    p.add_argument("--feet", type=float, default=0.1)
    p.add_argument("--act_bound", type=float, default=0.3)
    for k in ("dis", "motor", "imu", "contact", "ETG"):
        p.add_argument("--sensor_" + k, type=int, default=1)
    for k in ("footpose", "ETG_obs", "dynamic", "exforce"):
        p.add_argument("--sensor_" + k, type=int, default=0)
    p.add_argument("--sensor_noise", type=int, default=1)
    p.add_argument("--RNN_mode", type=str, default="None")
    p.add_argument("--agent_mode", type=str, default="None")
    p.add_argument("--enable_action_filter", type=int, default=0)
    p.add_argument("--x_noise", type=int, default=0)
    # ---- the reference's data file of BCtrain.py:226-227 is not in its tree: nominal dynamics unless a 48-vector is given
    p.add_argument("--dynamic_param", type=str, default="", help="PATH.npy: a 48-vector in [-1, 1] -> param2dynamic_dict -> every env (BCtrain.py:226-227)")
    # ---- batched engine (module constants of BCtrain.py:34-40, or the batched train.py)
    p.add_argument("--num_envs", type=int, default=4096)
    p.add_argument("--batch", type=int, default=1024)                         # BATCH_SIZE
    p.add_argument("--memory", type=float, default=1e7)                       # MEMORY_SIZE: 3.8 GB of float32 at 46 + 49 columns
    p.add_argument("--warmup", type=int, default=200)                         # WARMUP_STEPS
    p.add_argument("--train_per_steps", type=int, default=1024)               # TRAIN_PER_STEPS
    p.add_argument("--train_per_time", type=int, default=10)                  # TRAIN_PER_TIME
    p.add_argument("--eval_every_steps", type=float, default=1e4)             # EVAL_EVERY_STEPS
    p.add_argument("--eval_envs", type=int, default=1, help="envs of each evaluation episode (one episode each, no auto-reset)")
    p.add_argument("--terrain_grid", type=int, default=0, help=TERRAIN_GRID_HELP)
    p.add_argument("--dynamics_grid", type=int, default=0, help=DYNAMICS_GRID_HELP)
    p.add_argument("--graph_steps", type=int, default=64, help="BC updates per captured CUDA graph")
    p.add_argument("--seed", type=int, default=0)
    p.add_argument("--render_dir", type=str, default="", help="--eval 1: write env 0's camera image of every step to DIR/img{step}.png")
    p.add_argument("--render_width", type=int, default=640)
    p.add_argument("--render_height", type=int, default=480)
    p.add_argument("--save_state", type=int, default=0, help="1: write the whole training state (envs, student learner, BC ring, expert, gait, "
                   "generators, counters) to <outdir>/<suffix>/state.pt after every evaluation block and when --max_steps is reached, replacing the "
                   "previous file atomically")
    p.add_argument("--resume", type=str, default="", help="a state.pt of bctrain --save_state: continue that run with its arguments (bit for bit until "
                   "the first BC update, then as close as two uninterrupted runs: the learner sums with f32 atomics); only --max_steps, --outdir, "
                   "--suffix and --save_state may be given with other values")
    return p


RESUME_FREE = ("max_steps", "outdir", "suffix", "save_state", "resume")      # the flags a --resume may change


def check_supported(args):
    """Options the batched engine does not provide raise before any device work (the make_env rule: honoured or raised, never ignored)."""
    if args.agent_mode == "stack":
        raise NotImplementedError("--agent_mode stack: the stacked-history student is not provided")
    if args.RNN_mode not in ("None", "", None):
        raise NotImplementedError("--RNN_mode %s: recurrent observation modes are not provided" % args.RNN_mode)
    for k in ("footpose", "ETG_obs", "dynamic", "exforce"):
        if getattr(args, "sensor_" + k):
            raise NotImplementedError("--sensor_%s 1: this rlschool-only observation block is not provided" % k)
    for k in ("dis", "motor", "imu", "contact", "ETG"):
        if getattr(args, "sensor_" + k) != 1:
            raise NotImplementedError("--sensor_%s %d: the student's noise slices (BCtrain.py:55-58) assume the full 49-dim observation" % (k, getattr(args, "sensor_" + k)))
    if args.random_dynamic:
        raise NotImplementedError("--random_dynamic 1: per-episode dynamics randomisation is not provided")
    if args.random_force:
        raise NotImplementedError("--random_force 1: per-episode pushes are not provided in the batched env")
    if args.stand != 0:
        raise NotImplementedError("--stand %g: the stand reward term is not provided" % args.stand)
    if args.render:
        raise NotImplementedError("--render 1: there is no GUI window; --eval 1 --render_dir writes the camera frames")
    if args.x_noise and not args.eval:
        raise NotImplementedError("--x_noise 1 while training: the device auto-reset starts every episode at x = 0")


def act_bound_of(args):
    """BCtrain.py:238-243."""
    if args.act_mode == "pose":
        return np.array([0.1, 0.7, 0.7] * 4)
    if args.act_mode == "torque":
        return np.array([10.0] * 12)
    return np.array([args.act_bound] * 12)


def sweep_schedule(total, num_envs, train_per_steps, train_per_time, batch, memory, warmup, graph_steps):
    """The passes of the control step that takes the env-step count from `total` to `total + num_envs`: for every multiple m of
    train_per_steps crossed, train_per_time passes over the first size = min(m, memory) rows when size >= warmup.  Yields one
    (m, size, offsets, chunks) per pass: offsets = range(0, size - batch, batch) (BCtrain.py:132), chunks = the graph replays of
    graph_steps updates and the eager remainder that cover them ([G] * (K // G) + [K % G] when nonzero)."""
    for m in range((total // train_per_steps + 1) * train_per_steps, total + num_envs + 1, train_per_steps):
        size = min(m, memory)
        if size < warmup:
            continue
        offsets = bc.pass_offsets(size, batch)
        k = len(offsets)
        chunks = [graph_steps] * (k // graph_steps) + ([k % graph_steps] if k % graph_steps else [])
        for _ in range(train_per_time):
            yield m, size, offsets, chunks


def env_kwargs(args):
    reward = {"torso": args.torso, "up": args.up, "tau": args.tau, "feet": args.feet, "stand": args.stand}
    cfg, _ = quadrupedal_config(task=args.task_mode, motor_control_mode=args.act_mode, normal=args.normal, reward_param=reward, ETG=args.ETG,
                                ETG_T=args.ETG_T, reward_p=args.reward_p, ETG_H=args.ETG_H, vel_d=args.vel_d, step_y=args.step_y,
                                enable_action_filter=args.enable_action_filter, seed=args.seed,
                                sensor_mode={"dis": args.sensor_dis, "motor": args.sensor_motor, "imu": args.sensor_imu, "contact": args.sensor_contact,
                                             "ETG": args.sensor_ETG})
    return cfg


def make_vec_env(args, n, auto_reset, max_episode_steps=0):
    env = VecQuadrupedalEnv(n, auto_reset=auto_reset, max_episode_steps=max_episode_steps, **env_kwargs(args))
    return apply_dynamic_param(env, args.dynamic_param)


def main(argv=None):
    from . import run_state
    p = parser()
    args = p.parse_args(argv)
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        raise NotImplementedError("bctrain under torchrun (WORLD_SIZE %s): its BC update has no data-parallel path; run it on one GPU"
                                  % os.environ["WORLD_SIZE"])
    state = None
    if args.resume:
        state = run_state.load_state(p, args.resume, "bctrain")
        args = run_state.resume_args(p, parser, argv, state["args"], RESUME_FREE, (("--load", "load"), ("--ETG_path", "ETG_path"), ("--eval 1", "eval")),
                                     "the student, the expert, the gait and the training loop")
    if args.save_state and not args.outdir:
        p.error("--save_state 1 writes <outdir>/<suffix>/state.pt: it needs --outdir")
    check_supported(args)
    check_terrain_grid(p, args)
    check_dynamics_grid(p, args)
    torch.manual_seed(args.seed); np.random.seed(args.seed)
    # a resume takes the gait and the expert from the state, not from --ETG_path / --ref_agent, whose files may have changed since
    w, b = etg_of_path(args.ETG_path, args.ETG_T) if state is None else (state["w"], state["b"])
    bound = torch.as_tensor(act_bound_of(args), dtype=torch.float32, device="cuda")
    student = MujocoAgent(46, 12, seed=args.seed)
    if args.load and state is None:
        student.restore(args.load)
    if args.eval:
        return evaluate(args, student, w, b, bound)
    n, memory, every = args.num_envs, int(args.memory), int(args.eval_every_steps)
    expert = MujocoAgent(49, 12, seed=args.seed)
    if state is None:
        expert.restore(args.ref_agent)
    else:
        expert.load_state_dict(state["expert"])
    e_step = args.e_step
    env = make_vec_env(args, n, auto_reset=True, max_episode_steps=e_step + 1)
    # The evaluation env needs no snapshot: random_eval resets every env of it before each episode, and neither it nor the student's
    # evaluation noise (keyed by the step number) draws from a generator that lives across evaluations.
    eval_env = make_vec_env(args, args.eval_envs, auto_reset=False)
    learner = SACLearner(student, args.batch, actor_lr=ACTOR_LR, critic_lr=CRITIC_LR)
    rpm = bc.BCReplayMemory(memory, 46, 49, device=env.device)
    gen = torch.Generator(device=env.device).manual_seed(args.seed)
    outdir = os.path.join(args.outdir, args.suffix)
    os.makedirs(outdir, exist_ok=True)
    obs = env.reset(w, b).clone()
    noise = bool(args.sensor_noise)
    total, it, updates, test_flag, t0 = 0, 0, 0, 0, time.perf_counter()
    ret_acc = torch.zeros(n, device=env.device); ep_sum = torch.zeros((), device=env.device); ep_cnt = torch.zeros((), device=env.device)
    log = []
    run_args = dict(vars(args))                                                            # what a --save_state file records
    if state is not None:
        # the learner's bc_sweep graphs are captured again at its first sweep: a new learner holds none
        env.load_state_dict(state["env"]); learner.load_state_dict(state["learner"]); rpm.load_state_dict(state["rpm"])
        gen.set_state(state["gen"]); np.random.set_state(state["np_random"])
        obs.copy_(state["obs"]); ret_acc.copy_(state["ret_acc"]); ep_sum.copy_(state["ep_sum"]); ep_cnt.copy_(state["ep_cnt"])
        total, it, updates, test_flag, e_step = (state["loop"][k] for k in ("total", "it", "updates", "test_flag", "e_step"))
        torch.cuda.synchronize()                                                           # the CPU sources are freed on return

    def save_state():
        torch.cuda.synchronize()
        run_state.write_atomic(os.path.join(outdir, "state.pt"), {
            "command": "bctrain", "args": run_args, "env": env.state_dict(), "learner": learner.state_dict(), "rpm": rpm.state_dict(),
            "expert": expert.state_dict(), "w": np.array(w), "b": np.array(b), "gen": gen.get_state(), "np_random": np.random.get_state(),
            "obs": obs.cpu(), "ret_acc": ret_acc.cpu(), "ep_sum": ep_sum.cpu(), "ep_cnt": ep_cnt.cpu(),
            "loop": {"total": total, "it": it, "updates": updates, "test_flag": test_flag, "e_step": e_step}})
    while total < args.max_steps:
        warm = rpm.size() < args.warmup                                                       # BCtrain.py:102-105
        a_obs = rpm.observe(obs, it, noise=noise, append=True, seed=args.seed)             # BCtrain.py:98-99,120
        if warm:
            act = torch.rand(n, 12, device=env.device, generator=gen) * 2 - 1
        else:
            act = learner.actor.forward(a_obs, mode=1, seed=it + 1)[0][0]                  # agent.sample(agent_obs)
        nobs, rew, done, _ = env.step(act * bound)
        obs.copy_(nobs)
        fin = done.float()
        ret_acc.add_(rew); ep_sum.add_((ret_acc * fin).sum()); ep_cnt.add_(fin.sum()); ret_acc.mul_(1.0 - fin)
        losses, k_step = [], 0
        for m, size, offsets, _ in sweep_schedule(total, n, args.train_per_steps, args.train_per_time, args.batch, memory, args.warmup, args.graph_steps):
            if len(offsets):
                perm = torch.randperm(size, device=env.device, generator=gen)
                losses.append(learner.bc_sweep(rpm, expert, perm, len(offsets), seed=args.seed, graph_steps=args.graph_steps, pull=False) * len(offsets))
                k_step += len(offsets)
        total += n; it += 1
        if k_step:
            updates += k_step
            l = torch.stack(losses).sum(0) / k_step
            el = time.perf_counter() - t0
            rec = {"env_steps": total, "iters": it, "rpm_size": rpm.size(), "updates": k_step, "total_updates": updates,
                   "critic_loss": float(l[0]), "actor_loss": float(l[1]), "episode_return": float(ep_sum / ep_cnt) if float(ep_cnt) > 0 else None,
                   "e_step": e_step, "env_steps_per_s": total / el}
            ep_sum.zero_(); ep_cnt.zero_()
            log.append(rec); print(json.dumps(rec), flush=True)
        if (total + 1) // every >= test_flag:                                                 # BCtrain.py:299-316
            while (total + 1) // every >= test_flag:
                test_flag += 1
                rec = random_eval(args, learner, expert, eval_env, w, b, bound)
                rec.update({"eval_env_steps": total})
                log.append(rec); print(json.dumps(rec), flush=True)
            if e_step < E_STEP_MAX:
                e_step += E_STEP_GROWTH
                env.set_max_episode_steps(e_step + 1)
            learner.pull()
            student.save(os.path.join(outdir, "itr_%d.pt" % total))
            if args.save_state:
                save_state()
    if args.save_state:
        save_state()
    torch.cuda.synchronize()
    learner.pull()
    env.close(); eval_env.close()
    return log


def random_eval(args, learner, expert, env, w, b, bound):
    """run_random_eval (BCtrain.py:178-199): the student's deterministic episode on noisy obs[3:] and the expert's on the full obs, at most
    800 steps each; ref_ratio = student return / expert return."""
    noise = bool(args.sensor_noise)
    obs_mem = bc.BCReplayMemory(1, 46, 49, device=env.device)       # observe(append=False) never touches its ring

    def student(o, s):
        # noise keys of the evaluation steps: step words from 2^30 up, apart from the training steps' 0, 1, 2, ...
        return learner.actor.forward(obs_mem.observe(o, 1 << 30 | s, noise=noise, append=False, seed=args.seed), mode=0)[0][0]
    stu = run_evaluate_episodes(env, w, b, policy=student, act_bound=bound, max_step=RANDOM_EVAL_STEPS)
    ref = run_evaluate_episodes(env, w, b, policy=lambda o, s: expert.predict_batch(o), act_bound=bound, max_step=RANDOM_EVAL_STEPS)
    return {"eval_return": stu["mean_return"], "eval_length": stu["mean_length"], "ref_return": ref["mean_return"], "ref_length": ref["mean_length"],
            "ref_ratio": stu["mean_return"] / ref["mean_return"] if ref["mean_return"] != 0 else None, "terms": stu["terms"]}


def evaluate(args, student, w, b, bound):
    """--eval 1 --load X.pt: run_evaluate_episodes (BCtrain.py:147-176,317-326) — the student's deterministic episode, at most 600 steps, on
    its (noisy) obs[3:]; one JSON line; --render_dir writes img{step}.png of env 0.  With --terrain_grid 1 or --dynamics_grid 1, the
    records of train.evaluate_terrain_grid or evaluate_dynamics_grid, in which every setting's envs see the sensor noise and --x_noise
    offsets of this episode."""
    if args.terrain_grid or getattr(args, "dynamics_grid", 0):
        return evaluate_grid(args, student, w, b, bound)
    env = make_vec_env(args, args.eval_envs, auto_reset=False)
    obs_mem = bc.BCReplayMemory(1, 46, 49, device=env.device)
    xo = np.random.uniform(-0.1, 0.1, args.eval_envs) if args.x_noise else None
    r = run_evaluate_episodes(env, w, b, policy=lambda o, s: student.predict_batch(obs_mem.observe(o, s, noise=bool(args.sensor_noise), append=False, seed=args.seed)),
                              act_bound=bound, max_step=EVAL_STEPS, x_offset=xo, render=frame_writer(env, args) if args.render_dir else None)
    rec = {"eval_envs": args.eval_envs, "mean_return": r["mean_return"], "mean_length": r["mean_length"], "terms": r["terms"]}
    print(json.dumps(rec), flush=True)
    env.close()
    return rec


def evaluate_grid(args, student, w, b, bound):
    """--eval 1 with --terrain_grid 1 or --dynamics_grid 1.  b2q_bc_observe keys the student's noise by the observation row, so the noise
    of env j of a single-setting episode is drawn once per step on zero rows (0 + sigma * normal is the noise itself) and added to env j
    of every geometry or dynamics setting: the same float32 sum the kernel forms, so each setting's student sees that episode's
    observations."""
    n, noise = args.eval_envs, bool(args.sensor_noise)
    xo = np.random.uniform(-0.1, 0.1, n) if args.x_noise else None
    obs_mem = bc.BCReplayMemory(1, 46, 49, device="cuda")
    zero = torch.zeros(n, 49, device="cuda")

    def policy(o, s):
        if not noise:
            return student.predict_batch(obs_mem.observe(o, s, noise=False, append=False, seed=args.seed))
        z = obs_mem.observe(zero, s, noise=True, append=False, seed=args.seed)
        return student.predict_batch((o[:, 3:].reshape(-1, n, 46) + z).reshape(-1, 46))
    grid = evaluate_terrain_grid if args.terrain_grid else evaluate_dynamics_grid
    return grid(args, env_kwargs(args), w, b, policy=policy, act_bound=bound, max_step=EVAL_STEPS, x_offset=xo)


if __name__ == "__main__":
    main()
