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
from .train import EVAL_TERMS

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
    p.add_argument("--graph_steps", type=int, default=64, help="BC updates per captured CUDA graph")
    p.add_argument("--seed", type=int, default=0)
    p.add_argument("--render_dir", type=str, default="", help="--eval 1: write env 0's camera image of every step to DIR/img{step}.png")
    p.add_argument("--render_width", type=int, default=640)
    p.add_argument("--render_height", type=int, default=480)
    return p


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


def run_episodes(env, policy, w, b, act_bound, max_step, x_noise=0, render=None):
    """One episode per env (no auto-reset), at most max_step + 1 control steps (donef = steps > max_step, BCtrain.py:161).  Return,
    length and the per-term sums freeze at each env's first done (b2q_es_accumulate, as train.evaluate).  render(steps): per-step hook."""
    from . import _lib
    from ._config import INFO
    lib, dev, n, es, stream = _lib.load(), env.device, env.num_envs, env.obs.element_size(), env._stream()
    nt = len(EVAL_TERMS)
    cols = torch.tensor([INFO[k] for k in EVAL_TERMS], device=dev)
    alive = torch.ones(n, dtype=torch.uint8, device=dev)
    ret, length = torch.zeros(n, dtype=env.dtype, device=dev), torch.zeros(n, dtype=torch.int32, device=dev)
    t_alive, t_sum, t_len = torch.empty(nt, n, dtype=torch.uint8, device=dev), torch.zeros(nt, n, dtype=env.dtype, device=dev), torch.zeros(nt, n, dtype=torch.int32, device=dev)
    t_val = torch.empty(nt, n, dtype=env.dtype, device=dev)
    xo = np.random.uniform(-0.1, 0.1, n) if x_noise else None
    obs = env.reset(w, b, x_offset=xo)
    for steps in range(1, max_step + 2):
        obs, rew, done, info = env.step(policy(obs, steps) * act_bound, donef=steps > max_step)
        if render is not None:
            render(steps)
        t_val.copy_(info.index_select(1, cols).T)
        t_alive.copy_(alive.expand(nt, n))
        for j in range(nt):
            assert lib.b2q_es_accumulate(t_val[j].data_ptr(), done.data_ptr(), t_alive[j].data_ptr(), t_sum[j].data_ptr(), t_len[j].data_ptr(), n, es, stream) == 0
        assert lib.b2q_es_accumulate(rew.data_ptr(), done.data_ptr(), alive.data_ptr(), ret.data_ptr(), length.data_ptr(), n, es, stream) == 0
        if not bool(alive.any()):
            break
    return {"mean_return": float(ret.double().mean()), "mean_length": float(length.double().mean()),
            "terms": {k: float(t_sum[j].double().mean()) for j, k in enumerate(EVAL_TERMS)}}


def main(argv=None):
    args = parser().parse_args(argv)
    check_supported(args)
    torch.manual_seed(args.seed); np.random.seed(args.seed)
    w, b = etg_of_path(args.ETG_path, args.ETG_T)
    bound = torch.as_tensor(act_bound_of(args), dtype=torch.float32, device="cuda")
    student = MujocoAgent(46, 12, seed=args.seed)
    if args.load:
        student.restore(args.load)
    if args.eval:
        return evaluate(args, student, w, b, bound)
    n, memory, every = args.num_envs, int(args.memory), int(args.eval_every_steps)
    expert = MujocoAgent(49, 12, seed=args.seed)
    expert.restore(args.ref_agent)
    e_step = args.e_step
    env = make_vec_env(args, n, auto_reset=True, max_episode_steps=e_step + 1)
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
    torch.cuda.synchronize()
    learner.pull()
    env.close(); eval_env.close()
    return log


def random_eval(args, learner, expert, env, w, b, bound):
    """run_random_eval (BCtrain.py:178-199): the student's deterministic episode on noisy obs[3:] and the expert's on the full obs, at most
    800 steps each; ref_ratio = student return / expert return."""
    noise = bool(args.sensor_noise)
    obs_mem = bc.BCReplayMemory(1, 46, 49, device=env.device)       # observe(append=False) never touches its ring
    # noise keys of the evaluation steps: step words from 2^30 up, apart from the training steps' 0, 1, 2, ...
    stu = run_episodes(env, lambda o, s: learner.actor.forward(obs_mem.observe(o, 1 << 30 | s, noise=noise, append=False, seed=args.seed), mode=0)[0][0],
                       w, b, bound, RANDOM_EVAL_STEPS)
    ref = run_episodes(env, lambda o, s: expert.predict_batch(o), w, b, bound, RANDOM_EVAL_STEPS)
    return {"eval_return": stu["mean_return"], "eval_length": stu["mean_length"], "ref_return": ref["mean_return"], "ref_length": ref["mean_length"],
            "ref_ratio": stu["mean_return"] / ref["mean_return"] if ref["mean_return"] != 0 else None, "terms": stu["terms"]}


def evaluate(args, student, w, b, bound):
    """--eval 1 --load X.pt: run_evaluate_episodes (BCtrain.py:147-176,317-326) — the student's deterministic episode, at most 600 steps, on
    its (noisy) obs[3:]; one JSON line; --render_dir writes img{step}.png of env 0."""
    from .render import write_png
    env = make_vec_env(args, args.eval_envs, auto_reset=False)
    obs_mem = bc.BCReplayMemory(1, 46, 49, device=env.device)
    if args.render_dir:
        os.makedirs(args.render_dir, exist_ok=True)

    def frame(steps):
        rgba = env.get_camera_image(args.render_width, args.render_height, env_ids=[0])[0]
        write_png(os.path.join(args.render_dir, "img%d.png" % steps), rgba[0].cpu().numpy())
    rec = run_episodes(env, lambda o, s: student.predict_batch(obs_mem.observe(o, s, noise=bool(args.sensor_noise), append=False, seed=args.seed)),
                       w, b, bound, EVAL_STEPS, x_noise=args.x_noise, render=frame if args.render_dir else None)
    rec = {"eval_envs": args.eval_envs, **rec}
    print(json.dumps(rec), flush=True)
    env.close()
    return rec


if __name__ == "__main__":
    main()
