"""ETG-RL training loop on the GPU engine — the batched counterpart of ETGRL/train.py:252-449 (same phases, same flag names
where they exist): SAC episodes with one learner step per control step (train.py:163-169) over N parallel envs, and every
`ES_EVERY_STEPS` env steps an ES phase of `ES_TRAIN_STEPS` generations over the ETG control points (train.py:392-437).
Everything per-step stays on the device: obs -> fused MLP (wgmma) -> step kernel -> device replay -> SAC learn (CUDA graph).

    python -m paddlerobotics_b200.train --num_envs 4096 --max_steps 2000000 --ES 1
"""
import argparse
import json
import os
import time

import numpy as np
import torch

from .agent import MujocoAgent, SACLearner
from .env import VecQuadrupedalEnv, apply_dynamic_param
from .es import PopulationEvaluator, SimpleGA, solutions_to_etg_device
from .etg import ETG_layer, Opt_with_points
from .replay import ReplayMemory
from .terrain import make_terrain

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
    p.add_argument("--render_dir", type=str, default="", help="--eval: write env 0's camera image of every step to DIR/img{step}.png (train.py:196-199); empty = no frames")
    p.add_argument("--render_width", type=int, default=640)
    p.add_argument("--render_height", type=int, default=480)
    p.add_argument("--dynamic_param", type=str, default="", help="PATH.npy: a 48-vector in [-1, 1] (dynamic_train's dynamic_param{epoch}.npy) -> "
                   "param2dynamic_dict -> every env of training, the ES phase and --eval (train.py:302-303); empty = nominal dynamics")
    return p


def env_config(args):
    """The reward weights of the command line (train.py:255-261) go to BOTH the training env and the ES evaluator: ES must optimise the
    reward SAC is trained on."""
    return dict(w_torso=args.torso, w_feet=args.feet, w_up=args.up, w_tau=args.tau, w_badfoot=args.badfoot, w_footcontact=args.footcontact,
                heightfield=make_terrain(args.task_mode, step_y=args.step_y), stuck_termination=1, body_collisions=1,
                etg_foot_y_inset=args.step_y if args.task_mode == "balancebeam" else 0.0)


def make_envs(args, env_cfg, policy=None):
    """The training env and the ES phase's PopulationEvaluator (None without --ES), both on the --dynamic_param dynamics."""
    env = apply_dynamic_param(VecQuadrupedalEnv(args.num_envs, auto_reset=True, max_episode_steps=args.e_step, **env_cfg), args.dynamic_param)
    evaluator = None
    if args.ES:
        evaluator = PopulationEvaluator(args.popsize, args.es_rollouts, max_steps=args.e_step, policy=policy, act_bound=args.act_bound, **env_cfg)
        apply_dynamic_param(evaluator.env, args.dynamic_param)
    return env, evaluator


def main(argv=None):
    p = parser()
    args = p.parse_args(argv)
    torch.manual_seed(args.seed); np.random.seed(args.seed)
    n = args.num_envs
    layer = ETG_layer(args.ETG_T, 0.026, 20, 0.04, np.array([-np.pi / 2, 0]), 0.2, args.ETG_T)
    w0, b0, prior_points = Opt_with_points(ETG=layer, ETG_T=args.ETG_T, Footheight=args.footheight, Steplength=args.steplen)     # train.py:298-299
    w, b = w0, b0
    env_cfg = env_config(args)
    if args.eval:
        if not args.load:
            p.error("--eval 1 evaluates a checkpoint: it needs --load itr_*.pt")
        return evaluate(args, env_cfg)
    # the evaluator's policy reads `learner` when it runs, so it may be built before the learner
    env, evaluator = make_envs(args, env_cfg, policy=lambda o: learner.actor.forward(o)[0][0])
    agent = MujocoAgent(49, 12, seed=args.seed)
    ETG_best_param = np.zeros(12)                                                                                                 # ES_solver.get_best_param(), train.py:348
    if args.load:
        agent.restore(args.load)
        z = np.load(args.load[:-3] + ".npz")                                                                                      # train.py:439-441
        w, b, ETG_best_param = z["w"], z["b"], z["param"].reshape(-1)
    outdir = os.path.join(args.outdir, args.suffix) if args.outdir else ""
    if outdir:
        os.makedirs(outdir, exist_ok=True)
    ckpt_every = args.eval_every_steps or int(1e4) * n
    next_ckpt = ckpt_every
    learner = SACLearner(agent, args.batch, gamma=GAMMA, tau=TAU, alpha=ALPHA, actor_lr=ACTOR_LR, critic_lr=CRITIC_LR)
    rpm = ReplayMemory(args.memory, 49, 12, device_cursor=bool(args.graph_iter and args.overlap))
    solver = SimpleGA(12, sigma_init=args.sigma, sigma_decay=args.sigma_decay, sigma_limit=0.005, elite_ratio=0.1, weight_decay=0.005,
                      popsize=args.popsize, param=ETG_best_param.copy())                                                          # train.py:288-295
    obs = env.reset(w, b).clone()
    total, it, last_es, t0 = 0, 0, 0, time.perf_counter()
    s_learn = torch.cuda.Stream(device=env.device)
    ret_acc = torch.zeros(n, device=env.device); ep_rets = []; last_log = (0, 0.0)
    log = []
    # ---- one whole iteration as ONE CUDA graph (--graph_iter): everything step-dependent lives in device memory — the replay cursor, the learner's
    #      step counter (which also keys the rsample() noise), torch's graph-safe generator for the exploration noise — so the captured launches are
    #      valid for every later step.  The learner runs on its own stream inside the graph, beside the env step, exactly as in the eager loop below.
    iter_graph = None
    ep_sum = torch.zeros((), device=env.device); ep_cnt = torch.zeros((), device=env.device)
    def graph_iteration():
        cur = torch.cuda.current_stream()
        act = learner.actor.forward(obs, mode=1, eps=torch.randn(n, 12, device=env.device))[0][0]     # agent.sample(obs)
        batch_t = rpm.sample_batch(args.batch, out=learner.static_batch())
        s_learn.wait_stream(cur)
        with torch.cuda.stream(s_learn):
            learner.learn(*batch_t, graph=False, pull=False)
        nobs, rew, done, _ = env.step(act * args.act_bound)
        rpm.append(obs, act, rew, nobs, 1.0 - done.float())
        cur.wait_stream(s_learn)
        fin = done.float()
        ret_acc.add_(rew)
        ep_sum.add_((ret_acc * fin).sum()); ep_cnt.add_(fin.sum())
        ret_acc.mul_(1.0 - fin)
        obs.copy_(nobs)
    while total < args.max_steps:
        if iter_graph is not None:
            iter_graph.replay()
            rpm.advance(n)
            rew, done, losses = env.reward, env.done, learner.losses
            total += n; it += 1
            if it % args.log_every == 0 and float(ep_cnt) > 0:
                ep_rets.append(float(ep_sum / ep_cnt)); ep_sum.zero_(); ep_cnt.zero_()
        else:
            if rpm.size() < args.warmup_steps:
                act = torch.rand(n, 12, device=env.device) * 2 - 1                         # train.py:141-142
            else:
                act = learner.actor.forward(obs, mode=1, seed=it + 1)[0][0]               # agent.sample(obs)
            learning = rpm.size() >= args.warmup_steps
            if learning and args.overlap:
                # the learner step (latency-bound small kernels) runs on its own stream NEXT TO the env step (one warp per scheduler):
                # it samples transitions up to t-1 and its new weights are first used by the policy forward of step t+1, exactly as
                # in the sequential order, except that transition t itself joins the replay one update later
                batch_t = rpm.sample_batch(args.batch, out=learner.static_batch())
                s_learn.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(s_learn):
                    for x in batch_t:
                        x.record_stream(s_learn)
                    losses = learner.learn(*batch_t, graph=True, pull=False)
            nobs, rew, done, info = env.step(act * args.act_bound)
            rpm.append(obs, act, rew, nobs, 1.0 - done.float())                            # terminal = 1 - done, train.py:148-149,159
            if learning and args.overlap:
                torch.cuda.current_stream().wait_stream(s_learn)
            ret_acc += rew
            fin = done.bool()
            if it % args.log_every == 0 and bool(fin.any()):
                ep_rets.append(float(ret_acc[fin].mean()))
            ret_acc = torch.where(fin, torch.zeros_like(ret_acc), ret_acc)
            obs.copy_(nobs)
            total += n; it += 1
            if rpm.size() >= args.warmup_steps and not (learning and args.overlap):
                losses = learner.learn(*rpm.sample_batch(args.batch, out=learner.static_batch()), graph=True, pull=False)   # one update per control step, train.py:163-169
            if args.graph_iter and args.overlap and learning and it % args.log_every != 0:
                # warm-up is over and one eager learning iteration has run: capture the iteration once
                torch.cuda.synchronize()
                cap = torch.cuda.Stream(device=env.device)
                cap.wait_stream(torch.cuda.current_stream())
                iter_graph = torch.cuda.CUDAGraph()
                mirrors = (rpm._curr_pos, rpm._curr_size, rpm._samples)
                with torch.cuda.graph(iter_graph, stream=cap):
                    graph_iteration()
                rpm._curr_pos, rpm._curr_size, rpm._samples = mirrors     # capture records launches, it does not run them: the ring has not moved
                torch.cuda.current_stream().wait_stream(cap)
        if it % args.log_every == 0:
            torch.cuda.synchronize()
            el = time.perf_counter() - t0
            rate_int = (total - last_log[0]) / max(el - last_log[1], 1e-9); last_log = (total, el)
            rec = {"env_steps": total, "iters": it, "env_steps_per_s": total / el, "interval_env_steps_per_s": rate_int, "mean_step_reward": float(rew.mean()), "done_frac": float(done.float().mean()),
                   "episode_return": ep_rets[-1] if ep_rets else None,
                   "critic_loss": float(losses[0]) if rpm.size() >= args.warmup_steps else None, "actor_loss": float(losses[1]) if rpm.size() >= args.warmup_steps else None}
            log.append(rec); print(json.dumps(rec), flush=True)
        if outdir and total >= next_ckpt:                                               # agent.save + np.savez(w, b, param), train.py:386-390
            next_ckpt += ckpt_every
            learner.pull()
            agent.save(os.path.join(outdir, "itr_%d.pt" % total))
            np.savez(os.path.join(outdir, "itr_%d.npz" % total), w=w, b=b, param=ETG_best_param)
        if evaluator is not None and total - last_es >= args.es_every_steps and rpm.size() >= args.warmup_steps:
            last_es = total
            # the incumbent ETG seeds best_reward (train.py:395-396): a sampled individual replaces it only if it is actually better
            es_replay = rpm if args.es_rpm else None
            # popsize copies of ONE gait: only one episode goes to the replay (train.py:395)
            inc_fit, _ = evaluator.evaluate(np.repeat(np.asarray(w)[None], args.popsize, 0), np.repeat(np.asarray(b)[None], args.popsize, 0),
                                            replay=es_replay, record=np.arange(args.popsize) == 0)
            es_rows = [int(evaluator.rows)] if args.es_rpm else []
            inc = inc_fit.double().cpu().numpy()
            best_fit = float(np.nanmean(inc)) if np.isfinite(inc).any() else -np.inf
            best_param = ETG_best_param.copy()
            for gen in range(args.es_train_steps):                                     # train.py:397-418
                sol = solver.ask()
                ws, bs = solutions_to_etg_device(sol, prior_points, w0, b0, ETG_T=args.ETG_T)
                fit, mlen = evaluator.evaluate(ws.cpu().numpy(), bs.cpu().numpy(), replay=es_replay)
                fit_np = fit.double().cpu().numpy()
                fit_np = np.where(np.isfinite(fit_np), fit_np, -1e9)                    # a diverged rollout must lose, not poison tell()
                solver.tell(fit_np)
                if fit_np.max() > best_fit:
                    best_fit, best_param = float(fit_np.max()), np.asarray(sol[int(fit_np.argmax())]).copy()
                rec = {"ES_gen": gen, "fitness_max": float(fit_np.max()), "fitness_mean": float(fit_np.mean()), "mean_len": float(mlen.mean())}
                if args.es_rpm:
                    es_rows.append(int(evaluator.rows))
                    rec["rpm_rows"] = es_rows[-1]
                print(json.dumps(rec), flush=True)
            if args.es_rpm:
                # the masked appends advanced the ring's device cursor; one read brings the host mirrors level before the loop uses them
                rpm.sync_host()
                print(json.dumps({"ES_rpm_rows": sum(es_rows), "env_steps": total, "rpm_size": rpm.size()}), flush=True)
            ETG_best_param = best_param
            pts = prior_points + ETG_best_param.reshape(-1, 2)                          # train.py:433-437
            w, b, _ = Opt_with_points(ETG=layer, ETG_T=args.ETG_T, w0=w0, b0=b0, points=pts)
            solver.reset(ETG_best_param)
            obs.copy_(env.reset(w, b)); ret_acc.zero_()      # in place: the captured iteration graph reads and writes these tensors
    torch.cuda.synchronize()
    learner.pull()
    return log


EVAL_MAX_STEP = 600                                                         # run_evaluate_episodes(agent, env, 600, ...), train.py:445
EVAL_TERMS = ("torso", "feet", "up", "tau", "badfoot", "footcontact")       # the info terms summed per episode, train.py:202-207


def evaluate(args, env_cfg):
    """--eval 1: one deterministic episode per env of the restored agent and ETG (w, b) on the training env's config, at most
    EVAL_MAX_STEP + 1 control steps (the reference's loop breaks after step 601).  Each env's return, length and per-term sums are
    frozen at its first done by the ES evaluator's accumulator (b2q_es_accumulate).  Prints and returns one JSON record."""
    from . import _lib
    from ._config import INFO
    from .render import write_png
    agent = MujocoAgent(49, 12, seed=args.seed)
    agent.restore(args.load)
    z = np.load(args.load[:-3] + ".npz")                                                                                      # train.py:439-441
    w, b = z["w"], z["b"]
    n = args.eval_envs
    env = apply_dynamic_param(VecQuadrupedalEnv(n, auto_reset=False, **env_cfg), args.dynamic_param)
    lib, dev, es, stream = _lib.load(), env.device, env.obs.element_size(), env._stream()
    if args.render_dir:
        os.makedirs(args.render_dir, exist_ok=True)
    nt = len(EVAL_TERMS)
    cols = torch.tensor([INFO[k] for k in EVAL_TERMS], device=dev)
    alive = torch.ones(n, dtype=torch.uint8, device=dev)
    ret, length = torch.zeros(n, dtype=env.dtype, device=dev), torch.zeros(n, dtype=torch.int32, device=dev)
    # every term gets its own copy of `alive` per step (the accumulator clears it at done), so all sums freeze at the same step
    t_alive, t_sum, t_len = torch.empty(nt, n, dtype=torch.uint8, device=dev), torch.zeros(nt, n, dtype=env.dtype, device=dev), torch.zeros(nt, n, dtype=torch.int32, device=dev)
    t_val = torch.empty(nt, n, dtype=env.dtype, device=dev)
    obs = env.reset(w, b)
    for steps in range(1, EVAL_MAX_STEP + 2):
        act = agent.predict_batch(obs)                                                                        # agent.predict(obs), train.py:193
        obs, rew, done, info = env.step(act * args.act_bound, donef=steps > EVAL_MAX_STEP)
        if args.render_dir:
            rgba = env.get_camera_image(args.render_width, args.render_height, env_ids=[0])[0]
            write_png(os.path.join(args.render_dir, "img%d.png" % steps), rgba[0].cpu().numpy())
        t_val.copy_(info.index_select(1, cols).T)
        t_alive.copy_(alive.expand(nt, n))
        for j in range(nt):
            assert lib.b2q_es_accumulate(t_val[j].data_ptr(), done.data_ptr(), t_alive[j].data_ptr(), t_sum[j].data_ptr(), t_len[j].data_ptr(), n, es, stream) == 0
        assert lib.b2q_es_accumulate(rew.data_ptr(), done.data_ptr(), alive.data_ptr(), ret.data_ptr(), length.data_ptr(), n, es, stream) == 0
        if not bool(alive.any()):
            break
    rec = {"eval_envs": n, "mean_return": float(ret.double().mean()), "mean_length": float(length.double().mean()),
           "terms": {k: float(t_sum[j].double().mean()) for j, k in enumerate(EVAL_TERMS)}}
    print(json.dumps(rec), flush=True)
    env.close()
    return rec


if __name__ == "__main__":
    main()
