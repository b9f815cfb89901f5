"""ETG pretraining on the GPU engine — the batched counterpart of ETGRL/pretrain.py (same flags and defaults, pretrain.py:292-330).  ES over the
12 control-point offsets of the ETG (the open-loop gait), with no RL: the result is the `.npz` that `train --ETG_path`, `bctrain --ETG_path`
and deployment (through `env_test --save 1`) consume.

    setup:            SimpleGA(12, sigma, sigma_decay, sigma_limit=0.005, elite_ratio=0.1, weight_decay=0.005, popsize) from --ETG_path's
                      `param` (zeros without a file); the incumbent is evaluated once and seeds best_param / best_reward
    every round:      --es_train_steps generations of ask -> batched ETG fit (b2q_etg_fit) -> all popsize x es_rollouts envs roll out the zero
                      residual in lock step for up to 401 control steps (run_episode(env, 400)) with per-term sums and the velx success
                      count frozen at each env's first done (b2q_es_accumulate_terms) -> tell -> one JSON line
    after a round:    when env_steps crossed a multiple of --eval_every_steps: best_param is evaluated once (zero residual, at most 601 steps,
                      one episode per env of --eval_envs) and <outdir>/<suffix>/itr_<env_steps>.npz = {w, b, param = best_param}

The evaluator's env is train.py's ES-phase configuration (train.env_config, --dynamic_param), so a pretrained gait is scored on the reward
`train --ETG_path` goes on to optimise.  Fixes to the reference's loop: best_reward / best_param are seeded by the incumbent (they are
undefined there); env_steps counts the env steps the rollouts take (total_steps never advances there); the success count is kept per
episode (success_num is unbound there); the checkpoint's param is best_param, the one its (w, b) are fitted to (the reference saves the
never-updated ETG_best_param); a round that crosses several multiples evaluates once; the evaluation is the zero residual (the reference
calls an agent that does not exist).  --epsilon, --gamma, --random and --e_step are accepted and ignored, as in the reference.

    python -m paddlerobotics_b200.pretrain --task_mode stairstair --popsize 40 --outdir pretrain_log
    python -m paddlerobotics_b200.pretrain --outdir pretrain_log --save_state 1; python -m paddlerobotics_b200.pretrain --resume pretrain_log/exp0/state.pt --max_steps N
    python -m paddlerobotics_b200.pretrain --eval 1 --load pretrain_log/exp0/itr_160400.npz --render_dir frames
    python -m paddlerobotics_b200.train --task_mode stairstair --ETG_path pretrain_log/exp0/itr_160400.npz
    torchrun --nproc_per_node 8 -m paddlerobotics_b200.pretrain --popsize 256 --es_rollouts 16 --outdir pretrain_log

Under torchrun (WORLD_SIZE > 1) every rank seeds NumPy alike and asks the same population; it rolls out its contiguous shard of the
individuals, and one all-gather per generation (fitness, length, term sums and success rate) gives every rank the whole table, so every
rank tells the same fitness and the run computes what one GPU computes with the same --popsize and --es_rollouts.  --popsize must be
divisible by the ranks.  Rank 0 alone evaluates, prints and writes itr_*.npz and state.pt; a --resume loads the file on every rank.
"""
import argparse
import json
import os

import numpy as np

ES_TRAIN_STEPS = 10         # pretrain.py:37
EVAL_EVERY_STEPS = 10000    # pretrain.py:35
ES_MAX_STEP = 400           # run_episode(env, 400), pretrain.py:232: up to 401 control steps
EVAL_MAX_STEP = 600         # run_evaluate_episodes(agent, env, 600, ...), pretrain.py:264
SUCCESS_VELX = 0.3          # pretrain.py:147


def parser():
    from .dynamics_grid import HELP as DYNAMICS_GRID_HELP
    from .train import TERRAIN_GRID_HELP
    p = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    # ---- pretrain.py:292-329
    p.add_argument("--outdir", type=str, default="train_log")
    p.add_argument("--max_steps", type=int, default=int(1e7), help="env steps the ES rollouts may take in all")
    p.add_argument("--epsilon", type=float, default=0.4, help="accepted and ignored, as in the reference")
    p.add_argument("--gamma", type=float, default=0.95, help="accepted and ignored, as in the reference")
    p.add_argument("--sigma", type=float, default=0.02)
    p.add_argument("--sigma_decay", type=float, default=0.99)
    p.add_argument("--popsize", type=int, default=40)
    p.add_argument("--random_dynamic", type=int, default=0)
    p.add_argument("--random_force", type=int, default=0)
    p.add_argument("--task_mode", type=str, default="stairstair")
    p.add_argument("--step_y", type=float, default=0.05)
    p.add_argument("--load", type=str, default="", help="--eval 1: the .npz whose (w, b) is evaluated")
    p.add_argument("--eval", type=int, default=0, help="1: evaluate the --load gait instead of training (pretrain.py:278-289)")
    p.add_argument("--render", type=int, default=0)
    p.add_argument("--suffix", type=str, default="exp0")
    p.add_argument("--random", type=int, default=0, help="accepted and ignored, as in the reference")
    p.add_argument("--normal", type=int, default=1)
    p.add_argument("--vel_d", type=float, default=0.5)
    p.add_argument("--ETG_T", type=float, default=0.5)
    p.add_argument("--reward_p", type=float, default=5)
    p.add_argument("--footheight", type=float, default=0.1)
    p.add_argument("--steplen", type=float, default=0.05)
    p.add_argument("--ETG", type=int, default=1)
    p.add_argument("--ETG_T2", type=float, default=0.5)
    p.add_argument("--e_step", type=int, default=400, help="accepted and ignored, as in the reference (its episodes are 401 steps)")
    p.add_argument("--act_mode", type=str, default="traj")
    p.add_argument("--ETG_path", type=str, default="None", help="an .npz whose `param` starts the search; zeros when the file does not exist")
    p.add_argument("--ETG_H", type=int, default=20)
    p.add_argument("--stand", type=float, default=0)
    p.add_argument("--torso", type=float, default=1.5)
    p.add_argument("--up", type=float, default=0.6)
    p.add_argument("--tau", type=float, default=0.07)
    p.add_argument("--feet", type=float, default=0.3)
    p.add_argument("--badfoot", type=float, default=0.1)
    p.add_argument("--footcontact", type=float, default=0.1)
    p.add_argument("--enable_action_filter", type=int, default=0)
    p.add_argument("--x_noise", type=int, default=0)
    # ---- the module constants of pretrain.py:34-37, the data file of :192-193, and the batched engine
    p.add_argument("--es_train_steps", type=int, default=ES_TRAIN_STEPS, help="generations per round")
    p.add_argument("--es_rollouts", type=int, default=1, help="episodes per individual (the reference runs one)")
    p.add_argument("--eval_every_steps", type=int, default=EVAL_EVERY_STEPS, help="evaluation and itr_*.npz cadence in env steps")
    p.add_argument("--eval_envs", type=int, default=1, help="envs of each evaluation episode (one episode each, no auto-reset)")
    p.add_argument("--terrain_grid", type=int, default=0, help=TERRAIN_GRID_HELP)
    p.add_argument("--dynamics_grid", type=int, default=0, help=DYNAMICS_GRID_HELP)
    p.add_argument("--dynamic_param", type=str, default="", help="PATH.npy: a 48-vector in [-1, 1] -> param2dynamic_dict -> every env "
                   "(pretrain.py:192-193); empty = nominal dynamics")
    p.add_argument("--seed", type=int, default=0, help="seeds np.random before the solver is built")
    p.add_argument("--render_dir", type=str, default="", help="--eval 1: write env 0's camera image of every step to DIR/img{step}.png")
    p.add_argument("--render_width", type=int, default=640)
    p.add_argument("--render_height", type=int, default=480)
    p.add_argument("--save_state", type=int, default=0, help="1: write the whole search state to <outdir>/<suffix>/state.pt after every evaluation block "
                   "and when --max_steps is reached, replacing the previous file atomically")
    p.add_argument("--resume", type=str, default="", help="a state.pt of pretrain --save_state: continue that search bit for bit with its arguments; "
                   "only --max_steps, --outdir, --suffix, --save_state and --dist_backend may be given with other values")
    p.add_argument("--dist_backend", type=str, default="nccl", choices=("nccl", "gloo"), help="under torchrun: the process group's backend; gloo lets "
                   "several ranks share one GPU")
    return p


RESUME_FREE = ("max_steps", "outdir", "suffix", "save_state", "resume", "dist_backend")      # the flags a --resume may change


def check_supported(args):
    """Options the batched engine does not provide raise before any device work (the make_env rule: honoured or raised, never ignored)."""
    if args.random_dynamic:
        raise NotImplementedError("--random_dynamic 1: per-episode dynamics randomisation is not provided")
    if args.random_force:
        raise NotImplementedError("--random_force 1: per-episode pushes are not provided in the batched env")
    if args.x_noise:
        raise NotImplementedError("--x_noise 1: the ES rollouts start every episode at x = 0")
    if args.render:
        raise NotImplementedError("--render 1: there is no GUI window; --eval 1 --render_dir writes the camera frames")
    if args.stand != 0:
        raise NotImplementedError("--stand %g: the stand reward term is not provided" % args.stand)
    if args.ETG_H != 20:
        raise NotImplementedError("--ETG_H %d: the RBF layer width is fixed at 20 in the kernel" % args.ETG_H)
    if not args.ETG:
        raise NotImplementedError("--ETG 0: pretraining searches the ETG; without it there is nothing to search")
    if args.ETG_T2 != args.ETG_T:
        raise NotImplementedError("--ETG_T2 %g != --ETG_T %g: the second ETG period is not provided" % (args.ETG_T2, args.ETG_T))
    if args.act_mode != "traj":
        raise NotImplementedError("--act_mode %s: pretraining runs the trajectory mode only" % args.act_mode)


def env_config(args):
    """train.py's ES-phase configuration (train.env_config) with the reward and observation flags of this command."""
    from .train import env_config as train_env_config
    cfg = train_env_config(args)
    cfg.update(vel_d=float(args.vel_d), reward_p=float(args.reward_p), obs_normal=int(bool(args.normal)), action_filter=int(bool(args.enable_action_filter)),
               etg_T=float(args.ETG_T), etg_T2=float(args.ETG_T))
    return cfg


def eval_due(env_steps, test_flag, every):
    """The reference's `while (total_steps + 1) // EVAL_EVERY_STEPS >= test_flag: test_flag += 1` (pretrain.py:258-260), run once per
    round: (evaluate?, new test_flag).  The first round always evaluates; later rounds when env_steps crossed another multiple."""
    k = (int(env_steps) + 1) // int(every)
    if k >= test_flag:
        return True, k + 1
    return False, test_flag


def checkpoint_names(round_totals, every):
    """[(round index, itr_<env_steps>.npz)] for the env-step totals reached at the end of each round."""
    out, flag = [], 0
    for r, total in enumerate(round_totals):
        due, flag = eval_due(total, flag, every)
        if due:
            out.append((r, "itr_%d.npz" % int(total)))
    return out


def main(argv=None):
    from . import dist_run, run_state
    p = parser()
    args = p.parse_args(argv)
    rank, world, local = dist_run.ranks()
    state = None
    if args.resume:
        state = run_state.load_state(p, args.resume, "pretrain")
        args = run_state.resume_args(p, parser, argv, state["args"], RESUME_FREE, (("--load", "load"), ("--ETG_path", "ETG_path"), ("--eval 1", "eval")),
                                     "the solver, the incumbent and the search loop")
    if args.save_state and not args.outdir:
        p.error("--save_state 1 writes <outdir>/<suffix>/state.pt: it needs --outdir")
    if world > 1 and not args.eval:                 # after a --resume: the saved run's population is the one that is split
        dist_run.check_divisible(p, world, popsize=args.popsize)
    check_supported(args)
    if args.eval and not args.load:
        p.error("--eval 1 evaluates a gait: it needs --load X.npz")
    from .train import check_dynamics_grid, check_terrain_grid
    check_terrain_grid(p, args)
    check_dynamics_grid(p, args)
    if args.popsize < 1 or args.es_rollouts < 1 or args.es_train_steps < 1 or args.eval_every_steps < 1 or args.eval_envs < 1:
        p.error("--popsize, --es_rollouts, --es_train_steps, --eval_every_steps and --eval_envs must be positive")
    if not args.eval and int(args.popsize * 0.1) < 1:
        p.error("--popsize %d: SimpleGA's elite_ratio 0.1 needs a population of at least 10 to keep one parent" % args.popsize)
    if args.eval:
        return evaluate(args) if rank == 0 else []                     # --eval runs on rank 0 alone
    if world == 1:
        return pretrain(args) if state is None else pretrain(args, state)
    with dist_run.process_group(world, local, getattr(args, "dist_backend", "nccl")) as dev:     # a state file may predate the flag
        return pretrain(args, state, rank, world, dev)


def make_eval_env(args, cfg, device=0):
    from .env import VecQuadrupedalEnv, apply_dynamic_param
    return apply_dynamic_param(VecQuadrupedalEnv(args.eval_envs, device=device, auto_reset=False, **cfg), args.dynamic_param)


def evaluate(args):
    """--eval 1 --load X.npz: the file's (w, b) with the zero residual, one episode per env of --eval_envs, at most 601 steps; one JSON line;
    --render_dir writes img{step}.png of env 0 for every step taken (pretrain.py:278-289).  --terrain_grid 1 / --dynamics_grid 1: the
    records of train.evaluate_terrain_grid / evaluate_dynamics_grid."""
    from .train import evaluate_dynamics_grid, evaluate_terrain_grid, frame_writer, run_evaluate_episodes
    with np.load(args.load) as z:
        w, b = z["w"], z["b"]
    if args.terrain_grid:
        return evaluate_terrain_grid(args, env_config(args), w, b, policy=None, max_step=EVAL_MAX_STEP)
    if getattr(args, "dynamics_grid", 0):
        return evaluate_dynamics_grid(args, env_config(args), w, b, policy=None, max_step=EVAL_MAX_STEP)
    env = make_eval_env(args, env_config(args))
    r = run_evaluate_episodes(env, w, b, policy=None, max_step=EVAL_MAX_STEP, render=frame_writer(env, args) if args.render_dir else None)
    rec = {"eval_envs": args.eval_envs, **{k: v for k, v in r.items() if k != "per_env"}}
    print(json.dumps(rec), flush=True)
    env.close()
    return rec


def pretrain(args, state=None, rank=0, world=1, dev=0):
    """The search on this rank (device `dev`) of `world` ranks; returns the records rank 0 printed, [] on the other ranks.  `state`: a
    --save_state file to continue from (its solver, incumbent and counters replace the set-up)."""
    import torch
    import torch.distributed as dist
    from . import run_state
    from .env import apply_dynamic_param
    from .es import PopulationEvaluator, SimpleGA, solutions_to_etg_device
    from .etg import Opt_with_points
    from .train import EVAL_TERMS, etg_prior, initial_etg, run_evaluate_episodes
    np.random.seed(args.seed); torch.manual_seed(args.seed)
    layer, w0, b0, prior_points = etg_prior(args.ETG_T, args.footheight, args.steplen)
    if state is None:
        init, w_inc, b_inc = initial_etg(args)                                                                  # pretrain.py:171-177
    else:
        init = np.zeros(12)                              # the saved solver replaces it: a resume does not read --ETG_path again
    solver = SimpleGA(12, sigma_init=args.sigma, sigma_decay=args.sigma_decay, sigma_limit=0.005, elite_ratio=0.1, weight_decay=0.005,
                      popsize=args.popsize, param=init.copy())                                                  # pretrain.py:178-185
    cfg = env_config(args)
    evaluator = PopulationEvaluator(args.popsize, args.es_rollouts, max_steps=ES_MAX_STEP + 1, rank=rank, world=world, device=dev, policy=None, **cfg)
    apply_dynamic_param(evaluator.env, args.dynamic_param)
    eval_env = make_eval_env(args, cfg, device=dev) if rank == 0 else None
    outdir = os.path.join(args.outdir, args.suffix)
    if rank == 0:
        os.makedirs(outdir, exist_ok=True)
    pop = args.popsize

    def rollout(ws, bs):
        fit, mlen, tmean, succ = evaluator.evaluate(ws, bs, terms=EVAL_TERMS)
        steps = evaluator.len.sum()                               # the env steps these episodes took, over every rank's shard
        if world > 1:
            dist.all_reduce(steps)
        steps = int(steps)
        return fit.double().cpu().numpy(), mlen.double().cpu().numpy(), tmean.double().cpu().numpy(), succ.double().cpu().numpy(), steps

    # the incumbent seeds best_param / best_reward (the train.py:395-396 rule; both are undefined in the reference).  This evaluation is set-up:
    # env_steps counts the steps of the generations' rollouts only, so --max_steps bounds the search as the reference's total_steps would
    # A resume skips it: best_reward is in the state.  Every rollout and evaluation resets all envs of its handle and draws no random numbers,
    # so the envs carry nothing from one generation to the next and need no snapshot.
    if state is None:
        inc = rollout(np.repeat(np.asarray(w_inc)[None], pop, 0), np.repeat(np.asarray(b_inc)[None], pop, 0))[0]
        best_reward = float(np.nanmean(inc)) if np.isfinite(inc).any() else -np.inf
        best_param = init.copy()
        test_flag, es_step, env_steps = 0, 0, 0
    else:
        solver.load_state_dict(state["solver"])
        best_param, best_reward = np.array(state["best_param"]), state["best_reward"]
        test_flag, es_step, env_steps = (state["loop"][k] for k in ("test_flag", "es_step", "env_steps"))
    log = []
    run_args = dict(vars(args))                          # what a --save_state file records

    def save_state():
        if rank != 0:
            return
        run_state.write_atomic(os.path.join(outdir, "state.pt"), {
            "command": "pretrain", "args": run_args, "solver": solver.state_dict(), "best_param": np.array(best_param), "best_reward": best_reward,
            "loop": {"test_flag": test_flag, "es_step": es_step, "env_steps": env_steps}})
    while env_steps < args.max_steps:
        for _ in range(args.es_train_steps):                                                                   # pretrain.py:221-256
            sol = solver.ask()
            ws, bs = solutions_to_etg_device(sol, prior_points, w0, b0, ETG_T=args.ETG_T, device=dev)
            fit, mlen, tmean, succ, steps = rollout(ws.cpu().numpy(), bs.cpu().numpy())
            env_steps += steps
            fit = np.where(np.isfinite(fit), fit, -1e9)                  # a diverged rollout must lose, not poison tell()
            if fit.max() > best_reward:
                best_reward, best_param = float(fit.max()), np.asarray(sol[int(fit.argmax())]).copy()
            solver.tell(fit)
            es_step += 1
            mean_steps = float(mlen.mean())
            rec = {"ES_step": es_step, "fitness_max": float(np.max(fit)), "fitness_mean": float(np.mean(fit)), "fitness_min": float(np.min(fit)),
                   "fitness_std": float(np.std(fit)), "mean_len": mean_steps, "sigma": float(np.mean(solver.result()[3])), "best_reward": best_reward}
            for j, k in enumerate(EVAL_TERMS):
                ep = float(tmean[j].mean())                               # infos[key] += info[key] / popsize
                rec["episode_" + k], rec["mean_" + k] = ep, ep / mean_steps
            rec["success_rate"] = float(succ.mean())
            rec["env_steps"] = env_steps
            if rank == 0:
                log.append(rec); print(json.dumps(rec), flush=True)
        due, test_flag = eval_due(env_steps, test_flag, args.eval_every_steps)
        if due and rank == 0:                                                                                  # pretrain.py:258-277
            w, b, _ = Opt_with_points(ETG=layer, ETG_T=args.ETG_T, w0=w0, b0=b0, points=prior_points + best_param.reshape(-1, 2))
            r = run_evaluate_episodes(eval_env, w, b, policy=None, max_step=EVAL_MAX_STEP)
            path = os.path.join(outdir, "itr_%d.npz" % env_steps)
            np.savez(path, w=w, b=b, param=best_param)
            rec = {"env_steps": env_steps, "eval_return": r["mean_return"], "eval_length": r["mean_length"], "eval_success_rate": r["success_rate"],
                   "terms": r["terms"], "best_reward": best_reward, "checkpoint": os.path.basename(path)}
            log.append(rec); print(json.dumps(rec), flush=True)
            if args.save_state:
                save_state()
    if args.save_state:
        save_state()
    evaluator.env.close()
    if eval_env is not None:
        eval_env.close()
    return log


if __name__ == "__main__":
    main()
