"""Dynamics identification on the GPU engine — the batched counterpart of ETGRL/Dynamic_train.py and model/Dynamic_parallel_model.py
(same flags and defaults where they exist).  An ES solver searches the 48 dynamics parameters (param2dynamic_dict) whose simulated
replay of recorded gait tables best matches the real robot's joint-angle and body-rate statistics:

    every epoch:        ask -> every individual replays the `exp` and `ori` tables for 100 control steps (es.DynamicsEvaluator: one
                        env per individual and table, all in lock step) -> reward = mean over the two tables of 30 - loss -> tell ->
                        <outdir>/<suffix>/dynamic_param{epoch}.npy = result()[0] -> one JSON line
    every fifth epoch:  the current vector replays the `height` table -> one JSON line

The population is K x thread; individual i*K + j is the reference's actor i, slot j.  Under torchrun each rank evaluates its shard and
the rewards are all-gathered; only rank 0 writes, prints and runs the `height` evaluation.

Deviations: --gamma and --xparl are accepted and ignored (the reference ignores gamma; there is no xparl cluster).  --seed seeds NumPy's
global RNG, which the reference leaves unseeded.  In training, --load does not seed the solver: like the reference, every solver
starts from zeros.  --alg cma is refused: the reference's set_solver has no cma branch.

    python -m paddlerobotics_b200.dynamic_train --data_dir data/dynamic --alg ga --steps 10000
    python -m paddlerobotics_b200.dynamic_train --data_dir data/dynamic --save_state 1; python -m paddlerobotics_b200.dynamic_train --resume Dynamic/exp0/state.pt --steps N
    python -m paddlerobotics_b200.dynamic_train --eval 1 --load Dynamic/exp0/dynamic_param9027.npy
    python -m paddlerobotics_b200.dynamic_train --eval 1 --load Dynamic/exp0/dynamic_param9027.npy --dynamics_grid 1   # the landscape around it
    python -m paddlerobotics_b200.train --dynamic_param Dynamic/exp0/dynamic_param9027.npy     # train the expert on the result
"""
import argparse
import json
import os

import numpy as np

from .es import PEPG, OpenES, SimpleES, SimpleGA

NUM_PARAMS = 48
STEPS = 100                 # control steps per replay, Dynamic_parallel_model.py:59
SIGMA_DECAY = 0.9999        # ES_ParallelModel's default, :80
ALGS = ("ga", "ses", "pepg", "openes", "simples")
DATA_FILES = {"mean_dict": "mean_dict_5_18.npz", "exp": "gait_action_list_t0.3.npy", "ori": "gait_action_list_CPG_ori.npy",
              "height": "gait_action_list_CPG_height.npy"}           # Dynamic_train.py:10-17
STATS = ("_motor_mean", "_motor_std", "_drpy_mean", "_drpy_std")


def parser():
    p = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    # ---- Dynamic_train.py:20-31
    p.add_argument("--outdir", type=str, default="Dynamic")
    p.add_argument("--steps", type=int, default=10000, help="epochs")
    p.add_argument("--K", type=int, default=20, help="individuals per actor")
    p.add_argument("--load", type=str, default="", help="dynamic_param*.npy to evaluate with --eval 1 (training always starts from zeros)")
    p.add_argument("--eval", type=int, default=0, help="1: evaluate the --load vector on the height table")
    p.add_argument("--dynamics_grid", type=int, default=0, help="--eval 1: the identification landscape around the --load vector: each group of "
                   "its 48 parameters set alone to -1, -0.75, ..., 1, all 82 vectors scored in one batch on the height table (eval_reward) and "
                   "on the exp and ori tables (train_reward); one JSON line per vector and a summary")
    p.add_argument("--suffix", type=str, default="exp0")
    p.add_argument("--sigma", type=float, default=0.1)
    p.add_argument("--gamma", type=float, default=1, help="accepted and ignored, as in the reference")
    p.add_argument("--alg", type=str, default="ga", help=" ".join(ALGS))
    p.add_argument("--xparl", type=str, default="172.18.188.13:8007", help="accepted and ignored: ranks come from torchrun")
    p.add_argument("--thread", type=int, default=2, help="actors; the population is K x thread")
    # ---- the data the reference reads from fixed paths, and its RNG
    p.add_argument("--data_dir", type=str, default="data/dynamic", help="holds %s" % ", ".join(DATA_FILES.values()))
    p.add_argument("--seed", type=int, default=0, help="seeds np.random before the solver is built: every rank asks the same population")
    p.add_argument("--save_state", type=int, default=0, help="1: rank 0 writes the solver and the next epoch to <outdir>/<suffix>/state.pt after every "
                   "epoch with a height evaluation and after the last epoch, replacing the previous file atomically")
    p.add_argument("--resume", type=str, default="", help="a state.pt of dynamic_train --save_state: continue that search bit for bit with its arguments "
                   "(every rank loads it); only --steps, --outdir, --suffix and --save_state may be given with other values")
    return p


RESUME_FREE = ("steps", "outdir", "suffix", "save_state", "resume")      # the flags a --resume may change


def make_solver(alg, popsize, sigma, num_params=NUM_PARAMS, sigma_decay=SIGMA_DECAY):
    """ES_ParallelModel.set_solver (Dynamic_parallel_model.py:102-149): every solver starts from zeros."""
    if alg == "ga":
        return SimpleGA(num_params, sigma_init=sigma, sigma_decay=sigma_decay, sigma_limit=0.02, elite_ratio=0.1, weight_decay=0.005, popsize=popsize,
                        param=np.zeros(num_params))
    if alg == "ses":
        return PEPG(num_params, sigma_init=sigma, sigma_decay=sigma_decay, sigma_alpha=0.2, sigma_limit=0.02, elite_ratio=0.1, weight_decay=0.005,
                    popsize=popsize)
    if alg == "pepg":
        return PEPG(num_params, sigma_init=sigma, sigma_decay=sigma_decay, sigma_alpha=0.20, sigma_limit=0.02, learning_rate=0.01, learning_rate_decay=1.0,
                    learning_rate_limit=0.01, weight_decay=0.005, popsize=popsize)
    if alg == "openes":
        return OpenES(num_params, sigma_init=sigma, sigma_decay=sigma_decay, sigma_limit=0.02, learning_rate=0.01, learning_rate_decay=1.0,
                      learning_rate_limit=0.01, antithetic=True, weight_decay=0.005, popsize=popsize)
    if alg == "simples":
        return SimpleES(num_params, sigma_init=sigma, sigma_decay=sigma_decay, sigma_limit=0.02, weight_decay=0.005, popsize=popsize)
    raise ValueError("--alg %s: supported algorithms are %s" % (alg, ", ".join(ALGS)))


def evaluator_config():
    """The evaluators' env: rlschool.make_env('Quadrupedal', task="ground", render=False, ETG=0) (Dynamic_parallel_model.py:49), i.e.
    make_env's configuration with joint limits and knee contacts on and the analytic plane.  etg_enabled is left out: DynamicsEvaluator
    always passes etg_enabled=0 itself."""
    from .env import quadrupedal_config
    cfg, _ = quadrupedal_config(task="ground", ETG=0)
    cfg.pop("etg_enabled")
    return cfg


def load_data(data_dir):
    """(gait {exp, ori, height: [>=100, 12]}, mean_dict) from the reference's four files; ValueError naming the file that is missing
    or too short."""
    paths = {k: os.path.join(data_dir, f) for k, f in DATA_FILES.items()}
    for path in paths.values():
        if not os.path.isfile(path):
            raise ValueError("dynamics data file %s is missing" % path)
    with np.load(paths["mean_dict"]) as z:
        mean_dict = {k: np.asarray(z[k]) for k in z.files}
    gait = {}
    for key in ("exp", "ori", "height"):
        gait[key] = np.load(paths[key])
        if gait[key].ndim != 2 or gait[key].shape[0] < STEPS or gait[key].shape[1] != 12:
            raise ValueError("%s: a gait table must be [>= %d, 12], got %s" % (paths[key], STEPS, list(gait[key].shape)))
        for s in STATS:
            name, width = key + s, 12 if "motor" in s else 3
            if name not in mean_dict:
                raise ValueError("%s has no %r" % (paths["mean_dict"], name))
            if mean_dict[name].ndim != 2 or mean_dict[name].shape[0] < STEPS or mean_dict[name].shape[1] != width:
                raise ValueError("%s: %r must be [>= %d, %d], got %s" % (paths["mean_dict"], name, STEPS, width, list(mean_dict[name].shape)))
    return gait, mean_dict


def main(argv=None):
    from . import run_state
    p = parser()
    args = p.parse_args(argv)
    state = None
    if args.resume:
        state = run_state.load_state(p, args.resume, "dynamic_train")
        args = run_state.resume_args(p, parser, argv, state["args"], RESUME_FREE, (("--load", "load"), ("--eval 1", "eval")), "the solver and the epoch")
    if args.save_state and not args.outdir:
        p.error("--save_state 1 writes <outdir>/<suffix>/state.pt: it needs --outdir")
    if args.alg not in ALGS:
        p.error("--alg %s is not provided (the reference's set_solver has no %s branch); supported algorithms: %s" % (args.alg, args.alg, ", ".join(ALGS)))
    if args.eval and not args.load:
        p.error("--eval 1 evaluates a dynamics vector: it needs --load dynamic_param*.npy")
    if getattr(args, "dynamics_grid", 0) and not args.eval:          # a state file may predate the flag
        p.error("--dynamics_grid 1 evaluates the landscape around a dynamics vector: it needs --eval 1 --load dynamic_param*.npy")
    try:
        gait, mean_dict = load_data(args.data_dir)
    except ValueError as e:
        p.error(str(e))
    import torch
    import torch.distributed as dist
    rank, world, local = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("LOCAL_RANK", "0"))
    popsize = args.K * args.thread
    if popsize % world != 0:
        p.error("the population K x thread = %d must be divisible by the %d ranks" % (popsize, world))
    torch.cuda.set_device(local)
    own_group = world > 1 and not dist.is_initialized()
    if own_group:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    try:
        return run(args, gait, mean_dict, rank, world, local, state)
    finally:
        if own_group:
            dist.destroy_process_group()


def run(args, gait, mean_dict, rank, world, local, state=None):
    """The epochs (or the --eval evaluation) on this rank; returns the records rank 0 printed.  `state`: a --save_state file to continue
    from (its solver, NumPy's RNG included, and its next epoch).  The evaluators set every env's dynamics and reset it before each
    replay, so they carry nothing between epochs and need no snapshot."""
    from . import run_state
    from .es import DynamicsEvaluator
    popsize = args.K * args.thread
    cfg = evaluator_config()
    if args.eval and rank != 0:
        return []
    if args.eval and args.dynamics_grid:
        return landscape(args, gait, mean_dict, cfg, local)
    height = DynamicsEvaluator(1, gait, mean_dict, keys=("height",), steps=STEPS, device=local, **cfg) if rank == 0 else None

    def eval_height(param):
        return float(height.evaluate(np.asarray(param).reshape(1, NUM_PARAMS))[0])
    log = []
    if args.eval:                                                            # evaluate_episode(0), Dynamic_train.py:43-44
        rec = {"eval_reward": eval_height(np.load(args.load).reshape(-1))}
        print(json.dumps(rec), flush=True)
        height.env.close()
        return [rec]
    np.random.seed(args.seed)
    solver = make_solver(args.alg, popsize, args.sigma)
    start = 0
    if state is not None:
        solver.load_state_dict(state["solver"])
        start = int(state["epoch"])
    evaluator = DynamicsEvaluator(popsize, gait, mean_dict, keys=("exp", "ori"), steps=STEPS, rank=rank, world=world, device=local, **cfg)
    outdir = os.path.join(args.outdir, args.suffix)
    if rank == 0:
        os.makedirs(outdir, exist_ok=True)
    run_args = dict(vars(args))                                              # what a --save_state file records
    for epoch in range(start, args.steps):                                   # ES_ParallelModel.update / train, :152-190
        solutions = solver.ask()
        rewards = evaluator.evaluate(solutions).double().cpu().numpy()
        solver.tell(rewards)
        result = solver.result()
        if rank == 0:
            np.save(os.path.join(outdir, "dynamic_param%d.npy" % epoch), result[0])
            rec = {"epoch": epoch, "reward_max": float(np.max(rewards)), "reward_mean": float(np.mean(rewards)), "reward_min": float(np.min(rewards)),
                   "reward_std": float(np.std(rewards)), "best_reward": float(result[1]), "sigma": float(np.mean(result[3]))}
            log.append(rec); print(json.dumps(rec), flush=True)
            if epoch % 5 == 0 and epoch > 0:
                rec = {"epoch": epoch, "eval_reward": eval_height(result[0])}
                log.append(rec); print(json.dumps(rec), flush=True)
            if args.save_state and ((epoch % 5 == 0 and epoch > 0) or epoch == args.steps - 1):
                run_state.write_atomic(os.path.join(outdir, "state.pt"), {"command": "dynamic_train", "args": run_args, "solver": solver.state_dict(),
                                                                          "epoch": epoch + 1})
    evaluator.env.close()
    if height is not None:
        height.env.close()
    return log


COPIES = 8      # envs per vector and table in the landscape: one warp of the step kernel


def landscape(args, gait, mean_dict, cfg, device=0):
    """--eval 1 --load P.npy --dynamics_grid 1: the 82 vectors of dynamics_grid.swept_params(P) (P, then P with one group set to each
    level), scored in one batch by a DynamicsEvaluator on `height` (eval_reward, what --eval 1 reports) and one on `exp` and `ori`
    (train_reward, what the epochs maximise).  Every vector fills whole warps (COPIES envs per table): the evaluators' configuration has
    joint limits and knee contacts, whose general contact solve the step kernel switches per warp of 8 robots, so no other vector's
    robots can switch a vector's solve: its eval_reward is what --eval 1 --load of it reports (DESIGN §8i).  Prints one JSON line per vector and a summary: the centre's rewards and, per
    group, the level with the best train_reward and the range of train_reward over the levels (a flat group is one the data does not
    identify), most sensitive group first."""
    from . import dynamics_grid
    from .es import DynamicsEvaluator
    sols = np.repeat(dynamics_grid.swept_params(np.load(args.load).reshape(-1)), COPIES, 0)
    rewards = {}
    for name, keys in (("eval_reward", ("height",)), ("train_reward", ("exp", "ori"))):
        ev = DynamicsEvaluator(len(sols), gait, mean_dict, keys=keys, steps=STEPS, device=device, **cfg)
        rewards[name] = ev.evaluate(sols).double().cpu().numpy()[::COPIES]
        ev.env.close()
    recs = []
    for s, setting in enumerate(dynamics_grid.setting_records()):
        rec = dict(setting, eval_reward=float(rewards["eval_reward"][s]), train_reward=float(rewards["train_reward"][s]))
        recs.append(rec)
        print(json.dumps(rec), flush=True)
    summary = {"settings": len(recs), "load": args.load, "centre_eval_reward": recs[0]["eval_reward"], "centre_train_reward": recs[0]["train_reward"],
               "groups": dynamics_grid.group_summary(recs[1:], "train_reward", highest=True)}
    print(json.dumps(summary), flush=True)
    return recs + [summary]


if __name__ == "__main__":
    main()
