"""What one bctrain --save_state write and one --resume read cost on this GPU (DESIGN §8g):
    python scripts/bctrain_state_cost.py [--num_envs 4096] [--memory 10000000] [--fill 1000000,10000000]
bctrain's objects at the given size (train env, student learner, BC ring, expert) are saved and restored once after one warm-up round trip,
for every fill level of the BC ring (the state holds the ring up to its fill level; --memory rows is the largest state a run writes).  Each
part is timed with CUDA events around its state_dict / load_state_dict, and a host clock times the file write (write_atomic) and the file
read (torch.load).  The card's name and power limit are read in the same run.  The state file goes to a temporary directory."""
import argparse
import json
import os
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from paddlerobotics_b200 import bc, bctrain, run_state
from paddlerobotics_b200.agent import MujocoAgent, SACLearner
from train_state_cost import card, nbytes, timed


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--num_envs", type=int, default=4096)
    ap.add_argument("--memory", type=int, default=int(1e7))
    ap.add_argument("--fill", type=str, default="1000000,10000000", help="comma-separated fill levels of the BC ring")
    a = ap.parse_args()
    args = bctrain.parser().parse_args(["--num_envs", str(a.num_envs), "--memory", str(a.memory)])
    env = bctrain.make_vec_env(args, a.num_envs, auto_reset=True, max_episode_steps=args.e_step + 1)
    student, expert = MujocoAgent(46, 12), MujocoAgent(49, 12, seed=1)
    learner = SACLearner(student, args.batch, actor_lr=bctrain.ACTOR_LR, critic_lr=bctrain.CRITIC_LR)
    rpm = bc.BCReplayMemory(a.memory, 46, 49, device=env.device)
    gen = torch.Generator(device=env.device).manual_seed(0)
    w, b = bctrain.etg_of_path("None")
    obs = env.reset(w, b).clone()
    parts = {"env": env, "learner": learner, "rpm": rpm}
    rec = {"card": card(), "num_envs": a.num_envs, "memory": a.memory, "fills": []}
    for fill in [int(x) for x in a.fill.split(",")]:
        rpm.obs[:fill].normal_(generator=gen); rpm.ref_obs[:fill].normal_(generator=gen)
        rpm._pos, rpm._size = fill % a.memory, fill
        path = os.path.join(tempfile.mkdtemp(), "state.pt")
        for rnd in range(2):                              # round 0 warms up every path
            save, state = {}, {}
            for k, o in parts.items():
                state[k], dev_s, _ = timed(o.state_dict)
                save[k] = {"bytes": nbytes(state[k]), "event_s": dev_s}
            rest, dev_s, _ = timed(lambda: {"expert": expert.state_dict(), "w": np.array(w), "b": np.array(b), "gen": gen.get_state(),
                                            "np_random": np.random.get_state(), "obs": obs.cpu()})
            state.update(rest, command="bctrain")
            save["rest"] = {"bytes": nbytes(rest), "event_s": dev_s}
            t = time.perf_counter(); run_state.write_atomic(path, state); save["file_write_s"] = time.perf_counter() - t
            save["file_bytes"] = os.path.getsize(path)
            del state, rest
            load = {}
            t = time.perf_counter(); got = torch.load(path, map_location="cpu", weights_only=False); load["file_read_s"] = time.perf_counter() - t
            for k, o in parts.items():
                _, dev_s, _ = timed(lambda: o.load_state_dict(got[k]))
                load[k] = {"event_s": dev_s}
            _, dev_s, _ = timed(lambda: (expert.load_state_dict(got["expert"]), gen.set_state(got["gen"]), obs.copy_(got["obs"])))
            load["rest"] = {"event_s": dev_s}
            save["total_s"] = sum(v["event_s"] for v in save.values() if isinstance(v, dict)) + save["file_write_s"]
            load["total_s"] = sum(v["event_s"] for v in load.values() if isinstance(v, dict)) + load["file_read_s"]
            del got
        os.remove(path); os.rmdir(os.path.dirname(path))
        rec["fills"].append({"fill": fill, "save": save, "resume": load})
        print(json.dumps(rec["fills"][-1]), flush=True)
    print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
