#!/usr/bin/env python
"""Secondary measurements (not the driver's bench contract): BASELINE configs 2-5 building blocks on one GPU.
  python bench_extra.py            -> JSON lines: policy-in-the-loop rollout, MLP forward, SAC learn, ES generation, terrain."""
import json
import sys
import time

import numpy as np
import torch

sys.path.insert(0, __import__("os").path.dirname(__import__("os").path.abspath(__file__)))
from bench import etg_weights  # noqa: E402


def timed(fn, iters, warm=5):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    from paddlerobotics_b200.agent import MujocoAgent, SACLearner
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    from paddlerobotics_b200.es import PopulationEvaluator
    w, b = etg_weights()
    out = []
    # config 2 with the policy in the loop: obs -> fused MLP (wgmma) -> env.step, 4096 envs
    env = VecQuadrupedalEnv(4096, auto_reset=True); env.reset(w, b)
    ag = MujocoAgent(49, 12, seed=0)
    state = {"obs": env.obs}
    def roll():
        a = ag.predict_batch(state["obs"]); a.mul_(0.3); state["obs"] = env.step(a)[0]
    ms = timed(roll, 300, 20)
    out.append({"what": "rollout 4096 envs, policy in the loop (fused MLP + step kernel)", "ms_per_step": ms, "env_steps_per_s": 4096 / ms * 1e3})
    obs = torch.randn(4096, 49, device="cuda")
    ms = timed(lambda: ag.actor.forward(obs), 300, 20)
    out.append({"what": "actor MLP forward M=4096 (wgmma)", "ms": ms, "tflops": 2 * 4096 * (64 * 256 + 256 * 256 + 256 * 32) / ms / 1e9})
    obs8 = torch.randn(8192, 49, device="cuda")
    ms = timed(lambda: ag.actor.forward(obs8), 300, 20)
    out.append({"what": "actor MLP forward M=8192 (wgmma)", "ms": ms})
    env.close()
    # config 4: SAC update, batch 8192 (and the reference's 256)
    for B in (256, 8192):
        L = SACLearner(ag, B)
        d = lambda *s: torch.randn(*s, device="cuda")
        o, no, ac, r, t, e1, e2 = d(B, 49), d(B, 49), torch.rand(B, 12, device="cuda") * 2 - 1, d(B), torch.ones(B, device="cuda"), d(B, 12), d(B, 12)
        ms = timed(lambda: L.learn(o, ac, r, no, t, eps_next=e1, eps_cur=e2, pull=False), 50, 5)
        out.append({"what": "SAC learn (critic+actor fwd/bwd, Adam, Polyak) batch %d" % B, "ms": ms, "samples_per_s": B / ms * 1e3})
        ms = timed(lambda: L.learn(o, ac, r, no, t, eps_next=e1, eps_cur=e2, pull=False, graph=True), 50, 5)
        out.append({"what": "SAC learn from a CUDA graph, batch %d" % B, "ms": ms, "samples_per_s": B / ms * 1e3})
        L.close()
    # config 3 (one GPU's share at G=8): 32 individuals x 16 rollouts x 400 steps
    ev = PopulationEvaluator(32, 16, max_steps=400)
    W, Bb = np.repeat(w[None], 32, 0), np.repeat(b[None], 32, 0)
    t0 = time.perf_counter(); ev.evaluate(W, Bb); torch.cuda.synchronize(); dt = time.perf_counter() - t0
    out.append({"what": "ES generation share: 32 individuals x 16 rollouts x 400 steps (512 envs)", "s": dt, "env_steps_per_s": 512 * 400 / dt})
    ev.env.close()
    # config 5: height-field terrain (stairs-like), 4096 envs
    xs = np.arange(512) * 0.02 - 2.0
    hf = np.tile(np.floor(np.maximum(xs, 0) / 0.3) * 0.08, (512, 1))
    envt = VecQuadrupedalEnv(4096, auto_reset=True, heightfield=(hf, -2.0, -5.12, 0.02)); envt.reset(w, b)
    g = torch.Generator(device="cuda"); g.manual_seed(0)
    pool = torch.rand(16, 4096, 12, device="cuda", generator=g) * 0.6 - 0.3
    k = {"i": 0}
    def st():
        envt.step(pool[k["i"] % 16]); k["i"] += 1
    ms = timed(st, 300, 20)
    out.append({"what": "height-field terrain (0.08 m stairs every 0.3 m), 4096 envs", "ms_per_step": ms, "env_steps_per_s": 4096 / ms * 1e3})
    for o_ in out:
        print(json.dumps(o_))


if __name__ == "__main__":
    main()
