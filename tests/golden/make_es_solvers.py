"""Generates tests/golden/es_solvers.npz: the reference's dynamics-identification solvers (ETGRL/alg/es.py) built by the reference's own
ES_ParallelModel.set_solver (model/Dynamic_parallel_model.py:102-149, ast-extracted: the module imports rlschool and parl), driven
through ROUNDS ask/tell rounds with seeded fitness.

Run where the reference is installed (oracle/ref_shim.py):  python tests/golden/make_es_solvers.py
"""
import ast
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import ref_shim  # noqa: E402

ALGS = ("ga", "ses", "pepg", "openes", "simples")
NUM_PARAMS, K, THREAD, SIGMA, SIGMA_DECAY = 48, 20, 2, 0.1, 0.9999     # Dynamic_train.py defaults, ES_ParallelModel's sigma_decay
ROUNDS = 4


def fitness(sol, target, rng):
    """A smooth objective with seeded noise and a few exact ties (so the rank transforms see them)."""
    f = 30.0 - np.sum((sol - target) ** 2, axis=1) + rng.normal(0, 0.01, sol.shape[0])
    f[1::13] = f[0]
    return f


def main():
    ns = ref_shim.load()
    src = open(os.path.join(ns.REF, "model", "Dynamic_parallel_model.py")).read()
    env = {"np": np, "SimpleGA": ns.es.SimpleGA, "PEPG": ns.es.PEPG, "OpenES": ns.es.OpenES, "SimpleES": ns.es.SimpleES}
    for node in ast.parse(src).body:
        if isinstance(node, ast.ClassDef) and node.name == "ES_ParallelModel":
            for fn in node.body:
                if isinstance(fn, ast.FunctionDef) and fn.name == "set_solver":
                    exec(compile(ast.Module([fn], []), "Dynamic_parallel_model.py", "exec"), env)
    out = {"num_params": np.array(NUM_PARAMS), "popsize": np.array(K * THREAD), "sigma": np.array(SIGMA), "sigma_decay": np.array(SIGMA_DECAY)}
    target = np.random.default_rng(11).uniform(-0.3, 0.3, NUM_PARAMS)
    out["target"] = target
    for j, alg in enumerate(ALGS):
        model = types.SimpleNamespace(alg=alg, num_params=NUM_PARAMS, sigma=SIGMA, sigma_decay=SIGMA_DECAY, popsize=K * THREAD)
        np.random.seed(100 + j)
        env["set_solver"](model, param=np.zeros(NUM_PARAMS))         # ES_ParallelModel.__init__, :100
        rng = np.random.default_rng(200 + j)
        rec = {k: [] for k in ("solutions", "fitness", "best", "best_reward", "curr_best_reward", "sigma")}
        for _ in range(ROUNDS):
            sol = model.solver.ask()
            fit = fitness(sol, target, rng)
            model.solver.tell(fit.copy())
            r = model.solver.result()
            for k, v in zip(("solutions", "fitness", "best", "best_reward", "curr_best_reward", "sigma"), (sol, fit) + tuple(r[:4])):
                rec[k].append(np.array(v, copy=True))
        out["%s_seed" % alg] = np.array(100 + j)
        for k, v in rec.items():
            out["%s_%s" % (alg, k)] = np.array(v)
    np.savez_compressed(os.path.join(HERE, "es_solvers.npz"), **out)
    print("wrote", sorted(out.keys()))


if __name__ == "__main__":
    main()
