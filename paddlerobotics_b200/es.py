"""ES population evaluator (SURVEY §8 a15, §8e collective 1) and the host-side GA driver.

* `SimpleGA` keeps the reference's ask/tell contract and draws from NumPy's global RNG in the same order as
  ETGRL/alg/es.py:257-314, so that identically seeded runs produce identical populations on every rank (the reference's
  distributed variant relies on the same property: Dynamic_parallel_model.py:152-182).  The GA arithmetic stays on the
  host (12–48 parameters); what moves to the GPU is the rollout of the whole population.
* `PopulationEvaluator` replaces the serial loop `for solution in solutions: ... run_EStrain_episode(...)`
  (train.py:404-413): individual i owns `rollouts` consecutive envs of this rank's shard; all envs step in lock step
  inside the CUDA step kernel; per-env returns are frozen at the first `done`; fitness = mean over rollouts
  (`b2q_es_fitness`); shards are concatenated with ONE all-gather (NCCL on GPUs, gloo in the CPU tests).
"""
import ctypes as C

import numpy as np

from .etg import ETG_layer, Opt_with_points


def compute_weight_decay(weight_decay, model_param_list):
    grid = np.array(model_param_list)
    return -weight_decay * np.mean(grid * grid, axis=1)


class SimpleGA:
    """Elitist GA with Gaussian mutation; same constructor/ask/tell/reset semantics as the reference class."""

    def __init__(self, num_params, sigma_init=0.1, sigma_decay=0.999, sigma_limit=0.01, popsize=256, elite_ratio=0.1,
                 forget_best=False, weight_decay=0.01, param=None):
        self.num_params, self.popsize = num_params, int(popsize)
        self.sigma_init, self.sigma_decay, self.sigma_limit = sigma_init, sigma_decay, sigma_limit
        self.elite_ratio = elite_ratio
        self.elite_popsize = int(self.popsize * self.elite_ratio)
        self.sigma = sigma_init
        self.elite_params = np.zeros((self.elite_popsize, num_params))
        self.elite_rewards = np.zeros(self.elite_popsize)
        self.best_param = np.zeros(num_params) if param is None else param
        self.curr_best_param = self.best_param
        self.best_reward = 0
        self.first_iteration = True
        self.forget_best, self.weight_decay = forget_best, weight_decay

    def reset(self, param):
        self.best_param = np.copy(param)
        self.curr_best_param = np.copy(param)
        self.first_iteration = True

    def rms_stdev(self):
        return self.sigma

    def ask(self):
        # RNG draw order (global NumPy state): one randn block, then per child two parent picks and, after the first
        # generation, one uniform crossover mask.
        self.epsilon = np.random.randn(self.popsize, self.num_params) * self.sigma
        children = np.empty((self.popsize, self.num_params))
        parents = range(self.elite_popsize)
        for i in range(self.popsize):
            ia, ib = np.random.choice(parents), np.random.choice(parents)
            if self.first_iteration:
                base = self.best_param
            else:
                base = np.copy(self.elite_params[ia])
                take_b = np.where(np.random.rand(base.size) > 0.5)
                base[take_b] = self.elite_params[ib][take_b]
            children[i] = base + self.epsilon[i]
        self.solutions = children
        return children

    def tell(self, reward_table_result):
        assert len(reward_table_result) == self.popsize, "Inconsistent reward_table size reported."
        table = np.array(reward_table_result, dtype=np.float64)
        if self.weight_decay > 0:
            table += compute_weight_decay(self.weight_decay, self.solutions)
        if self.forget_best or self.first_iteration:
            reward, solution = table, self.solutions
        else:
            reward, solution = np.concatenate([table, self.elite_rewards]), np.concatenate([self.solutions, self.elite_params])
        idx = np.argsort(reward)[::-1][0:self.elite_popsize]
        self.elite_rewards, self.elite_params = reward[idx], solution[idx]
        self.curr_best_reward = self.elite_rewards[0]
        self.curr_best_param = np.copy(self.elite_params[0])
        if self.first_iteration or (self.curr_best_reward > self.best_reward):
            self.first_iteration = False
            self.best_reward = self.elite_rewards[0]
            self.best_param = np.copy(self.elite_params[0])
        if self.sigma > self.sigma_limit:
            self.sigma *= self.sigma_decay

    def current_param(self):
        return self.curr_best_param

    def set_mu(self, mu):
        pass

    def best_param_(self):
        return self.best_param

    def result(self):
        return (self.best_param, self.best_reward, self.curr_best_reward, self.sigma)


# ---- the gradient-style solvers of dynamics identification (Dynamic_parallel_model.py:102-149; ETGRL/alg/es.py:145-211,328-619).
#      Each keeps the reference's arithmetic order and dtypes, so an identically seeded run asks identical populations: the ranks are
#      float32, the Adam moments start as float32, and OpenES / PEPG move mu twice per tell (once directly, once through Adam).

def compute_centered_ranks(x):
    """Ranks of x (0 = smallest) mapped to [-0.5, 0.5] in float32; ties are broken by np.argsort's default order."""
    ranks = np.empty(x.size, dtype=int)
    ranks[x.ravel().argsort()] = np.arange(x.size)
    y = ranks.reshape(x.shape).astype(np.float32)
    y /= (x.size - 1)
    y -= .5
    return y


class Adam:
    """Adam ascent on `pi.mu`: update(g) moves pi.mu by -a·m/(sqrt(v)+eps) with the bias-corrected step a (beta1 0.99, beta2 0.999)."""

    def __init__(self, pi, stepsize, beta1=0.99, beta2=0.999, epsilon=1e-08):
        self.pi, self.stepsize, self.beta1, self.beta2, self.epsilon = pi, stepsize, beta1, beta2, epsilon
        self.t = 0
        self.m = np.zeros(pi.num_params, dtype=np.float32)
        self.v = np.zeros(pi.num_params, dtype=np.float32)

    def update(self, g):
        self.t += 1
        a = self.stepsize * np.sqrt(1 - self.beta2 ** self.t) / (1 - self.beta1 ** self.t)
        self.m = self.beta1 * self.m + (1 - self.beta1) * g
        self.v = self.beta2 * self.v + (1 - self.beta2) * (g * g)
        self.pi.mu = self.pi.mu + (-a * self.m / (np.sqrt(self.v) + self.epsilon))


class SimpleES:
    """Gaussian search around mu; tell() moves mu to the softmax(3·normalised reward)-weighted mean of the population."""

    def __init__(self, num_params, popsize=256, sigma_init=0.1, sigma_decay=0.999, sigma_limit=0.01, weight_decay=0.01, param=None):
        self.num_params, self.popsize = num_params, popsize
        self.sigma, self.sigma_decay, self.sigma_limit, self.weight_decay = sigma_init, sigma_decay, sigma_limit, weight_decay
        self.mu = np.zeros(num_params) if param is None else param
        self.best_mu = np.zeros(num_params) if param is None else param
        self.best_reward = 0
        self.first_iteration = True

    def ask(self):
        self.epsilon = np.random.randn(self.popsize, self.num_params)
        self.solutions = self.mu.reshape(1, self.num_params) + self.epsilon * self.sigma
        return self.solutions

    def tell(self, reward_table_result):
        assert len(reward_table_result) == self.popsize, "Inconsistent reward_table size reported."
        reward = np.array(reward_table_result)
        if self.weight_decay > 0:
            reward += compute_weight_decay(self.weight_decay, self.solutions)
        top = np.argsort(reward)[::-1][0]
        self.curr_best_reward, self.curr_best_mu = reward[top], self.solutions[top]
        if self.first_iteration or self.curr_best_reward > self.best_reward:
            self.first_iteration = False
            self.best_reward, self.best_mu = self.curr_best_reward, self.curr_best_mu
        if self.sigma > self.sigma_limit:
            self.sigma *= self.sigma_decay
        lo, spread = np.min(reward), np.max(reward) - np.min(reward)
        if spread > 1e-2:
            reward = 3 * (reward - lo) / spread
        e = np.exp(reward)
        weight = e / np.sum(e)
        self.mu = np.zeros(self.num_params)
        for i in range(self.popsize):               # sequential sum: the reference's order of additions
            self.mu += weight[i] * self.solutions[i]

    def result(self):
        return (self.best_mu, self.best_reward, self.curr_best_reward, self.sigma)


class OpenES:
    """OpenAI-ES: a Gaussian population around mu and a normalised-reward gradient step on mu."""

    def __init__(self, num_params, sigma_init=0.1, sigma_decay=0.999, sigma_limit=0.01, learning_rate=0.01, learning_rate_decay=0.9999,
                 learning_rate_limit=0.001, popsize=256, antithetic=False, weight_decay=0.01, rank_fitness=True, forget_best=True):
        self.num_params, self.popsize = num_params, popsize
        self.sigma, self.sigma_init, self.sigma_decay, self.sigma_limit = sigma_init, sigma_init, sigma_decay, sigma_limit
        self.learning_rate, self.learning_rate_decay, self.learning_rate_limit = learning_rate, learning_rate_decay, learning_rate_limit
        self.antithetic = antithetic
        if antithetic:
            assert popsize % 2 == 0, "Population size must be even"
            self.half_popsize = popsize // 2
        self.mu = np.zeros(num_params)
        self.best_mu = np.zeros(num_params)
        self.best_reward = 0
        self.first_iteration = True
        self.weight_decay, self.rank_fitness = weight_decay, rank_fitness
        self.forget_best = True if rank_fitness else forget_best
        self.optimizer = Adam(self, learning_rate)

    def ask(self):
        if self.antithetic:
            half = np.random.randn(self.half_popsize, self.num_params)
            self.epsilon = np.concatenate([half, -half])
        else:
            self.epsilon = np.random.randn(self.popsize, self.num_params)
        self.solutions = self.mu.reshape(1, self.num_params) + self.epsilon * self.sigma
        return self.solutions

    def tell(self, reward_table_result):
        assert len(reward_table_result) == self.popsize, "Inconsistent reward_table size reported."
        reward = np.array(reward_table_result)
        if self.rank_fitness:
            reward = compute_centered_ranks(reward)
        if self.weight_decay > 0:
            reward += compute_weight_decay(self.weight_decay, self.solutions)
        top = np.argsort(reward)[::-1][0]
        self.curr_best_reward, self.curr_best_mu = reward[top], self.solutions[top]
        if self.first_iteration or self.forget_best or self.curr_best_reward > self.best_reward:
            self.first_iteration = False
            self.best_reward, self.best_mu = self.curr_best_reward, self.curr_best_mu
        normalized = (reward - np.mean(reward)) / np.std(reward)
        change_mu = 1. / (self.popsize * self.sigma) * np.dot(self.epsilon.T, normalized)
        self.mu += self.learning_rate * change_mu
        self.optimizer.stepsize = self.learning_rate
        self.optimizer.update(-change_mu)
        if self.sigma > self.sigma_limit:
            self.sigma *= self.sigma_decay
        if self.learning_rate > self.learning_rate_limit:
            self.learning_rate *= self.learning_rate_decay

    def result(self):
        return (self.best_mu, self.best_reward, self.curr_best_reward, self.sigma)


class PEPG:
    """Parameter-exploring policy gradients: antithetic pairs mu ± eps with a per-parameter sigma that adapts, each step clipped to
    ±sigma_max_change·sigma; with elite_ratio > 0, mu moves by the mean offset of the elite instead of the Adam step."""

    def __init__(self, num_params, sigma_init=0.10, sigma_alpha=0.20, sigma_decay=0.999, sigma_limit=0.01, sigma_max_change=0.2, learning_rate=0.01,
                 learning_rate_decay=0.9999, learning_rate_limit=0.01, elite_ratio=0, popsize=256, average_baseline=True, weight_decay=0.01,
                 rank_fitness=True, forget_best=True):
        self.num_params, self.popsize = num_params, popsize
        self.sigma_init, self.sigma_alpha, self.sigma_decay, self.sigma_limit, self.sigma_max_change = sigma_init, sigma_alpha, sigma_decay, sigma_limit, sigma_max_change
        self.learning_rate, self.learning_rate_decay, self.learning_rate_limit = learning_rate, learning_rate_decay, learning_rate_limit
        self.average_baseline = average_baseline
        if average_baseline:
            assert popsize % 2 == 0, "Population size must be even"
            self.batch_size = popsize // 2
        else:
            assert popsize & 1, "Population size must be odd"
            self.batch_size = (popsize - 1) // 2
        self.elite_popsize = int(popsize * elite_ratio)
        self.use_elite = self.elite_popsize > 0
        self.mu = np.zeros(num_params)
        self.sigma = np.ones(num_params) * sigma_init
        self.best_mu = np.zeros(num_params)
        self.best_reward = 0
        self.first_iteration = True
        self.weight_decay, self.rank_fitness = weight_decay, rank_fitness
        self.forget_best = True if rank_fitness else forget_best
        self.optimizer = Adam(self, learning_rate)

    def ask(self):
        self.epsilon = np.random.randn(self.batch_size, self.num_params) * self.sigma.reshape(1, self.num_params)
        self.epsilon_full = np.concatenate([self.epsilon, -self.epsilon])
        eps = self.epsilon_full if self.average_baseline else np.concatenate([np.zeros((1, self.num_params)), self.epsilon_full])
        self.solutions = self.mu.reshape(1, self.num_params) + eps      # without the average baseline, member 0 is mu itself
        return self.solutions

    def tell(self, reward_table_result):
        assert len(reward_table_result) == self.popsize, "Inconsistent reward_table size reported."
        table = np.array(reward_table_result)
        if self.rank_fitness:
            table = compute_centered_ranks(table)
        if self.weight_decay > 0:
            table += compute_weight_decay(self.weight_decay, self.solutions)
        if self.average_baseline:
            base, reward = np.mean(table), table
        else:
            base, reward = table[0], table[1:]
        idx = np.argsort(reward)[::-1]
        if self.use_elite:
            idx = idx[0:self.elite_popsize]
        if self.average_baseline or reward[idx[0]] > base:
            self.curr_best_mu, self.curr_best_reward = self.mu + self.epsilon_full[idx[0]], reward[idx[0]]
        else:
            self.curr_best_mu, self.curr_best_reward = self.mu, base
        if self.first_iteration:
            self.sigma = np.ones(self.num_params) * self.sigma_init
        if self.first_iteration or self.forget_best or self.curr_best_reward > self.best_reward:
            self.first_iteration = False
            self.best_mu, self.best_reward = self.curr_best_mu, self.curr_best_reward
        eps, sigma = self.epsilon, self.sigma
        if self.use_elite:
            self.mu += self.epsilon_full[idx].mean(axis=0)
        else:
            change_mu = np.dot(reward[:self.batch_size] - reward[self.batch_size:], eps)
            self.optimizer.stepsize = self.learning_rate
            self.optimizer.update(-change_mu)
            self.mu += change_mu * self.learning_rate
        if self.sigma_alpha > 0:
            stdev_reward = 1.0 if self.rank_fitness else reward.std()
            S = (eps * eps - (sigma * sigma).reshape(1, self.num_params)) / sigma.reshape(1, self.num_params)
            rS = (reward[:self.batch_size] + reward[self.batch_size:]) / 2.0 - base
            change = self.sigma_alpha * (np.dot(rS, S) / (2 * self.batch_size * stdev_reward))
            change = np.maximum(np.minimum(change, self.sigma_max_change * self.sigma), -self.sigma_max_change * self.sigma)
            self.sigma += change
        if self.sigma_decay < 1:
            self.sigma[self.sigma > self.sigma_limit] *= self.sigma_decay
        if self.learning_rate_decay < 1 and self.learning_rate > self.learning_rate_limit:
            self.learning_rate *= self.learning_rate_decay

    def result(self):
        return (self.best_mu, self.best_reward, self.curr_best_reward, self.sigma)


def shard_range(n, rank, world):
    """Contiguous shard [lo, hi) of n units owned by `rank` (SURVEY §8e: GPU g owns [g·N/G,(g+1)·N/G))."""
    return (n * rank) // world, (n * (rank + 1)) // world


def solutions_to_etg(solutions, prior_points, w0, b0, ETG_T=0.5, etg_layer=None):
    """train.py:404-407: control-point deltas -> (w,b) per individual through Opt_with_points (host LS fit)."""
    layer = etg_layer or ETG_layer(ETG_T, 0.026, 20, 0.04, np.array([-np.pi / 2, 0]), 0.2, ETG_T)
    ws, bs = [], []
    for sol in solutions:
        pts = prior_points + np.asarray(sol).reshape(-1, 2)
        w, b, _ = Opt_with_points(ETG=layer, ETG_T=ETG_T, w0=w0, b0=b0, points=pts)
        ws.append(w); bs.append(b)
    return np.array(ws), np.array(bs)


def solutions_to_etg_device(solutions, prior_points, w0, b0, ETG_T=0.5, device=0, lamb=0.5, precision=1e-4):
    """Same as solutions_to_etg but batched on the GPU (b2q_etg_fit, SURVEY §8f-1): one thread per individual, float64."""
    import torch
    from . import _lib
    lib = _lib.load()
    layer = ETG_layer(ETG_T, 0.026, 20, 0.04, np.array([-np.pi / 2, 0]), 0.2, ETG_T)
    ts = [0.5 * ETG_T + 0.1, 0, 0.05, 0.1, 0.15, 0.2]
    obs = np.array([layer.update(t) for t in ts]).reshape(6, 20)
    dev = torch.device("cuda", int(device))
    t = lambda a: torch.as_tensor(np.ascontiguousarray(a, dtype=np.float64), device=dev)
    sol = t(np.asarray(solutions).reshape(-1, 12))
    pop = sol.shape[0]
    o, pp, w0t, b0t = t(obs), t(np.asarray(prior_points).reshape(6, 2)), t(np.asarray(w0).reshape(3, 20)), t(np.asarray(b0).reshape(3))
    w = torch.empty(pop, 3, 20, dtype=torch.float64, device=dev)
    b = torch.empty(pop, 3, dtype=torch.float64, device=dev)
    rc = lib.b2q_etg_fit(o.data_ptr(), pp.data_ptr(), sol.data_ptr(), w0t.data_ptr(), b0t.data_ptr(), float(lamb), float(precision), w.data_ptr(), b.data_ptr(), pop,
                         C.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
    assert rc == 0, rc
    return w, b


def all_gather_concat(local, world, rank, group=None):
    """One all-gather of equally sized shards; returns the concatenation on every rank (torch.distributed)."""
    import torch
    import torch.distributed as dist
    if world == 1:
        return local
    out = torch.empty((world * local.shape[0],) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(out, local.contiguous(), group=group)
    return out


def gather_fitness_and_length(fl, world, rank, group=None):
    """fl [2, pop_local] = this rank's [fitness | mean episode length] -> (fitness [pop], length [pop]) on every rank with ONE all-gather
    (SURVEY §8e collective 1: the two vectors travel packed)."""
    if world == 1:
        return fl[0], fl[1]
    g = all_gather_concat(fl.reshape(1, 2, fl.shape[1]), world, rank, group)     # [world, 2, pop_local]
    return g[:, 0, :].reshape(-1), g[:, 1, :].reshape(-1)


class PopulationEvaluator:
    """Evaluates this rank's shard of an ES population on its GPU and all-gathers the fitness vector."""

    def __init__(self, popsize, rollouts, max_steps=400, rank=0, world=1, device=0, policy=None, act_bound=0.3, precision="f32", **env_cfg):
        import torch
        from . import _lib
        from .env import VecQuadrupedalEnv
        if popsize % world != 0:
            raise ValueError("popsize must be divisible by the number of ranks (individuals are assigned whole to a GPU)")
        self.popsize, self.rollouts, self.max_steps, self.rank, self.world = popsize, rollouts, max_steps, rank, world
        self.lo, self.hi = shard_range(popsize, rank, world)
        self.pop_local = self.hi - self.lo
        self.n = self.pop_local * rollouts
        self.env = VecQuadrupedalEnv(self.n, device=device, precision=precision, auto_reset=False, **env_cfg)
        self.lib = _lib.load()
        dev, dt = self.env.device, self.env.dtype
        self.alive = torch.ones(self.n, dtype=torch.uint8, device=dev)
        self.ret = torch.zeros(self.n, dtype=dt, device=dev)
        self.len = torch.zeros(self.n, dtype=torch.int32, device=dev)
        self._fl = torch.zeros(2, self.pop_local, dtype=dt, device=dev)      # [fitness | mean length] packed: ONE all-gather per generation
        self.fitness, self.mean_len = self._fl[0], self._fl[1]
        self.policy, self.act_bound = policy, act_bound
        self.zero_act = torch.zeros(self.n, 12, dtype=dt, device=dev)
        self.es_launches = 0
        self.rows = None

    def evaluate(self, etg_w, etg_b, residual_noise=None, replay=None, record=None):
        """etg_w [pop,3,20], etg_b [pop,3] for the WHOLE population (identical on every rank); returns fitness[pop]
        (identical on every rank) and mean episode length[pop].

        replay: a ReplayMemory that receives the transitions whose reward enters the fitness (run_EStrain_episode with es_rpm,
        train.py:240-241): on every step, the rows of the envs still in their first episode, of the FIRST rollout of each recorded
        individual (the reference runs one episode per solution).  A row is (obs before the step, applied action / act_bound, reward,
        next obs, 1 - done).  record: bool [pop] over the whole population, default all.  Needs an f32 evaluator.  Afterwards
        `self.rows` (device int64 scalar) holds the number of rows this rank appended."""
        import torch
        if replay is not None and self.env.dtype != torch.float32:
            raise ValueError("evaluate(replay=...): the replay memory stores float32, so the evaluator must be built with precision='f32'")
        w = np.repeat(np.asarray(etg_w)[self.lo:self.hi], self.rollouts, axis=0)
        b = np.repeat(np.asarray(etg_b)[self.lo:self.hi], self.rollouts, axis=0)
        env = self.env
        obs = env.reset(w, b)
        self.alive.fill_(1); self.ret.zero_(); self.len.zero_()
        es = env.obs.element_size()
        stream = env._stream()
        if replay is not None:
            rec = np.ones(self.popsize, dtype=bool) if record is None else np.asarray(record, dtype=bool).reshape(self.popsize)
            rec_local = torch.as_tensor(rec[self.lo:self.hi].astype(np.uint8), device=env.device)
            keep = torch.zeros(self.pop_local, self.rollouts, dtype=torch.uint8, device=env.device)
            keep[:, 0] = rec_local                                  # rollout 0 of each recorded individual
            keep = keep.reshape(-1)
            mask, prev_obs = torch.empty_like(keep), torch.empty_like(env.obs)
            act_out, term, one = torch.empty_like(self.zero_act), torch.empty_like(self.ret), torch.ones_like(self.ret)
        for k in range(self.max_steps):
            if self.policy is not None:
                act = self.policy(obs) * self.act_bound            # agent.predict(obs) * action_bound, train.py:226-228
            else:
                act = self.zero_act
            if residual_noise is not None:
                act = act + residual_noise[k]
            if replay is not None:
                prev_obs.copy_(obs)                                 # env.step overwrites env.obs in place
            obs, rew, done, _ = env.step(act, donef=(k + 1 > self.max_steps))
            if replay is not None:                                  # the rows whose reward b2q_es_accumulate adds below
                torch.mul(self.alive, keep, out=mask)
                torch.div(act, self.act_bound, out=act_out)
                torch.sub(one, done, out=term)                      # terminal = 1 - done, train.py:229-230
                replay.append_masked(prev_obs, act_out, rew, obs, term, mask)
            rc = self.lib.b2q_es_accumulate(rew.data_ptr(), done.data_ptr(), self.alive.data_ptr(), self.ret.data_ptr(), self.len.data_ptr(),
                                            self.n, es, stream)
            assert rc == 0
            self.es_launches += 1
        rc = self.lib.b2q_es_fitness(self.ret.data_ptr(), self.len.data_ptr(), self.fitness.data_ptr(), self.mean_len.data_ptr(),
                                     self.pop_local, self.rollouts, es, stream)
        assert rc == 0
        self.es_launches += 1
        if replay is not None:
            self.rows = (self.len.reshape(self.pop_local, self.rollouts)[:, 0].long() * rec_local).sum()
        return gather_fitness_and_length(self._fl, self.world, self.rank)


DIVERGED_REWARD = -1e9      # the reward of an individual whose rollout went non-finite


class DynamicsEvaluator:
    """Sim-to-real dynamics identification on the GPU (SURVEY §8f-4): the population of 48-vectors is mapped through
    param2dynamic_dict to per-env dynamics rows; every individual replays the recorded gait tables (ETG off, action =
    table - pose_ori) for `steps` control steps and is scored against the recorded real-robot statistics with the
    reference's loss (RemoteESAgent.sample_episode / batch_sample_episodes, Dynamic_parallel_model.py:53-77).  Individuals
    are sharded over ranks exactly like the xparl actors (`solutions[i*K:(i+1)*K]`, :157-159) and the rewards all-gathered."""

    def __init__(self, popsize, gait, mean_dict, keys=("exp", "ori"), steps=100, rank=0, world=1, device=0, precision="f32", ring_depth=4, **env_cfg):
        import torch
        from . import _lib
        from .env import VecQuadrupedalEnv
        if popsize % world != 0:
            raise ValueError("popsize must be divisible by the number of ranks")
        self.popsize, self.keys, self.steps, self.rank, self.world = popsize, tuple(keys), steps, rank, world
        self.lo, self.hi = shard_range(popsize, rank, world)
        self.pop_local = self.hi - self.lo
        self.n = self.pop_local * len(self.keys)          # env index = key * pop_local + individual
        self.env = VecQuadrupedalEnv(self.n, device=device, precision=precision, etg_enabled=0, ring_depth=ring_depth, **env_cfg)
        self.lib = _lib.load()
        dev, dt = self.env.device, self.env.dtype
        pose = np.array([0, 0.9, -1.8] * 4)
        # per-step action table [steps, n, 12] and statistics [steps, keys, 15]
        act = np.stack([np.repeat((np.asarray(gait[k])[:steps] - pose)[:, None, :], self.pop_local, axis=1) for k in self.keys], axis=1).reshape(steps, self.n, 12)
        self.actions = torch.as_tensor(act, dtype=dt, device=dev)
        self.mean = [torch.as_tensor(np.concatenate([mean_dict[k + "_motor_mean"][:steps], mean_dict[k + "_drpy_mean"][:steps]], 1), dtype=dt, device=dev) for k in self.keys]
        self.std = [torch.as_tensor(np.concatenate([mean_dict[k + "_motor_std"][:steps], mean_dict[k + "_drpy_std"][:steps]], 1), dtype=dt, device=dev) for k in self.keys]
        self.acc = torch.zeros(self.n, 15, dtype=dt, device=dev)
        self.reward = torch.zeros(self.n, dtype=dt, device=dev)

    def evaluate(self, solutions):
        """solutions [pop,48] in [-1,1] (identical on every rank) -> reward [pop] = mean over the gait keys (identical on every rank);
        DIVERGED_REWARD for an individual whose rollout is non-finite."""
        import torch
        from .etg import param2dynamic_rows
        rows = param2dynamic_rows(np.asarray(solutions)[self.lo:self.hi])          # the rows of param2dynamic_dict, bit for bit
        env = self.env
        env.set_dynamics(np.tile(rows, (len(self.keys), 1)))          # env.reset(hardset=False, dynamic_param=...) :55
        env.reset()
        self.acc.zero_()
        es, stream, pl = env.obs.element_size(), env._stream(), self.pop_local
        for t in range(self.steps):
            _, _, _, info = env.step(self.actions[t], donef=False)
            for ki in range(len(self.keys)):
                sl = slice(ki * pl, (ki + 1) * pl)
                rc = self.lib.b2q_dyn_accumulate(info[sl].data_ptr(), self.mean[ki][t].data_ptr(), self.std[ki][t].data_ptr(), self.acc[sl].data_ptr(), pl, es, stream)
                assert rc == 0
        assert self.lib.b2q_dyn_finish(self.acc.data_ptr(), self.steps, self.reward.data_ptr(), self.n, es, stream) == 0
        local = self.reward.reshape(len(self.keys), pl).mean(0)        # (reward1 + reward2) / 2, :73
        # a row whose robot diverges (light legs: the settle already ends in NaN) must rank last, not poison tell(): argsort puts NaN
        # first in descending order, which would make the diverged individual the elite (same convention as train.py's ES phase)
        local = torch.where(torch.isfinite(local), local, torch.full_like(local, DIVERGED_REWARD))
        return all_gather_concat(local.contiguous(), self.world, self.rank)
