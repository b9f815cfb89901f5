"""The step kernel on the GPU against the float64 oracle over the full dynamics-randomisation range (tests/full_range.py), in both
precisions: diverging rows behave as the oracle's and leave the other envs of their handle bit-identical, every finite row matches the
oracle teacher-forced, and dynamics identification ranks a diverged individual last.

Each bound is about 4x the largest error measured on an H100 80GB HBM3 (400 W power limit); the measured value sits beside it.  The
checks themselves are those of tests/test_emu_full_range.py."""
import os

import numpy as np
import pytest

import f32_cases as F
import full_range as FR
import test_emu_full_range as E

pytestmark = pytest.mark.gpu

# float64: the conditioning rule of tests/test_emu_full_range.py, error <= F64_EXCESS x 4-ulp sensitivity + F64_BOUND on every step
F64_BOUND = 1e-12                   # errors are 2.5e-13 on every row up to friction 3; the largest, 1.2e-4 (fric_10.2), is 0.90x its
                                    # 4-ulp sensitivity of 1.8e-4 there, as the emulated device code's 3.3e-5 is 0.30x on the same step
F64_EXCESS = 4.0                    # measured 1.01 (draw_17)
F64_RESET_BOUND = 1e-7              # the H100's (FMA-contracted) float64 settle vs the oracle's: measured 2.3e-8 (draw_08, friction 6.6)
F32_BOUND = {"low": 4.4e-4,         # measured 1.1e-4
             "high": 5.7e-2}        # measured 1.4e-2 (draw_17, friction 7.6, on a step whose oracle f32-input sensitivity is 4.6e-3)
F32_RESET_BOUND = 8.3e-3            # float32 settle vs float64 settle: measured 2.1e-3 (draw_08, friction 6.6)
EXCESS = 1600.0                     # the conditioning rule of tests/test_gpu_f32_parity.py; measured multiple over the full range: 238


@pytest.fixture(scope="module")
def torch_cuda():
    import torch
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    return torch


def _np(t):
    return t.detach().double().cpu().numpy()


class _Gpu:
    def __init__(self, env):
        self.env = env

    def set_state(self, s):
        self.env.set_state(s)

    def get_state(self):
        return _np(self.env.get_state())

    def step(self, a):
        ob, rw, dn, inf = self.env.step(a)
        return _np(ob), _np(rw), dn.cpu().numpy(), _np(inf)


@pytest.mark.parametrize("precision", ["f32", "f64"])
def test_diverging_rows_agree_with_oracle(torch_cuda, etg_stable, precision):
    """Every row of the set in one handle: the reset is non-finite exactly for the oracle's diverging rows, and the first step reports
    done and the nan info column (9) exactly where the oracle does."""
    from oracle import oracle as O
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    w, b = etg_stable
    fin, div = FR.row_set()
    names = list(fin) + list(div)
    rows = np.stack([fin.get(n, div.get(n)) for n in names])
    env = VecQuadrupedalEnv(len(names), precision=precision)
    env.set_dynamics(rows)
    ob0 = _np(env.reset(w, b))
    a = E._actions(len(names), 1)[0]
    _, _, dn1, inf1 = _Gpu(env).step(a)
    env.close()
    assert [n for n, x in zip(names, ~np.isfinite(ob0).all(1)) if x] == list(div)
    for i, n in enumerate(names):
        o = O.OracleEnv(O.default_config(), rows[i])
        o.reset(w, b)
        _, _, do, io = o.step(a[i])
        assert bool(dn1[i]) == do and inf1[i, 9] == io[9], (n, dn1[i], do, inf1[i, 9], io[9])
        assert (n in div) == bool(inf1[i, 9]) and (n not in div or dn1[i])


@pytest.mark.parametrize("precision", ["f32", "f64"])
def test_mixed_handle_diverging_rows_leave_the_others_bit_identical(torch_cuda, etg_stable, precision):
    """N = 21 (two full warps and a ragged one), a diverging row in each: the finite envs' reset, steps with auto-reset, masked
    set_dynamics and masked reset are bit-identical to a handle whose diverging rows are replaced by the nominal row."""
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    w, b = etg_stable

    def make(rows):
        env = VecQuadrupedalEnv(21, precision=precision, auto_reset=True)
        env.set_dynamics(rows)
        g = _Gpu(env)
        return (env, g.step, g.get_state, lambda r, mk: env.set_dynamics(r, env_mask=mk),
                lambda w_, b_, mk, xo: _np(env.reset(w_, b_, env_mask=mk, x_offset=xo)))

    E.check_mixed(E.mixed_sequence(make, w, b))


def test_f64_teacher_forced_every_finite_row(torch_cuda, etg_stable):
    """All finite rows in one handle (N = 70), each env against its own oracle, as tests/test_emu_full_range.py runs them."""
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    w, b = etg_stable
    envs = []

    def make(rows):
        env = VecQuadrupedalEnv(len(rows), precision="f64")
        envs.append(env)
        env.set_dynamics(rows)
        return _Gpu(env), _np(env.reset(w, b))

    res = E.f64_all_rows(make, w, b)
    envs[0].close()
    E.check_f64(*res, F64_BOUND, F64_EXCESS, F64_RESET_BOUND)


def _f32_rows(env, names, rows, w, b, keep=None):
    """Teacher-forced f32 run of a handle already holding `rows`; checks every env in `keep` (default all) as check_f32 does."""
    ob0 = _np(env.reset(w, b))
    oracles = [F.make_oracle({}, None, w, b, rows[i], env_id=i) for i in range(len(names))]
    FR.adopt_reset_orientation([o for o, _ in oracles], _np(env.get_state()))
    rec = F.teacher_forced(_Gpu(env), [o for o, _ in oracles], E._actions(len(names)), F.flag_columns({}))
    for i in (range(len(names)) if keep is None else keep):
        ri = [r for r in rec if r[1] == i]
        cls = E.friction_class(rows[i])
        print("%-18s fric %5.2f lat %2.0f ms  reset %.3g  %s" % (names[i], rows[i][24], 1e3 * rows[i][25],
                                                           np.abs(ob0[i] - oracles[i][1]).max() / max(1.0, np.abs(oracles[i][1]).max()),
                                                           F.summary(cls, [r for r in ri if r[0] >= FR.warmup_steps(rows[i][25])])))
        E.check_f32(names[i], rows[i], ob0[i], oracles[i][1], ri, F32_BOUND[cls], EXCESS, F32_RESET_BOUND)


def test_f32_teacher_forced_every_finite_row(torch_cuda, etg_stable):
    """Every finite row as a single-env handle, the float32 product kernel against the float64 oracle."""
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    w, b = etg_stable
    fin, _ = FR.row_set()
    for name, row in fin.items():
        env = VecQuadrupedalEnv(1)
        env.set_dynamics(row[None, :])
        _f32_rows(env, [name], row[None, :], w, b)
        env.close()


def test_f32_teacher_forced_mixed_handle(torch_cuda, etg_stable):
    """The N = 21 handle with a diverging row in each warp: its finite envs against their oracles, in float32."""
    from paddlerobotics_b200.env import VecQuadrupedalEnv
    w, b = etg_stable
    rows = E.mixed_rows()[0]
    env = VecQuadrupedalEnv(21)
    env.set_dynamics(rows)
    _f32_rows(env, ["mixed_%02d" % i for i in range(21)], rows, w, b, keep=np.setdiff1d(np.arange(21), E.MIXED_DIVERGING))
    env.close()


def test_dynamics_identification_ranks_diverged_individuals_last(torch_cuda, golden):
    """Full-range individuals, finite and diverging mixed: the diverging ones score es.DIVERGED_REWARD in both precisions, SimpleGA.tell
    never makes them elite or best, and the finite ones' float64 rewards equal oracle rollouts scored with the reference's loss (the
    horizon, 10 control steps, keeps even the friction-9 rows non-chaotic: free-running float64 agrees to 1e-8 there)."""
    from oracle import oracle as O
    from paddlerobotics_b200.es import DIVERGED_REWARD, DynamicsEvaluator, SimpleGA
    from paddlerobotics_b200.etg import dynamic_dict_to_row, param2dynamic_dict

    def loss_np(drpy, motor, md, key):          # numpy restatement of Dynamic_parallel_model.py:29-41
        lm = np.max(np.mean((motor - md[key + "_motor_mean"]) ** 2 / md[key + "_motor_std"] ** 2, axis=0))
        ld = np.max(np.mean((drpy - md[key + "_drpy_mean"]) ** 2 / md[key + "_drpy_std"] ** 2, axis=0))
        return (ld + lm) / 2.0

    T = 10
    tab = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gait_action_list_CPG_stairstair7_12_3.npy")) + np.array([0, 0.9, -1.8] * 4)
    gait = {"exp": tab[:T], "ori": tab[100:100 + T]}
    rng = np.random.default_rng(0)
    md = {}
    for k in ("exp", "ori"):
        md[k + "_motor_mean"] = gait[k] + rng.normal(0, 0.02, (T, 12)); md[k + "_motor_std"] = rng.uniform(0.05, 0.1, (T, 12))
        md[k + "_drpy_mean"] = rng.normal(0, 0.2, (T, 3)); md[k + "_drpy_std"] = rng.uniform(0.3, 0.6, (T, 3))
    x = np.random.default_rng(FR.SEED).uniform(-1, 1, (FR.NDRAW, 48))      # the draws of full_range.drawn_rows
    fin, div = FR.row_set()
    pick = [1, 0, 3, 2, 22, 5, 8, 17]                                      # draw_01 / 03 / 05 diverge; 02, 08, 17, 22 have friction 6.6-9.7
    sols = x[pick]
    diverged = np.array(["draw_%02d" % i in div for i in pick])
    assert diverged.sum() == 3 and all(("draw_%02d" % i in fin) for i, d in zip(pick, diverged) if not d)
    for precision in ("f64", "f32"):
        ev = DynamicsEvaluator(len(pick), gait, md, steps=T, precision=precision)
        rew = ev.evaluate(sols).double().cpu().numpy()
        ev.env.close()
        print(precision, "rewards", np.round(rew, 4))
        assert np.isfinite(rew).all() and (rew[diverged] == DIVERGED_REWARD).all() and (rew[~diverged] > DIVERGED_REWARD).all(), rew
        np.random.seed(0)
        ga = SimpleGA(48, popsize=len(pick), elite_ratio=0.25, weight_decay=0.0)
        ga.ask()
        ga.solutions = sols
        ga.tell(rew)
        assert np.isfinite(ga.elite_rewards).all() and ga.best_reward > DIVERGED_REWARD
        assert not any(np.array_equal(p, s) for p in ga.elite_params for s in sols[diverged])
        assert set(np.argsort(rew)[:3]) == set(np.nonzero(diverged)[0])
        if precision == "f64":
            ref = np.zeros(len(pick))
            pose = np.array([0, 0.9, -1.8] * 4)
            for i in np.nonzero(~diverged)[0]:
                row = dynamic_dict_to_row(param2dynamic_dict(sols[i]))
                for k in ("exp", "ori"):
                    o = O.OracleEnv(O.default_config(etg_enabled=0), row); o.reset()
                    motor, drpy = [], []
                    for t in range(T):
                        _, _, _, info = o.step(gait[k][t] - pose)
                        motor.append(info[42:54]); drpy.append(info[39:42])
                    ref[i] += (30 - loss_np(np.array(drpy), np.array(motor), md, k)) / 2.0
            assert np.abs(rew[~diverged] - ref[~diverged]).max() < 1e-6, (rew, ref)


def test_dynamics_identification_ranks_a_nan_loss_column_diverged(torch_cuda):
    """An individual whose rollout is finite but whose accumulated loss has NaN in ONE of its 15 columns (one joint angle, or one body
    rate) is non-finite only through b2q_dyn_finish's maxima: it must score es.DIVERGED_REWARD.  With a NaN-dropping max (fmax) its
    reward came out finite from the other 14 columns, so it could become the elite.  The untouched individuals keep their rewards."""
    from paddlerobotics_b200.es import DIVERGED_REWARD, DynamicsEvaluator
    T = 5
    tab = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gait_action_list_CPG_stairstair7_12_3.npy")) + np.array([0, 0.9, -1.8] * 4)
    gait = {"exp": tab[:T], "ori": tab[100:100 + T]}
    rng = np.random.default_rng(1)
    md = {}
    for k in ("exp", "ori"):
        md[k + "_motor_mean"] = gait[k] + rng.normal(0, 0.02, (T, 12)); md[k + "_motor_std"] = rng.uniform(0.05, 0.1, (T, 12))
        md[k + "_drpy_mean"] = rng.normal(0, 0.2, (T, 3)); md[k + "_drpy_std"] = rng.uniform(0.3, 0.6, (T, 3))
    sols = rng.uniform(-0.2, 0.2, (4, 48))

    class Poisoned:
        """The library, except that dyn_finish first sets acc[env, col] = value for each entry of `poison`."""

        def __init__(self, lib, acc, poison):
            self.lib, self.acc, self.poison = lib, acc, poison

        def __getattr__(self, name):
            return getattr(self.lib, name)

        def b2q_dyn_finish(self, *args):
            for env, col, value in self.poison:
                self.acc[env, col] = value
            return self.lib.b2q_dyn_finish(*args)

    for precision in ("f32", "f64"):
        ev = DynamicsEvaluator(4, gait, md, steps=T, precision=precision)
        clean = ev.evaluate(sols).double().cpu().numpy()
        assert np.isfinite(clean).all() and (clean > DIVERGED_REWARD).all(), clean
        # env = key * pop + individual: individual 1's joint-angle column 4 on the "exp" gait, individual 2's body-rate column 13 on "ori"
        ev.lib = Poisoned(ev.lib, ev.acc, [(1, 4, float("nan")), (4 + 2, 13, float("nan"))])
        rew = ev.evaluate(sols).double().cpu().numpy()
        ev.env.close()
        assert rew[1] == DIVERGED_REWARD and rew[2] == DIVERGED_REWARD, (precision, rew)
        assert rew[0] == clean[0] and rew[3] == clean[3], (precision, rew, clean)
