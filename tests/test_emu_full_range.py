"""The step kernel's device code in CPU emulation (tests/emu) against the float64 oracle over the full dynamics-randomisation range
(tests/full_range.py): rows that diverge at settle behave as the oracle's do and leave the other envs of their handle untouched, and
every finite row matches the oracle teacher-forced, in float64 and float32.

The emulator builds without FMA contraction and with exact division and square root, so its float32 errors are not the H100's; bounds
are about 4x the largest error measured here (measured value beside each)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import emu  # noqa: E402
import f32_cases as F  # noqa: E402
import full_range as FR  # noqa: E402
from oracle import oracle as O  # noqa: E402

STEPS = 12
HIGH_FRICTION = 3.0     # above it the feet stick and a control step is ill-conditioned (see DESIGN.md, "Full-range dynamics rows")

# float64, teacher-forced, all finite rows in one handle: on every step and measure, error <= F64_EXCESS x (the oracle's response to a
# 4-ulp perturbation of its input state and action, F.ulps) + F64_BOUND.  A well-conditioned step is held to the plain bound; a step
# where the feet stick and the oracle itself moves by up to 1.8e-4 under that perturbation is held to the multiple.
F64_BOUND = 1e-12       # errors are 2.5e-13 typical; the largest, 3.3e-5 (fric_10.2, step 8), is 0.30x its sensitivity of 1.8e-4
F64_EXCESS = 3.2        # measured 0.80 (draw_17)
# float32, teacher-forced, per friction class
F32_BOUND = {"low": 3.0e-4,     # measured 7.3e-5
             "high": 2.7e-2}    # measured 6.8e-3 (draw_17, friction 7.6, on a step where the oracle itself moves by 4.6e-3 under f32-rounded inputs)
# every f32 step is also held to the oracle's conditioning, error <= EXCESS x sensitivity + F.FLOOR, as tests/test_emu_f32.py does;
# measured multiple over the full range: 347
EXCESS = 2800.0
RESET_BOUND = 6e-3      # reset observation, float32 settle vs float64 settle (500 free substeps): measured 1.5e-3 (draw_22, friction 9.0)


class _Emu:
    """The emulator with the GPU env's call shapes, float64 numpy out."""

    def __init__(self, e):
        self.e = e

    def set_state(self, s):
        self.e.set_state(s)

    def get_state(self):
        return self.e.get_state().astype(np.float64)

    def step(self, a):
        return tuple(x.astype(np.float64) for x in self.e.step(a))


def _actions(n, steps=STEPS, seed=1):
    rng = np.random.default_rng(seed)
    return [rng.uniform(-0.2, 0.2, (n, 12)) for _ in range(steps)]


def test_full_range_row_set():
    """The set holds both classes, and no single clipped extreme diverges on its own: divergence needs several light links together."""
    fin, div = FR.row_set()
    print("full-range rows: %d finite, %d diverging at settle: %s" % (len(fin), len(div), sorted(div)))
    assert len(fin) >= 60 and len(div) >= 4
    assert all(name.startswith("draw_") for name in div)
    for r in div.values():                     # leg masses back to nominal: every diverging row settles
        fixed = r.copy()
        fixed[33:36] = 1.0
        assert FR.settles_finite(fixed)


@pytest.mark.parametrize("precision", [0, 1])
def test_diverging_rows_agree_with_oracle(etg_stable, precision):
    """Every row of the set in one handle: the reset is non-finite exactly for the oracle's diverging rows, and the first step reports
    done and the nan info column (9) exactly where the oracle does."""
    w, b = etg_stable
    fin, div = FR.row_set()
    names = list(fin) + list(div)
    rows = np.stack([fin.get(n, div.get(n)) for n in names])
    e = emu.EmuEnv(len(names), precision)
    e.set_dynamics(rows)
    ob0 = e.reset(w, b).astype(np.float64)
    a = _actions(len(names), 1)[0]
    ob1, rw1, dn1, inf1 = e.step(a)
    e.close()
    bad = ~np.isfinite(ob0).all(1)
    assert [n for n, x in zip(names, bad) if x] == list(div)
    for i, n in enumerate(names):
        o = O.OracleEnv(O.default_config(), rows[i])
        assert np.isfinite(o.reset(w, b)).all() == (n in fin), n
        _, _, do, io = o.step(a[i])
        assert bool(dn1[i]) == do and inf1[i, 9] == io[9], (n, dn1[i], do, inf1[i, 9], io[9])
        assert (n in div) == bool(inf1[i, 9]) and (n not in div or dn1[i])


MIXED_DIVERGING = (1, 5, 9, 14, 17, 20)   # N = 21 as on the GPU: two full warps of 8 robots and a ragged one, diverging rows in each


def mixed_rows():
    """(rows, rows with the diverging ones replaced by the nominal row, a second set for masked set_dynamics, its mask)."""
    fin, div = FR.row_set()
    f, d = list(fin.values()), list(div.values())
    rows, it_f, it_d = [], iter(f[:15]), iter(d)
    for i in range(21):
        rows.append(next(it_d) if i in MIXED_DIVERGING else next(it_f))
    rows = np.stack(rows)
    clean = rows.copy()
    clean[list(MIXED_DIVERGING)] = FR._nominal()
    mask = np.arange(21) % 4 == 1                               # envs 1, 5, 9, 13, 17: diverging and finite
    rows2 = rows.copy()
    rows2[mask] = np.stack([d[(i + 2) % len(d)] if i in MIXED_DIVERGING else f[15 + i] for i in np.nonzero(mask)[0]])
    clean2 = rows2.copy()
    clean2[list(MIXED_DIVERGING)] = FR._nominal()
    return rows, clean, rows2, clean2, mask


def mixed_sequence(make, w, b):
    """Reset, 4 steps with auto-reset, masked set_dynamics + masked reset, 4 more steps, on a handle from `make(rows)`; returns the
    outputs of every call (each [21, ...]) for the handle with the diverging rows ("mixed") and the one without ("clean")."""
    rows, clean, rows2, clean2, mask = mixed_rows()
    out = {}
    for tag, r1, r2 in (("mixed", rows, rows2), ("clean", clean, clean2)):
        env, step, state, set_dyn, reset = make(r1)
        xo = np.linspace(-0.05, 0.05, 21)
        res = [(reset(w, b, None, xo),)]
        acts = _actions(21, 8, seed=7)
        for k in range(4):
            res.append(step(acts[k]) + (state(),))
        set_dyn(r2, mask)
        res.append((state(), reset(w, b, mask, xo)))
        for k in range(4, 8):
            res.append(step(acts[k]) + (state(),))
        env.close()
        out[tag] = res
    return out


def check_mixed(out):
    """Finite envs bit-identical with and without the diverging rows beside them; the diverging envs report done and nan on every
    step (auto-reset puts them back on their non-finite snapshot)."""
    keep = np.setdiff1d(np.arange(21), MIXED_DIVERGING)
    for c, (x, y) in enumerate(zip(out["mixed"], out["clean"])):
        for p, q in zip(x, y):
            assert np.array_equal(np.asarray(p)[keep], np.asarray(q)[keep]), c
    for c, x in enumerate(out["mixed"]):
        if len(x) == 5:                                          # a step: obs, reward, done, info, state
            assert np.asarray(x[2])[list(MIXED_DIVERGING)].all() and (np.asarray(x[3])[list(MIXED_DIVERGING), 9] == 1).all(), c
            assert np.isfinite(np.asarray(x[0])[keep]).all(), c


@pytest.mark.parametrize("precision", [0, 1])
def test_mixed_handle_diverging_rows_leave_the_others_bit_identical(etg_stable, precision):
    w, b = etg_stable

    def make(rows):
        e = emu.EmuEnv(21, precision, auto_reset=1)
        e.set_dynamics(rows)
        f = lambda a: e.step(a)
        return (e, f, e.get_state, lambda r, m: e.set_dynamics(r, mask=m.astype(np.uint8)),
                lambda w_, b_, m, xo: e.reset(w_, b_, mask=None if m is None else m.astype(np.uint8), x_offset=xo))

    check_mixed(mixed_sequence(make, w, b))


def run_row(precision, row, w, b):
    e = emu.EmuEnv(1, precision)
    e.set_dynamics(row[None, :])
    ob0 = e.reset(w, b)[0].astype(np.float64)
    o, oo = F.make_oracle({}, None, w, b, row)
    FR.adopt_reset_orientation([o], e.get_state())
    rec = F.teacher_forced(_Emu(e), [o], _actions(1), F.flag_columns({}))
    e.close()
    return ob0, oo, rec


def f64_all_rows(make, w, b):
    """All finite rows in one handle from `make(rows)` (an engine for the teacher-forced runner), stepped teacher-forced against one
    oracle each with the same actions on the GPU and in emulation; the sensitivity is the oracle's response to 4-ulp input changes.
    Returns (names, rows, reset observations, oracle reset observations, records)."""
    fin, _ = FR.row_set()
    names, rows = list(fin), np.stack(list(fin.values()))
    eng, ob0 = make(rows)
    oracles = [F.make_oracle({}, None, w, b, rows[i], env_id=i) for i in range(len(names))]
    FR.adopt_reset_orientation([o for o, _ in oracles], eng.get_state())
    rec = F.teacher_forced(eng, [o for o, _ in oracles], _actions(len(names)), F.flag_columns({}), perturb=F.ulps)
    return names, rows, ob0, [oo for _, oo in oracles], rec


def check_f64(names, rows, ob0, oo, rec, bound, excess, reset_bound):
    """The reset on its own (the two settles); contact flags, done and the fall flag bit-exact; and error <= excess x sensitivity + bound
    on every measure of every step from the first one whose delayed observation reads only teacher-forced steps, on q-dot before it."""
    worst_all = 0.0
    for i, n in enumerate(names):
        ri = [r for r in rec if r[1] == i]
        wu = FR.warmup_steps(rows[i][25])
        reset = np.abs(ob0[i] - oo[i]).max() / max(1.0, np.abs(oo[i]).max())
        checked = [(r[0], m, r[2][m], r[3][m]) for r in ri for m in (F.METRICS if r[0] >= wu else ("qd",))]
        ex = max((e - bound) / max(s_, 1e-300) for _, _, e, s_ in checked)
        print("%-18s fric %5.2f lat %2.0f ms  reset %.3g  worst rel %.3g  4-ulp sensitivity %.3g  excess over %.0e %.3g" % (
            n, rows[i][24], 1e3 * rows[i][25], reset, max(c[2] for c in checked), max(c[3] for c in checked), bound, ex))
        worst_all = max(worst_all, ex)
        assert reset <= reset_bound, (n, reset)
        for k, i_, mm in ((r[0], r[1], r[4]) for r in ri):
            assert mm is None, (n, k, mm)
        for k, m, e, s_ in checked:
            assert e <= excess * s_ + bound, (n, k, m, e, s_)
    print("f64 full range, %d rows: worst multiple of the 4-ulp sensitivity above %.0e: %.3g" % (len(names), bound, worst_all))


def check_f32(name, row, ob0, oo, rec, bound, excess, reset_bound=RESET_BOUND):
    """Reset compared on its own (the two settles); then every step: contact flags, done and the fall flag bit-exact, and from the first
    step whose delayed observation reads only teacher-forced steps on, every measure within `bound` and the conditioning rule.  On the
    warm-up steps before it (FR.warmup_steps) the q-dot error, which the history does not enter, is held to the conditioning rule."""
    assert np.abs(ob0 - oo).max() / max(1.0, np.abs(oo).max()) <= reset_bound, name
    wu = FR.warmup_steps(row[25])
    for k, i, err, sens, mm in rec:
        assert mm is None, (name, k, mm)
        metrics = F.METRICS if k >= wu else ("qd",)
        for m in metrics:
            assert err[m] <= bound or k < wu, (name, k, m, err[m])
            assert err[m] <= excess * sens[m] + F.FLOOR, (name, k, m, err[m], sens[m])


def friction_class(row):
    return "high" if row[24] > HIGH_FRICTION else "low"


def test_f64_teacher_forced_every_finite_row(etg_stable):
    """All finite rows in one handle (N = 70), each env against its own oracle: the layout and actions of the GPU test."""
    w, b = etg_stable

    def make(rows):
        e = emu.EmuEnv(len(rows), 1)
        e.set_dynamics(rows)
        return _Emu(e), e.reset(w, b).astype(np.float64)

    check_f64(*f64_all_rows(make, w, b), F64_BOUND, F64_EXCESS, 1e-9)


def test_f32_teacher_forced_every_finite_row(etg_stable):
    w, b = etg_stable
    fin, _ = FR.row_set()
    for name, row in fin.items():
        ob0, oo, rec = run_row(0, row, w, b)
        post = [r for r in rec if r[0] >= FR.warmup_steps(row[25])]
        print("%-18s fric %5.2f lat %2.0f ms  reset %.3g  %s" % (name, row[24], 1e3 * row[25], np.abs(ob0 - oo).max() / max(1.0, np.abs(oo).max()),
                                                           F.summary(friction_class(row), post)))
        check_f32(name, row, ob0, oo, rec, F32_BOUND[friction_class(row)], EXCESS)
