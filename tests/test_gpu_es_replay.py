"""The ES phase's rollouts in the replay memory (run_EStrain_episode with --es_rpm, ETGRL/train.py:213-249,395): the masked ring append
on the device cursor (b2q_rpm_append_masked_cursor), ReplayMemory.append_masked in both cursor modes, PopulationEvaluator.evaluate(replay=)
and train.py --es_rpm."""
import json

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

OD, AD = 49, 12


class RingModel:
    """Sequential `x[mask]` appends into a ring of the same capacity, in torch."""

    def __init__(self, cap, device):
        import torch
        self.cap, self.pos, self.size = cap, 0, 0
        self.data = [torch.zeros(cap, OD, device=device), torch.zeros(cap, AD, device=device), torch.zeros(cap, device=device),
                     torch.zeros(cap, OD, device=device), torch.zeros(cap, device=device)]

    def append(self, rows, mask=None):
        import torch
        rows = rows if mask is None else [x[mask.bool()] for x in rows]
        m = rows[0].shape[0]
        slots = (self.pos + torch.arange(m, device=rows[0].device)) % self.cap
        for d, x in zip(self.data, rows):
            d[slots] = x
        self.pos, self.size = (self.pos + m) % self.cap, min(self.size + m, self.cap)


def _ring(rpm):
    return [rpm.obs, rpm.action, rpm.reward, rpm.next_obs, rpm.terminal]


def _rows(n, g):
    import torch
    return [torch.randn(n, OD, device="cuda", generator=g), torch.rand(n, AD, device="cuda", generator=g) * 2 - 1, torch.randn(n, device="cuda", generator=g),
            torch.randn(n, OD, device="cuda", generator=g), (torch.rand(n, device="cuda", generator=g) > 0.1).float()]


@pytest.mark.parametrize("device_cursor", [False, True])
@pytest.mark.parametrize("n", [1, 31, 160, 4097])
@pytest.mark.parametrize("density", [0.0, 0.3, 1.0])
def test_masked_append_equals_sequential_boolean_index_appends(device_cursor, n, density):
    import torch
    from paddlerobotics_b200.replay import ReplayMemory
    cap = n + n // 3 + 2                                     # 12 appends of density 0.3 wrap the ring about 2.7 times
    rpm = ReplayMemory(cap, OD, AD, device_cursor=device_cursor)
    model = RingModel(cap, "cuda")
    g = torch.Generator(device="cuda"); g.manual_seed(n * 10 + int(density * 10))
    first = _rows(n, g)
    rpm.append(*first); model.append(first)
    rpm.sample_batch(8)                                      # the sample counter is 1 and must stay 1
    for k in range(12):
        rows = _rows(n, g)
        if k == 6:                                           # a plain append between masked ones reads the mirrors the masked ones advanced
            rpm.append(*rows); model.append(rows)
            continue
        mask = torch.rand(n, device="cuda", generator=g) < density
        if k % 2:
            mask = mask.to(torch.uint8) * 7                  # any nonzero byte is valid
        rpm.append_masked(*rows, mask)
        model.append(rows, mask)
    torch.cuda.synchronize()
    for got, want in zip(_ring(rpm), model.data):
        assert torch.equal(got, want)
    assert rpm.size() == model.size and (rpm._curr_pos, rpm._curr_size, rpm._samples) == (model.pos, model.size, 1)
    cursor = rpm.cursor if device_cursor else rpm._masked_cursor
    assert cursor.tolist() == [model.pos, model.size, 1]
    if density == 0.0:
        assert (model.pos, model.size) == ((2 * n) % cap, min(2 * n, cap))     # only the two plain appends moved the ring


def test_masked_append_replays_from_a_graph_with_new_mask_contents():
    import torch
    from paddlerobotics_b200.replay import ReplayMemory
    n, cap = 300, 1000
    eager, graphed = ReplayMemory(cap, OD, AD, device_cursor=True), ReplayMemory(cap, OD, AD, device_cursor=True)
    g = torch.Generator(device="cuda"); g.manual_seed(5)
    rows = _rows(n, g)
    mask = torch.zeros(n, dtype=torch.uint8, device="cuda")
    def fill():
        for x, y in zip(rows, _rows(n, g)):
            x.copy_(y)
        mask.copy_((torch.rand(n, device="cuda", generator=g) < 0.7).to(torch.uint8))
    fill(); eager.append_masked(*rows, mask); graphed.append_masked(*rows, mask)      # eager call first (warm-up)
    torch.cuda.synchronize()
    gr = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream(); side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.graph(gr, stream=side):
        graphed.append_masked(*rows, mask)
    torch.cuda.current_stream().wait_stream(side)
    total = int(mask.sum())
    for _ in range(5):
        fill()
        total += int(mask.sum())
        eager.append_masked(*rows, mask)
        gr.replay()
    graphed.sync_host(); eager.sync_host()
    for x, y in zip(_ring(eager), _ring(graphed)):
        assert torch.equal(x, y)
    assert total > cap                                       # the replays wrapped the ring
    assert graphed.cursor.tolist() == eager.cursor.tolist() == [total % cap, cap, 0]
    assert (graphed._curr_pos, graphed._curr_size) == (eager._curr_pos, eager._curr_size) == (total % cap, cap)


def test_masked_append_rejects_rows_beyond_capacity_and_mismatched_rows():
    import torch
    from paddlerobotics_b200.replay import ReplayMemory
    rpm = ReplayMemory(16, OD, AD, device_cursor=True)
    g = torch.Generator(device="cuda"); g.manual_seed(0)
    with pytest.raises(AssertionError):
        rpm.append_masked(*_rows(17, g), torch.ones(17, dtype=torch.uint8, device="cuda"))
    with pytest.raises(ValueError):
        rpm.append_masked(*_rows(8, g), torch.ones(7, dtype=torch.uint8, device="cuda"))
    assert rpm.cursor.tolist() == [0, 0, 0] and rpm.size() == 0


POP, ROLL, T, ACT_BOUND = 6, 2, 60, 0.3


@pytest.fixture(scope="module")
def es_case(etg_stable):
    """pop 6 x 2 rollouts x 60 steps on the gentle gait; per-individual noise from 0 to 1 rad: the quiet ones walk all 60 steps, the
    loud ones fall within a few steps.  Returns the gait, the noise and the per-step rows recorded in Python with the fitness kernels'
    alive flags (alive before this step's accumulation)."""
    import torch
    from paddlerobotics_b200.es import PopulationEvaluator
    w, b = etg_stable
    W, B = np.repeat(np.asarray(w)[None], POP, 0), np.repeat(np.asarray(b)[None], POP, 0)
    scale = torch.tensor([0.0, 0.05, 0.2, 0.3, 0.5, 1.0], device="cuda").repeat_interleave(ROLL)
    g = torch.Generator(device="cuda"); g.manual_seed(11)
    noise = torch.randn(T, POP * ROLL, 12, device="cuda", generator=g) * scale[None, :, None]
    ev = PopulationEvaluator(POP, ROLL, max_steps=T, act_bound=ACT_BOUND)
    fit, mlen = ev.evaluate(W, B, residual_noise=noise)
    fit, mlen, lens = fit.clone(), mlen.clone(), ev.len.clone()
    env = ev.env
    obs = env.reset(np.repeat(W, ROLL, 0), np.repeat(B, ROLL, 0))
    alive = torch.ones(POP * ROLL, dtype=torch.bool, device="cuda")
    steps = []
    for k in range(T):
        act = ev.zero_act + noise[k]
        o0 = obs.clone()
        obs, rew, done, _ = env.step(act)
        steps.append((o0, act / ACT_BOUND, rew.clone(), obs.clone(), 1.0 - done.float(), alive.clone()))
        alive &= ~done.bool()
    return dict(ev=ev, W=W, B=B, noise=noise, fit=fit, mlen=mlen, lens=lens, steps=steps)


def _expected(case, record):
    import torch
    keep = torch.zeros(POP, ROLL, dtype=torch.bool, device="cuda")
    keep[:, 0] = torch.as_tensor(record, device="cuda")
    keep = keep.reshape(-1)
    return [torch.cat([s[j][s[5] & keep] for s in case["steps"]]) for j in range(5)]


def test_evaluator_stores_exactly_the_fitness_transitions(es_case):
    import torch
    from paddlerobotics_b200.replay import ReplayMemory
    ev, lens = es_case["ev"], es_case["lens"]
    assert bool((lens < 20).any()) and bool((lens == T).any()), lens.tolist()              # some fall early, some walk the whole episode
    rpm = ReplayMemory(4000, OD, AD)
    fit, mlen = ev.evaluate(es_case["W"], es_case["B"], residual_noise=es_case["noise"], replay=rpm)
    assert torch.equal(fit, es_case["fit"]) and torch.equal(mlen, es_case["mlen"])        # the fitness path is untouched
    want = _expected(es_case, [True] * POP)
    m = want[0].shape[0]
    assert m == int(lens.reshape(POP, ROLL)[:, 0].sum()) == int(ev.rows) == rpm.size()
    for got, x in zip(_ring(rpm), want):
        assert torch.equal(got[:m], x)
    assert not bool(rpm.obs[m:].any())


def test_evaluator_records_only_the_selected_individual(es_case):
    import torch
    from paddlerobotics_b200.replay import ReplayMemory
    ev, lens = es_case["ev"], es_case["lens"]
    record = [False, False, False, True, False, False]
    rpm = ReplayMemory(4000, OD, AD, device_cursor=True)
    fit, _ = ev.evaluate(es_case["W"], es_case["B"], residual_noise=es_case["noise"], replay=rpm, record=record)
    assert torch.equal(fit, es_case["fit"])
    want = _expected(es_case, record)
    m = int(lens[3 * ROLL])
    assert want[0].shape[0] == m == int(ev.rows) == rpm.size() and rpm.cursor.tolist() == [m, m, 0]
    for got, x in zip(_ring(rpm), want):
        assert torch.equal(got[:m], x)


def test_evaluator_replay_needs_float32():
    from paddlerobotics_b200.es import PopulationEvaluator
    from paddlerobotics_b200.replay import ReplayMemory
    ev = PopulationEvaluator(2, 1, max_steps=2, precision="f64")
    with pytest.raises(ValueError):
        ev.evaluate(np.zeros((2, 3, 20)), np.zeros((2, 3)), replay=ReplayMemory(16, OD, AD))
    ev.env.close()


@pytest.mark.parametrize("graph_iter", [1, 0])
def test_train_loop_es_rpm_feeds_the_replay(graph_iter, monkeypatch, capsys):
    """--es_rpm 1: the ES phases' rows join the replay; the count printed per generation is popsize x mean episode length, the ring's
    fill level after each phase is the SAC rows plus the ES rows so far, and after the SAC steps that follow the last phase the host
    mirrors still count every row and (captured iteration) equal the device cursor."""
    from paddlerobotics_b200 import train
    made = []

    class Recorded(train.ReplayMemory):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            made.append(self)
    monkeypatch.setattr(train, "ReplayMemory", Recorded)
    pop, n, max_steps = 10, 256, 6400                                                    # SimpleGA keeps int(0.1 * popsize) >= 1 elites
    log = train.main(["--num_envs", str(n), "--batch", "256", "--warmup_steps", "2048", "--log_every", "5", "--max_steps", str(max_steps),
                      "--es_every_steps", "2560", "--es_train_steps", "1", "--popsize", str(pop), "--es_rollouts", "1", "--e_step", "100",
                      "--task_mode", "ground", "--es_rpm", "1", "--graph_iter", str(graph_iter)])
    lines = [json.loads(l) for l in capsys.readouterr().out.splitlines() if l.startswith("{")]
    es_total, gen_rows, phases = 0, [], 0
    for r in lines:
        if "ES_gen" in r:                                                                  # one generation per phase
            assert r["rpm_rows"] == pytest.approx(pop * r["mean_len"], abs=1e-3) and r["rpm_rows"] > 0   # mean_len: a float32 mean
            gen_rows.append(r["rpm_rows"])
        elif "ES_rpm_rows" in r:
            phases += 1
            assert len(gen_rows) == 1 and 1 <= r["ES_rpm_rows"] - gen_rows[0] <= 100      # plus one incumbent episode of at most e_step steps
            es_total += r["ES_rpm_rows"]; gen_rows = []
            assert r["rpm_size"] == r["env_steps"] + es_total                              # every SAC row plus every ES row so far
    assert phases == 2 and not gen_rows                                                    # at 2560 and 5120 env steps
    assert all("ES_gen" not in r and "ES_rpm_rows" not in r for r in log)
    losses = [r["critic_loss"] for r in log if r["critic_loss"] is not None] + [r["actor_loss"] for r in log if r["actor_loss"] is not None]
    assert len(losses) >= 2 and np.isfinite(losses).all()
    (rpm,) = made
    assert not rpm._stale and (rpm._curr_pos, rpm._curr_size) == (max_steps + es_total,) * 2   # mirrors kept by append / advance after the phases
    assert (rpm.cursor is not None) == bool(graph_iter)
    if graph_iter:                                                                         # and the captured iteration's device cursor agrees
        assert rpm.cursor.tolist()[:2] == [rpm._curr_pos, rpm._curr_size]
