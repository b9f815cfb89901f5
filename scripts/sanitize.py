"""Small invocation of every kernel in libb2q.so for compute-sanitizer (memcheck / racecheck / initcheck):
    compute-sanitizer --tool memcheck  python scripts/sanitize.py
    compute-sanitizer --tool racecheck python scripts/sanitize.py
"""
import ctypes as C, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from paddlerobotics_b200.env import VecQuadrupedalEnv
from paddlerobotics_b200.etg import ETG_layer, Opt_with_points
from paddlerobotics_b200.agent import MujocoAgent, SACLearner
from paddlerobotics_b200.replay import ReplayMemory
from paddlerobotics_b200.es import PopulationEvaluator

layer = ETG_layer(0.5, 0.026, 20, 0.04, np.array([-np.pi / 2, 0]), 0.2, 0.5)
w, b, _ = Opt_with_points(ETG=layer, ETG_T=0.5, Footheight=0.1, Steplength=0.05)
rng = np.random.default_rng(0)
hf = (rng.random((32, 32)) * 0.03).astype(np.float64)
for kw in (dict(num_envs=13), dict(num_envs=16, precision="f64"), dict(num_envs=24, auto_reset=True, action_filter=1, max_episode_steps=3),
           dict(num_envs=8, heightfield=(hf, -1.0, -1.0, 0.1)), dict(num_envs=40, threads_per_block=128),
           # round-2 paths: reduced sensor layout + noise + stuck / body-collision epilogue; the FEAT variant (joint-limit rows in shared
           # memory, TORQUE mode, base push, damping) in f32 and f64
           dict(num_envs=13, sensor_motor=2, sensor_imu=2, obs_normal=0, noise_stdev=(0.01, 0.05, 0.1, 0.02, 0.04), stuck_termination=1, body_collisions=1, auto_reset=True),
           dict(num_envs=11, joint_limits=1, knee_contacts=1, external_force=1, base_damping=(0.04, 0.02, 0.04, 0.01)), dict(num_envs=9, joint_limits=1, precision="f64"),
           dict(num_envs=8, motor_mode=1), dict(num_envs=8, motor_mode=2),
           # height-field far edges: the field ends 0.35 m behind the robot in x and y, so every foot lies beyond both far edges (the
           # cell index is clamped to nx - 2 / ny - 2; in f32, nx - 1.000001 rounds to nx - 1)
           dict(num_envs=13, heightfield=(hf[:24, :24], -1.5, -1.5, 0.05)), dict(num_envs=13, heightfield=(hf[:24, :24], -1.5, -1.5, 0.05), precision="f64")):
    env = VecQuadrupedalEnv(**kw)
    n = env.num_envs
    env.reset(w, b)
    a = (rng.random((n, 12)) * 0.6 - 0.3)
    if kw.get("motor_mode") == 2:                                # HYBRID: (q*, kp, qd*, kd, tau_ff) per motor
        a5 = np.zeros((n, 12, 5)); a5[:, :, 0] = np.array([0.0, 0.9, -1.8] * 4) + a; a5[:, :, 1] = 100.0; a5[:, :, 3] = 1.5; a = a5.reshape(n, 60)
    if kw.get("joint_limits"):
        a[:, 2::3] = 1.2; a[:, 0::3] = 0.9                       # into the stops: the shared-memory 24-row solve runs
    if kw.get("external_force"):
        env.set_external_force(rng.uniform(-10, 10, (n, 3)))
    if kw.get("noise_stdev"):
        env.reset(w, b, x_offset=rng.uniform(-0.1, 0.1, n))
    for _ in range(4):
        env.step(torch.as_tensor(a, device="cuda", dtype=env.dtype))
    env.step_host(a.astype(np.float32 if env.dtype == torch.float32 else np.float64))
    s = env.get_state(); env.set_state(s)
    env.reset(w, b, env_mask=(np.arange(n) % 2 == 0))
    torch.cuda.synchronize(); env.close()

agent = MujocoAgent(49, 12, seed=0)
obs = torch.randn(200, 49, device="cuda")
agent.predict(np.zeros(49, np.float32)); agent.sample(np.zeros(49, np.float32))
learner = SACLearner(agent, 256)
learner.actor.forward(obs, mode=1, seed=3)
rpm = ReplayMemory(4096, 49, 12)
for _ in range(3):
    rpm.append(torch.randn(512, 49, device="cuda"), torch.rand(512, 12, device="cuda") * 2 - 1, torch.randn(512, device="cuda"), torch.randn(512, 49, device="cuda"), torch.ones(512, device="cuda"))
for _ in range(2):
    learner.learn(*rpm.sample_batch(256), graph=False)
flat = SACLearner(agent, 256, sync="flat")
flat.learn(*rpm.sample_batch(256), graph=False)
# explicit-noise path, the graph path on the learner's static inputs (counter-RNG noise), behaviour cloning (given-target critic head, plain Adam)
learner.learn(*rpm.sample_batch(256), eps_next=torch.randn(256, 12, device="cuda"), eps_cur=torch.randn(256, 12, device="cuda"), graph=False)
g2 = SACLearner(MujocoAgent(49, 12, seed=1), 256)
for _ in range(2):
    g2.learn(*rpm.sample_batch(256, out=g2.static_batch()), graph=True, pull=False)
expert = MujocoAgent(49, 12, seed=2)
learner.bc_learn(torch.randn(256, 49, device="cuda"), torch.randn(256, 49, device="cuda"), expert)
# a non-default learner (A = 1: the runtime-dimension actor head, 32-thread dy blocks, one tile) and a full-width (in_dim 64) MLP on a
# partial last tile
small = SACLearner(MujocoAgent(3, 1, seed=3), 128)
small.learn(torch.randn(128, 3, device="cuda"), torch.rand(128, 1, device="cuda") * 2 - 1, torch.randn(128, device="cuda"), torch.randn(128, 3, device="cuda"), torch.ones(128, device="cuda"))
from paddlerobotics_b200.agent import FusedMLP
wide = FusedMLP(64, 2, 2)
for i in range(2):
    wide.set_weights(i, torch.randn(256, 64, device="cuda") * 0.1, torch.zeros(256, device="cuda"), torch.randn(256, 256, device="cuda") * 0.05,
                     torch.zeros(256, device="cuda"), torch.randn(2, 256, device="cuda") * 0.05, torch.zeros(2, device="cuda"))
wide.forward(torch.randn(129, 52, device="cuda"), in2=torch.randn(129, 12, device="cuda"), mode=1, seed=5)
ev = PopulationEvaluator(4, 2, max_steps=5)
ev.evaluate(np.repeat(w[None], 4, 0), np.repeat(b[None], 4, 0))
# masked appends on the device cursor: a partial mask whose rows cross the ring's wrap (100 rows, 60 valid, from position 4050 of 4096),
# then the ES evaluator feeding a host-cursor ring
mrpm = ReplayMemory(4096, 49, 12, device_cursor=True)
mrpm.cursor[0] = 4050
mrpm.append_masked(torch.randn(100, 49, device="cuda"), torch.rand(100, 12, device="cuda"), torch.randn(100, device="cuda"), torch.randn(100, 49, device="cuda"),
                   torch.ones(100, device="cuda"), torch.arange(100, device="cuda") % 5 < 3)
mrpm.sync_host()
ev.evaluate(np.repeat(w[None], 4, 0), np.repeat(b[None], 4, 0), replay=rpm)
# masked append with several 256-row chunks per CTA (n = 131073: tiles of 288 rows), cap == n, then a mask 3 bytes past a word boundary
# (count_valid's byte-wise head), both through ReplayMemory.append_masked
n = 131073
big = ReplayMemory(n, 49, 12, device_cursor=True)
big.cursor[0] = 7
big.append_masked(torch.randn(n, 49, device="cuda"), torch.rand(n, 12, device="cuda"), torch.randn(n, device="cuda"), torch.randn(n, 49, device="cuda"),
                  torch.ones(n, device="cuda"), torch.rand(n, device="cuda") < 0.5)
mbuf = torch.ones(1003, dtype=torch.uint8, device="cuda")
big.append_masked(torch.randn(1000, 49, device="cuda"), torch.rand(1000, 12, device="cuda"), torch.randn(1000, device="cuda"), torch.randn(1000, 49, device="cuda"),
                  torch.ones(1000, device="cuda"), mbuf[3:])
big.sync_host()
# ES fitness with 33 rollouts per individual: lane 0 runs the strided loop twice
evr = PopulationEvaluator(3, 33, max_steps=2)
evr.evaluate(np.repeat(w[None], 3, 0), np.repeat(b[None], 3, 0))
# behaviour cloning: student observation with noise into a ring that wraps (capacity not a multiple of n), without a ring; the gather cursor
# past the end of its permutation; bc_sweep with graph replays and an eager remainder (counter-RNG BC update)
from paddlerobotics_b200.bc import BCReplayMemory
bcm = BCReplayMemory(1001, 46, 49)
bcm._pos = 700
bcm.observe(torch.randn(513, 49, device="cuda"), 3)
bcm.observe(torch.randn(37, 49, device="cuda"), 4, noise=False, append=False)
bcur = torch.tensor([1001 - 20], dtype=torch.int64, device="cuda")
bcm.gather_cursor(torch.randperm(1001, device="cuda"), bcur, torch.empty(128, 46, device="cuda"), torch.empty(128, 49, device="cuda"))
bcl = SACLearner(MujocoAgent(46, 12, seed=4), 128)
bcl.bc_sweep(bcm, expert, torch.randperm(1001, device="cuda"), 7, seed=1, graph_steps=3)
# fused episode statistics: a partial last block (n = 300) in both precisions with terms and a count, ncols = 0 with a NULL count, and the
# evaluator's terms path
from paddlerobotics_b200 import _lib
from paddlerobotics_b200.es import EpisodeStats
for dt in (torch.float32, torch.float64):
    for terms, cc in ((("torso", "feet", "up", "tau", "badfoot", "footcontact"), "velx"), ((), None)):
        st = EpisodeStats(_lib.load(), 300, dt, torch.device("cuda"), terms, count_col=cc)
        st.step(torch.randn(300, device="cuda", dtype=dt), (torch.rand(300, device="cuda") < 0.3).to(torch.uint8), torch.randn(300, 56, device="cuda", dtype=dt),
                C.c_void_p(torch.cuda.current_stream().cuda_stream))
ev.evaluate(np.repeat(w[None], 4, 0), np.repeat(b[None], 4, 0), terms=("torso", "up"))
# training episode statistics: a partial last block (n = 300) in both precisions with the six terms and a count, with 16 terms, and with none
from paddlerobotics_b200.es import TrainEpisodeStats
for dt in (torch.float32, torch.float64):
    for terms, cc in ((("torso", "feet", "up", "tau", "badfoot", "footcontact"), "velx"), (("torso",) * 16, "velx"), ((), None)):
        ts = TrainEpisodeStats(_lib.load(), 300, torch.device("cuda"), terms, count_col=cc)
        for _ in range(3):
            ts.step(torch.randn(300, device="cuda", dtype=dt), (torch.rand(300, device="cuda") < 0.3).to(torch.uint8), torch.randn(300, 56, device="cuda", dtype=dt),
                    C.c_void_p(torch.cuda.current_stream().cuda_stream))
        ts.take(); ts.restart()
# deployment rehearsal: both kernels in both precisions on a partial last block (13 envs x 12 columns), counters past the table (NaN rows),
# a record shorter than the rollout, and no ETG block
from paddlerobotics_b200 import deploy
for prec in ("f32", "f64"):
    for kw in (dict(), dict(sensor_etg=0, sensor_dis=0)):
        env = VecQuadrupedalEnv(13, precision=prec, etg_enabled=0, **kw)
        tab = torch.randn(4, 12, device="cuda", dtype=env.dtype)
        rec_o, rec_a = torch.empty(3, env.observation_dim, device="cuda", dtype=env.dtype), torch.empty(3, 12, device="cuda", dtype=env.dtype)
        act = torch.empty(13, 12, device="cuda", dtype=env.dtype)
        obs = env.reset()
        for _ in range(6):
            deploy.deploy_obs(env, tab, 4, obs, rec_o)
            deploy.deploy_act(env, torch.rand(13, 12, device="cuda") * 2 - 1, 0.3, tab, 4, act, rec_a)
            obs = env.step(act)[0]
        torch.cuda.synchronize(); env.close()
torch.cuda.synchronize()
print("sanitizer script done")
