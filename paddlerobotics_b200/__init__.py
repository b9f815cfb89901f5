"""paddlerobotics_b200 — H100-native batched A1 simulator + rollout engine: drop-in for the per-step hot path of
PaddleRobotics QuadrupedalRobots/ETGRL (env.reset/env.step, agent.predict/sample, ES population fitness).

Python here is only the host-side mirror of the reference's call surface; all per-step arithmetic runs in
hand-written sm_90a CUDA reached through the C ABI in include/b2q.h (csrc/libb2q.so).  There is no CPU fallback.
"""
__version__ = "0.1.0"
