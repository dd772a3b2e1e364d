"""seed_rl_b200: H100-native (sm_90a) hot path of a SEED-RL V-trace learner.

Mirrors the reference's module layout for the path it replaces:
  common.vtrace, common.parametric_distribution, common.utils,
  dmlab.networks (ImpalaDeep), agents.vtrace.learner, grpc.
All device math runs in hand-written CUDA behind include/seedrl_b200.h.
"""
__version__ = '0.1.0'
