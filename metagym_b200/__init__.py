"""metagym_b200 -- H100-native batched engine for MetaGym's quadrotor and MetaMaze hot paths.

Public surface (mirrors the reference's gym.Env classes with a leading batch axis):
    BatchedQuadrotor            <- metagym.quadrotor.Quadrotor            (metagym/quadrotor/env.py:30)
    BatchedMetaMaze2D           <- metagym.metamaze.MetaMaze2D            (metagym/metamaze/envs/maze_env.py:155)
    BatchedMetaMazeDiscrete3D   <- metagym.metamaze.MetaMazeDiscrete3D    (metagym/metamaze/envs/maze_env.py:16)
    BatchedMetaMazeContinuous3D <- metagym.metamaze.MetaMazeContinuous3D  (metagym/metamaze/envs/maze_env.py:85)
All arithmetic runs in libmgb200.so (hand-written sm_90a CUDA, C ABI in include/mgb200.h); there is no CPU path.
"""
from ._lib import MgbError  # noqa: F401
from .registration import register_envs  # noqa: F401

__version__ = "0.2.0"

register_envs()     # no-op without gym / gymnasium (metagym/quadrotor/__init__.py:20-32, metagym/metamaze/__init__.py:21-54)


def __getattr__(name):
    # lazy: importing the package must not require torch/CUDA (the ABI tests only dlopen the library)
    if name in ("BatchedQuadrotor", "Quadrotor"):
        from . import quadrotor
        return getattr(quadrotor, name)
    if name in ("BatchedMetaMaze2D", "BatchedMetaMazeDiscrete3D", "BatchedMetaMazeContinuous3D", "MetaMaze2D",
                "MetaMazeDiscrete3D", "MetaMazeContinuous3D", "TaskConfig", "MazeTaskSampler"):
        from . import metamaze
        return getattr(metamaze, name)
    if name in ("MLPPolicy", "GRUPolicy", "LSTMPolicy", "PolicyPopulation"):
        from . import policy
        return getattr(policy, name)
    raise AttributeError(name)
