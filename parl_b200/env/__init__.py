"""``parl.env`` for the hot path: VectorEnv with the reference's auto-reset contract for host gym-API
envs, and the device-resident vector envs that replace it on the H100."""
from .vector_env import VectorEnv
from .device_envs import AtariSynthVectorEnv, MujocoSynthVectorEnv, CartPoleVectorEnv
from .compat_wrappers import CompatWrapper
from . import atari_wrappers, mujoco_wrappers, compat_wrappers
from .host_bridge import HostEnvBridge

__all__ = ['VectorEnv', 'CompatWrapper', 'AtariSynthVectorEnv', 'MujocoSynthVectorEnv', 'CartPoleVectorEnv',
           'atari_wrappers', 'mujoco_wrappers', 'compat_wrappers', 'HostEnvBridge']
