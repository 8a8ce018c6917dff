"""parl_b200 — a H100-native actor-learner RL engine behind PaddlePaddle/PARL's API.

Keeps ``parl.Model / Algorithm / Agent``, ``parl.algorithms.{IMPALA,A2C,PPO,DQN,DDQN,PolicyGradient}``
and the ``parl.remote_class`` / ``parl.connect`` decorator surface; the hot path (vectorised env
stepping, action sampling, return scans, losses and their gradients, clip + Adam) runs in
hand-written sm_90a kernels behind the C ABI of include/parl_b200.h.

``import parl_b200 as parl`` or ``parl_b200.install_as_parl()`` (then ``import parl`` resolves here).
"""
import sys

__version__ = '0.1.0'

from .core import Model, Algorithm, Agent          # noqa: E402
from . import algorithms                           # noqa: E402
from . import utils                                # noqa: E402
from . import env                                  # noqa: E402
from . import remote                               # noqa: E402
from .remote import remote_class, connect          # noqa: E402

__all__ = ['Model', 'Algorithm', 'Agent', 'algorithms', 'utils', 'env', 'remote', 'remote_class', 'connect',
           'install_as_parl']


def install_as_parl():
    """Register this package under the name ``parl`` so unmodified reference scripts
    (``import parl``, ``from parl.utils import logger``, ``from parl.env.vector_env import VectorEnv`` ...)
    drop in."""
    me = sys.modules[__name__]
    sys.modules['parl'] = me
    prefix = __name__ + '.'
    for name, mod in list(sys.modules.items()):
        if name.startswith(prefix):
            sys.modules['parl.' + name[len(prefix):]] = mod
    return me
