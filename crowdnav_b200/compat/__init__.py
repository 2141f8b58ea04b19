"""Reference-facing surface: the names the reference's callers import, backed by the CUDA engine.

    import crowdnav_b200.compat as compat
    compat.install()                       # aliases crowd_sim.* / crowd_nav.utils.explorer in sys.modules, registers gym id
    import gym, crowd_sim
    env = gym.make('CrowdSim-v0')          # -> crowdnav_b200.compat.crowd_sim_env.CrowdSim

After install() the reference's own drivers (crowd_nav/test.py:64-109) run unchanged against the CUDA path: `from
crowd_sim.envs.utils.robot import Robot`, `from crowd_sim.envs.policy.orca import ORCA`, `from crowd_nav.utils.explorer
import Explorer`, `from crowd_sim.envs.utils.info import *` all resolve to the modules below. If `gym` is not importable
a minimal registry with register()/make() is provided under that name (the reference only uses those two calls).
"""
import sys
import types

from . import agents, crowd_sim_env, explorer, policies
from . import statetypes as state_types
from .crowd_sim_env import CrowdSim

_ENV_ID = 'CrowdSim-v0'
_registry = {}


def make(env_id=_ENV_ID):
    if env_id != _ENV_ID:
        raise KeyError(env_id)
    return CrowdSim()


def _module(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


def install(force_gym_shim=False, numpy_stream=False):
    """numpy_stream=True: CrowdSim.reset leaves np.random in the state the reference's reset leaves it in (the case's seed
    advanced by the scene generator's draws), so the reference's own policies explore from the reference's stream. The
    hand-placed debug scene (test case -1) is not seeded by the reference either: numpy's state is left alone there."""
    t = state_types
    crowd_sim_env.NUMPY_STREAM = bool(numpy_stream)
    _module('crowd_sim')
    _module('crowd_sim.envs', CrowdSim=CrowdSim)
    _module('crowd_sim.envs.crowd_sim', CrowdSim=CrowdSim)
    _module('crowd_sim.envs.utils')
    _module('crowd_sim.envs.utils.action', ActionXY=t.ActionXY, ActionRot=t.ActionRot)
    _module('crowd_sim.envs.utils.state', FullState=t.FullState, ObservableState=t.ObservableState, JointState=t.JointState)
    _module('crowd_sim.envs.utils.info', Timeout=t.Timeout, ReachGoal=t.ReachGoal, Danger=t.Danger, Collision=t.Collision,
            Nothing=t.Nothing, __all__=['Timeout', 'ReachGoal', 'Danger', 'Collision', 'Nothing'])
    _module('crowd_sim.envs.utils.agent', Agent=agents.Agent)
    _module('crowd_sim.envs.utils.human', Human=agents.Human)
    _module('crowd_sim.envs.utils.robot', Robot=agents.Robot)
    _module('crowd_sim.envs.policy')
    _module('crowd_sim.envs.policy.policy', Policy=policies.Policy)
    _module('crowd_sim.envs.policy.orca', ORCA=policies.ORCA)
    _module('crowd_sim.envs.policy.linear', Linear=policies.Linear)
    _module('crowd_sim.envs.policy.policy_factory', policy_factory=policies.policy_factory)
    if 'crowd_nav' not in sys.modules:
        _module('crowd_nav'); _module('crowd_nav.utils')
    _module('crowd_nav.utils.explorer', Explorer=explorer.Explorer, average=explorer.average)
    try:
        if force_gym_shim:
            raise ImportError
        import gym
        from gym.envs.registration import register
        try:
            register(id=_ENV_ID, entry_point='crowdnav_b200.compat.crowd_sim_env:CrowdSim')
        except Exception:       # already registered
            pass
    except ImportError:
        g = _module('gym', make=make, register=lambda id, entry_point=None, **kw: _registry.__setitem__(id, entry_point),
                    Env=object)
        _module('gym.envs'); _module('gym.envs.registration', register=g.register)
    return sys.modules['crowd_sim']
