"""Device-native env kinds and how a creator callable maps to one.

The reference passes ``env_creator`` callables to ``vector.make`` and the backend calls each one N times
(vector.py:79).  The B200 backend instead asks the creator which native kind it stands for and builds ONE
device-resident multi-env (the PufferEnv seam, pufferlib/environment.py:1-21).  A creator is recognised by a
``b200_kind`` attribute (ours) or by name for the reference's own ``make_squared``, ``make_memory``, ...
(pufferlib/environments/ocean/environment.py:28-72), so the reference's creator can be passed unchanged.

A kind may have several agents per env (multiagent: two); the backend reads that number from the library
(pb_env_agents_per_env) and sizes every row buffer by agents, as the reference's vectorisers do (vector.py:85-92).
"""
import math
import operator

from pufferlib_b200.exceptions import APIUsageError

KNOWN_BY_NAME = {'make_squared': 'squared', 'make_breakout': 'breakout', 'make_snake': 'snake', 'make_pong': 'pong',
                 'make_memory': 'memory', 'make_password': 'password', 'make_stochastic': 'stochastic',
                 'make_bandit': 'bandit', 'make_multiagent': 'multiagent', 'make_breakout_pixels': 'breakout_pixels'}

# Kinds whose reference env draws from a process-global RNG stream (CPython's `random` for squared, numpy's
# `np.random` for memory and bandit): their results depend on which envs share a process, so the B200 backend gives
# every `num_workers` worker its own shard and stream, as the reference's Multiprocessing backend does.
GLOBAL_STREAM_KINDS = frozenset({'squared', 'memory', 'bandit'})

# The reference creators' parameters (positional order) and defaults, ocean/environment.py:33-46, 67-70
OCEAN_PARAMS = {
    'memory': (('mem_length', 2), ('mem_delay', 2)),
    'password': (('password_length', 5),),
    'stochastic': (('p', 0.7), ('horizon', 100)),
    'bandit': (('num_actions', 10), ('reward_scale', 1), ('reward_noise', 1)),
}


def _ocean_values(kind, args, kwargs):
    params = OCEAN_PARAMS[kind]
    if len(args or ()) > len(params):
        raise APIUsageError(f'{kind}: at most {len(params)} positional args')
    vals = dict(params)
    vals.update(zip((n for n, _ in params), args or ()))
    for name, _ in params:
        if name in kwargs:
            vals[name] = kwargs.pop(name)
    return vals


def _int_in(kind, name, v, lo, hi):
    try:
        v = operator.index(v)
    except TypeError:
        raise APIUsageError(f'{kind}: {name} must be an integer, got {v!r}')
    if not lo <= v <= hi:
        raise APIUsageError(f'{kind}: {name} must be in [{lo}, {hi}] on the device, got {v}')
    return v


def _finite(kind, name, v):
    try:
        v = float(v)
    except (TypeError, ValueError):
        raise APIUsageError(f'{kind}: {name} must be a number, got {v!r}')
    if not math.isfinite(v):
        raise APIUsageError(f'{kind}: {name} must be finite, got {v}')
    return v


def resolve(creator, args, kwargs):
    """-> (kind name, iparam list of 8 ints) for pb_env_config."""
    kind, iparam, _ = resolve_config(creator, args, kwargs)
    return kind, iparam


def resolve_config(creator, args, kwargs):
    """-> (kind name, iparam list of 8 ints, dparam list of floats) for pb_env_create_ex."""
    kind = getattr(creator, 'b200_kind', None)
    if kind is None:
        kind = KNOWN_BY_NAME.get(getattr(creator, '__name__', ''), None)
    if kind is None:
        raise APIUsageError(
            f'env creator {creator!r} has no device-native kind: the B200 backend only runs '
            f'{sorted(set(KNOWN_BY_NAME.values()))} (no CPU fallback)')
    kwargs = dict(kwargs or {})
    iparam, dparam = [0] * 8, []
    if kind == 'squared':
        names = ('distance_to_target', 'num_targets')
        vals = dict(zip(names, args or ()))
        vals.update({k: kwargs.pop(k) for k in list(kwargs) if k in names})
        if vals.get('num_targets', 1) != 1:
            raise APIUsageError('squared: only num_targets=1 (the reference default) is implemented on the device')
        iparam[0] = int(vals.get('distance_to_target', 3))
    elif kind == 'breakout':
        iparam[0] = int(kwargs.pop('max_ticks', 0))
    elif kind == 'snake':
        iparam[0] = int(kwargs.pop('max_ticks', 0))
    elif kind == 'breakout_pixels':
        if args:
            raise APIUsageError(f'breakout_pixels: takes max_ticks as a keyword only, got args {list(args)}')
        if 'max_ticks' in kwargs:      # the tick counter is 16 bits of the packed state
            iparam[0] = _int_in(kind, 'max_ticks', kwargs.pop('max_ticks'), 1, 65535)
    elif kind == 'pong':
        iparam[0] = int(kwargs.pop('max_score', 0))
        iparam[1] = int(kwargs.pop('max_ticks', 0))
    elif kind == 'multiagent':
        if args or kwargs:      # make_multiagent() takes no arguments (ocean/environment.py:69-72)
            raise APIUsageError(f'multiagent: takes no arguments, got args {list(args or ())} kwargs {sorted(kwargs)}')
    elif kind in OCEAN_PARAMS:
        v = _ocean_values(kind, args, kwargs)
        if kind == 'memory':
            iparam[0] = _int_in(kind, 'mem_length', v['mem_length'], 1, 64)
            iparam[1] = _int_in(kind, 'mem_delay', v['mem_delay'], 0, 1024) + 1
        elif kind == 'password':
            iparam[0] = _int_in(kind, 'password_length', v['password_length'], 1, 128)
        elif kind == 'stochastic':
            dparam = [_finite(kind, 'p', v['p'])]       # horizon is accepted and ignored: make_stochastic passes 100
        else:
            iparam[0] = _int_in(kind, 'num_actions', v['num_actions'], 1, 1 << 15)
            dparam = [_finite(kind, 'reward_scale', v['reward_scale']), _finite(kind, 'reward_noise', v['reward_noise'])]
    if kwargs:
        raise APIUsageError(f'{kind}: unexpected env kwargs {sorted(kwargs)}')
    return kind, iparam, dparam


def _creator(kind):
    def make(*args, **kwargs):
        raise APIUsageError(
            f"'{kind}' is a device-native env: pass this creator to pufferlib_b200.vector.make(..., "
            f'backend=pufferlib_b200.vector.B200); it cannot be instantiated on the CPU')
    make.__name__ = 'make_' + kind
    make.b200_kind = kind
    return make
