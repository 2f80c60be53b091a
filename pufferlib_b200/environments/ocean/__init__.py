"""Mirror of pufferlib.environments.ocean (reference: ocean/environment.py:6-26): ``env_creator(name)``.

memory, password, stochastic, bandit and multiagent are the reference's ocean test envs (multiagent has two agents
per env, so its vecenv has 2 * num_envs agent rows); spaces, performance and performance_empiric have no device
form."""
from pufferlib_b200.environments import _creator

make_squared = _creator('squared')
make_breakout = _creator('breakout')
make_snake = _creator('snake')
make_pong = _creator('pong')
make_memory = _creator('memory')
make_password = _creator('password')
make_stochastic = _creator('stochastic')
make_bandit = _creator('bandit')
make_multiagent = _creator('multiagent')

_CREATORS = {'squared': make_squared, 'breakout': make_breakout, 'snake': make_snake, 'pong': make_pong,
             'memory': make_memory, 'password': make_password, 'stochastic': make_stochastic, 'bandit': make_bandit,
             'multiagent': make_multiagent}


def env_creator(name='squared'):
    try:
        return _CREATORS[name]
    except KeyError:
        raise ValueError('Invalid environment name')
