"""Which update path train() takes, and what it computes, across the minibatch forms and update engines:

    python tests/experimental/check_train_paths.py --out DIR [--repo ROOT] [--only NAME ...]
    python tests/experimental/check_train_paths.py --compare DIR_A DIR_B

For every configuration below the trainer is built from fixed seeds and `evaluate(); train()` runs three times.  Each
train() records the minibatch form (data.train_minibatch_path), the recurrent path, whether the hand-written update ran
and on the fused kernel, the train graph state, the project kernels launched from Python during the call
(pb_launch_count), those a captured update graph holds and the epochs run.  The final parameters, Adam moments and losses go to
DIR/<name>.npz, the records to DIR/records.json.  --repo imports pufferlib_b200 from another checkout, so two versions
can be run on the same machine and compared.

--compare: the records must be identical; the parameter, moment and loss differences are printed per configuration (the
single-pass GAE composes its tile aggregates in a timing-dependent order, so two runs of the same code can differ in the
last bits of fp32 sums: compare against the spread of two runs of one version)."""
import argparse
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))


def config(env, n, h, **kw):
    import pufferlib_b200
    cfg = dict(seed=1, torch_deterministic=True, env=env, batch_size=n * h, bptt_horizon=16, minibatch_size=n * h // 4,
               cpu_offload=False, device='cuda', compile=False, learning_rate=2.5e-4, gamma=0.99, gae_lambda=0.95,
               update_epochs=2, norm_adv=True, clip_coef=0.1, clip_vloss=True, vf_clip_coef=0.1, vf_coef=0.5,
               ent_coef=0.01, max_grad_norm=0.5, target_kl=None, anneal_lr=False, total_timesteps=10 ** 9)
    cfg.update(kw)
    return pufferlib_b200.namespace(**cfg)


# name -> (env, num_envs, horizon, policy kind, policy options, config overrides)
CASES = {
    'direct': ('breakout', 64, 128, 'mlp', {}, {}),
    'direct_graph': ('breakout', 64, 128, 'mlp', {}, dict(cuda_graph=True)),
    'slabs_kernel_chain': ('breakout', 64, 128, 'mlp', {}, dict(fused_update=False)),
    'snake_uint8_chain': ('snake', 64, 64, 'mlp', dict(fused_sample=False), {}),
    'autograd_slabs': ('breakout', 64, 128, 'mlp', {}, dict(manual_update=False)),
    'gathered': ('breakout', 64, 128, 'mlp', {}, dict(zero_copy_minibatches=False)),
    'reference_loss': ('breakout', 64, 128, 'mlp', {}, dict(fused_loss=False)),
    'no_slab_layout': ('breakout', 64, 48, 'mlp', {}, dict(minibatch_size=64 * 48 // 2)),     # h / bptt = 3, 2 minibatches
    'target_kl': ('breakout', 64, 128, 'mlp', {}, dict(target_kl=0.02)),
    'raw_advantages_direct': ('breakout', 64, 128, 'mlp', {}, dict(norm_adv=False)),
    'pong_conv': ('pong', 64, 32, 'conv', {}, dict(bptt_horizon=8, minibatch_size=64 * 32 // 2)),
    'lstm_segments': ('breakout', 256, 64, 'lstm', {}, dict(minibatch_size=256 * 64 // 2)),
    'lstm_segments_graph': ('breakout', 256, 64, 'lstm', {}, dict(minibatch_size=256 * 64 // 2, cuda_graph=True)),
    'lstm_gathered': ('breakout', 256, 64, 'lstm', {}, dict(minibatch_size=256 * 64 // 2, zero_copy_minibatches=False)),
    'lstm_cudnn_hidden64': ('squared', 64, 16, 'lstm', dict(fused_update=False, hidden=64),
                            dict(bptt_horizon=8, minibatch_size=64 * 16 // 2)),
    'fast_path_off_slabs': ('breakout', 64, 128, 'mlp', dict(fast_path=False), {}),    # model(obs) + fused_ppo_loss
    'squared_heads16_graph': ('squared', 64, 64, 'mlp', {}, dict(cuda_graph=True)),      # Discrete(8): 16-row chain
    'lstm_cudnn_graph': ('squared', 64, 16, 'lstm', dict(fused_update=False, hidden=64),
                         dict(bptt_horizon=8, minibatch_size=64 * 16 // 2, cuda_graph=True)),
    # LSTMWrapper(Convolutional, 512, 512), the Atari LSTM policy: the 'cudnn_conv' engine on segment views
    'conv_lstm': ('pong', 64, 32, 'conv_lstm', {}, dict(bptt_horizon=8, minibatch_size=64 * 32 // 2)),
    'conv_lstm_graph': ('pong', 64, 32, 'conv_lstm', {}, dict(bptt_horizon=8, minibatch_size=64 * 32 // 2, cuda_graph=True)),
    # target_kl on the autograd engines; 1e-6 stops after the first epoch
    'lstm_target_kl': ('breakout', 256, 64, 'lstm', {}, dict(minibatch_size=256 * 64 // 2, target_kl=0.02)),
    'lstm_target_kl_stop_graph': ('breakout', 256, 64, 'lstm', {},
                                  dict(minibatch_size=256 * 64 // 2, target_kl=1e-6, cuda_graph=True)),
    'autograd_target_kl': ('breakout', 64, 128, 'mlp', {}, dict(manual_update=False, target_kl=0.02)),
    'autograd_target_kl_stop_graph': ('breakout', 64, 128, 'mlp', {},
                                      dict(manual_update=False, target_kl=1e-6, cuda_graph=True)),
    'target_kl_stop_graph': ('breakout', 64, 128, 'mlp', {}, dict(target_kl=1e-6, cuda_graph=True)),
}


def build(env, n, h, kind, pol_kw, cfg_kw):
    import torch
    import pufferlib_b200.vector as pvec
    from pufferlib_b200 import clean_pufferl, models
    from pufferlib_b200.environments import ocean
    from pufferlib_b200.frameworks import cleanrl
    vec = pvec.make(ocean.env_creator(env), num_envs=n, backend=pvec.B200)
    torch.manual_seed(0)
    if kind == 'conv_lstm':             # as tests/test_gpu_conv_lstm.py builds it
        net = models.LSTMWrapper(vec.driver_env, models.Convolutional(vec.driver_env), input_size=512, hidden_size=512)
        pol = cleanrl.RecurrentPolicy(net, seed=3)
    elif kind == 'lstm':
        hid = pol_kw.get('hidden', 128)
        net = models.LSTMWrapper(vec.driver_env, models.Default(vec.driver_env, hidden_size=hid), input_size=hid,
                                 hidden_size=hid)
        pol = cleanrl.RecurrentPolicy(net, fused_sample=True, seed=3, fused_update=pol_kw.get('fused_update', True))
    else:
        net = models.Convolutional(vec.driver_env) if kind == 'conv' else models.Default(vec.driver_env)
        if 'fast_path' in pol_kw:
            net.fast_path = pol_kw['fast_path']
        pol = cleanrl.Policy(net, fused_sample=pol_kw.get('fused_sample', kind == 'mlp'), seed=7)
    return clean_pufferl.create(config(env, n, h, **cfg_kw), vec, pol.cuda())


def run_case(name, out_dir):
    import torch
    from pufferlib_b200 import _native, clean_pufferl
    data = build(*CASES[name])
    lib, records = _native.lib(), []
    for _ in range(3):
        clean_pufferl.evaluate(data)
        torch.cuda.synchronize()
        l0 = lib.pb_launch_count()
        clean_pufferl.train(data)
        torch.cuda.synchronize()
        mu = data.manual_update
        records.append(dict(
            minibatch_path=data.train_minibatch_path, recurrent_path=data.train_recurrent_path,
            manual_update=mu is not None, used_fused=bool(mu.used_fused) if mu is not None else None,
            train_graph_state=data.train_graph_state, launches_from_python=int(lib.pb_launch_count() - l0),
            graph_launches=int(data.train_graph_launches), epochs_run=data.train_epochs_run))
    arrays = {f'param/{k}': v.detach().float().cpu().numpy() for k, v in data.policy.state_dict().items()}
    names = {id(p): k for k, p in data.policy.named_parameters()}
    for p, st in data.optimizer.state.items():
        for k in ('exp_avg', 'exp_avg_sq', 'step'):
            arrays[f'adam/{names[id(p)]}/{k}'] = st[k].detach().float().cpu().numpy()
    arrays['losses'] = np.array([getattr(data.losses, k) for k in ('policy_loss', 'value_loss', 'entropy', 'old_approx_kl',
                                                                   'approx_kl', 'clipfrac', 'explained_variance')])
    np.savez(os.path.join(out_dir, name + '.npz'), **arrays)
    clean_pufferl.close(data)
    return records


def compare(a, b):
    ra, rb = (json.load(open(os.path.join(d, 'records.json'))) for d in (a, b))
    same = True
    worst = {'param': 0.0, 'adam': 0.0, 'losses': 0.0}
    for name in sorted(set(ra) | set(rb)):
        if ra.get(name) != rb.get(name):
            same = False
            print(f'{name}: RECORDS DIFFER\n  {ra.get(name)}\n  {rb.get(name)}')
            continue
        za, zb = (np.load(os.path.join(d, name + '.npz')) for d in (a, b))
        diff = {'param': 0.0, 'adam': 0.0, 'losses': 0.0}
        for k in za.files:
            d = float(np.nanmax(np.abs(za[k].astype(np.float64) - zb[k].astype(np.float64)), initial=0.0))
            diff[k.split('/')[0]] = max(diff[k.split('/')[0]], d)
        for k in worst:
            worst[k] = max(worst[k], diff[k])
        paths = [(r['minibatch_path'], r['recurrent_path'], r['manual_update'], r['used_fused'], r['train_graph_state'],
                  r['launches_from_python'], r['graph_launches'], r['epochs_run']) for r in ra[name]]
        print(f'{name}: records identical {paths}; max |diff| param {diff["param"]:.3e} adam {diff["adam"]:.3e} '
              f'losses {diff["losses"]:.3e}')
    print(json.dumps({'records_identical': same, 'max_abs_diff': worst}))
    return same


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out')
    ap.add_argument('--repo', default=os.path.dirname(os.path.dirname(HERE)))
    ap.add_argument('--only', nargs='*', default=None)
    ap.add_argument('--compare', nargs=2, metavar=('DIR_A', 'DIR_B'))
    args = ap.parse_args()
    if args.compare:
        sys.exit(0 if compare(*args.compare) else 1)
    sys.path.insert(0, os.path.abspath(args.repo))
    import torch
    import pufferlib_b200
    assert os.path.dirname(os.path.dirname(os.path.abspath(pufferlib_b200.__file__))) == os.path.abspath(args.repo)
    torch.cuda.set_device(0)
    os.makedirs(args.out, exist_ok=True)
    records = {}
    for name in args.only or CASES:
        records[name] = run_case(name, args.out)
        print(name, records[name], flush=True)
    json.dump(records, open(os.path.join(args.out, 'records.json'), 'w'), indent=1)


if __name__ == '__main__':
    main()
