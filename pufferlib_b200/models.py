"""Policies for the configs in BASELINE.json: PyTorch modules, dense GEMMs on cuBLAS/cuDNN (tensor cores).

Same architecture and call convention as the reference (adjacent to the hot path, not rewritten):
  Default        reference pufferlib/models.py:12-62   Linear(prod(obs)->hidden)+ReLU; heads hidden->n_act, ->1
  Convolutional  reference pufferlib/models.py:113-157 NatureCNN for (S,84,84) uint8, S = framestack (atari/torch.py:8-18)
  layer_init     reference pufferlib/pytorch.py:193-199
"""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional  # noqa: F401


class _DefaultMLPFunction(torch.autograd.Function):
    """models.Default as one autograd node on the device fast path.

    forward : hidden = relu(x @ W_enc^T + b_enc)  -- bias + ReLU fused into the cuBLASLt GEMM epilogue;
              out    = hidden @ W_cat^T + b_cat    -- both heads in ONE R-column GEMM (n_act logits, value, zero pad;
                                                      R = 8 for n_act <= 7, 16 for n_act <= 15, 32 for n_act <= 31:
                                                      Default.head_matrix).
    backward: pb_mlp_tail_backward_ex reads `hidden` once and produces dPre (heads dX + ReLU backward), dW_heads,
              db_heads and db_enc; the dense dW_enc = dPre^T @ x stays on cuBLAS tensor cores.  x (the observations) has
              no grad.
    """

    @staticmethod
    def forward(ctx, x, w_enc, b_enc, w_dec, b_dec, w_val, b_val, model):
        n_act, hid = w_dec.shape
        if x.dim() == 3:
            # slab form [G, R, F]: G equally spaced row slabs of the rollout buffer (a strided VIEW, see
            # Experience.flatten_batch_slabs) -- one GEMM per slab writes its part of the contiguous hidden layer,
            # the observations are never gathered into a minibatch copy
            g_, r_, _ = x.shape
            hidden = x.new_empty(g_ * r_, hid)
            for g in range(g_):
                torch._addmm_activation(b_enc, x[g], w_enc.t(), use_gelu=False, out=hidden[g * r_:(g + 1) * r_])
        else:
            try:
                hidden = torch._addmm_activation(b_enc, x, w_enc.t(), use_gelu=False)
            except (AttributeError, RuntimeError):
                hidden = torch.relu(torch.addmm(b_enc, x, w_enc.t()))
        # the head matrix of Default.head_matrix, cached only when no parameter records gradients
        # (torch.is_grad_enabled() is always False inside Function.forward: decide from the inputs that need gradients)
        w_cat, b_cat = model.head_matrix(cache=not any(ctx.needs_input_grad[1:7]))
        out = torch.addmm(b_cat, hidden, w_cat.t())
        ctx.save_for_backward(x, hidden, w_cat)
        ctx.n_act = n_act
        return out

    @staticmethod
    def backward(ctx, dout):
        from pufferlib_b200 import _native
        x, hidden, w_cat = ctx.saved_tensors
        n_act, (m, hid), rows = ctx.n_act, hidden.shape, w_cat.shape[0]
        dout = dout.contiguous()
        dpre = torch.empty_like(hidden)
        grads = torch.empty(rows * hid + hid + rows, dtype=torch.float32, device=x.device)
        lib = _native.lib()
        ws = torch.empty(lib.pb_mlp_tail_workspace_bytes_ex(m, hid, rows), dtype=torch.uint8, device=x.device)
        _native.check(lib.pb_mlp_tail_backward_ex(_native.ptr(dout), dout.stride(0), _native.ptr(w_cat),
                                                  _native.ptr(hidden), m, hid, _native.ptr(dpre), _native.ptr(grads),
                                                  _native.ptr(ws), ws.numel(), rows, _native.stream_ptr()))
        dw_cat = grads[:rows * hid].view(rows, hid)
        db_enc = grads[rows * hid:(rows + 1) * hid]
        db_cat = grads[(rows + 1) * hid:]
        # dW_enc = dPre^T @ x is one 128x128 output tile with K = M: as a batched GEMM over 64 K-slices (+ a 64-way sum)
        # gives the library GEMM enough parallel work at this shape (slab form: K-slices per slab)
        dw_enc = _gemm_tn(dpre, x)
        return (None, dw_enc, db_enc, dw_cat[:n_act], db_cat[:n_act], dw_cat[n_act:n_act + 1],
                db_cat[n_act:n_act + 1], None)


# hidden sizes the hand-written kernels are built for (pb_policy_mlp_sample, pb_mlp_tail_backward_ex): 128 * k, k <= 4
FAST_HIDDEN = (128, 256, 384, 512)
# LSTM sizes H (input size = hidden size = the inner Default's hidden size) of the fused recurrent kernels
# (pb_policy_lstm_sample, pb_lstm_bptt_*)
FUSED_LSTM_HIDDEN = (128, 256)


def _slab_split(g_, r_, split=64):
    """K-slices per slab in the slab form of _gemm_tn: split / G, halved until they divide R."""
    sp = max(1, split // g_)
    while r_ % sp:
        sp //= 2
    return sp


def _gemm_tn(a, b, split=64, out=None, part=None):
    """a^T @ b for a [M, Na], b [M, Nb] with unit column stride (row slices of wider rows are fine): a small output with
    K = M, so for large M a batched GEMM over `split` K-slices plus a sum gives the library GEMM enough parallel work.
    b may also be G equally strided row slabs [G, R, Nb] (a strided view of the rollout buffer) with a = [G*R, Na] in
    slab-major order: then the K-slices tile each slab (_slab_split), every slab's batched GEMM writes its partial
    products into one buffer (or `part`, [G * _slab_split(G, R, split), Na, Nb]) and one sum reduces them into `out`."""
    if b.dim() == 3:
        g_, r_, nb = b.shape
        sp = _slab_split(g_, r_, split)
        if part is None:
            part = b.new_empty(g_ * sp, a.shape[1], nb)
        for g in range(g_):
            torch.bmm(a[g * r_:(g + 1) * r_].view(sp, r_ // sp, a.shape[1]).transpose(1, 2), b[g].view(sp, r_ // sp, nb),
                      out=part[g * sp:(g + 1) * sp])
        return torch.sum(part, 0, out=out)
    m = a.shape[0]
    if m % split == 0 and m // split >= 256:
        return torch.bmm(a.view(split, m // split, -1).transpose(1, 2), b.view(split, m // split, -1)).sum(0)
    return a.t() @ b


class _LSTMBPTTFunction(torch.autograd.Function):
    """LSTMWrapper(models.Default) over a minibatch of bptt segments as one autograd node (the fused recurrent update).

    forward : pb_lstm_bptt_forward -- encoder, LSTM cell over the T steps and both heads; returns the packed head output
              out [B*T, R] (n_act logits | value | zero pad, rows b*T + t) and the final state (h_T, c_T) [B, H], and
              keeps the saved-activation rows [B*T, 8H] for the backward (H = 128 or 256: LSTMWrapper.fused_supported).
    backward: pb_lstm_bptt_backward -- dz (the gate pre-activations) and dPre (the encoder pre-activation) in reverse
              time; the weight gradients are library GEMMs on those buffers (_gemm_tn).  The observations and the initial
              state get no gradient; neither does the final state (train() hands it on detached).
    x is either the gathered minibatch [B, T, F] or the segment view [E, G, T, F] of Experience.segment_obs (segment
    b = e*G + g, read in place from the rollout buffer; pb_lstm_bptt_forward_rows / _backward_rows).  The segment view
    writes dPre in the order of its G observation slabs [G, T*E] so that dW_enc is the slab form of _gemm_tn; every
    other buffer, and the state, keep row order b*T + t."""

    @staticmethod
    def forward(ctx, x, h0, c0, ops, w_enc, b_enc, w_ih, w_hh, b_ih, b_hh, w_dec, b_dec, w_val, b_val):
        from pufferlib_b200 import _native
        w_enc_p, b_enc_p, w_gates, b_gates, w_cat, b_cat, w_gates_t = ops
        n_act, seg, hid = w_dec.shape[0], x.dim() == 4, w_hh.shape[1]
        bsz, steps, feats = (x.shape[0] * x.shape[1],) + tuple(x.shape[2:]) if seg else x.shape
        m = bsz * steps
        out = x.new_empty(m, w_cat.shape[0])
        h_out, c_out = x.new_empty(bsz, hid), x.new_empty(bsz, hid)
        saved = x.new_empty(m, 8 * hid)
        P, lib = _native.ptr, _native.lib()
        if seg:
            _native.check(lib.pb_lstm_bptt_forward_rows(
                P(x), feats, bsz, steps, x.shape[1], x.stride(0), x.stride(1), x.stride(2), P(h0), P(c0), P(w_enc_p),
                P(b_enc_p), P(w_gates), P(b_gates), P(w_cat), P(b_cat), hid, hid, n_act, P(out), P(h_out), P(c_out),
                P(saved), _native.stream_ptr()))
        else:
            _native.check(lib.pb_lstm_bptt_forward(
                P(x), x.stride(1), feats, bsz, steps, P(h0), P(c0), P(w_enc_p), P(b_enc_p), P(w_gates), P(b_gates),
                P(w_cat), P(b_cat), hid, hid, n_act, P(out), P(h_out), P(c_out), P(saved), _native.stream_ptr()))
        ctx.save_for_backward(x, c0, saved, w_gates_t, w_cat)
        ctx.n_act = n_act
        ctx.mark_non_differentiable(h_out, c_out)
        return out, h_out, c_out

    @staticmethod
    def backward(ctx, dout, _dh, _dc):
        from pufferlib_b200 import _native
        x, c0, saved, w_gates_t, w_cat = ctx.saved_tensors
        n_act, seg, hid = ctx.n_act, x.dim() == 4, saved.shape[1] // 8
        bsz, steps, feats = (x.shape[0] * x.shape[1],) + tuple(x.shape[2:]) if seg else x.shape
        m = bsz * steps
        dout = dout.contiguous()
        dz = x.new_empty(m, 4 * hid)
        dpre = x.new_empty(m, hid)
        P, lib = _native.ptr, _native.lib()
        if seg:       # dPre row (e, g, t) -> (g*T + t)*E + e: slab g holds the rows of observation slab g, (t, e) order
            e_, g_ = x.shape[:2]
            _native.check(lib.pb_lstm_bptt_backward_rows(
                P(dout), P(saved), P(c0), P(w_gates_t), P(w_cat), bsz, steps, hid, hid, n_act, g_, hid, hid * steps * e_,
                hid * e_, P(dz), P(dpre), _native.stream_ptr()))
            x_rows = x.permute(1, 2, 0, 3).view(g_, steps * e_, feats)     # [G, T*E, F] slabs, a view (forward_packed_seq)
        else:
            _native.check(lib.pb_lstm_bptt_backward(
                P(dout), P(saved), P(c0), P(w_gates_t), P(w_cat), bsz, steps, hid, hid, n_act, P(dz), P(dpre),
                _native.stream_ptr()))
            x_rows = x.reshape(m, feats)
        dw_gates = _gemm_tn(dz, saved[:, :2 * hid])        # dz^T [e | h_prev] = [dW_ih | dW_hh]
        db_gates = dz.sum(0)
        dw_enc = _gemm_tn(dpre, x_rows)
        dw_cat = _gemm_tn(dout, saved[:, 7 * hid:])         # dOut^T h
        db_cat = dout.sum(0)
        # b_ih and b_hh get the same gradient, as separate tensors (their .grad must not alias)
        return (None, None, None, None, dw_enc, dpre.sum(0), dw_gates[:, :hid], dw_gates[:, hid:], db_gates,
                db_gates.clone(), dw_cat[:n_act], db_cat[:n_act], dw_cat[n_act:n_act + 1], db_cat[n_act:n_act + 1])


def _round_tf32(w):
    """fp32 -> nearest TF32 value (ties away from zero: cvt.rna), kept as fp32 bits."""
    bits = w.detach().contiguous().view(torch.int32)
    return ((bits + 0x1000) & ~0x1FFF).view(torch.float32)


def layer_init(layer, std=np.sqrt(2), bias_const=0.0):
    torch.nn.init.orthogonal_(layer.weight, std)
    torch.nn.init.constant_(layer.bias, bias_const)
    return layer


class Default(nn.Module):
    def __init__(self, env, hidden_size=128):
        super().__init__()
        self.encoder = nn.Linear(int(np.prod(env.single_observation_space.shape)), hidden_size)
        self.decoder = layer_init(nn.Linear(hidden_size, env.single_action_space.n), std=0.01)
        self.value_head = nn.Linear(hidden_size, 1)
        self.fast_path = True     # fused forward epilogues + pb_mlp_tail_backward (CUDA, FAST_HIDDEN, <= 31 actions)
        self._head_cache = {}

    def invalidate_cache(self):
        """Call after the parameters changed (clean_pufferl does: optimizer post-step hook, start of evaluate, end of
        train)."""
        self._head_cache.clear()

    def head_matrix(self, cache=None):
        """(w_cat [R, H], b_cat [R]): n_act logit rows | value row | zero padding up to R = 8 rows for n_act <= 7, 16 for
        n_act <= 15, 32 for n_act <= 31 (the row counts the kernels are built for), the next multiple of 8 past that.
        Cached until invalidate_cache() when `cache` is true (default: under no_grad); built anew otherwise, since fused
        optimizers do not bump tensor._version and the cache cannot see an optimizer step."""
        if cache is None:
            cache = not torch.is_grad_enabled()
        key = (self.decoder.weight.data_ptr(), torch.cuda.is_current_stream_capturing())
        if cache and self._head_cache.get('key') == key:
            return self._head_cache['w'], self._head_cache['b']
        n_act, hid = self.decoder.weight.shape
        rows = next((r for r in (8, 16, 32) if n_act + 1 <= r), -(-(n_act + 1) // 8) * 8)
        with torch.no_grad():
            w_cat = self.decoder.weight.new_zeros(rows, hid)
            w_cat[:n_act] = self.decoder.weight
            w_cat[n_act] = self.value_head.weight[0]
            b_cat = self.decoder.weight.new_zeros(rows)
            b_cat[:n_act] = self.decoder.bias
            b_cat[n_act] = self.value_head.bias[0]
        if cache:
            self._head_cache.update(key=key, w=w_cat, b=b_cat)
        return w_cat, b_cat

    def encoder_weight_tf32(self):
        """The encoder weight rounded to TF32 (_round_tf32) for pb_policy_mlp_sample, which feeds the bits straight to
        the tensor cores; cached with the head matrix (same invalidation)."""
        cache = self._head_cache
        key = (self.encoder.weight.data_ptr(), torch.cuda.is_current_stream_capturing())
        if not torch.is_grad_enabled() and cache.get('ekey') == key:
            return cache['wenc']
        w = _round_tf32(self.encoder.weight)
        if not torch.is_grad_enabled():
            cache['ekey'], cache['wenc'] = key, w
        return w

    def _fast_ok(self, x):
        n_act, hid = self.decoder.weight.shape
        return self.fast_path and x.is_cuda and hid in FAST_HIDDEN and n_act + 1 <= 32 and not x.requires_grad

    def forward_packed(self, observations):
        """-> (out [M, R], n_act) with logits = out[:, :n_act], value = out[:, n_act] (zero padding after; R = 8 for
        n_act <= 7, 16 for n_act <= 15, 32 for n_act <= 31), or None when the fast path does not apply.  Lets the fused
        PPO loss hand back ONE [M, R] gradient."""
        x = observations.view(observations.shape[0], -1)
        if not self._fast_ok(x):
            return None
        out = _DefaultMLPFunction.apply(x.float().contiguous(), self.encoder.weight, self.encoder.bias,
                                        self.decoder.weight, self.decoder.bias, self.value_head.weight,
                                        self.value_head.bias, self)
        return out, self.decoder.weight.shape[0]

    def forward_packed_slabs(self, slabs):
        """forward_packed for a minibatch given as [G, R, features] row slabs (a strided view of the rollout
        observations; Experience.slab_obs): rows of the result are slab-major.  None when the fast path does not apply."""
        if slabs.dim() > 3:
            slabs = slabs.flatten(2)          # [G, R, *obs] -> [G, R, features] (a view: obs dims are contiguous)
        if slabs.dim() != 3 or not self._fast_ok(slabs) or slabs.stride(2) != 1 or slabs.stride(1) != slabs.shape[2]:
            return None
        out = _DefaultMLPFunction.apply(slabs.float(), self.encoder.weight, self.encoder.bias,
                                        self.decoder.weight, self.decoder.bias, self.value_head.weight,
                                        self.value_head.bias, self)
        return out, self.decoder.weight.shape[0]

    def forward(self, observations):
        packed = self.forward_packed(observations)
        if packed is not None:
            out, n_act = packed
            return out[:, :n_act], out[:, n_act:n_act + 1]
        hidden, lookup = self.encode_observations(observations)
        return self.decode_actions(hidden, lookup)

    def encode_observations(self, observations):
        batch_size = observations.shape[0]
        observations = observations.view(batch_size, -1)
        return torch.relu(self.encoder(observations.float())), None

    def decode_actions(self, hidden, lookup, concat=True):
        # both heads out of ONE GEMM (same parameters, same math as two nn.Linear calls): the value head is a
        # 1-column GEMV that would otherwise re-read `hidden`
        n_act = self.decoder.out_features
        pad = (-(n_act + 1)) % 8          # zero rows up to a multiple of 8 columns: keeps the aligned GEMM kernels
        w = torch.cat([self.decoder.weight, self.value_head.weight, hidden.new_zeros(pad, hidden.shape[1])], dim=0)
        b = torch.cat([self.decoder.bias, self.value_head.bias, hidden.new_zeros(pad)], dim=0)
        out = torch.nn.functional.linear(hidden, w, b)
        return out[:, :n_act], out[:, n_act:n_act + 1]


class LSTMWrapper(nn.Module):
    """Recurrent wrapper around a policy that defines encode_observations / decode_actions (reference:
    pufferlib/models.py:64-111): obs [B, *obs] or [B, T, *obs] -> encode -> nn.LSTM (cuDNN) over T -> decode.
    Returns (logits, value, state)."""

    def __init__(self, env, policy, input_size=128, hidden_size=128, num_layers=1):
        super().__init__()
        self.obs_shape = tuple(env.single_observation_space.shape)
        self.policy = policy
        self.input_size = input_size
        self.hidden_size = hidden_size
        self.recurrent = nn.LSTM(input_size, hidden_size, num_layers)
        for name, param in self.recurrent.named_parameters():
            if 'bias' in name:
                nn.init.constant_(param, 0)
            elif 'weight' in name:
                nn.init.orthogonal_(param, 1.0)
        self._fused_cache = {}

    def invalidate_cache(self):
        """Call after the parameters changed (clean_pufferl does: optimizer post-step hook, start of evaluate, end of
        train).  Clears the packed operands of fused_operands() and the inner policy's cache."""
        self._fused_cache.clear()
        if hasattr(self.policy, 'invalidate_cache'):
            self.policy.invalidate_cache()

    def fused_supported(self, x):
        """Can pb_policy_lstm_sample run this model on observations x?  One LSTM layer with bias, input size = hidden
        size = H with H in FUSED_LSTM_HIDDEN, a models.Default inner policy with an H-unit encoder and <= 15 actions,
        fp32 CUDA observations of <= 128 features."""
        rnn, inner = self.recurrent, self.policy
        H = rnn.hidden_size
        if not (isinstance(inner, Default) and rnn.num_layers == 1 and rnn.bias and H in FUSED_LSTM_HIDDEN
                and rnn.input_size == H and getattr(rnn, 'proj_size', 0) == 0):
            return False
        n_act, hid = inner.decoder.weight.shape
        feats = int(np.prod(self.obs_shape))
        return (tuple(inner.encoder.weight.shape) == (H, feats) and hid == H and n_act <= 15 and feats <= 128
                and x.is_cuda and x.dtype == torch.float32 and rnn.weight_ih_l0.dtype == torch.float32)

    def fused_operands(self):
        """The packed operands of pb_policy_lstm_sample (layouts in include/pufferlib_b200.h), for H = hidden size:
        (w_enc [H, 136] TF32, b_enc [H], w_gates [H/8 * 32, 2H + 8] TF32 in chunk order, b_gates [4H] = b_ih + b_hh
        in chunk order, w_cat [8 or 16, H], b_cat).  Cached under no_grad, keyed like Default.head_matrix."""
        cache = self._fused_cache
        rnn, inner = self.recurrent, self.policy
        key = (inner.encoder.weight.data_ptr(), rnn.weight_ih_l0.data_ptr(), rnn.weight_hh_l0.data_ptr(),
               inner.decoder.weight.data_ptr(), torch.cuda.is_current_stream_capturing())
        if not torch.is_grad_enabled() and cache.get('key') == key:
            return cache['ops']
        with torch.no_grad():
            w, H = inner.encoder.weight, rnn.hidden_size
            w_enc = w.new_zeros(H, 136)
            w_enc[:, :w.shape[1]] = _round_tf32(w)
            # chunk ch, row 8j + u <- gate j of unit 8ch + u = row Hj + 8ch + u of [W_ih | W_hh]
            dev = w.device
            order = (torch.arange(4, device=dev)[None, :, None] * H + torch.arange(H // 8, device=dev)[:, None, None] * 8
                     + torch.arange(8, device=dev)[None, None, :]).reshape(-1)
            w_gates = w.new_zeros(H // 8 * 32, 2 * H + 8)
            w_gates[:, :2 * H] = _round_tf32(torch.cat([rnn.weight_ih_l0, rnn.weight_hh_l0], dim=1)[order])
            b_gates = (rnn.bias_ih_l0 + rnn.bias_hh_l0)[order].contiguous()
            w_cat, b_cat = inner.head_matrix()
            ops = (w_enc, inner.encoder.bias.detach(), w_gates, b_gates, w_cat, b_cat)
        if not torch.is_grad_enabled():
            cache['key'], cache['ops'] = key, ops
        return ops

    def gate_weights_transposed(self):
        """The gate weights for the backward product of pb_lstm_bptt_backward: [H/8 * 2H, 40] TF32 (cvt.rna); chunk ch,
        row n, column 8j + u = row Hj + 8ch + u, column n of [W_ih | W_hh]; columns 32..39 zero.  Cached under
        no_grad, keyed like fused_operands."""
        cache = self._fused_cache
        rnn = self.recurrent
        key = (rnn.weight_ih_l0.data_ptr(), rnn.weight_hh_l0.data_ptr(), torch.cuda.is_current_stream_capturing())
        if not torch.is_grad_enabled() and cache.get('tkey') == key:
            return cache['wt']
        with torch.no_grad():
            H = rnn.hidden_size
            w = _round_tf32(torch.cat([rnn.weight_ih_l0, rnn.weight_hh_l0], dim=1))      # [4H, 2H]
            wt = w.new_zeros(H // 8, 2 * H, 40)
            # w.view(4, H/8, 8, 2H)[j, ch, u, n] = row Hj + 8ch + u -> [ch, n, 8j + u]
            wt[:, :, :32] = w.view(4, H // 8, 8, 2 * H).permute(1, 3, 0, 2).reshape(H // 8, 2 * H, 32)
            wt = wt.view(H // 8 * 2 * H, 40)
        if not torch.is_grad_enabled():
            cache['tkey'], cache['wt'] = key, wt
        return wt

    def forward_packed_seq(self, x, state=None):
        """The training forward over bptt segments on the fused kernels (pb_lstm_bptt_forward / _backward):
        x [B, T, *obs], or the strided segment view [E, G, T, *obs] of Experience.segment_obs with segment b = e*G + g
        (B = E*G; read in place, pb_lstm_bptt_forward_rows / _backward_rows); state (h, c) of shape [1, B, H] (detached)
        or None (zeros), H the hidden size.  -> (out [B*T, R], n_act, (h_T, c_T) [1, B, H]) with logits = out[:, :n_act],
        value = out[:, n_act], rows b*T + t in both cases; or None when the fast path does not apply (fused_supported
        fails, the inner Default's fast_path is off, or the layout is not one the kernel reads).  The packed operands are
        rebuilt on every call that records gradients."""
        nd = len(self.obs_shape)
        if x.dim() not in (nd + 2, nd + 3) or tuple(x.shape[x.dim() - nd:]) != self.obs_shape:
            return None
        if not (self.fused_supported(x) and getattr(self.policy, 'fast_path', False)):
            return None
        lead = x.shape[:x.dim() - nd]
        bsz, steps = int(np.prod(lead[:-1])), lead[-1]
        if bsz == 0:
            return None
        if len(lead) == 3:
            try:           # rows of equal stride in each of E, G, T; the [G, T*E] observation slabs of dW_enc are a view
                x3 = x.view(*lead, -1)
                x3.permute(1, 2, 0, 3).view(lead[1], steps * lead[0], -1)
            except RuntimeError:
                return None
            if x3.stride(3) != 1:
                return None
        else:
            x3 = x.reshape(bsz, steps, -1)
            if x3.stride(2) != 1 or x3.stride(0) != steps * x3.stride(1):
                return None                     # rows (b, t) must be equally spaced
        h0 = c0 = None
        if state is not None:
            h0, c0 = state
            for s in (h0, c0):
                if (tuple(s.shape) != (1, bsz, self.recurrent.hidden_size) or s.dtype != torch.float32 or s.device != x.device
                        or s.requires_grad):
                    return None
            h0, c0 = h0[0].contiguous(), c0[0].contiguous()
        inner, rnn = self.policy, self.recurrent
        ops = self.fused_operands() + (self.gate_weights_transposed(),)
        out, h, c = _LSTMBPTTFunction.apply(
            x3, h0, c0, ops, inner.encoder.weight, inner.encoder.bias, rnn.weight_ih_l0, rnn.weight_hh_l0,
            rnn.bias_ih_l0, rnn.bias_hh_l0, inner.decoder.weight, inner.decoder.bias, inner.value_head.weight,
            inner.value_head.bias)
        return out, inner.decoder.weight.shape[0], (h.unsqueeze(0), c.unsqueeze(0))

    def forward(self, x, state):
        nd = len(self.obs_shape)
        if tuple(x.shape[-nd:]) != self.obs_shape or x.dim() not in (nd + 1, nd + 2):
            raise ValueError('Invalid input tensor shape', x.shape)
        batch, steps = (x.shape[0], 1) if x.dim() == nd + 1 else (x.shape[0], x.shape[1])
        if state is not None:
            assert state[0].shape[1] == state[1].shape[1] == batch
        hidden, lookup = self.policy.encode_observations(x.reshape(batch * steps, *self.obs_shape))
        return self._recur(hidden, lookup, batch, steps, state)

    def forward_segments(self, x, state):
        """forward for the training minibatch read in place: x the segment view [E, G, T, *obs] of
        Experience.segment_obs (segment b = e*G + g, B = E*G segments of T steps), state (h, c) [1, B, H] or None.
        The inner policy's encode_segments reads the view (models.Convolutional: conv1's kernel on the frame stacks where
        they lie); the LSTM and the heads are those of forward.  -> (logits, value, state) with rows b*T + t, what
        forward gives for the gathered copy [B, T, *obs]; None when the inner policy cannot encode the view.  The view
        is never reshaped (that would copy the observations)."""
        nd = len(self.obs_shape)
        encode = getattr(self.policy, 'encode_segments', None)
        if encode is None or x.dim() != nd + 3 or tuple(x.shape[3:]) != self.obs_shape:
            return None
        batch, steps = x.shape[0] * x.shape[1], x.shape[2]
        if state is not None:
            assert state[0].shape[1] == state[1].shape[1] == batch
        hidden = encode(x)
        if hidden is None:
            return None
        return self._recur(hidden, None, batch, steps, state)

    def _recur(self, hidden, lookup, batch, steps, state):
        """The LSTM over hidden [B*T, input_size] (rows b*T + t) from state, then the inner policy's heads."""
        assert hidden.shape == (batch * steps, self.input_size)
        seq = hidden.reshape(batch, steps, self.input_size).transpose(0, 1)       # [T, B, F] for nn.LSTM
        seq, state = self.recurrent(seq, state)
        flat = seq.transpose(0, 1).reshape(batch * steps, self.hidden_size)
        logits, value = self.policy.decode_actions(flat, lookup)
        return logits, value, state


_CONV1_FRAME = 84 * 84     # bytes of one 84 x 84 uint8 frame; a frame stack of S frames is S of them
_CONV1_FRAMES = (1, 4)     # the frame-stack depths S conv1's kernels take (framestack=1 with an LSTM, 4 without)


class _Conv1U8Function(torch.autograd.Function):
    """relu(conv1(x / 255) + b) of NatureCNN (Conv2d(S, 32, 8, stride=4) on (S, 84, 84) uint8 frame stacks, S = 1 or
    4) as one autograd node: pb_conv1_u8_forward_ex reads the uint8 rows in place and writes y [M, 32, 20, 20]; the
    backward (pb_conv1_u8_wgrad_ex) takes the ReLU's gradient rule and the weight and bias gradients from y, dy and the
    same bytes.  x gets no gradient (conv1 is the first layer), so only y is saved beside it.
    x is either rows [M, S, 84, 84] or the segment view [E, G, T, S, 84, 84] of Experience.segment_obs (segment
    b = e*G + g; pb_conv1_u8_forward_rows_ex / _wgrad_rows_ex), whose y rows are b*T + t.  The view itself is saved, not
    a copy."""

    @staticmethod
    def _segments(x):
        """(batch, steps, groups, stride_e, stride_g, stride_t) of a segment view, in bytes.  A dimension of size 1 is
        never stepped over, so its stride is whatever torch reports; it is passed as one S-frame row, which the kernel
        accepts."""
        e_, g_, steps = x.shape[:3]
        row = x.shape[3] * _CONV1_FRAME
        st = [x.stride(i) if x.shape[i] > 1 else row for i in range(3)]
        return e_ * g_, steps, g_, st[0], st[1], st[2]

    @staticmethod
    def forward(ctx, x, w, b):
        from pufferlib_b200 import _native
        P, lib = _native.ptr, _native.lib()
        seg = x.dim() == 6
        m = x.shape[0] * x.shape[1] * x.shape[2] if seg else x.shape[0]
        frames = x.shape[-3]
        y = torch.empty(m, 32, 20, 20, dtype=torch.float32, device=x.device)
        if seg:
            _native.check(lib.pb_conv1_u8_forward_rows_ex(frames, P(x), *_Conv1U8Function._segments(x), P(w), P(b), P(y),
                                                          _native.stream_ptr()))
        else:
            _native.check(lib.pb_conv1_u8_forward_ex(frames, P(x), x.stride(0), m, P(w), P(b), P(y),
                                                     _native.stream_ptr()))
        ctx.save_for_backward(x, y)
        return y

    @staticmethod
    def backward(ctx, dy):
        from pufferlib_b200 import _native
        x, y = ctx.saved_tensors
        dy = dy.contiguous()
        m, lib, P = y.shape[0], _native.lib(), _native.ptr
        frames = x.shape[-3]
        dw = torch.empty(32, frames, 8, 8, dtype=torch.float32, device=x.device)
        db = torch.empty(32, dtype=torch.float32, device=x.device)
        ws = torch.empty(lib.pb_conv1_u8_wgrad_workspace_bytes(m), dtype=torch.uint8, device=x.device)
        if x.dim() == 6:
            _native.check(lib.pb_conv1_u8_wgrad_rows_ex(frames, P(x), *_Conv1U8Function._segments(x), P(y), P(dy), P(dw),
                                                        P(db), P(ws), ws.numel(), _native.stream_ptr()))
        else:
            _native.check(lib.pb_conv1_u8_wgrad_ex(frames, P(x), x.stride(0), m, P(y), P(dy), P(dw), P(db), P(ws),
                                                   ws.numel(), _native.stream_ptr()))
        return None, dw, db


class _ConvReLUTF32Function(torch.autograd.Function):
    """relu(conv(x, w) + b) of NatureCNN's conv2 (layer 2: Conv2d(32, 64, 4, stride=2) on [M, 32, 20, 20]) or conv3
    (layer 3: Conv2d(64, 64, 3, stride=1) on [M, 64, 9, 9]) as one autograd node on TF32 tensor cores
    (pb_nature_conv_forward).  The backward takes the ReLU's gradient rule from y and returns dx
    (pb_nature_conv_dgrad) and dw, db (pb_nature_conv_wgrad), each only when autograd asks for it.  x and y are saved:
    for conv2, x is conv1's y, which _Conv1U8Function keeps anyway."""

    SHAPES = {2: ((32, 20, 20), (64, 9, 9)), 3: ((64, 9, 9), (64, 7, 7))}

    @staticmethod
    def forward(ctx, x, w, b, layer):
        from pufferlib_b200 import _native
        m = x.shape[0]
        y = torch.empty(m, *_ConvReLUTF32Function.SHAPES[layer][1], dtype=torch.float32, device=x.device)
        _native.check(_native.lib().pb_nature_conv_forward(layer, _native.ptr(x), m, _native.ptr(w), _native.ptr(b),
                                                           _native.ptr(y), _native.stream_ptr()))
        ctx.layer = layer
        ctx.save_for_backward(x, w, y)
        return y

    @staticmethod
    def backward(ctx, dy):
        from pufferlib_b200 import _native
        x, w, y = ctx.saved_tensors
        dy = dy.contiguous()
        m, lib, layer, P = x.shape[0], _native.lib(), ctx.layer, _native.ptr
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty_like(x)
            _native.check(lib.pb_nature_conv_dgrad(layer, P(y), P(dy), P(w), m, P(dx), _native.stream_ptr()))
        if ctx.needs_input_grad[1] or ctx.needs_input_grad[2]:
            dw = torch.empty_like(w)
            db = torch.empty(w.shape[0], dtype=torch.float32, device=x.device)
            ws = torch.empty(lib.pb_nature_conv_wgrad_workspace_bytes(layer, m), dtype=torch.uint8, device=x.device)
            _native.check(lib.pb_nature_conv_wgrad(layer, P(x), P(y), P(dy), m, P(dw), P(db), P(ws), ws.numel(),
                                                   _native.stream_ptr()))
        return (dx, dw if ctx.needs_input_grad[1] else None, db if ctx.needs_input_grad[2] else None, None)


class Convolutional(nn.Module):
    def __init__(self, env, *args, framestack=4, flat_size=64 * 7 * 7, input_size=512, hidden_size=512,
                 output_size=512, channels_last=False, downsample=1, **kwargs):
        super().__init__()
        self.channels_last = channels_last
        self.downsample = downsample
        self.fast_path = True     # conv1 + ReLU on the uint8 frames in place (_Conv1U8Function) where _conv1_u8_ok holds,
                                  # then conv2, conv3 (_ConvReLUTF32Function) where _trunk_ok holds too
        self.network = nn.Sequential(
            layer_init(nn.Conv2d(framestack, 32, 8, stride=4)), nn.ReLU(),
            layer_init(nn.Conv2d(32, 64, 4, stride=2)), nn.ReLU(),
            layer_init(nn.Conv2d(64, 64, 3, stride=1)), nn.ReLU(),
            nn.Flatten(),
            layer_init(nn.Linear(flat_size, hidden_size)), nn.ReLU(),
        )
        self.actor = layer_init(nn.Linear(output_size, env.single_action_space.n), std=0.01)
        self.value_fn = layer_init(nn.Linear(output_size, 1), std=1)

    def forward(self, observations):
        hidden, lookup = self.encode_observations(observations)
        return self.decode_actions(hidden, lookup)

    def _conv1_u8_ok(self, x):
        """Can pb_conv1_u8_forward_ex run the first layer on x?  CUDA uint8 [M, S, 84, 84] with every row one contiguous
        frame stack (rows 16-byte aligned), channels-first frames at full resolution, and the stock
        Conv2d(S, 32, 8, stride=4) + ReLU with fp32 parameters first, S = framestack = 1 or 4."""
        return x.dim() == 4 and x.stride(0) % 16 == 0 and self._frames_ok(x)

    def _conv1_segments_ok(self, x):
        """The same for a segment view [E, G, T, S, 84, 84] (Experience.segment_obs) and pb_conv1_u8_forward_rows_ex:
        every frame stack contiguous, and each of E, G, T that is stepped over (size > 1) a multiple of 16 bytes and at
        least one frame stack (S * 7056 bytes) apart."""
        return (x.dim() == 6 and self._frames_ok(x)
                and all(x.stride(i) % 16 == 0 and x.stride(i) >= x.shape[3] * _CONV1_FRAME
                        for i in range(3) if x.shape[i] > 1))

    def _frames_ok(self, x):
        """_conv1_u8_ok's conditions on the trailing (S, 84, 84) dimensions of x, S = conv1's in_channels = 1 or 4, and
        on the module."""
        conv = self.network[0]
        if not (self.fast_path and not self.channels_last and self.downsample == 1 and x.is_cuda
                and x.dtype == torch.uint8 and x.dim() >= 3 and x.shape[-3] in _CONV1_FRAMES
                and tuple(x.shape[-2:]) == (84, 84) and tuple(x.stride()[-3:]) == (7056, 84, 1)
                and x.data_ptr() % 16 == 0):
            return False
        return (type(conv) is nn.Conv2d and type(self.network[1]) is nn.ReLU and conv.in_channels == x.shape[-3]
                and conv.out_channels == 32 and conv.kernel_size == (8, 8) and conv.stride == (4, 4)
                and conv.padding == (0, 0) and conv.dilation == (1, 1) and conv.groups == 1
                and conv.padding_mode == 'zeros' and conv.bias is not None
                and conv.weight.dtype == conv.bias.dtype == torch.float32 and conv.weight.is_contiguous()
                and conv.weight.data_ptr() % 16 == 0)

    def _trunk_ok(self):
        """Can _ConvReLUTF32Function run network[2:6] (after conv1 ran on the uint8 frames)?  Only where torch would let
        cuDNN run these convolutions in TF32 (torch.backends.cudnn.allow_tf32): with it off the user asked for fp32
        convolutions and gets them.  network[2:6] must be the stock Conv2d(32, 64, 4, stride=2), ReLU,
        Conv2d(64, 64, 3, stride=1), ReLU with bias, no padding, fp32 contiguous 16-byte aligned weights."""
        if not torch.backends.cudnn.allow_tf32:
            return False
        net = self.network
        if not (type(net[3]) is nn.ReLU and type(net[5]) is nn.ReLU):
            return False
        for conv, cin, ks, stride in ((net[2], 32, 4, 2), (net[4], 64, 3, 1)):
            if not (type(conv) is nn.Conv2d and conv.in_channels == cin and conv.out_channels == 64
                    and conv.kernel_size == (ks, ks) and conv.stride == (stride, stride) and conv.padding == (0, 0)
                    and conv.dilation == (1, 1) and conv.groups == 1 and conv.padding_mode == 'zeros'
                    and conv.bias is not None and conv.weight.dtype == conv.bias.dtype == torch.float32
                    and conv.weight.is_cuda and conv.weight.is_contiguous() and conv.bias.is_contiguous()
                    and conv.weight.data_ptr() % 16 == 0 and conv.bias.data_ptr() % 4 == 0):
                return False
        return True

    def encode_observations(self, observations):
        if self.channels_last:
            observations = observations.permute(0, 3, 1, 2)
        if self.downsample > 1:
            observations = observations[:, :, ::self.downsample, ::self.downsample]
        if observations.shape[0] > 0 and self._conv1_u8_ok(observations):
            conv = self.network[0]
            return self._after_conv1(_Conv1U8Function.apply(observations, conv.weight, conv.bias)), None
        return self.network(observations.float() / 255.0), None

    def encode_segments(self, view):
        """encode_observations for the bptt segments of a training minibatch read in place: the segment view
        [E, G, T, S, 84, 84] of Experience.segment_obs (segment b = e*G + g) -> hidden [E*G*T, 512] in row order b*T + t,
        what encode_observations gives for the gathered copy [E*G*T, S, 84, 84] of the same rows, bit for bit.  None when
        conv1's kernel cannot read the view (_conv1_segments_ok) or it is empty; the view is never reshaped (that would
        copy it)."""
        if view.dim() != 6 or view.numel() == 0 or not self._conv1_segments_ok(view):
            return None
        conv = self.network[0]
        return self._after_conv1(_Conv1U8Function.apply(view, conv.weight, conv.bias))

    def _after_conv1(self, y1):
        """network[2:] on conv1's output y1 [M, 32, 20, 20]: conv2 and conv3 on _ConvReLUTF32Function where _trunk_ok."""
        if self._trunk_ok():
            y2 = _ConvReLUTF32Function.apply(y1, self.network[2].weight, self.network[2].bias, 2)
            y3 = _ConvReLUTF32Function.apply(y2, self.network[4].weight, self.network[4].bias, 3)
            return self.network[6:](y3)
        return self.network[2:](y1)

    def decode_actions(self, flat_hidden, lookup, concat=None):
        return self.actor(flat_hidden), self.value_fn(flat_hidden)
