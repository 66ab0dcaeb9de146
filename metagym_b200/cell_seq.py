"""Masked-reset cell sequences (mgb_rnn_seq_forward / mgb_rnn_seq_backward; DESIGN.md "Fused unroll"): h_t of a GRU or
LSTM cell over T given steps of N envs, whose memory is zeroed after the steps where ``wipe`` is set, as a
differentiable torch op.  GRUPolicy.unroll and LSTMPolicy.unroll run their cell through it; only the recurrence runs in
the CUDA kernels, and everything batched over the T N rows (the input, the head, the weight gradients) stays in torch.
"""
import ctypes

import torch
from torch.autograd.function import once_differentiable

from . import _lib

CTA = _lib.RNN_SEQ_CTA_ENVS


def smem_bytes(gates, H, n_in):
    """(forward, backward) bytes of dynamic shared memory per CTA of a cell of `gates` gates (3: GRU, 4: LSTM), H units
    and n_in inputs: the forward's staged cell (units rounded up to 8) and columns x, c, h, h; the backward's weight_hh,
    rows padded to 16, 32 or 64 floats, and two H columns."""
    Hp = -(-H // 8) * 8
    C = H if gates == 4 else 0
    fwd = 4 * (gates * Hp * (n_in + H) + 2 * gates * Hp + (n_in + C + 2 * H) * CTA)
    HA = 16 if H <= 16 else 32 if H <= 32 else 64
    return fwd, 4 * (gates * H * HA + 2 * H * CTA)


def fits(cell):
    """True when the kernels run `cell`: float32 parameters on a CUDA device whose opt-in shared memory holds both
    footprints.  Anything else unrolls through the torch loop."""
    w = cell.weight_ih
    if w.dtype != torch.float32 or w.device.type != "cuda":
        return False
    gates = w.shape[0] // cell.hidden_size
    optin = torch.cuda.get_device_properties(w.device).shared_memory_per_block_optin
    return max(smem_bytes(gates, cell.hidden_size, cell.input_size)) <= optin


def _packed(w_ih, w_hh, b_ih, b_hh):
    """The cell part of the packed buffer from the live parameters: weight_ih, weight_hh, bias_ih, bias_hh."""
    G = w_ih.shape[0]
    zeros = w_ih.new_zeros(G)
    return torch.cat([w_ih.reshape(-1), w_hh.reshape(-1), zeros if b_ih is None else b_ih,
                      zeros if b_hh is None else b_hh])


def _call(fn, seq, device):
    with torch.cuda.device(device):
        _lib.check(fn(ctypes.byref(seq), _lib.current_stream(torch, device)))


def _struct(code, H, params, X, wipe, state0, h, gates=None):
    T, n_in, N = X.shape
    return _lib.RnnSeq(code, H, n_in, T, N, params.data_ptr(), X.data_ptr(), wipe.data_ptr(), state0.data_ptr(),
                       h.data_ptr(), _lib.ptr(gates), None, None, None, None)


def forward(code, H, params, X, wipe, state0, save=False):
    """h [T, N, H] (and the saved gates [T, S, H, N] with save) of the cell packed in `params` on X [T, in, N], wipe
    [T, N] bool and state0 [N, HC]: mgb_rnn_seq_forward.  No autograd."""
    T, _, N = X.shape
    h = torch.empty((T, N, H), dtype=torch.float32, device=X.device)
    gates = None
    if save:
        S = 4 if code == _lib.RNN_CELL_GRU else 5
        gates = torch.empty((T, S, H, N), dtype=torch.float32, device=X.device)
    _call(_lib.load().mgb_rnn_seq_forward, _struct(code, H, params, X, wipe, state0, h, gates), X.device)
    return h, gates


def previous_h(h, wipe, h0):
    """[T, N, H]: the h each step read, h0 [N, H] at t = 0, then h_{t-1} [N, H], zeros where wipe[t-1]."""
    hprev = torch.cat([h0[None], h[:-1]], 0)
    if h.shape[0] > 1:
        hprev[1:].masked_fill_(wipe[:-1, :, None], 0.)
    return hprev


class CellSequence(torch.autograd.Function):
    """h = CellSequence.apply(code, H, X, wipe, state0, weight_ih, weight_hh, bias_ih, bias_hh): the cell over T steps
    with gradients to state0 [N, HC] and the four parameters (bias None for a cell without bias).  X and wipe are data:
    they get no gradient."""

    @staticmethod
    def forward(ctx, code, H, X, wipe, state0, w_ih, w_hh, b_ih, b_hh):
        params = _packed(w_ih, w_hh, b_ih, b_hh)
        state0 = state0.contiguous()
        h, gates = forward(code, H, params, X, wipe, state0, save=True)
        ctx.save_for_backward(X, wipe, state0, params, h, gates)
        ctx.code, ctx.H = code, H
        ctx.bias = (b_ih is not None, b_hh is not None)
        return h

    @staticmethod
    @once_differentiable
    def backward(ctx, dh):
        X, wipe, state0, params, h, gates = ctx.saved_tensors
        code, H = ctx.code, ctx.H
        gru = code == _lib.RNN_CELL_GRU
        T, n_in, N = X.shape
        GH = (3 if gru else 4) * H
        dgi = torch.empty((T, GH, N), dtype=torch.float32, device=X.device)
        dghn = torch.empty((T, H, N), dtype=torch.float32, device=X.device) if gru else None
        dstate0 = torch.empty_like(state0)
        dh = dh.contiguous()
        seq = _struct(code, H, params, X, wipe, state0, h, gates)
        seq.dh_dev, seq.dgi_dev, seq.dghn_dev, seq.dstate0_dev = (dh.data_ptr(), dgi.data_ptr(), _lib.ptr(dghn),
                                                                  dstate0.data_ptr())
        _call(_lib.load().mgb_rnn_seq_backward, seq, X.device)
        hprev = previous_h(h, wipe, state0[:, :H])
        dW_ih = torch.matmul(dgi, X.transpose(1, 2)).sum(0)
        db_ih = dgi.sum((0, 2))
        if gru:
            dW_hh = torch.cat([torch.matmul(dgi[:, :2 * H], hprev).sum(0), torch.matmul(dghn, hprev).sum(0)])
            db_hh = torch.cat([db_ih[:2 * H], dghn.sum((0, 2))])
        else:
            dW_hh = torch.matmul(dgi, hprev).sum(0)
            db_hh = db_ih
        return (None, None, None, None, dstate0 if ctx.needs_input_grad[4] else None, dW_ih, dW_hh,
                db_ih if ctx.bias[0] else None, db_hh if ctx.bias[1] else None)


def run(cell, code, X, wipe, state0):
    """h [T, N, H] of `cell` (an nn.GRUCell or nn.LSTMCell of code MGB_RNN_CELL_*) over X [T, in, N] float32, wipe
    [T, N] bool and state0 [N, HC]: through CellSequence when autograd has something to reach, else one forward launch
    that saves nothing."""
    H = cell.hidden_size
    args = (cell.weight_ih, cell.weight_hh, cell.bias_ih, cell.bias_hh)
    if torch.is_grad_enabled() and (state0.requires_grad or any(p is not None and p.requires_grad for p in args)):
        return CellSequence.apply(code, H, X, wipe, state0, *args)
    with torch.no_grad():
        return forward(code, H, _packed(*args), X, wipe, state0.contiguous())[0]
