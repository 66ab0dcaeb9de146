"""NumPy restatements of the critic rollouts' GAE (include/mgb200.h "value heads and GAE"): the float32 recursion the
launch runs, bit for bit, and the float64 textbook GAE it approximates."""
import numpy as np


def gae_f32(rew, cut, truncated, value, value_last, final_value, gamma, lam):
    """(adv, ret) [T, N] float32 exactly as the kernel's epilogue computes them: every operation is one float32
    operation rounded to nearest (NumPy float32 scalar arithmetic never contracts), r_t is the reward rounded once to
    float32.  final_value is read only where cut & truncated."""
    f = np.float32
    rew = np.asarray(rew).astype(np.float32)
    cut = np.asarray(cut).astype(bool)
    truncated = np.asarray(truncated).astype(bool)
    value = np.asarray(value, np.float32)
    final_value = np.asarray(final_value, np.float32)
    T, N = value.shape
    g = f(gamma)
    gl = f(g * f(lam))
    adv = np.empty((T, N), np.float32)
    ret = np.empty((T, N), np.float32)
    nv_next = np.asarray(value_last, np.float32).copy()
    A = np.zeros(N, np.float32)
    zero = np.zeros(N, np.float32)
    for t in range(T - 1, -1, -1):
        nv = np.where(cut[t], np.where(truncated[t], final_value[t], zero), nv_next).astype(np.float32)
        delta = ((rew[t] + g * nv).astype(np.float32) - value[t]).astype(np.float32)
        A = (delta + np.where(cut[t], zero, (gl * A).astype(np.float32))).astype(np.float32)
        adv[t] = A
        ret[t] = (A + value[t]).astype(np.float32)
        nv_next = value[t]
    return adv, ret


def gae_f64(rew, cut, truncated, value, value_last, final_value, gamma, lam):
    """Textbook GAE in float64: delta_t = r_t + gamma V_next - V_t, A_t = delta_t + gamma lam A_{t+1}, with the
    recursion cut where the memory is wiped and V_next the terminal value of a truncated episode (0 when it ended)."""
    rew = np.asarray(rew, np.float64)
    value = np.asarray(value, np.float64)
    T, N = value.shape
    adv = np.zeros((T, N))
    nxt_v, nxt_a = np.asarray(value_last, np.float64), np.zeros(N)
    for t in range(T - 1, -1, -1):
        c = np.asarray(cut[t], bool)
        boot = np.where(np.asarray(truncated[t], bool), np.asarray(final_value[t], np.float64), 0.0)
        v_next = np.where(c, boot, nxt_v)
        delta = rew[t] + gamma * v_next - value[t]
        adv[t] = delta + np.where(c, 0.0, gamma * lam * nxt_a)
        nxt_v, nxt_a = value[t], adv[t]
    return adv, adv + value
