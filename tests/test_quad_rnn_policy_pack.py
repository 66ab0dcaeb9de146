"""CPU: GRUPolicy and LSTMPolicy with dist="gaussian" pack a cell and a Gaussian head into the layout the recurrent
quadrotor rollout reads (include/mgb200.h, mgb_quad_rollout_rnn): the cell, the head with its optional value row, then
log_std [4].  They refuse what that rollout cannot run, the maze refuses them and the quadrotor refuses categorical
ones, and unroll() recomputes a rollout's means and log-probabilities with the raw-action feedback, with gradients
reaching log_std."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
nn = torch.nn

D = 19      # velocity_control


def make_head(H, width, act=nn.Tanh):
    if not width:
        return nn.Linear(H, 4)
    return nn.Sequential(nn.Linear(H, width), act(), nn.Linear(width, 4))


def head_linears(head):
    return [head] if isinstance(head, nn.Linear) else [m for m in head if isinstance(m, nn.Linear)]


def hand_packed(cell, head, value, log_std, mean=None, std=None):
    """The packed buffer from the header's list: weight_ih (obs columns divided by std), weight_hh, bias_ih (minus
    W_obs mean / std), bias_hh, each head layer's W and b with the value row appended to the last, then log_std."""
    f = lambda t: t.detach().double().numpy()                   # noqa: E731
    Wi, bi = f(cell.weight_ih).copy(), f(cell.bias_ih).copy()
    if mean is not None:
        bi = bi - Wi[:, :D] @ (mean / std)
        Wi[:, :D] = Wi[:, :D] / std
    parts = [Wi.ravel(), f(cell.weight_hh).ravel(), bi, f(cell.bias_hh)]
    lins = head_linears(head)
    for k, m in enumerate(lins):
        W, b = f(m.weight), f(m.bias)
        if k == len(lins) - 1 and value is not None:
            W, b = np.concatenate([W, f(value.weight)]), np.concatenate([b, f(value.bias)])
        parts += [W.ravel(), b]
    parts.append(np.zeros(4) if log_std is None else np.asarray(log_std, np.float64))
    return np.concatenate(parts).astype(np.float32)


def policy_classes():
    from metagym_b200.policy import GRUPolicy, LSTMPolicy
    return {"gru": (GRUPolicy, nn.GRUCell, 3), "lstm": (LSTMPolicy, nn.LSTMCell, 4)}


@pytest.mark.parametrize("kind", ["gru", "lstm"])
@pytest.mark.parametrize("width", [0, 16])
@pytest.mark.parametrize("value", [False, True], ids=["actor", "critic"])
@pytest.mark.parametrize("norm", [False, True], ids=["raw", "normalised"])
def test_gaussian_pack_layout(kind, width, value, norm):
    Pol, Cell, gates = policy_classes()[kind]
    torch.manual_seed(3)
    H = 24
    cell, head = Cell(D + 5, H), make_head(H, width)
    vh = nn.Linear(width or H, 1) if value else None
    ls = torch.tensor([-0.5, -0.25, 0.0, 0.25])
    mean, std = (np.linspace(-1, 1, D), np.linspace(0.5, 2.0, D)) if norm else (None, None)
    pol = Pol(cell, head, log_std=ls, dist="gaussian", device="cpu", value=vh, obs_mean=mean, obs_std=std)
    want = hand_packed(cell, head, vh, ls.numpy(), mean, std)
    assert pol.numel == want.size
    assert np.array_equal(pol.params.numpy(), want)
    assert np.array_equal(pol.params.numpy()[-4:], ls.numpy())
    assert pol.has_log_std and pol.dist == "gaussian" and pol.obs_dim == D
    assert pol.state_dim == (gates - 2) * H + 5          # H + 5 (GRU) or 2H + 5 (LSTM): the categorical layout's
    s = pol.struct()
    assert (s.hidden, s.feedback, s.reset, s.head_hidden, s.head_width) == (H, 1, 0, int(width > 0), width)
    # without log_std the buffer still ends with four zeros, and only deterministic rollouts may use it
    p0 = Pol(cell, head, dist="gaussian", device="cpu", value=vh, obs_mean=mean, obs_std=std)
    assert not p0.has_log_std and p0.numel == pol.numel and not p0.params[-4:].any()
    assert np.array_equal(p0.params.numpy()[:-4], want[:-4])
    # the categorical policy of the same modules is this buffer without log_std
    pc = Pol(cell, head, device="cpu", value=vh, obs_mean=mean, obs_std=std)
    assert pc.numel == pol.numel - 4 and np.array_equal(pc.params.numpy(), want[:-4])


@pytest.mark.parametrize("kind", ["gru", "lstm"])
def test_update_log_std_in_place(kind):
    Pol, Cell, _ = policy_classes()[kind]
    torch.manual_seed(4)
    pol = Pol(Cell(D + 5, 8), make_head(8, 0), dist="gaussian", device="cpu")
    buf = pol.params
    ls = torch.tensor([0.1, 0.2, 0.3, 0.4])
    pol.update(log_std=ls)
    assert pol.params is buf and pol.has_log_std
    assert np.array_equal(buf.numpy()[-4:], ls.numpy())
    before = buf.clone()
    pol.update(Cell(D + 5, 8))
    assert pol.params is buf and np.array_equal(buf.numpy()[-4:], ls.numpy())
    assert not torch.equal(buf[:-4], before[:-4])
    with pytest.raises(ValueError):
        pol.update(log_std=torch.zeros(3))
    assert np.array_equal(buf.numpy()[-4:], ls.numpy())


def test_refusals():
    from metagym_b200.policy import GRUPolicy, LSTMPolicy, PolicyPopulation
    H = 8
    bad = [
        lambda: GRUPolicy(nn.GRUCell(D + 5, H), make_head(H, 0), dist="beta", device="cpu"),
        lambda: GRUPolicy(nn.GRUCell(D + 5, H), make_head(H, 0), dist="gaussian", hidden_reset="task", device="cpu"),
        lambda: LSTMPolicy(nn.LSTMCell(D + 5, H), make_head(H, 0), dist="gaussian", hidden_reset="task", device="cpu"),
        lambda: GRUPolicy(nn.GRUCell(D + 5, H), make_head(H, 0), log_std=torch.zeros(3), dist="gaussian",
                          device="cpu"),
    ]
    for k, make in enumerate(bad):
        with pytest.raises(ValueError):
            make()
            print("not refused: case %d" % k)
    with pytest.raises(TypeError):          # as before: a categorical LSTMPolicy takes no log_std
        LSTMPolicy(nn.LSTMCell(D + 5, H), make_head(H, 0), log_std=torch.zeros(4), device="cpu")
    cat = GRUPolicy(nn.GRUCell(D + 5, H), make_head(H, 0), device="cpu")
    with pytest.raises(ValueError):
        cat.update(log_std=torch.zeros(4))
    # a population keeps one distribution and one log_std presence
    g = GRUPolicy(nn.GRUCell(D + 5, H), make_head(H, 0), log_std=torch.zeros(4), dist="gaussian", device="cpu")
    g0 = GRUPolicy(nn.GRUCell(D + 5, H), make_head(H, 0), dist="gaussian", device="cpu")
    c = GRUPolicy(nn.GRUCell(D + 5, H), make_head(H, 0), device="cpu")
    for members in ([g, c], [g, g0]):
        with pytest.raises(ValueError):
            PolicyPopulation(members)
    assert PolicyPopulation([g, GRUPolicy(nn.GRUCell(D + 5, H), make_head(H, 0), log_std=torch.ones(4),
                                          dist="gaussian", device="cpu")]).dist == "gaussian"


class _FakeEnv(object):
    """The attributes the rollouts read before they reach the device: the cross-env refusals come first."""
    num_envs, obs_dim, need_reset, _torch, device = 64, D, False, torch, torch.device("cpu")


def test_cross_env_refusals():
    from metagym_b200.metamaze import BatchedMetaMaze2D
    from metagym_b200.policy import GRUPolicy, LSTMPolicy, PolicyPopulation
    from metagym_b200.quadrotor import BatchedQuadrotor
    H = 8
    gauss = LSTMPolicy(nn.LSTMCell(D + 5, H), make_head(H, 0), dist="gaussian", device="cpu")
    cat = GRUPolicy(nn.GRUCell(D + 5, H), make_head(H, 0), device="cpu")
    env = _FakeEnv()
    for p in (gauss, PolicyPopulation.from_template(gauss, 2)):
        with pytest.raises(ValueError, match="Gaussian"):
            BatchedMetaMaze2D.rollout(env, 4, policy=p, state=torch.zeros(64, p.state_dim))
    for p in (cat, PolicyPopulation.from_template(cat, 2)):
        with pytest.raises(ValueError, match="categorical"):
            BatchedQuadrotor.rollout(env, 4, policy=p, state=torch.zeros(64, p.state_dim))
    with pytest.raises(ValueError, match="carried state"):
        BatchedQuadrotor.rollout(env, 4, policy=gauss)


def fake_rollout(T, N, S, seed):
    g = torch.Generator().manual_seed(seed)
    done = (torch.rand((T, N), generator=g) < 0.2).to(torch.uint8)
    done[T // 2, :] = 1                                     # every env resets mid-chunk
    return {"obs0": torch.randn((N, D), generator=g),
            "obs": torch.randn((T, N, D), generator=g),
            "act": torch.randn((T, N, 4), generator=g) * 3 + 7,
            "rew": torch.randn((T, N), generator=g),
            "done": done,
            "state0": torch.randn((N, S), generator=g)}


def hand_unroll(kind, cell, head, value, log_std, out):
    """A float64 loop written from the contract: x_t = [obs_t, a_{t-1}, r_{t-1}] from the state row at t = 0, the
    torch cell equations, mean = head(h_t), logp of the Gaussian; the whole row is zeroed at every done, else it
    carries (h, c) and the raw action and reward."""
    f = lambda t: t.detach().double().numpy()                  # noqa: E731
    Wi, Wh, bi, bh = f(cell.weight_ih), f(cell.weight_hh), f(cell.bias_ih), f(cell.bias_hh)
    H = cell.hidden_size
    lins = head_linears(head)
    T, N = out["done"].shape
    obs = np.concatenate([out["obs0"].numpy()[None], out["obs"].numpy()[:-1]]).astype(np.float64)
    st = out["state0"].numpy().astype(np.float64)
    nm = H if kind == "gru" else 2 * H
    mem, fb = st[:, :nm].copy(), st[:, nm:].copy()
    sig = lambda v: 1.0 / (1.0 + np.exp(-v))                   # noqa: E731
    means, logp, vals = np.zeros((T, N, 4)), np.zeros((T, N)), np.zeros((T, N))
    ls = np.asarray(log_std, np.float64)
    for t in range(T):
        for e in range(N):
            x = np.concatenate([obs[t, e], fb[e]])
            gi, gh = Wi @ x + bi, Wh @ mem[e, :H] + bh
            if kind == "gru":
                r, z = sig(gi[:H] + gh[:H]), sig(gi[H:2 * H] + gh[H:2 * H])
                n = np.tanh(gi[2 * H:] + r * gh[2 * H:])
                h = (1 - z) * n + z * mem[e, :H]
                new = h
            else:
                v = gi + gh
                i, fg, g, o = sig(v[:H]), sig(v[H:2 * H]), np.tanh(v[2 * H:3 * H]), sig(v[3 * H:])
                c = fg * mem[e, H:] + i * g
                h = o * np.tanh(c)
                new = np.concatenate([h, c])
            y = h
            for k, m in enumerate(lins):
                y_in = y
                y = f(m.weight) @ y + f(m.bias)
                if k < len(lins) - 1:
                    y = np.tanh(y)
            vals[t, e] = (f(value.weight) @ y_in + f(value.bias))[0]
            a = out["act"][t, e].numpy().astype(np.float64)
            means[t, e] = y
            zz = (a - y) / np.exp(ls)
            logp[t, e] = np.sum(-0.5 * zz * zz - ls) - 2 * np.log(2 * np.pi)
            if out["done"][t, e]:
                mem[e], fb[e] = 0.0, 0.0
            else:
                mem[e] = new
                fb[e] = np.concatenate([a, [float(out["rew"][t, e])]])
    return means, logp, vals


@pytest.mark.parametrize("kind", ["gru", "lstm"])
@pytest.mark.parametrize("width", [0, 6])
def test_unroll_reference_against_hand_loop(kind, width):
    Pol, Cell, _ = policy_classes()[kind]
    torch.manual_seed(11)
    H, T, N = 5, 10, 4
    cell, head = Cell(D + 5, H).double(), make_head(H, width).double()
    value = nn.Linear(width or H, 1).double()
    log_std = torch.tensor([-0.3, 0.1, 0.4, -0.7], dtype=torch.float64, requires_grad=True)
    pol = Pol(cell, head, log_std=log_std, dist="gaussian", device="cpu", value=value)
    out = fake_rollout(T, N, pol.state_dim, seed=5)
    mean, logp, v = pol._unroll_reference(out, value=True)
    assert mean.shape == (T, N, 4) and logp.shape == (T, N) and mean.dtype == torch.float64
    ref_mean, ref_logp, ref_v = hand_unroll(kind, cell, head, value, log_std.detach().numpy(), out)
    assert np.abs(mean.detach().numpy() - ref_mean).max() < 1e-12
    assert np.abs(logp.detach().numpy() - ref_logp).max() < 1e-12
    assert np.abs(v.detach().numpy() - ref_v).max() < 1e-12
    # unroll() of a float64 cell is the reference loop
    m2, l2 = pol.unroll(out)
    assert torch.equal(m2, mean) and torch.equal(l2, logp)
    # the feedback is the raw action: one-hot feedback would give other means after the first step
    out2 = dict(out, act=out["act"] + 1.0)
    m3, _ = pol._unroll_reference(out2)
    assert (m3[1:] - mean[1:]).abs().max() > 1e-6 and torch.equal(m3[0], mean[0])
    # gradients reach the cell, the head, the value head and the caller's log_std tensor
    (logp.sum() + mean.pow(2).sum() + v.sum()).backward()
    assert log_std.grad is not None and log_std.grad.abs().sum() > 0
    for name, p in (list(cell.named_parameters()) + list(head.named_parameters())
                    + list(value.named_parameters())):
        assert p.grad is not None and p.grad.abs().sum() > 0, name
    # d logp / d log_std_k = sum over (t, e) of (z_k^2 - 1)
    z = (out["act"].double() - mean.detach()) / log_std.detach().exp()
    want = (z * z - 1).sum((0, 1)) + 0.0
    log_std.grad = None
    logp2 = pol._unroll_reference(out)[1]
    logp2.sum().backward()
    assert torch.allclose(log_std.grad, want, rtol=1e-12, atol=1e-9)
