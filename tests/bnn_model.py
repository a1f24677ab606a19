"""Exact numpy restatement of the device Bayesian neural network (robo_b200/csrc/gpk_bnn.cuh) — TEST INFRASTRUCTURE ONLY.

pybnn, the library robo/models/wrapper_bohamiann.py wraps, is not available, so the model is stated here, in gpk_bnn.cuh
and in DESIGN §1 row a28 (a restatement, not checked against pybnn):

* Network: Linear(D, 50) . tanh . Linear(50, 50) . tanh . Linear(50, 1) plus a scalar log-variance lv.  theta holds
  W1 (50 x D), b1, W2 (50 x 50), b2, W3 (50), b3, lv: P = 50 D + 2652.  Initial W_l = xi / sqrt(fan_in) with xi the
  chain's step -1 normals, biases 0, lv = log(1e-2).
* Data: X per column and y scaled to zero mean and unit population std (sums in ascending row order).
* Batches of B rows: epoch e visits the rows in the ranks of (Philox word 0 of (row, e, counter, TAG_ORDER), row).
* Loss L = nll - lvp / N - wp / N, gradient G = N dL/dtheta in the order ``grad`` states.
* Adaptive SGHMC (``step``), a network kept after step s when s > burn_in and (s - burn_in) % keep_every == 0.
* Predict: m = mean f_k, v = mean (f_k - m)^2 + mean exp(lv_k), then un-scaled.

numpy's elementwise float64 operations round each product, sum and quotient once, like the kernel's __dmul_rn /
__dadd_rn / __ddiv_rn, and every sum below runs in the kernel's order, so given the device's normals (gpk_bnn_draws)
the chain is the device's bit for bit.  ``predict_ld`` evaluates the predictive moments in extended precision with an
error bound for the device's fp64 scoring pass; ``torch_*`` restate the loss and the update in torch (float64) as
pybnn writes them, as an independent check and as the host arm of tools/bnn_bench.py.
"""
import numpy as np

from tests.cmaes_model import exp
from tests.de_model import _philox

H = 50
TAG_NOISE, TAG_ORDER = 0x424E0001, 0x424E0002
LOG_LV0, LOG_1EM6 = -4.605170185988091, -13.815510557964274
LR, MDECAY, EPS, KEEP_EVERY, BATCH = 1e-2, 0.05, 1e-10, 100, 20


def n_params(D):
    return H * D + 2652


def layout(D):
    """Slices of W1, b1, W2, b2, W3, b3, lv in theta."""
    o = [0, H * D, H * D + H, H * D + H + H * H, H * D + 2 * H + H * H, H * D + 3 * H + H * H]
    return dict(W1=slice(o[0], o[1]), b1=slice(o[1], o[2]), W2=slice(o[2], o[3]), b2=slice(o[3], o[4]),
                W3=slice(o[4], o[5]), b3=o[5], lv=o[5] + 1)


def tanh(x):
    """gpk_bnn_tanh: |x| < 2^-8 by the degree-7 Taylor polynomial, otherwise sign(x) (1 - t) / (1 + t), t = exp(-2|x|)."""
    x = np.asarray(x, dtype=np.float64)
    ax = np.fabs(x)
    x2 = x * x
    small = x + x * (x2 * (-0.3333333333333333 + x2 * (0.13333333333333333 - 0.05396825396825397 * x2)))
    t = exp(-2.0 * ax)
    r = (1.0 - t) / (1.0 + t)
    big = np.where(x < 0.0, -r, np.where(x > 0.0, r, x))
    return np.where(ax < 0.00390625, small, big)


def _seq(rows, start=None):
    """Sum over the first axis in ascending order from +0.0 (or from `start`), one rounding per addition."""
    acc = np.zeros_like(rows[0]) if start is None else np.array(start, dtype=np.float64)
    for r in rows:
        acc = acc + r
    return acc


def normalise(X, y):
    """(Xs, ys, x_mean, x_std, y_mean, y_std) as gpk_bnn_set_data computes them; ValueError where the device refuses."""
    X = np.asarray(X, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64).ravel()
    n = X.shape[0]
    if n < 2:
        raise ValueError("need n >= 2 training points to normalise the data")

    def stats(V):
        m = _seq(V) / float(n)
        return m, np.sqrt(_seq([(v - m) * (v - m) for v in V]) / float(n))
    xm, xs = stats(X)
    if not np.all(xs > 0.0):
        raise ValueError("an input column is constant; it cannot be normalised")
    ym, ysd = stats(y[:, None])
    if not ysd[0] > 0.0:
        raise ValueError("y is constant; it cannot be normalised")
    return (X - xm) / xs, (y - ym[0]) / ysd[0], xm, xs, float(ym[0]), float(ysd[0])


def epoch_order(seed, counter, e, N):
    rows = np.arange(N, dtype=np.uint64)
    keys = _philox(seed, rows, e, counter, TAG_ORDER)[0]
    return np.lexsort((rows, keys))


def batch_rows(seed, counter, s, N, B, cache=None):
    """The rows of step s's batch."""
    nb = (N + B - 1) // B
    e, bi = divmod(s, nb)
    if cache is not None:
        if cache.get("e") != e:
            cache["e"], cache["order"] = e, epoch_order(seed, counter, e, N)
        order = cache["order"]
    else:
        order = epoch_order(seed, counter, e, N)
    return order[bi * B:min(N, (bi + 1) * B)]


def init_theta(D, xi):
    L = layout(D)
    th = np.zeros(n_params(D))
    th[L["W1"]] = xi[L["W1"]] * (1.0 / np.sqrt(float(D)))
    sc2 = 1.0 / np.sqrt(float(H))
    th[L["W2"]] = xi[L["W2"]] * sc2
    th[L["W3"]] = xi[L["W3"]] * sc2
    th[L["lv"]] = LOG_LV0
    return th


def grad(theta, xb, yb, N):
    """G = N dL/dtheta on the batch (xb (B_t, D), yb (B_t,)) in gpk_bnn_chain_kernel's order."""
    Bt, D = xb.shape
    L = layout(D)
    W1 = theta[L["W1"]].reshape(H, D)
    b1 = theta[L["b1"]]
    W2 = theta[L["W2"]].reshape(H, H)
    b2 = theta[L["b2"]]
    W3 = theta[L["W3"]]
    b3, lv = theta[L["b3"]], theta[L["lv"]]
    a1 = np.broadcast_to(b1, (Bt, H)).copy()
    for k in range(D):
        a1 = a1 + W1[:, k][None, :] * xb[:, k][:, None]
    h1 = tanh(a1)
    a2 = np.broadcast_to(b2, (Bt, H)).copy()
    for k in range(H):
        a2 = a2 + W2[:, k][None, :] * h1[:, k][:, None]
    h2 = tanh(a2)
    f = np.full(Bt, b3)
    for j in range(H):
        f = f + W3[j] * h2[:, j]
    ev = float(exp(lv))
    s2, c = ev + 1e-16, float(N) / float(Bt)
    q = (yb - f) / s2
    df = -(c * q)
    u = 0.5 - 0.5 * ((q * q) * ev)
    g = np.zeros_like(theta)
    g[L["W3"]] = _seq(df[:, None] * h2)
    g[L["b3"]] = _seq(df)
    g[L["lv"]] = c * _seq(u) + (lv - LOG_1EM6) / 0.01
    d2 = (df[:, None] * W3[None, :]) * (1.0 - h2 * h2)
    acc = np.zeros((Bt, H))
    for j in range(H):
        acc = acc + d2[:, j][:, None] * W2[j][None, :]
    d1 = acc * (1.0 - h1 * h1)
    g[L["W2"]] = _seq(d2[:, :, None] * h1[:, None, :]).ravel()
    g[L["b2"]] = _seq(d2)
    g[L["W1"]] = _seq(d1[:, :, None] * xb[:, None, :]).ravel()
    g[L["b1"]] = _seq(d1)
    return g + theta / float(len(theta))


def step(theta, st, G, xi, adapt, lr=LR, mdecay=MDECAY, eps=EPS):
    """One adaptive-SGHMC update of theta and the state dict (p, tau, g, vhat) in place; returns theta."""
    if adapt:
        tau, g, v = st["tau"], st["g"], st["vhat"]
        r = 1.0 / (tau + 1.0)
        st["tau"] = (tau - (tau * (g * g)) / (v + eps)) + 1.0
        st["g"] = (g - g * r) + r * G
        st["vhat"] = (v - v * r) + r * (G * G)
    lr2 = lr * lr
    minv = 1.0 / (np.sqrt(st["vhat"]) + eps)
    ns2 = ((2.0 * lr2) * mdecay) * minv - lr2 * lr2
    st["p"] = ((st["p"] - (lr2 * minv) * G) - mdecay * st["p"]) + np.sqrt(np.fmax(ns2, 1e-16)) * xi
    return theta + st["p"]


def kept(s, burn_in, keep_every):
    return s > burn_in and (s - burn_in) % keep_every == 0


def chain(Xs, ys, seed, counter, normals, lr=LR, mdecay=MDECAY, eps=EPS, burn_in=0, num_steps=1,
          keep_every=KEEP_EVERY, batch=BATCH):
    """The whole chain on the scaled data; normals(step) gives the P normals of a step (-1: initialisation).
    -> (samples (S, P), final state dict(theta, p, tau, g, vhat))."""
    N, D = Xs.shape
    P = n_params(D)
    theta = init_theta(D, normals(-1))
    st = dict(p=np.zeros(P), tau=np.ones(P), g=np.ones(P), vhat=np.ones(P))
    cache, out = {}, []
    for s in range(num_steps):
        rows = batch_rows(seed, counter, s, N, batch, cache)
        G = grad(theta, Xs[rows], ys[rows], N)
        theta = step(theta, st, G, normals(s), s + 1 <= burn_in, lr, mdecay, eps)
        if kept(s, burn_in, keep_every):
            out.append(theta.copy())
    st["theta"] = theta
    return np.array(out).reshape(-1, P), st


def n_kept(burn_in, num_steps, keep_every):
    return (num_steps - 1 - burn_in) // keep_every if num_steps - 1 > burn_in else 0


def forward_ld(samples, Xs):
    """f (S, M) and lv (S,) of every network at the scaled rows Xs, in np.longdouble, with the magnitude of each f's
    rounding error bound for an fp64 evaluation (sums of |terms| through the layers)."""
    LD = np.longdouble
    S, P = samples.shape
    M, D = Xs.shape
    L = layout(D)
    u = LD(2.0) ** -53
    x = Xs.astype(LD)
    F, E = np.empty((S, M), dtype=LD), np.empty((S, M), dtype=LD)
    for k in range(S):
        th = samples[k].astype(LD)
        W1, b1 = th[L["W1"]].reshape(H, D), th[L["b1"]]
        W2, b2 = th[L["W2"]].reshape(H, H), th[L["b2"]]
        W3, b3 = th[L["W3"]], th[L["b3"]]
        a1 = x @ W1.T + b1
        e1 = (D + 2) * u * (np.fabs(x) @ np.fabs(W1).T + np.fabs(b1)) + 4 * u
        h1 = np.tanh(a1)
        a2 = h1 @ W2.T + b2
        e2 = (H + 2) * u * (np.fabs(h1) @ np.fabs(W2).T + np.fabs(b2)) + e1 @ np.fabs(W2).T + 4 * u
        h2 = np.tanh(a2)
        F[k] = h2 @ W3 + b3
        E[k] = (H + 2) * u * (np.fabs(h2) @ np.fabs(W3) + np.fabs(b3)) + e2 @ np.fabs(W3)
    return F, samples[:, L["lv"]].astype(LD), E


def predict_ld(samples, X, xm, xs, ym, ysd):
    """(m, v, bound_m, bound_v): the predictive moments in np.longdouble and bounds on the device's fp64 error."""
    LD = np.longdouble
    u = LD(2.0) ** -53
    S = samples.shape[0]
    Xs = (np.asarray(X, dtype=np.float64).astype(LD) - xm) / xs
    F, lv, E = forward_ld(samples, Xs)
    m = F.mean(axis=0)
    dev = F - m
    vs = (dev * dev).mean(axis=0) + np.exp(lv).mean()
    emax = E.max(axis=0) + (S + 4) * u * np.fabs(F).max(axis=0)
    bm = emax + 4 * u * np.fabs(m)
    bv = 2 * np.fabs(dev).mean(axis=0) * (2 * emax) + 4 * emax * emax + (S + 8) * u * vs
    ysd_ld = LD(ysd)
    return m * ysd_ld + LD(ym), vs * ysd_ld * ysd_ld, 4 * (bm * ysd_ld + 4 * u * np.fabs(m * ysd_ld + LD(ym))), \
        4 * bv * ysd_ld * ysd_ld


# ---- torch restatement (pybnn's formulation): loss, autograd gradient, update, the whole training loop ---------------
def torch_net(D, theta):
    """The reference's get_default_network structure with theta's values."""
    import torch
    from robo_b200.models.wrapper_bohamiann import get_default_network
    net = get_default_network(D)
    L = layout(D)
    t = torch.as_tensor(theta, dtype=torch.float64)
    with torch.no_grad():
        net[0].weight.copy_(t[L["W1"]].reshape(H, D))
        net[0].bias.copy_(t[L["b1"]])
        net[2].weight.copy_(t[L["W2"]].reshape(H, H))
        net[2].bias.copy_(t[L["b2"]])
        net[4].weight.copy_(t[L["W3"]].reshape(1, H))
        net[4].bias.copy_(t[L["b3"]:L["b3"] + 1])
        net[5].bias.copy_(t[L["lv"]:L["lv"] + 1].reshape(1, 1))
    return net


def torch_loss(net, xb, yb, N):
    import torch
    out = net(xb)
    f, lv = out[:, 0], out[:, 1]
    nll = -torch.mean(-0.5 * (yb - f) ** 2 / (torch.exp(lv) + 1e-16) - 0.5 * lv)
    lvp = torch.mean(-(lv - np.log(1e-6)) ** 2 / 0.02 - 0.5 * np.log(0.01))
    params = list(net.parameters())
    P = sum(p.numel() for p in params)
    wp = -0.5 * sum(torch.sum(p ** 2) for p in params) / P
    return nll - lvp / N - wp / N


def torch_grad(theta, xb, yb, N):
    """N dL/dtheta by torch.autograd, in theta's order."""
    import torch
    D = xb.shape[1]
    net = torch_net(D, theta)
    loss = torch_loss(net, torch.as_tensor(xb), torch.as_tensor(yb), N)
    loss.backward()
    g = [net[0].weight.grad.ravel(), net[0].bias.grad, net[2].weight.grad.ravel(), net[2].bias.grad,
         net[4].weight.grad.ravel(), net[4].bias.grad, net[5].bias.grad.ravel()]
    return N * torch.cat(g).numpy()


def torch_step(p, G, st, xi, adapt, lr=LR, mdecay=MDECAY, eps=EPS):
    """The adaptive-SGHMC update of one torch parameter tensor p (gradient G, state tensors st, noise xi)."""
    import torch
    with torch.no_grad():
        if adapt:
            r = 1.0 / (st["tau"] + 1.0)
            st["tau"] = st["tau"] - st["tau"] * st["g"] * st["g"] / (st["vhat"] + eps) + 1.0
            st["g"] = st["g"] - st["g"] * r + r * G
            st["vhat"] = st["vhat"] - st["vhat"] * r + r * G * G
        minv = 1.0 / (torch.sqrt(st["vhat"]) + eps)
        lr2 = lr * lr
        s2 = 2.0 * lr2 * mdecay * minv - lr2 * lr2
        st["p"] = st["p"] - lr2 * minv * G - mdecay * st["p"] + torch.sqrt(torch.clamp(s2, min=1e-16)) * xi
        p.add_(st["p"])


def torch_train(X, y, seed, lr=LR, mdecay=MDECAY, eps=EPS, burn_in=None, num_steps=None, keep_every=KEEP_EVERY,
                batch=BATCH):
    """pybnn's training loop restated in torch on the host (float64): a shuffled batch loader looped forever, the loss
    above, adaptive SGHMC per parameter tensor.  -> (samples (S, P), normalisation) for ``predict_samples``."""
    import torch
    Xs, ys, xm, xs, ym, ysd = normalise(X, y)
    N, D = Xs.shape
    if burn_in is None:
        burn_in, num_steps = 100 * N, 100 * N + 10000
    gen = torch.Generator().manual_seed(int(seed))
    torch.manual_seed(int(seed))
    from robo_b200.models.wrapper_bohamiann import get_default_network
    net = get_default_network(D)
    params = list(net.parameters())
    state = [dict(p=torch.zeros_like(p), tau=torch.ones_like(p), g=torch.ones_like(p), vhat=torch.ones_like(p))
             for p in params]
    Xt, yt = torch.as_tensor(Xs), torch.as_tensor(ys)
    out, s, order = [], 0, None
    while s < num_steps:
        order = torch.randperm(N, generator=gen)
        for b0 in range(0, N, batch):
            if s >= num_steps:
                break
            rows = order[b0:b0 + batch]
            net.zero_grad()
            torch_loss(net, Xt[rows], yt[rows], N).backward()
            for p, st in zip(params, state):
                xi = torch.randn(p.shape, generator=gen, dtype=torch.float64)
                torch_step(p, N * p.grad, st, xi, s + 1 <= burn_in, lr, mdecay, eps)
            if kept(s, burn_in, keep_every):
                out.append(torch.cat([p.detach().ravel() for p in params]).numpy().copy())
            s += 1
    return np.array(out), (xm, xs, ym, ysd)


def predict_samples(samples, X, xm, xs, ym, ysd):
    """(m, v) in float64 (host evaluation of the same moments)."""
    m, v, _, _ = predict_ld(samples, X, xm, xs, ym, ysd)
    return m.astype(np.float64), v.astype(np.float64)
