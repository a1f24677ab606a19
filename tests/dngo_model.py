"""Exact numpy restatement of the device DNGO training (robo_b200/csrc/gpk_dngo.cuh) — TEST INFRASTRUCTURE ONLY.

pybnn's dngo.py is not available, so the model is stated here, in gpk_dngo.cuh and in DESIGN §1 row a29 (a restatement,
not checked against pybnn):

* Network: Linear(D, 50) . tanh . Linear(50, 50) . tanh . Linear(50, 50) . tanh . Linear(50, 1) in fp64.  theta holds
  W1 (50 x D), b1, W2 (50 x 50), b2, W3 (50 x 50), b3, W4 (50), b4: P = 50 D + 5201.  Every entry of a layer with fan_in
  inputs starts at (2 u - 1) / sqrt(fan_in), u the 53-bit uniform of Philox words 0, 1 of (p, 0, counter, TAG_INIT).
* Data: with a flag on, X per column / y scaled to zero mean and unit population std (gpk_bnn_set_data's code).
* Batches: B = min(batch, N); epoch e visits the rows in the ranks of (Philox word 0 of (row, e, counter, TAG_ORDER),
  row) in floor(N / B) full batches, the remainder dropped.
* Loss: the batch's mean squared error; ``grad`` states the gradient's order.
* Adam (``adam``): torch's single-tensor update with beta^t kept as running products.
* Theta: the third tanh layer over the scaled training rows.

numpy's elementwise float64 operations round each product, sum, quotient and square root once, like the kernel's
__dmul_rn / __dadd_rn / __ddiv_rn / __dsqrt_rn, and every sum below runs in the kernel's order, so ``train`` is the
device's training bit for bit.  ``predict_ld`` evaluates the predictive mixture per hyper-sample in extended precision
with an error bound for the device's fp64 scoring pass (which uses the collapsed form).  ``torch_*`` restate the network,
its gradient and the training loop in torch (float64) as pybnn writes them, as an independent check and as the host arm
of tools/dngo_bench.py.
"""
import numpy as np

from tests.bnn_model import _seq, tanh
from tests.de_model import _philox, _u01

H = 50
TAG_INIT, TAG_ORDER = 0x444E0001, 0x444E0002
BETA1, BETA2, ADAM_EPS = 0.9, 0.999, 1e-8
LR, BATCH, EPOCHS = 0.01, 10, 500


def n_params(D):
    return H * D + 5201


def layout(D):
    """Slices of W1, b1, W2, b2, W3, b3, W4 and the index of b4 in theta."""
    o = np.cumsum([0, H * D, H, H * H, H, H * H, H, H])
    names = ("W1", "b1", "W2", "b2", "W3", "b3", "W4")
    L = {k: slice(int(o[i]), int(o[i + 1])) for i, k in enumerate(names)}
    L["b4"] = int(o[7])
    return L


def unpack(theta, D):
    L = layout(D)
    return (theta[L["W1"]].reshape(H, D), theta[L["b1"]], theta[L["W2"]].reshape(H, H), theta[L["b2"]],
            theta[L["W3"]].reshape(H, H), theta[L["b3"]], theta[L["W4"]], theta[L["b4"]])


def normalise(X, y, normalize_input=True, normalize_output=True):
    """(Xs, ys, x_mean, x_std, y_mean, y_std) as gpk_dngo_set_data computes them; ValueError where the device refuses.
    A side whose flag is off is used as given, with mean 0 and std 1."""
    X = np.asarray(X, dtype=np.float64)
    y = np.asarray(y, dtype=np.float64).ravel()
    n, D = X.shape
    if (normalize_input or normalize_output) and n < 2:
        raise ValueError("need n >= 2 training points to normalise the data")

    def stats(V):
        m = _seq(V) / float(n)
        return m, np.sqrt(_seq([(v - m) * (v - m) for v in V]) / float(n))
    if normalize_input:
        xm, xs = stats(X)
        if not np.all(xs > 0.0):
            raise ValueError("an input column is constant; it cannot be normalised")
        Xs = (X - xm) / xs
    else:
        xm, xs, Xs = np.zeros(D), np.ones(D), X.copy()
    if normalize_output:
        ym, ysd = (float(v[0]) for v in stats(y[:, None]))
        if not ysd > 0.0:
            raise ValueError("y is constant; it cannot be normalised")
        ys = (y - ym) / ysd
    else:
        ym, ysd, ys = 0.0, 1.0, y.copy()
    return Xs, ys, xm, xs, ym, ysd


def init_theta(D, seed, counter):
    p = np.arange(n_params(D), dtype=np.uint64)
    w = _philox(seed, p, 0, counter, TAG_INIT)
    u = _u01(w[0], w[1])
    bound = np.where(p < layout(D)["W2"].start, 1.0 / np.sqrt(float(D)), 1.0 / np.sqrt(float(H)))
    return (2.0 * u - 1.0) * bound


def epoch_order(seed, counter, e, N):
    rows = np.arange(N, dtype=np.uint64)
    keys = _philox(seed, rows, e, counter, TAG_ORDER)[0]
    return np.lexsort((rows, keys))


def batches(seed, counter, e, N, B):
    """The row lists of epoch e's full batches."""
    order = epoch_order(seed, counter, e, N)
    return [order[b * B:(b + 1) * B] for b in range(N // B)]


def forward(theta, xb):
    """h1, h2, h3 (rows x 50) and f (rows) in gpk_dngo_train_kernel's order."""
    W1, b1, W2, b2, W3, b3, W4, b4 = unpack(theta, xb.shape[1])
    hs, h = [], xb
    for W, b in ((W1, b1), (W2, b2), (W3, b3)):
        a = np.broadcast_to(b, (xb.shape[0], H)).copy()
        for k in range(W.shape[1]):
            a = a + W[:, k][None, :] * h[:, k][:, None]
        h = tanh(a)
        hs.append(h)
    f = np.full(xb.shape[0], b4)
    for j in range(H):
        f = f + W4[j] * h[:, j]
    return hs[0], hs[1], hs[2], f


def features(theta, Xs):
    """Theta (rows x 50) of the scaled rows Xs."""
    return forward(theta, Xs)[2]


def grad(theta, xb, yb):
    """dL/dtheta of the batch's mean squared error in gpk_dngo_train_kernel's order."""
    B, D = xb.shape
    L = layout(D)
    W1, b1, W2, b2, W3, b3, W4, b4 = unpack(theta, D)
    h1, h2, h3, f = forward(theta, xb)
    df = (2.0 * (f - yb)) / float(B)
    g = np.zeros_like(theta)
    g[L["W4"]] = _seq(df[:, None] * h3)
    g[L["b4"]] = _seq(df)
    d = (df[:, None] * W4[None, :]) * (1.0 - h3 * h3)
    for W, hin, oW, ob in ((W3, h2, "W3", "b3"), (W2, h1, "W2", "b2")):
        acc = np.zeros((B, H))
        for j in range(H):
            acc = acc + d[:, j][:, None] * W[j][None, :]
        g[L[oW]] = _seq(d[:, :, None] * hin[:, None, :]).ravel()
        g[L[ob]] = _seq(d)
        d = acc * (1.0 - hin * hin)
    g[L["W1"]] = _seq(d[:, :, None] * xb[:, None, :]).ravel()
    g[L["b1"]] = _seq(d)
    return g


def adam(theta, st, G, lr=LR):
    """One Adam step of theta and the state dict (m, v, t, p1, p2) in place; returns theta."""
    st["t"] += 1
    st["p1"] = st["p1"] * BETA1
    st["p2"] = st["p2"] * BETA2
    st["m"] = st["m"] + (1.0 - BETA1) * (G - st["m"])
    st["v"] = st["v"] * BETA2 + ((1.0 - BETA2) * G) * G
    ss = lr / (1.0 - st["p1"])
    den = np.sqrt(st["v"]) / np.sqrt(1.0 - st["p2"]) + ADAM_EPS
    return theta - ss * (st["m"] / den)


def adam_state(P):
    return dict(m=np.zeros(P), v=np.zeros(P), t=0, p1=1.0, p2=1.0)


def train(Xs, ys, seed, counter, lr=LR, batch=BATCH, epochs=EPOCHS):
    """The whole training on the scaled data -> (theta, Adam state dict, Theta)."""
    N, D = Xs.shape
    B = min(batch, N)
    theta = init_theta(D, seed, counter)
    st = adam_state(len(theta))
    for e in range(epochs):
        for rows in batches(seed, counter, e, N, B):
            theta = adam(theta, st, grad(theta, Xs[rows], ys[rows]), lr)
    return theta, st, features(theta, Xs)


def predict_ld(theta, models, hypers, X, xm, xs, ym, ysd):
    """(m, v, bound_m, bound_v): the mixture's mean and full variance over the k hyper-samples, each sample's mu_i =
    phi^T m_i and var_i = 1 / beta_i + phi^T S_i phi evaluated in np.longdouble, and bounds on the device's fp64 error
    (its features through fma and libdevice tanh, the collapse's k-term sums, Q's Cholesky factor and the quadratic form),
    from the magnitudes of the terms."""
    LD = np.longdouble
    u = LD(2.0) ** -53
    M = np.array([m for m, _ in models], dtype=LD)
    S = np.array([s for _, s in models], dtype=LD)
    ib = LD(1.0) / np.asarray(hypers, dtype=np.float64)[:, 1].astype(LD)
    k = len(models)
    Xl = (np.asarray(X, dtype=np.float64).astype(LD) - xm) / xs
    D = Xl.shape[1]
    W1, b1, W2, b2, W3, b3 = (a.astype(LD) for a in unpack(theta, D)[:6])
    e, h, fan = None, Xl, D
    for W, b in ((W1, b1), (W2, b2), (W3, b3)):
        a = h @ W.T + b
        en = (fan + 2) * u * (np.fabs(h) @ np.fabs(W).T + np.fabs(b)) + 4 * u
        if e is not None:
            en = en + e @ np.fabs(W).T
        h, e, fan = np.tanh(a), en, H
    phi, ephi = h, e
    mu = phi @ M.T                                            # (rows, k)
    qi = np.einsum("rj,ijl,rl->ri", phi, S, phi)
    var = ib[None, :] + qi
    m = mu.mean(axis=1)
    dev = mu - m[:, None]
    v = (dev * dev).mean(axis=1) + var.mean(axis=1)
    pa = np.fabs(phi)
    mbar = M.mean(axis=0)
    Q = S.mean(axis=0) + np.einsum("ia,ib->ab", M - mbar, M - mbar) / k
    Rl = np.linalg.cholesky(Q.astype(np.float64)).astype(LD)
    RR = np.fabs(Rl) @ np.fabs(Rl).T
    Qa = np.fabs(S).mean(axis=0) + np.einsum("ia,ib->ab", np.fabs(M - mbar), np.fabs(M - mbar)) / k
    g = (2 * H + k + 16) * u
    bm = pa @ np.fabs(mbar) * g + ephi @ np.fabs(mbar) + (k + 2) * u * (pa @ np.fabs(M).mean(axis=0))
    quad = np.einsum("rj,jl,rl->r", pa, RR + Qa, pa)
    bv = g * (quad + ib.mean()) + 2 * ephi * np.fabs(phi @ Q) @ np.ones(H) + (ephi * ephi) @ np.ones(H) * np.abs(Q).max()
    bv = bv + 4 * u * v
    ys = LD(ysd)
    return m * ys + LD(ym), v * ys * ys, 4 * (bm * ys + 4 * u * np.fabs(m * ys + LD(ym))), 4 * bv * ys * ys


# ---- torch restatement (pybnn's formulation): network, autograd gradient, Adam, the whole training loop -------------
def torch_net(D, theta=None):
    """The network as a torch module (float64), with theta's values when given."""
    import torch
    net = torch.nn.Sequential(torch.nn.Linear(D, H), torch.nn.Tanh(), torch.nn.Linear(H, H), torch.nn.Tanh(),
                              torch.nn.Linear(H, H), torch.nn.Tanh(), torch.nn.Linear(H, 1)).double()
    if theta is not None:
        t = torch.as_tensor(np.asarray(theta, dtype=np.float64))
        with torch.no_grad():
            off = 0
            for p in net.parameters():
                p.copy_(t[off:off + p.numel()].reshape(p.shape))
                off += p.numel()
    return net


def torch_flat(net, grads=False):
    import torch
    return torch.cat([(p.grad if grads else p).detach().ravel() for p in net.parameters()]).numpy().copy()


def torch_loss(net, xb, yb):
    import torch
    return torch.nn.functional.mse_loss(net(xb)[:, 0], yb)


def torch_grad(theta, xb, yb):
    """dL/dtheta by torch.autograd, in theta's order."""
    import torch
    net = torch_net(xb.shape[1], theta)
    torch_loss(net, torch.as_tensor(xb), torch.as_tensor(yb)).backward()
    return torch_flat(net, grads=True)


def torch_train(X, y, seed, lr=LR, batch=BATCH, epochs=EPOCHS, normalize_input=True, normalize_output=True):
    """pybnn's training loop restated in torch on the host (float64): nn.Linear's default initialisation, a fresh
    permutation per epoch in full batches of min(batch, N) rows, the mean squared error, torch.optim.Adam.
    -> (theta, Theta, normalisation)."""
    import torch
    Xs, ys, xm, xs, ym, ysd = normalise(X, y, normalize_input, normalize_output)
    N, D = Xs.shape
    B = min(batch, N)
    torch.manual_seed(int(seed))
    gen = torch.Generator().manual_seed(int(seed))
    net = torch_net(D)
    opt = torch.optim.Adam(net.parameters(), lr=lr, foreach=False)
    Xt, yt = torch.as_tensor(Xs), torch.as_tensor(ys)
    for _ in range(epochs):
        order = torch.randperm(N, generator=gen)
        for b0 in range(0, N - B + 1, B):
            rows = order[b0:b0 + B]
            opt.zero_grad()
            torch_loss(net, Xt[rows], yt[rows]).backward()
            opt.step()
    with torch.no_grad():
        Theta = net[:6](Xt).numpy().copy()
    return torch_flat(net), Theta, (xm, xs, ym, ysd)
