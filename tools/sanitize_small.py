"""Small end-to-end pass over every kernel for compute-sanitizer runs."""
import os, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from robo_b200 import _lib
from robo_b200 import kernels as K

rng = np.random.RandomState(0)
N, D, M = 300, 3, 700
X, y, Xs = rng.rand(N, D), rng.rand(N), rng.rand(M, D)
f = K.Product(K.ConstantKernel(0.1, ndim=D), K.Matern52Kernel(np.array([0.3, 0.5, 0.8]), ndim=D)).flatten()
h = _lib.Handle(0)
h.set_option("chunk", 256)
h.set_data(X, y)
h.set_input_bounds(np.zeros(D), np.ones(D))
h.set_output_transform(True, 0.5, 2.0)
h.set_kernel(f["family"], f["log_amp"], f["axis"], f["group"], f["log_metric"])
print("fit", h.fit(1e-3 + 1.25e-12, float(y.mean())))
r = h.acq(Xs, _lib.ACQ_EI, float(y.min()), 0.0, want_values=True, want_moments=True)
print(" acq best", r["best_idx"], r["best_val"], "neg", r["n_negative"])
for kind in (_lib.ACQ_LOG_EI, _lib.ACQ_PI, _lib.ACQ_LCB):
    h.acq(Xs[:300], kind, float(y.min()), 0.1)
mu, cov = h.predict_cov(Xs[:150])
g = h.nll_grad(1e-3, D)
pg = h.predict_grad(Xs[:5], _lib.ACQ_EI, float(y.min()), 0.0)
bx, bv, bi = h.maximize_random(7, 0, 1000, 700, np.zeros(D), np.ones(D), X[0], 0.1, _lib.ACQ_EI, float(y.min()), 0.0)
km = h.kernel_matrix(Xs[:40], X[:50])
print(" cov", cov.shape, "grad", np.round(g, 3), "dmu", pg["dmu"].shape, "max idx", bi, km.shape)
# incremental refit: 300 -> 310 rows inside the last 128-row block (NP = 384)
X2, y2 = np.vstack([X, rng.rand(10, D)]), np.concatenate([y, rng.rand(10)])
print(" append", h.fit_append(X2, y2, 1e-3 + 1.25e-12, float(y2.mean())), h.predict(Xs[:64])[0][:2])
h.close()
# round-2 kernels: int8 contraction (digit builder, several chunks), depth-2 trailing updates, fused multi-model
# scoring, raw posterior covariance
Xb = rng.rand(2304, D)
hs = []
for opts in ({"ozaki": 1}, {"ozaki": 0, "depth2": 1},
             # int8 contraction variants: one tile per CTA / persistent walk
             {"ozaki": 1, "ozpersist": 0}, {"ozaki": 1, "ozpersist": 1}):
    h = _lib.Handle(0)
    for k, v in opts.items():
        h.set_option(k, v)
    h.set_option("chunk", 1024)
    Xt, yt = (X, y) if len(hs) < 2 else (X[:250], y[:250])       # 250 rows = 2 row blocks: the CTA-pair kernels apply
    h.set_data(Xt, yt)
    h.set_kernel(f["family"], f["log_amp"], f["axis"], f["group"], f["log_metric"])
    for _ in range(2):
        ll = h.fit(1e-3 + 1.25e-12, float(yt.mean()))
    r = h.acq(Xb, _lib.ACQ_EI, float(y.min()), 0.0, want_values=True, want_moments=True)
    t = h.timings()
    print(opts, "fit", ll, "best", r["best_idx"], "oz launches", t["launches_ozaki"], "variant", t["ozaki_kernel_variant"])
    mu, cov = h.posterior_cov(Xs[:100])
    hs.append(h)
rm = _lib.acq_multi(hs[:2], Xs[:300], 0, _lib.ACQ_EI, [float(y.min())] * 2, 0.0, want_argmax=True)
rp = _lib.acq_multi(hs[:2], Xs[:300], 1)
print("multi", rm["best_idx"], rp["var"][:2])
for h in hs:
    h.close()
# information gain per unit cost: mean-only prediction, Fabolas transform, entropy change on two objective / cost pairs,
# the ratio, the mean over pairs and the device arg-max
pairs = []
for i in range(4):
    h = _lib.Handle(0)
    h.set_data(X, y if i < 2 else 0.1 * y)
    h.set_kernel(f["family"], f["log_amp"], f["axis"], f["group"], f["log_metric"])
    h.fit(1e-3 + 1.25e-12, float(y.mean()))
    pairs.append(h)
print("mean only", pairs[2].predict_mean(Xb)[:2], pairs[2].predict_mean(Xs[:70])[:2])
zb = np.hstack([rng.rand(20, D - 1), np.ones((20, 1))])
W = np.linspace(-2.0, 2.0, 40)
for h in pairs[:2]:
    h.es_update(zb, rng.rand(20), 1e-3, W, np.zeros(D), np.ones(D))
Xc = np.vstack([Xb, -np.ones((1, D))])
for bo, bc in ((_lib.BASIS_ONE_MINUS_S_SQ, _lib.BASIS_S), (_lib.BASIS_S, _lib.BASIS_ONE_MINUS_S_SQ)):
    r = _lib.es_cost_multi(pairs[:2], pairs[2:], Xc, np.zeros(D - 1), np.ones(D - 1), bo, bc, 0.1)
    print("es cost", r["best_idx"], r["values"][-1])
print("es cost random", _lib.maximize_random_es_cost(pairs[:1], pairs[2:3], 7, 1000, 700, np.zeros(D), np.ones(D), X[0],
                                                     0.1, np.zeros(D - 1), np.ones(D - 1), 1, 0, 0.0)[2])
for h in pairs:
    h.close()
# entropy search at N = 257 (two 256-row tiles of the sigma kernel) and Nb = 64: the read-back of var, sigma and U, and
# the entropy change itself (the dH kernel's full lane loop and all eight warps over the representer points)
h = _lib.Handle(0)
h.set_data(X[:257], y[:257])
h.set_kernel(f["family"], f["log_amp"], f["axis"], f["group"], f["log_metric"])
h.fit(1e-3 + 1.25e-12, float(y[:257].mean()))
h.es_update(rng.rand(64, D), rng.rand(64), 1e-3, W, np.zeros(D), np.ones(D))
var, sig = h.es_moments(Xs[:50])
print("es moments", var[:2], sig.shape, h.es_get_u().shape, "dH", h.es_compute(Xs[:50])[:2])
h.close()
# hyper-parameter sampling: the per-theta log-posterior (kernel, Cholesky, prior in one CTA) and a short stretch-move run
from robo_b200.priors import DefaultPrior
h = _lib.Handle(0)
h.set_data(X[:150], y[:150])
h.set_kernel(f["family"], f["log_amp"], f["axis"], f["group"], f["log_metric"])
_lib.set_hyper_model(h, f["slots"], len(f["axis"]), float(y.mean()), 1.25e-12, _lib.PRIOR_DEFAULT,
                     [1.0, 0.0, -10.0, 2.0, 0.1, 0.0, 0.0])
p0 = DefaultPrior(D + 2, rng=np.random.RandomState(0)).sample_from_prior(10)
print("hyper lnpost", _lib.hyper_lnpost(h, p0)[0][:3], "run", _lib.sample_hypers(h, p0, 5, 3)["n_accepted"])
h.close()
# multi-start L-BFGS: the stencil and step kernels over three starts (one clipped onto a corner), with maxcor = 2 so the
# pair ring wraps, on an acquisition and on the posterior objective
h = _lib.Handle(0)
h.set_data(X[:100], y[:100])
h.set_kernel(f["family"], f["log_amp"], f["axis"], f["group"], f["log_metric"])
h.fit(1e-3 + 1.25e-12, float(y[:100].mean()))
x0 = rng.rand(3, D)
x0[1] = 2.0
r = _lib.maximize_lbfgs([h], _lib.ACQ_LOG_EI, [float(y[:100].min())], 0.0, x0, np.zeros(D), np.ones(D), maxcor=2,
                        maxiter=8)
print("lbfgs", r["nfev"], r["status"],
      _lib.maximize_lbfgs([h], _lib.OBJ_MEAN_STD, None, 0.0, x0, np.zeros(D), np.ones(D), maxiter=8)["status"])
# CMA-ES: the init, sample and update kernels (the Jacobi sweeps included) over two runs, and the draws kernel
r = _lib.maximize_cmaes([h], _lib.ACQ_LOG_EI, [float(y[:100].min())], 0.0, 5, rng.rand(D), np.zeros(D), np.ones(D),
                        n_func_evals=300, restarts=1)
print("cmaes", r["nit"], r["stop"], _lib.cmaes_draws(h, 5, 1, 0, 2, 6, D).shape)
# DIRECT: the init, select, divide and result kernels over a run that ends on its budget
r = _lib.maximize_direct([h], _lib.ACQ_LOG_EI, [float(y[:100].min())], 0.0, np.zeros(D), np.ones(D), n_func_evals=200)
print("direct", r["nit"], r["nfev"], _lib.DIRECT_STOP_NAMES[r["stop"]])
h.close()
# Bayesian linear regression: features, Gram reduction, log-posterior, sampler half-steps, fit and the predictive pass
# (quadratic basis, F = 7), scored directly and through DIRECT
h = _lib.Handle(0)
_lib.blr_set_data(h, X[:60], y[:60], _lib.BLR_QUADRATIC, (0.1, -10.0, 0.1))
p0 = np.column_stack([-9.0 + 0.1 * rng.randn(6), 2.0 + rng.rand(6)])
r = _lib.blr_sample(h, 3, p0, 4)
print("blr lnpost", _lib.blr_lnpost(h, p0)[:2], "run", r["n_accepted"])
_lib.blr_fit(h, np.exp(r["pos"]))
print("blr predict", h.predict(Xs[:300])[1][:2], "acq", h.acq(Xs[:300], _lib.ACQ_EI, float(y.min()), 0.0)["best_idx"])
r = _lib.maximize_direct([h], _lib.ACQ_EI, [float(y.min())], 0.0, np.zeros(D), np.ones(D), n_func_evals=100)
print("blr direct", r["nit"], r["nfev"])
h.close()
# random forest: draws, growth (bootstrap and Fisher-Yates), the node read-back and upload, the predictive pass, scored
# directly and through DIRECT
h = _lib.Handle(0)
_lib.rf_set_data(h, X[:60], y[:60])
_lib.rf_fit(h, 3, 0, 33, 0, True, True)
t = _lib.rf_trees(h)
_lib.rf_fit(h, 3, 1, 5, 40, False, False)
_lib.rf_set_trees(h, t, True)
print("rf nodes", t["n_nodes"][:3], "predict", h.predict(Xs[:300])[1][:2],
      "acq", h.acq(Xs[:300], _lib.ACQ_EI, float(y.min()), 0.0)["best_idx"])
r = _lib.maximize_direct([h], _lib.ACQ_EI, [float(y.min())], 0.0, np.zeros(D), np.ones(D), n_func_evals=100)
print("rf direct", r["nit"], r["nfev"])
h.close()
# Bayesian neural network: the chain (burn-in, cut-over, keeps), its draws, the sample read-back and upload, the
# predictive pass over a ragged tile, scored directly and through DIRECT
h = _lib.Handle(0)
_lib.bnn_set_data(h, X[:23], y[:23])
_lib.bnn_train(h, 5, 0, 1e-2, 0.05, 1e-10, 4, 30, 5, 20)
Zb = _lib.bnn_draws(h, 5, 0, -1, 3)
_lib.bnn_set_samples(h, _lib.bnn_samples(h))
print("bnn samples", _lib.bnn_dims(h), "draws", Zb[0, :2], "predict", h.predict(Xs[:300])[1][:2],
      "acq", h.acq(Xs[:300], _lib.ACQ_EI, float(y.min()), 0.0)["best_idx"])
r = _lib.maximize_direct([h], _lib.ACQ_EI, [float(y.min())], 0.0, np.zeros(D), np.ones(D), n_func_evals=100)
print("bnn direct", r["nit"], r["nfev"])
h.close()
# DNGO: the training (a dropped remainder), Theta and the regression's products, its sampler and fit, the collapsed
# predictive over a ragged tile, the net read-back and upload, scored directly and through DIRECT
h = _lib.Handle(0)
_lib.dngo_set_data(h, X[:23], y[:23], True, True, (0.1, -10.0, 0.1))
_lib.dngo_train(h, 5, 0, 1e-2, 10, 3)
Pd = _lib.blr_sample(h, 3, np.c_[rng.uniform(-3, 1, 6), rng.uniform(0, 5, 6)], 4)["pos"]
_lib.dngo_fit(h, np.exp(Pd))
_lib.dngo_set_net(h, _lib.dngo_net(h))
_lib.dngo_fit(h, np.exp(Pd))
print("dngo", _lib.dngo_dims(h), "features", _lib.dngo_features(h, Xs[:3])[0, :2], "predict",
      h.predict(Xs[:300])[1][:2], "acq", h.acq(Xs[:300], _lib.ACQ_EI, float(y.min()), 0.0)["best_idx"])
r = _lib.maximize_direct([h], _lib.ACQ_EI, [float(y.min())], 0.0, np.zeros(D), np.ones(D), n_func_evals=100)
print("dngo direct", r["nit"], r["nfev"])
h.close()
# hyper-parameters at large N, blocked path: the log-posterior across two 128-row blocks in three chunks of at most two
# thetas (1 MiB of matrix and P strip each), the sampler and the optimiser
h = _lib.Handle(0)
h.set_option("hyper_batch_bytes", 2 * 1100000)
h.set_data(X[:150], y[:150])
h.set_kernel(f["family"], f["log_amp"], f["axis"], f["group"], f["log_metric"])
_lib.set_hyper_model(h, f["slots"], len(f["axis"]), float(y[:150].mean()), 1.25e-12)
Th = np.c_[rng.uniform(-1, 1, (5, 4)), rng.uniform(-6, -2, 5)]
print("hyper blocked", _lib.hyper_lnpost_blocked(h, Th)[0][:2],
      _lib.sample_hypers_blocked(h, Th[[0, 1, 2, 3, 4, 0, 1, 2, 3, 4]], 2, 5)["lnpost"][:2],
      _lib.optimize_hypers_blocked(h, Th[0], maxiter=3)["f"])
h.close()
h = _lib.moments_handle()
print(h.acq_moments(rng.randn(100), rng.rand(100) + 0.1, _lib.ACQ_LOG_EI, 0.0, 0.0)[0][:3])
print(h.reduce_models(rng.rand(4, 50), rng.rand(4, 50))[1][:3])
print("done")
