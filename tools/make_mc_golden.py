#!/usr/bin/env python
"""Write tests/golden/mc_pmin.npz by running the reference's own joint_pmin (robo/util/mc_part.py) with
numpy.random.multivariate_normal patched to return a given draw matrix F (Nf x Nb), so that the device kernel's
restatement (tests/mc_model.py) can be checked against the reference on the same draws.

Run where the reference tree is available, with ROBO_REFERENCE naming its root (the directory that holds robo/):
    ROBO_REFERENCE=/path/to/RoBO python tools/make_mc_golden.py
Only inputs and outputs are kept; no reference code enters the repository.

Cases: Np = 1 and Np > 1; Nb = 2, 50 and 64; means so large that every draw rounds away, which makes exact ties
(numpy.argmin's first index wins) and clamps the other points to 1e-70; a singular V that needs the jitter ladder.
"""
import importlib.util
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("ROBO_REFERENCE")
OUT = os.path.join(ROOT, "tests", "golden", "mc_pmin.npz")


def _load_reference():
    if not REF:
        raise SystemExit("set ROBO_REFERENCE to the root of the reference tree (the directory that holds robo/)")
    spec = importlib.util.spec_from_file_location("ref_mc_part", os.path.join(REF, "robo", "util", "mc_part.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _spd(nb, rng):
    A = rng.randn(nb, nb)
    return A @ A.T / nb + 0.05 * np.eye(nb)


def _cases():
    rng = np.random.RandomState(2024)
    out = []
    for nb, np_, nf in [(2, 1, 400), (2, 5, 300), (50, 1, 120), (50, 20, 40), (64, 1, 80), (64, 9, 30)]:
        out.append(("spd_nb%d_np%d" % (nb, np_), rng.randn(nb, np_) * 0.3, _spd(nb, rng), nf))
    out.append(("ties_clamp", np.array([[5e17], [1e17], [1e17], [3e17]]), np.eye(4), 300))
    V = _spd(6, rng)
    V[4], V[:, 4] = V[2], V[:, 2]                           # a duplicated row: singular, climbs the jitter ladder
    out.append(("singular", rng.randn(6, 3) * 0.1, V, 250))
    out.append(("rank_one", np.zeros((3, 1)), np.ones((3, 3)), 200))
    return out


def main():
    ref = _load_reference()
    data = {}
    names = []
    for name, m, V, nf in _cases():
        nb = m.shape[0]
        F = np.random.RandomState(len(names) + 7).randn(nf, nb)          # the reference's layout: Nf x Nb
        orig = np.random.multivariate_normal
        np.random.multivariate_normal = lambda mean, cov, size: F.copy()
        try:
            pmin = ref.joint_pmin(m, V, nf)
        finally:
            np.random.multivariate_normal = orig
        names.append(name)
        data[name + "/m"], data[name + "/V"], data[name + "/F"], data[name + "/pmin"] = m, V, F, pmin
    data["names"] = np.array(names)
    np.savez_compressed(OUT, **data)
    print("wrote", OUT, names)


if __name__ == "__main__":
    main()
