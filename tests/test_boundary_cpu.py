"""CPU-only checks of the drop-in boundary: the C-ABI library builds, loads and exports every
symbol include/gpk.h declares; host-side logic of the george-compatible kernels; and the
product never falls back to a CPU path (it must fail loudly without a GPU)."""
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    src = open(os.path.join(ROOT, "include", "gpk.h")).read()
    return sorted(set(re.findall(r"\b(gpk_[a-z_0-9]+)\s*\(", src)))


def test_library_builds_and_exports_every_declared_symbol():
    from robo_b200 import _lib
    lib = _lib.load()
    declared = _declared_symbols()
    assert len(declared) >= 20
    for name in declared:
        assert hasattr(lib, name), "libgpk.so does not export %s" % name
    assert set(declared) == set(_lib.exported_symbols())
    assert b"sm_90a" in lib.gpk_version()


def test_library_is_sm90a_with_tma_dmma_and_wgmma():
    """the built cubin must be Hopper-native: TMA (UTMALDG) staging, DMMA and int8 warpgroup MMA (IGMMA) tensor ops."""
    import subprocess
    from robo_b200 import _lib
    _lib.load()
    out = subprocess.run(["cuobjdump", "-sass", _lib.library_path()], stdout=subprocess.PIPE,
                         stderr=subprocess.STDOUT, text=True).stdout
    if "sm_90a" not in out and "SM90" not in out.upper():
        pytest.skip("cuobjdump not available")
    assert "UTMALDG" in out and "DMMA" in out and "SYNCS" in out and "IGMMA" in out


def test_no_cpu_fallback_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from robo_b200 import _lib
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        _lib.Handle(0)
    from robo_b200.models.gaussian_process import GaussianProcess
    from robo_b200 import kernels as K
    m = GaussianProcess(K.Matern52Kernel(np.ones(2), ndim=2), normalize_input=False)
    with pytest.raises(RuntimeError):
        m.train(np.random.rand(5, 2), np.random.rand(5), do_optimize=False)


def test_product_never_imports_oracle():
    for dirpath, _, files in os.walk(os.path.join(ROOT, "robo_b200")):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle", src, re.M), f


def test_kernel_algebra_matches_george_layout():
    from robo_b200 import kernels as K
    k = 2 * K.Matern52Kernel(np.ones(3), ndim=3)          # fmin/bayesian_optimization.py:79-81
    assert len(k) == 4
    np.testing.assert_allclose(k.get_parameter_vector(), [np.log(2.0 / 3), 0, 0, 0])
    k.set_parameter_vector([0.3, -1, -2, -3])
    np.testing.assert_allclose(k[:], [0.3, -1, -2, -3])
    f = k.flatten()
    assert f["family"] == 0 and f["group"] == [0, 0, 0] and f["axis"] == [0, 1, 2]
    assert f["log_amp"] == pytest.approx(0.3) and f["log_metric"] == [-1, -2, -3]
    # fabolas.py:104-110: product of 1-D kernels, one group per axis
    k = 1
    for d in range(3):
        k *= K.Matern52Kernel(np.ones([1]) * 0.01, ndim=4, axes=d)
    f = k.flatten()
    assert len(k) == 4 and f["group"] == [0, 1, 2] and f["axis"] == [0, 1, 2]
    assert f["log_amp"] == pytest.approx(np.log(1.0 / 4))
    import copy
    k2 = copy.deepcopy(k)
    k2.set_parameter_vector([0.0, 1.0, 2.0, 3.0])
    assert k[1] == pytest.approx(np.log(0.01)) and k2[1] == 1.0
    with pytest.raises(NotImplementedError):
        (K.Matern52Kernel(1.0, ndim=1) + K.Matern52Kernel(2.0, ndim=1)).flatten()
    iso = K.ExpSquaredKernel(0.5, ndim=3)
    assert len(iso) == 1 and iso.flatten()["log_metric"] == [np.log(0.5)] * 3


def test_model_api_surface_matches_reference():
    import inspect
    from robo_b200.models.gaussian_process import GaussianProcess
    sig = inspect.signature(GaussianProcess.__init__)
    names = list(sig.parameters)[1:]
    assert names[:9] == ["kernel", "prior", "noise", "use_gradients", "normalize_output",
                         "normalize_input", "lower", "upper", "rng"]
    assert sig.parameters["noise"].default == 1e-3 and sig.parameters["normalize_input"].default is True
    for meth in ["train", "predict", "nll", "grad_nll", "optimize", "predict_variance", "sample_functions",
                 "get_incumbent", "get_noise", "update", "get_json_data"]:
        assert callable(getattr(GaussianProcess, meth))
    from robo_b200 import kernels as K
    m = GaussianProcess(K.Matern52Kernel(np.ones(2), ndim=2))
    with pytest.raises(Exception, match="Model has to be trained first!"):
        m.predict(np.zeros((3, 2)))
    with pytest.raises(AssertionError):
        m.train(np.zeros((3, 2)), np.zeros((4,)))


def test_bench_reference_arm_contract_and_loud_failure_without_gpu():
    """bench.py --impl reference prints the contract's JSON line from the oracle port on the host cores; the product arm
    must refuse to run without a CUDA device (no CPU fallback)."""
    import json
    import subprocess
    import sys
    import torch
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0"],
                         capture_output=True, text=True, timeout=900, cwd=root)
    assert out.returncode == 0, out.stderr[-2000:]
    line = json.loads(out.stdout.strip().splitlines()[-1])
    assert line["impl"] == "reference" and line["unit"] == "EI evals/s" and line["higher_is_better"] is True
    assert line["steps"] == 1 and line["n_gpus"] == 1 and line["value"] > 0
    assert line["e2e"] == {"value": line["value"], "unit": "EI evals/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert line["cpu_baseline"]["kind"] == "port" and line["cpu_baseline"]["cores"] >= 1
    if not torch.cuda.is_available():
        out = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--steps", "1", "--warmup", "0"],
                             capture_output=True, text=True, timeout=600, cwd=root)
        assert out.returncode != 0 and "CUDA" in (out.stderr + out.stdout)

