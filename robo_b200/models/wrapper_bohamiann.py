"""WrapperBohamiann — RoBO's Bayesian neural network (robo/models/wrapper_bohamiann.py) on the GPU, without pybnn.

Same constructor arguments, ``train(X, y)``, ``predict(X_test)`` and ``get_incumbent`` as the reference.  pybnn's source
is not available, so the network and its sampler are restated (robo_b200/csrc/gpk_bnn.cuh states them step by step,
DESIGN §1 row a28): the wrapper's D -> 50 -> 50 -> 1 tanh network with a homoscedastic log-variance, inputs and targets
normalised, sampled by adaptive SGHMC with the wrapper's chain length (100 N burn-in steps, then 10,000 more, one
network kept every 100 steps: 99 networks).  ``train`` runs the whole chain on the device in one launch; ``predict``
and every device acquisition score candidates in one pass over the kept networks.

Only the default architecture runs on the device: ``get_net`` other than this module's ``get_default_network`` raises
TypeError, and ``use_double_precision=False`` raises ValueError (the device chain is fp64).  ``verbose`` is accepted
and unused: the chain prints nothing.

Random numbers: ``__init__`` takes one draw from ``rng`` (np.random when None) to seed the chain's Philox stream, and
every ``train`` advances a counter, so each train starts a fresh chain (pybnn's ``continue_training=False``).

Pickling and deepcopy drop the device handle; the kept networks are read back once per ``train`` and a copy re-uploads
them with the training set, so it predicts bit-identically.
"""
import numpy as np

from robo_b200 import _lib
from robo_b200.models.base_model import BaseModel

LR, MDECAY, EPS, KEEP_EVERY, BATCH = 1e-2, 0.05, 1e-10, 100, 20


def get_default_network(input_dimensionality):
    """The reference's network as a torch module (wrapper_bohamiann.py:10-34), for users who want it on the host; the
    device builds the same architecture itself.  torch is imported here only."""
    import torch

    class AppendLayer(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.bias = torch.nn.Parameter(torch.full((1, 1), float(np.log(1e-2)), dtype=torch.float64))

        def forward(self, x):
            return torch.cat((x, self.bias * torch.ones_like(x)), dim=1)

    net = torch.nn.Sequential(
        torch.nn.Linear(input_dimensionality, 50), torch.nn.Tanh(),
        torch.nn.Linear(50, 50), torch.nn.Tanh(),
        torch.nn.Linear(50, 1),
        AppendLayer()).double()
    for m in net:
        if isinstance(m, torch.nn.Linear):
            torch.nn.init.kaiming_normal_(m.weight, mode="fan_in", nonlinearity="linear")
            torch.nn.init.constant_(m.bias, 0.0)
    return net


def chain_settings(n):
    """(burn_in, num_steps) of the wrapper's chain on n training points (wrapper_bohamiann.py:63-68)."""
    return 100 * n, 100 * n + 10000


class WrapperBohamiann(BaseModel):

    def __init__(self, get_net=get_default_network, lr=1e-2, use_double_precision=True, verbose=True, rng=None,
                 device=0):
        if get_net is not get_default_network:
            raise TypeError("WrapperBohamiann: the device builds only the default network (get_default_network)")
        if not use_double_precision:
            raise ValueError("WrapperBohamiann: the device chain runs in double precision only")
        self.lr = float(lr)
        self.verbose = verbose
        self.rng = rng if rng is not None else np.random
        self.seed = int(self.rng.randint(2 ** 31 - 1))
        self.counter = 0
        self.X = None
        self.y = None
        self.samples = None
        self.device = int(device)
        self._handle = None

    # ---- device state: the handle does not survive pickling / deepcopy; _ready_handle re-uploads the networks -------
    def __getstate__(self):
        st = self.__dict__.copy()
        st["_handle"] = None
        return st

    def _upload(self):
        if self._handle is None:
            self._handle = _lib.Handle(self.device)
        _lib.bnn_set_data(self._handle, self.X, self.y)
        return self._handle

    def _ready_handle(self):
        """The handle with the kept networks resident (scoring entry points take it)."""
        if self.samples is None:
            raise ValueError("WrapperBohamiann: train the model first")
        if self._handle is None:
            _lib.bnn_set_samples(self._upload(), self.samples)
        return self._handle

    def train(self, X, y, **kwargs):
        """Sample the network on X (N, D) and y (N,) with the wrapper's chain (wrapper_bohamiann.py:61-68)."""
        self.X = X
        self.y = y
        X = np.asarray(X, dtype=np.float64)
        y = np.asarray(y, dtype=np.float64).ravel()
        if X.ndim != 2 or X.shape[0] != y.size:
            raise ValueError("WrapperBohamiann: X must be (N, D) and y (N,)")
        if X.shape[0] > _lib.BNN_MAX_N:
            raise ValueError("WrapperBohamiann: %d training points exceed GPK_BNN_MAX_N = %d"
                             % (X.shape[0], _lib.BNN_MAX_N))
        if X.shape[1] > _lib.BNN_MAX_D:
            raise ValueError("WrapperBohamiann: %d input dimensions exceed GPK_BNN_MAX_D = %d"
                             % (X.shape[1], _lib.BNN_MAX_D))
        self.samples = None
        h = self._upload()
        burn_in, num_steps = chain_settings(X.shape[0])
        _lib.bnn_train(h, self.seed, self.counter, self.lr, MDECAY, EPS, burn_in, num_steps, KEEP_EVERY, BATCH)
        self.counter += 1
        self.samples = _lib.bnn_samples(h)

    def predict(self, X_test, **kwargs):
        """Predictive mean and variance over the kept networks at every row: one device pass."""
        return self._ready_handle().predict(np.asarray(X_test, dtype=np.float64))
