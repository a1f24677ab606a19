"""RandomForest — RoBO's random forest (robo/models/random_forest.py) on the GPU, without the pyrfr package.

Same constructor, attributes (``X``, ``y``, ``rng``, ``n_points_per_tree``) and methods as the reference.  pyrfr's
source is not available, so the forest it grows is restated (robo_b200/csrc/gpk_rf.cuh states it step by step, DESIGN
§1 row a25): bagged CART regression trees on the residual sum of squares, every feature tried at every node, no depth
limit.  ``train`` grows every tree on the device in one call (gpk_rf_fit); ``predict`` and every device acquisition
score candidates in one pass with a warp per candidate walking all trees, where the reference loops predict_mean_var
over the rows in Python.

Random numbers: as the reference, ``__init__`` takes one ``rng.randint(1000)`` to seed the forest's engine and
``__setstate__`` one more; nothing else reads ``rng``, so a BO run sharing it draws the same numbers for everything
else.  The engine is a counter-based Philox stream keyed by that seed whose counter advances once per ``train``, as
pyrfr's engine advances from fit to fit; a copy starts a new engine, as the reference's does.

Pickling and deepcopy drop the device handle; the trees are read back once per ``train`` and a copy re-uploads them,
so it predicts bit-identically.  ``predict_each_tree`` and ``sample_functions`` are the reference's stubs, and
``compute_oob_error`` is stored and otherwise unused (RoBO never reads the OOB error).
"""
import numpy as np

from robo_b200 import _lib
from robo_b200.models.base_model import BaseModel


class RandomForest(BaseModel):

    def __init__(self, num_trees=30, do_bootstrapping=True, n_points_per_tree=0, compute_oob_error=False,
                 return_total_variance=True, rng=None, device=0):
        if rng is None:
            self.rng = np.random.RandomState()
        else:
            self.rng = rng
        self.seed = int(self.rng.randint(1000))
        self.counter = 0
        self.n_points_per_tree = n_points_per_tree
        self.num_trees = int(num_trees)
        self.do_bootstrapping = bool(do_bootstrapping)
        self.compute_oob_error = compute_oob_error
        self.return_total_variance = bool(return_total_variance)
        if not 1 <= self.num_trees <= _lib.RF_MAX_T:
            raise ValueError("RandomForest: num_trees must lie in 1 .. GPK_RF_MAX_T = %d" % _lib.RF_MAX_T)
        if int(n_points_per_tree) < 0:
            raise ValueError("RandomForest: n_points_per_tree must be >= 0")
        self.X = None
        self.y = None
        self.trees = None
        self.device = int(device)
        self._handle = None

    # ---- device state: the handle does not survive pickling / deepcopy; _ready_handle re-uploads the trees ----------
    def __getstate__(self):
        st = self.__dict__.copy()
        st["_handle"] = None
        return st

    def __setstate__(self, st):
        self.__dict__.update(st)
        # random_forest.py:122-124: a new engine from the copy's rng
        self.seed = int(st["rng"].randint(1000))
        self.counter = 0

    def _upload(self):
        if self._handle is None:
            self._handle = _lib.Handle(self.device)
        _lib.rf_set_data(self._handle, self.X, self.y)
        return self._handle

    def _ready_handle(self):
        """The handle with the trained forest resident (scoring entry points take it)."""
        if self.trees is None:
            raise ValueError("RandomForest: train the model first")
        if self._handle is None:
            _lib.rf_set_trees(self._upload(), self.trees, self.return_total_variance)
        return self._handle

    def train(self, X, y, **kwargs):
        """Grow the forest on X (N, D) and y (N,) (random_forest.py:59-83)."""
        self.X = X
        self.y = y
        X = np.asarray(X, dtype=np.float64)
        y = np.asarray(y, dtype=np.float64).ravel()
        if X.ndim != 2 or X.shape[0] != y.size:
            raise ValueError("RandomForest: X must be (N, D) and y (N,)")
        if X.shape[0] > _lib.RF_MAX_N:
            raise ValueError("RandomForest: %d training points exceed GPK_RF_MAX_N = %d" % (X.shape[0], _lib.RF_MAX_N))
        if X.shape[1] > _lib.RF_MAX_D:
            raise ValueError("RandomForest: %d input dimensions exceed GPK_RF_MAX_D = %d" % (X.shape[1], _lib.RF_MAX_D))
        n_t = int(self.n_points_per_tree) if self.n_points_per_tree != 0 else X.shape[0]
        if not self.do_bootstrapping and n_t > X.shape[0]:
            raise ValueError("RandomForest: without bootstrapping a tree cannot take %d of %d points" % (n_t, X.shape[0]))
        self.trees = None
        h = self._upload()
        _lib.rf_fit(h, self.seed, self.counter, self.num_trees, n_t, self.do_bootstrapping,
                    self.return_total_variance)
        self.counter += 1
        self.trees = _lib.rf_trees(h)

    def predict(self, X_test, **kwargs):
        """Mean and variance over the trees at every row (random_forest.py:85-109): one device pass."""
        return self._ready_handle().predict(np.asarray(X_test, dtype=np.float64))

    def predict_each_tree(self, X_test, **args):
        pass

    def sample_functions(self, X_test, n_funcs=1):
        pass
