from .random_sampling import RandomSampling  # noqa: F401
from .device_random_sampling import DeviceRandomSampling  # noqa: F401
from .differential_evolution import DifferentialEvolution  # noqa: F401
from .scipy_optimizer import SciPyOptimizer  # noqa: F401
from .cmaes import CMAES  # noqa: F401
from .direct import Direct  # noqa: F401
from .grid_search import GridSearch  # noqa: F401
