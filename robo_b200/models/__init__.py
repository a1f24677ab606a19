from .gaussian_process import GaussianProcess  # noqa: F401
from .gaussian_process_mcmc import GaussianProcessMCMC  # noqa: F401
from .fabolas_gp import FabolasGP, FabolasGPMCMC  # noqa: F401
from .mtbo_gp import MTBOGP, MTBOGPMCMC  # noqa: F401
from .bayesian_linear_regression import BayesianLinearRegression  # noqa: F401
from .random_forest import RandomForest  # noqa: F401
from .wrapper_bohamiann import WrapperBohamiann  # noqa: F401
from .dngo import DNGO  # noqa: F401
