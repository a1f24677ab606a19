"""Fabolas's incumbent (robo/util/incumbent_estimation.py: projected_incumbent_estimation): every observed configuration
is moved to the environment value ``proj_value`` (s = 1: the whole dataset) and the one with the lowest predicted mean
wins.  The prediction is the model's device ``predict``."""
import numpy as np


def projected_incumbent_estimation(model, X, proj_value=1):
    """-> (the winning row of X extended by proj_value, its predicted mean)."""
    X_env = np.hstack([X, np.full((X.shape[0], 1), proj_value, dtype=np.float64)])
    mean = model.predict(X_env)[0]
    i = int(np.argmin(mean))
    return X_env[i], mean[i]
