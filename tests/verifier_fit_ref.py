"""float64 reference of the verifier fit (train_verifier_model, openwakeword/custom_verifier_model.py:95-113 of the
original project) that the CPU and GPU tests compare the device fit against."""
import numpy as np


def fit_verifier_f64(features, labels, C=0.001, gtol=1e-13, max_iter=100):
    """train_verifier_model's fit restated in float64: StandardScaler's statistics as scikit-learn computes them (mean,
    population variance by its correction formula, scale 1 for the features it treats as constant), then the exact
    minimiser of 1/2 |w|^2 + C sum_i log(1 + exp(-s_i (w.z_i + b))) (intercept unpenalised) by Newton's method with
    dense solves, run until max |gradient| / (C n) <= gtol (scikit-learn's scaling of the gradient).
    features [N, n_in, 96] or [N, D]; labels [N] of two classes.  -> dict mean, var, scale, coef [D], intercept, iters."""
    x = np.asarray(features, np.float64).reshape(len(features), -1)
    y = np.asarray(labels).ravel()
    classes = np.unique(y)
    assert classes.size == 2, "two classes"
    t = (y == classes[1]).astype(np.float64)
    n, D = x.shape
    mean = x.sum(axis=0) / n
    dev = x - mean
    var = ((dev ** 2).sum(axis=0) - dev.sum(axis=0) ** 2 / n) / n
    eps = np.finfo(np.float64).eps
    const = var <= n * eps * var + (n * mean * eps) ** 2
    scale = np.where(const, 1.0, np.sqrt(var))
    z = np.hstack([dev / scale, np.ones((n, 1))])
    theta = np.zeros(D + 1)
    reg = np.ones(D + 1)
    reg[-1] = 0.0
    it = 0
    for it in range(1, max_iter + 1):
        m = z @ theta
        p = 0.5 * (1.0 + np.tanh(0.5 * m))
        g = reg * theta + C * (z.T @ (p - t))
        if np.abs(g).max() / (C * n) <= gtol:
            it -= 1
            break
        H = np.diag(reg) + C * (z.T * (p * (1.0 - p))) @ z
        theta = theta - np.linalg.solve(H, g)
    return {"mean": mean, "var": var, "scale": scale, "coef": theta[:D], "intercept": float(theta[D]), "iters": it}


def linear_proba(mean, scale, coef, intercept, features):
    """P(positive) of the standardized linear model in float64: features [n, n_in, 96] or [n, D] -> [n]."""
    x = np.asarray(features, np.float64).reshape(len(features), -1)
    zs = ((x - mean) / scale) @ coef + intercept
    return 0.5 * (1.0 + np.tanh(0.5 * zs))
