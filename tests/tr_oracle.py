"""NumPy restatement of one TREGO region (trieste/acquisition/rule.py:1585-1703, 1923-2035), written from the reference
and independent of trieste_b200/rule.py: the state after the first initialisation is global mode with eps = zeta * widths
and an infinite best value; ``update`` takes the best observation over the whole dataset."""
import numpy as np


class TregoRegion:
    def __init__(self, lower, upper, beta=0.7, kappa=1e-4, zeta=0.5, min_eps=1e-2):
        self.glo = np.asarray(lower, dtype=np.float64)
        self.gup = np.asarray(upper, dtype=np.float64)
        self.beta, self.kappa, self.min_eps = beta, kappa, min_eps
        self.eps = zeta * (self.gup - self.glo)
        self.is_global = True
        self.y_best = np.inf
        self.centre = None
        self.lower, self.upper = self.glo, self.gup

    def update(self, X: np.ndarray, y: np.ndarray) -> None:
        i = int(np.argmin(y[:, 0]))
        volume = np.prod(self.upper - self.lower)
        success = bool(y[i, 0] < self.y_best - self.kappa * volume)
        if not self.is_global:  # the size only moves after a local step
            self.eps = self.eps / self.beta if success else self.eps * self.beta
        if success:
            self.centre, self.y_best = X[i], float(y[i, 0])
        self.is_global = success or not self.is_global
        if self.is_global:
            self.lower, self.upper = self.glo, self.gup
        else:
            self.lower = np.maximum(self.glo, self.centre - self.eps)
            self.upper = np.minimum(self.gup, self.centre + self.eps)
        if np.any(self.eps < self.min_eps):
            raise AssertionError("the region would re-initialise at a random centre: run fewer steps")

    def sample(self, n: int, seed: int) -> np.ndarray:
        u = np.random.default_rng(seed).uniform(size=(n, len(self.glo)))
        return self.lower + u * (self.upper - self.lower)
