"""A minimal import-level stand-in for `lightfm` (test infrastructure only).  It is NOT LightFM: it does no training.

It lets the unmodified RecTools `LightFMWrapperModel` (rectools/models/lightfm.py) import, "fit" and recommend where the
real package is not installed, so that tests can inject the factors they need (small biases, a dominant user bias,
heavy-tailed item norms) and rank them.  It covers exactly these calls:

* `LightFM(no_components, k, n, learning_schedule, loss, learning_rate, rho, epsilon, item_alpha, user_alpha, max_sampled,
  random_state)`: every argument kept as an attribute of the same name (the wrapper's `_get_config` reads them), the
  seed also as `initial_random_state`;
* `fit_partial(interactions, user_features=None, item_features=None, sample_weight=None, epochs=1, num_threads=1,
  verbose=False)`: on the first call fills `user_embeddings` / `item_embeddings` (n_features x `no_components`) and
  `user_biases` / `item_biases` (n_features), float32, from a generator seeded with `random_state`.  n_features is the
  number of columns of the feature matrix, or the number of users / items of `interactions` without one.  Later calls
  keep the arrays (tests overwrite them);
* `get_user_representations(features=None)` / `get_item_representations(features=None)`: lightfm's documented semantics,
  `(features @ biases, features @ embeddings)`, and the raw arrays when `features` is None.
"""
from __future__ import annotations

import typing as tp

import numpy as np
from scipy import sparse

__version__ = "0.0.0+stub"


class LightFM:  # pylint: disable=too-many-instance-attributes
    def __init__(self, no_components: int = 10, k: int = 5, n: int = 10, learning_schedule: str = "adagrad",
                 loss: str = "logistic", learning_rate: float = 0.05, rho: float = 0.95, epsilon: float = 1e-6,
                 item_alpha: float = 0.0, user_alpha: float = 0.0, max_sampled: int = 10, random_state: tp.Any = None) -> None:
        self.no_components = no_components
        self.k = k
        self.n = n
        self.learning_schedule = learning_schedule
        self.loss = loss
        self.learning_rate = learning_rate
        self.rho = rho
        self.epsilon = epsilon
        self.item_alpha = item_alpha
        self.user_alpha = user_alpha
        self.max_sampled = max_sampled
        self.random_state = random_state
        self.initial_random_state = random_state
        self.user_embeddings: tp.Optional[np.ndarray] = None
        self.item_embeddings: tp.Optional[np.ndarray] = None
        self.user_biases: tp.Optional[np.ndarray] = None
        self.item_biases: tp.Optional[np.ndarray] = None

    def fit_partial(self, interactions: tp.Any, user_features: tp.Any = None, item_features: tp.Any = None,
                    sample_weight: tp.Any = None, epochs: int = 1, num_threads: int = 1, verbose: bool = False) -> "LightFM":  # pylint: disable=unused-argument
        if self.user_embeddings is None:
            n_users, n_items = interactions.shape
            n_user_features = n_users if user_features is None else user_features.shape[1]
            n_item_features = n_items if item_features is None else item_features.shape[1]
            seed = self.random_state if isinstance(self.random_state, (int, np.integer)) else 0
            rng = np.random.default_rng(seed)
            nc = self.no_components
            self.user_embeddings = ((rng.random((n_user_features, nc)) - 0.5) / nc).astype(np.float32)
            self.item_embeddings = ((rng.random((n_item_features, nc)) - 0.5) / nc).astype(np.float32)
            self.user_biases = (0.1 * rng.standard_normal(n_user_features)).astype(np.float32)
            self.item_biases = (0.1 * rng.standard_normal(n_item_features)).astype(np.float32)
        return self

    def fit(self, interactions: tp.Any, **kwargs: tp.Any) -> "LightFM":
        self.user_embeddings = self.item_embeddings = self.user_biases = self.item_biases = None
        return self.fit_partial(interactions, **kwargs)

    @staticmethod
    def _represent(features: tp.Any, biases: np.ndarray, embeddings: np.ndarray) -> tp.Tuple[np.ndarray, np.ndarray]:
        if features is None:
            return biases, embeddings
        features = sparse.csr_matrix(features, dtype=np.float32)
        return features @ biases, features @ embeddings

    def get_user_representations(self, features: tp.Any = None) -> tp.Tuple[np.ndarray, np.ndarray]:
        return self._represent(features, self.user_biases, self.user_embeddings)

    def get_item_representations(self, features: tp.Any = None) -> tp.Tuple[np.ndarray, np.ndarray]:
        return self._represent(features, self.item_biases, self.item_embeddings)
