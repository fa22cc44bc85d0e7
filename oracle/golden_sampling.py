"""TEST INFRASTRUCTURE - how tests/golden/make_model_golden.py keeps its fixture small, shared with the tests that read it.

* Variables are not stored: the generator hands the reference graph variables that are a seeded function of the variable's
  TF name, shape and the mean / std of the reference's own initializer, and stores only those statistics.
* Large outputs (gradients, Adam deltas, logits, intermediates) are stored at a fixed seeded sample of their entries.
"""
from __future__ import annotations

import zlib

import numpy as np


def preset_variable(name: str, shape, mean: float, std: float) -> np.ndarray:
    """float32 value of variable `name`: mean + std * N(0, 1) from a generator seeded by the name; biases, beta and gamma
    (zero- or one-initialised in TF) get N(0, 0.1) on top so that they count."""
    rs = np.random.RandomState(zlib.crc32(name.encode()) & 0x7fffffff)
    a = float(mean) + float(std) * rs.standard_normal(tuple(int(s) for s in shape))
    if name.endswith('bias') or name.endswith('beta_center') or name.endswith('gamma_scale'):
        a = a + rs.normal(0, 0.1, a.shape)
    return a.astype(np.float32)


def preset_variables(d, case: str) -> dict:
    """{TF name: value} of the variables of golden case `case` (d: the loaded model_golden.npz)."""
    P = case + '/'
    return {str(n): preset_variable(str(n), [s for s in shp if s >= 0], *st)
            for n, st, shp in zip(d[P + 'var_names'], d[P + 'var_stats'], d[P + 'var_shapes'])}


def sample_index(n: int, k: int) -> np.ndarray:
    """Sorted fixed sample of k of the flat indices [0, n) (all of them when n <= k)."""
    if n <= k:
        return np.arange(n)
    return np.sort(np.random.RandomState(n).choice(n, k, replace=False))
