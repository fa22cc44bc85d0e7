"""TEST INFRASTRUCTURE - specification of the dropout masks of the H100 NAR path (numpy).

The reference applies tf.layers.dropout to the three feature tensors (nar_model.py:338-340, :351-353, :367-369), to
the FC1 output (:417-419) and wraps every RNN cell in DropoutWrapper(output_keep_prob) (:1330-1333).  TF's stateful
random ops are not reproducible, so - exactly like the negative sampler (oracle/sampler_ref.py) - the masks are
DEFINED by a counter-based generator that the CUDA kernel (csrc/misc.cu: dropout_rows_kernel) and this file share:

  Philox4x32-10, key = (seed_lo, seed_hi ^ 0x5DEECE66), counter = (col >> 2, row_key_lo,
  (row_key_hi & 0xFFFFFF) | tensor_id << 24, step); the draw of element (row, col) is output word (col & 3);
  the element is KEPT iff draw < floor(keep_prob * 2^32) and then scaled by 1 / keep_prob (tf.nn.dropout).

  tensor_id 1 clicked-item feature rows, 2 positive rows, 3 negative rows, 4 FC1 output, 8 + i output of RNN layer i
  row_key   flat position b*T + t (b = GLOBAL session index), negatives: (b*T + t) * K + k
  col       feature rows: column in the INTERNAL (HBM) column order of chameleon_recsys_b200.plan.FeaturePlan;
            FC1 / RNN: unit index
Only tests/, __graft_entry__.smoke() and bench.py's reference legs may import this module.
"""
from __future__ import annotations

import numpy as np

from .sampler_ref import philox4x32_10

TID_X_IN, TID_X_POS, TID_X_NEG, TID_FC1, TID_RNN0 = 1, 2, 3, 4, 8
KEY_XOR = 0x5DEECE66


def keep_mask(seed: int, step: int, tensor_id: int, row_key, n_cols: int, keep_prob: float) -> np.ndarray:
    """bool [*row_key.shape, n_cols]: which elements survive."""
    rk = np.asarray(row_key, dtype=np.uint64)[..., None]
    col = np.arange(n_cols, dtype=np.uint64)
    c0 = (col >> np.uint64(2)).astype(np.uint32)
    c1 = (rk & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    c2 = (((rk >> np.uint64(32)) & np.uint64(0xFFFFFF)) | np.uint64(tensor_id << 24)).astype(np.uint32)
    k0 = seed & 0xFFFFFFFF
    k1 = ((seed >> 32) & 0xFFFFFFFF) ^ KEY_XOR
    w = philox4x32_10(np.broadcast_to(c0, np.broadcast_shapes(c1.shape, c0.shape)), c1, c2, np.uint32(step & 0xFFFFFFFF), k0, k1)
    sel = (col & np.uint64(3)).astype(np.int64)
    draws = np.choose(np.broadcast_to(sel, w[0].shape), [w[0], w[1], w[2], w[3]])
    thr = np.uint64(int(np.floor(keep_prob * 4294967296.0)))
    return draws.astype(np.uint64) < thr
