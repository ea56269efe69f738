"""float64 restatement of Spark ML 2.4's `LSHModel.approxSimilarityJoin(datasetA, datasetB, threshold)` for the
BucketedRandomProjectionLSH of `oracle/lsh.py`, as Spark plans it: explode each side's hash vector into (table,
bucket) rows, equi-join A and B on (table, bucket), `distinct()` over the (rowA, rowB) pairs, add the distance and keep
`distCol < threshold`.  DESIGN.md section 4.14 gives the semantics.

THIS IS THE READABLE SPEC, NOT PRODUCT.  Restated from memory of Spark's source, like the rest of `oracle/lsh.py`; it
shares no step with the device algorithm (no sort of bucket ids, no first-table rule).  Ids are unique within each
side, so Spark's distinct over row structs is distinct over (id_a, id_b); the order Spark leaves open is (id_a,
id_b) ascending here.
"""
from __future__ import annotations

import numpy as np

from oracle.lsh import transform


def approx_similarity_join(ids_a, x_a, ids_b, x_b, uv, bucket_length, threshold):
    """Every (a, b) sharing a bucket in at least one table, once, with sqrt(sum_d (x_a - x_b)^2) < threshold (summed
    over d ascending from 0.0 in double).  Returns (ids_a int32 [P], ids_b int32 [P], distances float64 [P]) by
    (id_a, id_b) ascending."""
    uv = np.asarray(uv, np.float64)
    xa = np.asarray(x_a, np.float32).astype(np.float64).reshape(-1, uv.shape[1])
    xb = np.asarray(x_b, np.float32).astype(np.float64).reshape(-1, uv.shape[1])
    ids_a, ids_b = np.asarray(ids_a, np.int64), np.asarray(ids_b, np.int64)
    L, nb = uv.shape[0], xb.shape[0]
    ha, hb = transform(xa, uv, bucket_length), transform(xb, uv, bucket_length)
    # explode B and build the join's hash side: (table, bucket) -> B rows (Python's float keys: -0.0 == 0.0)
    build = {}
    for r in range(nb):
        for j in range(L):
            build.setdefault((j, float(hb[r, j])), []).append(r)
    # explode A and probe
    pa, pb = [np.zeros(0, np.int64)], [np.zeros(0, np.int64)]
    for r in range(xa.shape[0]):
        for j in range(L):
            rows = build.get((j, float(ha[r, j])))
            if rows:
                pa.append(np.full(len(rows), r, np.int64))
                pb.append(np.asarray(rows, np.int64))
    # distinct (rowA, rowB)
    pair = np.unique(np.concatenate(pa) * nb + np.concatenate(pb))
    a, b = pair // max(nb, 1), pair % max(nb, 1)
    acc = np.zeros(len(pair))
    for d in range(uv.shape[1]):
        diff = xa[a, d] - xb[b, d]
        acc = acc + diff * diff
    dist = np.sqrt(acc)
    keep = dist < threshold
    a, b, dist = a[keep], b[keep], dist[keep]
    order = np.lexsort((ids_b[b], ids_a[a]))
    return ids_a[a[order]].astype(np.int32), ids_b[b[order]].astype(np.int32), dist[order]
