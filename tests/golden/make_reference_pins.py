"""Regenerate tests/golden/reference_pins.npz from a checkout of the reference project.

    python tests/golden/make_reference_pins.py <reference checkout>

What the reference-pinning tests of tests/test_oracle_golden.py compare against, stored so that
they run without the reference:

* `head_sha256` / `head_bytes` - SHA-256 of the first bytes of the reference's
  `sampledata/testSamples.csv`, as many as `samples_head.csv` holds;
* `label`, `graph_output` - the label column of all 22 440 rows of that file and what the
  serialised `modeldata/neuralcf/002` serving graph (oracle/savedmodel_graph.py) outputs for them;
* `sample_index`, `sample_movieId`, `sample_userId` - a fixed seeded sample of 2000 of those rows,
  with `user_ids` / `user_rows` the neuralcf/002 user-table rows the sample and the edge cases need;
* `edge_*` - what the graph does with out-of-range ids, the last valid ids and the "missing" id -1.

and tests/golden/bundle_pins.npz: for `modeldata/neuralcf/002` and `modeldata/MLPRec/005`, the
`variables.index` file as it is and the byte ranges of `variables.data-00000-of-00001` that hold the
model variables, the user tables only at the rows of the users the stored weight fixtures hold
(`<name>__index`, `__size`, `__offsets`, `__lengths`, `__bytes`): enough to rebuild a sparse copy of
the variables directory that the TF-free bundle reader reads like the original.
"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from oracle import savedmodel_graph as SG                            # noqa: E402
from sparrowrecsys_b200 import bundle                                # noqa: E402
from sparrowrecsys_b200.features import load_samples_csv            # noqa: E402

USER_TABLE = "layer_with_weights-1/userId_embedding.Sembedding_weights/.ATTRIBUTES/VARIABLE_VALUE"

N_SAMPLE = 2000


def raises(g, feats):
    try:
        g.run(feats)
    except ValueError:
        return True
    return False


def pins(webroot):
    out = {}
    with open(os.path.join(HERE, "samples_head.csv"), "rb") as f:
        n = len(f.read())
    with open(os.path.join(webroot, "sampledata/testSamples.csv"), "rb") as f:
        out["head_sha256"] = np.array(hashlib.sha256(f.read(n)).hexdigest())
    out["head_bytes"] = np.array(n, np.int64)
    full = load_samples_csv(os.path.join(webroot, "sampledata/testSamples.csv"))
    g = SG.ServingGraph(os.path.join(webroot, "modeldata/neuralcf/002"), bundle.read_variables)
    mid, uid = np.asarray(full["movieId"]), np.asarray(full["userId"])
    out["label"] = np.asarray(full["label"]).astype(np.uint8)
    out["graph_output"] = g.run({"movieId": mid, "userId": uid})[:, 0].astype(np.float32)
    idx = np.sort(np.random.default_rng(0).choice(len(mid), N_SAMPLE, replace=False)).astype(np.int32)
    out["sample_index"], out["sample_movieId"], out["sample_userId"] = idx, mid[idx], uid[idx]
    edge_users = np.array([7, 8, 30000], np.int32)
    W = bundle.load_neuralcf(os.path.join(webroot, "modeldata/neuralcf/002"))
    users = np.unique(np.concatenate([uid[idx], edge_users]))
    out["user_ids"], out["user_rows"] = users, W["userId_embedding"][users].astype(np.float32)
    out["edge_raises_movie_1001"] = np.array(raises(g, {"movieId": np.array([5, 1001]), "userId": np.array([7, 7])}))
    out["edge_raises_user_30001"] = np.array(raises(g, {"movieId": np.array([5, 5]), "userId": np.array([7, 30001])}))
    out["edge_last_valid"] = g.run({"movieId": np.array([5, 1000]), "userId": np.array([7, 30000])})[:, 0]
    out["edge_missing_movie"] = g.run({"movieId": np.array([-1]), "userId": np.array([7])})[:, 0]
    pair = {"movieId": np.array([3, 9]), "userId": np.array([7, 8])}
    out["edge_full_equals_partial"] = np.array(np.array_equal(g.run(pair), g.run(pair, full=False)))
    out["edge_pair_output"] = g.run(pair)[:, 0]
    return out


def bundle_pins(webroot):
    out = {}
    for name, rel in (("neuralcf_002", "modeldata/neuralcf/002"), ("mlprec_005", "modeldata/MLPRec/005")):
        vdir = os.path.join(webroot, rel, "variables")
        with open(os.path.join(vdir, "variables.index"), "rb") as f:
            out[name + "__index"] = np.frombuffer(f.read(), np.uint8)
        with open(os.path.join(vdir, "variables.data-00000-of-00001"), "rb") as f:
            blob = f.read()
        users = np.load(os.path.join(HERE, name + ".npz"))["user_ids"]
        ranges = []
        for key, e in bundle.read_index(os.path.join(vdir, "variables.index")).items():
            if e["dtype"] != bundle._DTYPE_FLOAT32 or e["shard"] != 0 or ".OPTIMIZER_SLOT" in key \
                    or key.startswith("optimizer/") or key.startswith("keras_api/"):
                continue
            if key == USER_TABLE:
                row = 4 * e["shape"][1]
                ranges += [(e["offset"] + int(u) * row, row) for u in users]
            else:
                ranges.append((e["offset"], e["size"]))
        out[name + "__size"] = np.array(len(blob), np.int64)
        out[name + "__offsets"] = np.array([o for o, _ in ranges], np.int64)
        out[name + "__lengths"] = np.array([n for _, n in ranges], np.int64)
        out[name + "__bytes"] = np.frombuffer(b"".join(blob[o:o + n] for o, n in ranges), np.uint8)
    return out


if __name__ == "__main__":
    webroot = os.path.join(sys.argv[1], "src/main/resources/webroot")
    np.savez_compressed(os.path.join(HERE, "reference_pins.npz"), **pins(webroot))
    np.savez_compressed(os.path.join(HERE, "bundle_pins.npz"), **bundle_pins(webroot))
