"""Host-side pieces of bench.py that need no GPU: the contract of the JSON line depends on them."""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def test_synthetic_ids_survive_the_float32_round_trip_of_the_graph():
    """DIN.py:95,125 feeds the movie ids through float32: the last ids of a 10^8 vocabulary round UP to the
    vocabulary size (TF would assert).  The generator must not draw them - the first cfg-5 sweep of round 2 failed
    on exactly those ids - and must leave small vocabularies alone."""
    from sparrowrecsys_b200.features import synthetic_features
    from sparrowrecsys_b200.spec import baseline_spec
    big = baseline_spec("cfg5_din")
    f = synthetic_features(big, 2048, seed=3, uniform_history=True)
    keys = ["movieId"] + ["userRatedMovie%d" % (k + 1) for k in range(big.hist_len)]
    ids = np.concatenate([np.asarray(f[k]) for k in keys]).astype(np.int64)
    assert ids.max() > 2 ** 26                                    # the whole vocabulary is in play
    assert ids.astype(np.float32).astype(np.int64).max() < big.n_movies
    z = synthetic_features(big, 2048, seed=3)                     # Zipf tail is clipped the same way
    zid = np.concatenate([np.asarray(z[k]) for k in keys]).astype(np.int64)
    assert zid.astype(np.float32).astype(np.int64).max() < big.n_movies
    small = baseline_spec("cfg3_din")
    g = synthetic_features(small, 4096, seed=3, uniform_history=True)
    assert int(np.asarray(g["movieId"]).max()) <= small.n_movies - 1
    assert int(np.asarray(g["movieId"]).max()) > small.n_movies - 200   # ... and still reaches the top of it


def test_tiled_dataset_holds_the_same_rows_in_other_orders():
    import bench
    from sparrowrecsys_b200.features import encode_batch, synthetic_features
    from sparrowrecsys_b200.spec import baseline_spec
    spec = baseline_spec("cfg3_din")
    enc = encode_batch(spec, synthetic_features(spec, 64, seed=5))
    big = bench.tile_encoded(enc, 3, np.random.default_rng(0))
    assert big.B == 3 * 64 and big.hist.shape == (192, enc.hist.shape[1])
    assert np.array_equal(big.hist[:64], enc.hist)                # replica 0 is the original order
    key = lambda e, lo, hi: sorted(map(tuple, np.column_stack([e.movie_id[lo:hi], e.user_id[lo:hi], e.hist[lo:hi]])))
    assert key(big, 64, 128) == key(enc, 0, 64) == key(big, 128, 192)
    assert not np.array_equal(big.hist[64:128], enc.hist)         # ... permuted
    assert bench.tile_encoded(enc, 1, np.random.default_rng(0)) is enc


def test_both_arms_print_the_same_config():
    import bench
    a = bench.parse_args(["--workload", "cfg3_din"])
    b = bench.parse_args(["--workload", "cfg3_din", "--impl", "reference"])
    from sparrowrecsys_b200.spec import baseline_spec
    spec = baseline_spec("cfg3_din")
    assert bench.shared_config(a, spec, 1) == bench.shared_config(b, spec, 1)
    c = bench.shared_config(a, spec, 4)
    assert c["global_batch"] == 4 * c["batch_per_gpu"] and "workload" in c
    assert not bench.parse_args(["--workload", "cfg5_din"]).no_graph      # every workload replays a CUDA graph
    assert bench.parse_args(["--workload", "cfg5_din", "--no-graph"]).no_graph
    assert not bench.parse_args([]).no_graph


def test_stdout_of_the_reference_arm_is_one_json_line():
    """stdout carries the JSON line and nothing else, even when libraries print banners there."""
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--batch", "64",
                        "--steps", "2", "--warmup", "1"], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.strip()]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["unit"] == "inferences/s" and d["value"] > 0
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["cpu_baseline"]["kind"] == "port"
    assert d["dtype"] == "f32" and d["higher_is_better"] is True


def test_dump_outputs_writes_float32_scores_and_a_fixed_sample_above_the_limit(tmp_path, monkeypatch):
    import bench
    small = np.random.default_rng(1).random((3, 5), dtype=np.float32)
    bench.dump_outputs(str(tmp_path / "a"), small)
    got = np.load(tmp_path / "a" / "scores.npy")
    assert got.dtype == np.float32 and np.array_equal(got, small)
    assert not (tmp_path / "a" / "scores_index.npy").exists()
    monkeypatch.setattr(bench, "DUMP_LIMIT_BYTES", 64)              # 8 values + their indices
    big = np.arange(1000, dtype=np.float32).reshape(10, 100)
    for d in ("b", "c"):
        bench.dump_outputs(str(tmp_path / d), big)
    idx, vals = np.load(tmp_path / "b" / "scores_index.npy"), np.load(tmp_path / "b" / "scores.npy")
    assert len(idx) == 8 and np.array_equal(vals, big.reshape(-1)[idx])
    assert np.array_equal(idx, np.load(tmp_path / "c" / "scores_index.npy"))   # the same sample every run
    assert vals.nbytes + idx.nbytes <= 64
