"""
Golden vectors for the tuner's trial (tangram/mapping_parameter_tuning.py) from the REAL reference.

Needs a Tangram checkout: the one next to this repository, or the one TANGRAM_REFERENCE names (as oracle/build_ref.py):
    python tests/golden/make_tuning_golden.py

The unmodified reference mapping_parameter_tuning.py is loaded by path as `tangram.mapping_parameter_tuning`, next to
the reference `tangram.mapping_optimizer` (also by path); `tangram.utils` and `tangram.spatial_weights` are empty stub
modules (the trial does not use them) and `ray.train` is a stub whose `report` captures the metrics dict.  Writes
tests/golden/tuning.npz:
  metric cases  m_<name>_cube (R x N x V float32) and the reference's pearson_corr / vote_entropy / consensus_entropy
  trial cases   t_<name>_*: the global numpy seed set before the call, the 12 data entries, the config, the five reported
                metrics, and per run the reference mapping's argmax and top-two gap (to recognise near-ties)
"""
import contextlib
import importlib.util
import io
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle.tangram_oracle import synthetic_inputs, grid_graph, spatial_weights_from_graph  # noqa: E402

REF = os.environ.get("TANGRAM_REFERENCE") or os.path.join(os.path.dirname(ROOT), "reference")
METRICS = ["cell_map_consistency", "cell_map_agreement", "cell_map_certainty", "gene_expr_consistency",
           "gene_expr_correctness"]


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


def load_reference():
    """-> (tangram.mapping_parameter_tuning, tangram.mapping_optimizer, list the reported dicts land in)."""
    pkg = types.ModuleType("tangram")
    pkg.__path__ = []
    sys.modules["tangram"] = pkg
    for stub in ("utils", "spatial_weights"):
        sys.modules["tangram." + stub] = types.ModuleType("tangram." + stub)
    reports = []
    ray = types.ModuleType("ray")
    ray_train = types.ModuleType("ray.train")
    ray_train.report = reports.append
    ray.train = ray_train
    sys.modules["ray"], sys.modules["ray.train"] = ray, ray_train
    mo = _load("tangram.mapping_optimizer", os.path.join(REF, "tangram", "mapping_optimizer.py"))
    mpt = _load("tangram.mapping_parameter_tuning", os.path.join(REF, "tangram", "mapping_parameter_tuning.py"))
    return mpt, mo, reports


def softmax_cube(rng, R, N, V):
    """Seeded softmax mappings with the awkward cases: exact argmax ties (also against later columns), exact zeros, a
    column that is zero in every run, a row on which all runs agree."""
    x = rng.normal(0, 2.5, (R, N, V))
    x[:, 1] = x[0, 1]                                   # row 1: identical in every run
    P = np.exp(x - x.max(axis=2, keepdims=True))
    P = (P / P.sum(axis=2, keepdims=True)).astype(np.float32)
    for r in range(R):
        for i in range(2, N, 5):                        # exact tie of the row maximum with another column
            j = int(P[r, i].argmax())
            k = (j + 1 + (i * 7 + r) % (V - 1)) % V
            P[r, i, k] = P[r, i, j]
        P[r, 3::4, rng.integers(0, V, 4)] = 0.0         # exact zeros
    P[:, 4, : V // 3] = 0.0                             # zero in every run: entr(0) = 0 in the consensus
    return P


METRIC_CASES = {"r2_37x129": (2, 37, 129, 1), "r3_37x129": (3, 37, 129, 2), "r3_64x200": (3, 64, 200, 3),
                "r5_29x131": (5, 29, 131, 4)}


def trial_case(name):
    if name == "default":
        N, V, K, T, seed = 300, 200, 80, 0, 21
        config = {"learning_rate": 0.1, "num_epochs": 60}
    else:
        N, V, K, T, seed = 280, 196, 80, 5, 22
        config = {"learning_rate": 0.1, "num_epochs": 80, "lambda_d": 0.8, "lambda_g2": 0.3, "lambda_r": 1e-6,
                  "lambda_neighborhood_g1": 0.9, "lambda_ct_islands": 0.2, "lambda_getis_ord": 0.6}
    inp = synthetic_inputs(N, V, K, seed=seed, n_types=T)
    train_idx = np.arange(0, K - 20)
    val_idx = np.arange(K - 25, K)                       # overlaps the training genes by five
    vw = nf = sw = ct = None
    if T:
        conn, dist = grid_graph(V)
        vw = spatial_weights_from_graph(conn, dist, True, True).toarray()
        nf = spatial_weights_from_graph(conn, dist, False, False).toarray()
        sw = spatial_weights_from_graph(conn, dist, False, True).toarray()
        ct = inp["ct_encode"]
    data = [inp["S"], inp["G"], None, inp["d"], "cpu", None, vw, ct, nf, sw, train_idx, val_idx]
    return data, config, 1000 + seed


DATA_KEYS = ["S", "G", "d_source", "d", "device", "print_each", "voxel_weights", "ct_encode", "neighborhood_filter",
             "spatial_weights", "train_genes_idx", "val_genes_idx"]


def main():
    mpt, mo, reports = load_reference()
    torch.set_num_threads(1)             # fixed summation order for the stored numbers
    save = {}
    for name, (R, N, V, seed) in METRIC_CASES.items():
        cube = softmax_cube(np.random.default_rng(seed), R, N, V)
        save[f"m_{name}_cube"] = cube
        save[f"m_{name}_pearson"] = mpt.pearson_corr(cube)
        save[f"m_{name}_vote"] = mpt.vote_entropy(cube)
        save[f"m_{name}_consensus"] = mpt.consensus_entropy(cube)

    outputs = []
    base_train = mo.Mapper.train

    def recording_train(self, *a, **kw):                  # keeps each run's mapping for the argmax record
        out, hist = base_train(self, *a, **kw)
        outputs.append(out)
        return out, hist

    mo.Mapper.train = recording_train
    for name in ("default", "spatial"):
        data, config, seed = trial_case(name)
        outputs.clear()
        reports.clear()
        np.random.seed(seed)
        with contextlib.redirect_stdout(io.StringIO()):
            mpt.train_multiple_Mapper(config, data)
        rep = reports[0]
        p = f"t_{name}_"
        save[p + "seed"] = np.array(seed)
        for k, v in zip(DATA_KEYS, data):
            if isinstance(v, np.ndarray):
                save[p + "in_" + k] = v
        for k, v in config.items():
            save[p + "cfg_" + k] = np.array(v)
        save[p + "metrics"] = np.array([float(rep[m]) for m in METRICS])
        srt = np.sort(np.stack(outputs), axis=2)
        save[p + "argmax"] = np.stack(outputs).argmax(axis=2).astype(np.int32)
        save[p + "gap"] = (srt[:, :, -1] - srt[:, :, -2]).astype(np.float32)
        print(name, dict(zip(METRICS, save[p + "metrics"])))
    path = os.path.join(HERE, "tuning.npz")
    np.savez_compressed(path, **save)
    print("->", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
