"""Per-epoch validation inside the training loop (tgb200_set_validation, Mapper.train(val_each=)).

_val_loss_fn (mapping_optimizer.py:311-356) of the mapping after the update of every validated epoch goes to history columns
12-15 of that epoch's row, without leaving the device.  Checked here:

* against the path it replaces, written out in the tests: one `run(1)` per epoch and `validation_terms()` after each validated
  one.  The training history, the mapping and all four values are bit-identical (the same kernels on the same forward);
* against float64 formulas of _val_loss_fn recomputed from the device's own Y_ext and M, including a gene whose predicted
  column norm is clamped at eps; validation_terms() on that mapping equals the history row bit for bit;
* exactly: columns 12-15 are 0 with validation off and NaN on the rows it does not fill, the call is refused inside a step
  and on a sharded handle, epochs that are not validated cost no launch in fp32 / bf16x3, and a validated train() call
  makes no allocation, copy to the host or host sync beyond those of the same call without validation.

Observed on an H100 80GB HBM3 (700 W power limit): against float64 the four values stay within 0.003 of their bounds.
"""
import collections
import contextlib
import io

import numpy as np
import pytest

from oracle.tangram_oracle import synthetic_inputs

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
EPS = 1e-8
LR = 0.1


def _engine(precision, mode="cells", N=600, V=300, K=90, seed=0, mask=None, S=None, **lam):
    from tangram_b200 import _lib
    from tangram_b200.engine import Engine
    inp = synthetic_inputs(N, V, K, seed=seed, clusters=mode == "clusters")
    if S is not None:
        inp["S"] = S
    if mode == "constrained":
        e = Engine(N, V, K, precision=precision, density_mode=_lib.DENSITY_CELLS, constrained=True, lambda_d=1.0,
                   lambda_count=1.0, lambda_f_reg=1.0, target_count=float(V), **lam)
    else:
        e = Engine(N, V, K, precision=precision, lambda_d=1.0,
                   density_mode=_lib.DENSITY_SOURCE if mode == "clusters" else _lib.DENSITY_CELLS, **lam)
    e.set_expression(inp["S"], inp["G"])
    e.set_density(inp["d"], inp.get("d_source"))
    rng = np.random.default_rng(seed + 1)
    e.set_mapping(rng.standard_normal((N, V)).astype(np.float32))
    if mode == "constrained":
        e.set_filter(rng.standard_normal(N).astype(np.float32))
    if mask is not None:
        e.set_loss_genes(mask)
    return e, inp


def _old_path(e, n, every):
    """What Mapper.train(val_each=every) did before: one epoch per call, validation_terms() after each validated one."""
    vals = {}
    for t in range(n):
        e.run(1, LR)
        if t % every == 0:
            vals[t] = e.validation_terms()
    return vals


def _new_path(e, n, every, chunks):
    e.set_validation(every)
    assert sum(chunks) == n
    for c in chunks:
        e.run(c, LR)
    e.set_validation(0)


def _result(e):
    N, V = e.cfg.n_cells, e.cfg.n_voxels
    M = np.empty((N, V), dtype=np.float32)
    e.get_state(M)
    P = e.get_mapping(np.empty((N, V), dtype=np.float32))
    return e.history(), M, P


def _check_against_old(h_new, M_new, P_new, h_old, M_old, P_old, vals, n, every):
    assert np.array_equal(h_new[:, :12], h_old[:, :12], equal_nan=True), "training history differs"
    assert np.array_equal(M_new, M_old), "final M differs"
    assert np.array_equal(P_new, P_old), "final mapping differs"
    assert h_new.shape[0] == n
    for t in range(n):
        row = h_new[t, 12:16]
        if t % every:
            assert np.all(np.isnan(row)), (t, row)
        else:
            assert np.array_equal(row, vals[t]), (t, row, vals[t])
    assert np.all(h_old[:, 12:16] == 0.0)


# (mode, lambdas, masked, n, every, chunks of the new path)
CASES = {
    "cells-every1-split": ("cells", {}, False, 7, 1, (3, 4)),
    "clusters-every3": ("clusters", {}, False, 8, 3, (8,)),
    "constrained-every1": ("constrained", {}, False, 5, 1, (2, 3)),
    "cells-mask-g2-entropy-every3": ("cells", dict(lambda_g2=1.0, lambda_r=1e-3), True, 7, 3, (2, 5)),
    "clusters-mask-every100": ("clusters", {}, True, 6, 100, (6,)),
    "cells-l1l2-every1": ("cells", dict(lambda_l1=1e-6, lambda_l2=1e-6), False, 4, 1, (4,)),
}


def _mask(K, seed=3):
    a = np.random.default_rng(seed).random(K) < 0.6
    a[0] = True
    return a


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("precision", ["fp32", "bf16x3", "bf16"])
def test_matches_one_epoch_loop(precision, case):
    mode, lam, masked, n, every, chunks = CASES[case]
    K = 90
    mask = _mask(K) if masked else None
    e_old, _ = _engine(precision, mode, K=K, mask=mask, **lam)
    vals = _old_path(e_old, n, every)
    e_new, _ = _engine(precision, mode, K=K, mask=mask, **lam)
    _new_path(e_new, n, every, chunks)
    _check_against_old(*_result(e_new), *_result(e_old), vals, n, every)


@pytest.mark.parametrize("chunks", ["2", "4"])
@pytest.mark.parametrize("every", [1, 3])
def test_matches_one_epoch_loop_bf16_pipeline(chunks, every, monkeypatch):
    """bf16 with the three-stream cell-chunk pipeline: the validated epochs run their exact row pass after the update on the
    work stream, and the next forward is not issued ahead of it."""
    monkeypatch.setenv("TGB200_CHUNKS", chunks)
    N, V, K, n = 4200, 260, 70, 8
    e_old, _ = _engine("bf16", N=N, V=V, K=K, seed=5)
    assert int(e_old.debug("shape")[4]) == int(chunks)
    vals = _old_path(e_old, n, every)
    e_new, _ = _engine("bf16", N=N, V=V, K=K, seed=5)
    _new_path(e_new, n, every, (n,))
    _check_against_old(*_result(e_new), *_result(e_old), vals, n, every)


def test_mapper_train_val_each_matches_one_epoch_loop():
    """Mapper.train(val_each=) reads the validated rows into the reference's val_* lists, with prints every 4 epochs."""
    from tangram_b200 import Mapper
    inp = synthetic_inputs(500, 240, 60, seed=8)
    M0 = np.random.default_rng(9).standard_normal((500, 240)).astype(np.float32)
    kw = dict(S=inp["S"], G=inp["G"], d=inp["d"], lambda_d=1.0, lambda_g2=1.0, device="cuda:0", M0=M0)
    a = Mapper(**kw)
    with contextlib.redirect_stdout(io.StringIO()) as out_a:
        P_a, h_a = a.train(10, print_each=4, val_each=3)
    b = Mapper(**kw)
    vals = _old_path(b._engine, 10, 3)
    h_b = b._engine.history()
    assert [float(x) for x in h_a["total_loss"]] == [float(x) for x in h_b[:, 0]]
    assert np.array_equal(P_a, b.train(0, print_each=None)[0])
    assert len(out_a.getvalue().splitlines()) == 3
    for c, key in enumerate(["val_total_loss", "val_gene_sim", "val_sp_sparsity_weighted_sim", "val_entropy"]):
        ref = [float(vals[t][c]) for t in sorted(vals)]
        assert len(h_a[key]) == len(ref) == 4
        assert h_a[key] == ref, key
    a.train(2, print_each=None)                                        # validation is off again after the call
    h = a._engine.history()
    assert np.all(np.isfinite(h[:10:3, 12:16])) and np.all(np.isnan(h[1:10:3, 12:16]))
    assert np.all(h[10:, 12:16] == 0.0)


def _softmax64(M):
    M = M - M.max(axis=1, keepdims=True)
    E = np.exp(M)
    return E / E.sum(axis=1, keepdims=True)


def _val_float64(Y, G, M, act):
    """_val_loss_fn (:311-356) in float64 from Y_ext's gene columns, G and M, over the genes flagged in `act`."""
    Ya, Ga = Y[:, act], G[:, act]
    cos_k = (Ya * Ga).sum(0) / (np.maximum(np.linalg.norm(Ya, axis=0), EPS) * np.maximum(np.linalg.norm(Ga, axis=0), EPS))
    gv = cos_k.mean()
    cos_j = (Ya * Ga).sum(1) / (np.maximum(np.linalg.norm(Ya, axis=1), EPS) * np.maximum(np.linalg.norm(Ga, axis=1), EPS))
    vg = cos_j.mean()
    w = (Ga != 0).sum(0) / G.shape[0]
    sp = (cos_k * w).sum() / w.sum()
    P = _softmax64(M)
    plogp = np.where(P > 0, P * np.log(np.where(P > 0, P, 1.0)), 0.0)
    ent = -plogp.sum(1).mean() / np.log(M.shape[1])
    return np.array([gv + vg, gv, sp, ent]), cos_k


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("precision", ["fp32", "bf16x3", "bf16"])
def test_against_float64(precision, masked):
    """The four values of the last validated epoch against float64 from the device's own Y_ext and M, with the
    test_stages_gpu.py-style bound 4 n u max(1, |ref|): n = V + K for the cosine terms (the column and row reductions and
    the mean over genes), n = V + N for the entropy (the row pass and the sum over cells).  Gene 2's S column is scaled to
    1e-10, so its predicted column norm (about 4e-9) is clamped at eps; its cosine enters the sparsity-weighted score."""
    N, V, K = 700, 260, 75
    inp = synthetic_inputs(N, V, K, seed=11)
    S = inp["S"].copy()
    S[:, 2] = S[:, 2] * 1e-10 + 1e-10
    act = _mask(K, seed=4) if masked else np.ones(K, dtype=bool)
    act[2] = True
    e, inp = _engine(precision, N=N, V=V, K=K, seed=11, S=S, mask=act if masked else None, lambda_g2=0.0)
    e.set_validation(1)
    e.run(3, LR)                     # the last epoch of a call runs the separate forward: Y_ext and M are its inputs
    got = e.history()[-1, 12:16].astype(np.float64)
    Ke, ld = (int(x) for x in e.debug("shape")[:2])
    Y = e.debug("Y").reshape(V, Ke)[:, :K].astype(np.float64)
    M = e.debug("M").reshape(N, ld)[:, :V].astype(np.float64)
    ref, cos_k = _val_float64(Y, inp["G"].astype(np.float64), M, act)
    assert np.linalg.norm(Y[:, 2]) < EPS, "gene 2 must be clamped"
    assert abs(cos_k[int(np.flatnonzero(act).tolist().index(2))]) > 0.05
    n = np.array([V + K, V + K, V + K, V + N], dtype=np.float64)
    bound = 4 * n * U * np.maximum(1.0, np.abs(ref))
    ratio = np.abs(got - ref) / bound
    print(f"[validation] {precision} masked={masked}: |err| / bound {np.array2string(ratio, precision=3)}")
    assert np.all(ratio <= 1.0), (got, ref, ratio)
    assert np.array_equal(e.validation_terms(), e.history()[-1, 12:16])


def test_columns_off_zero_and_skipped_rows_nan():
    e, _ = _engine("bf16x3", N=300, V=200, K=40)
    e.run(3, LR)
    assert np.all(e.history()[:, 12:16] == 0.0)
    e.set_validation(2)
    e.run(5, LR)
    h = e.history()[3:]
    for t in range(5):
        assert np.all(np.isnan(h[t, 12:16])) == bool(t % 2), (t, h[t, 12:16])
        assert np.all(np.isfinite(h[t, 12:16])) == (t % 2 == 0)
    e.set_validation(0)
    e.run(2, LR)
    assert np.all(e.history()[-2:, 12:16] == 0.0)


def test_refused_inside_a_step_and_on_a_sharded_handle():
    from tangram_b200 import _lib
    from tangram_b200.engine import Engine
    e, _ = _engine("fp32", N=300, V=200, K=40)
    e.step_begin()
    with pytest.raises(_lib.TangramB200Error, match="error -3"):
        e.set_validation(1)
    e.step_end(LR)
    e.set_validation(1)
    e.step_begin()
    e.step_end(LR)                   # step_begin / step_end validate too: epoch 0
    assert np.all(np.isfinite(e.history()[-1, 12:16]))
    with pytest.raises(_lib.TangramB200Error, match="error -1"):
        e.set_validation(-1)
    inp = synthetic_inputs(300, 200, 40, seed=0)
    s = Engine(300, 200, 40, n_cells_global=600, precision="fp32")
    s.set_expression(inp["S"], inp["G"])
    with pytest.raises(_lib.TangramB200Error, match="error -4"):
        s.set_validation(1)
    s.set_validation(0)


@pytest.mark.parametrize("precision", ["fp32", "bf16x3"])
def test_no_launch_on_epochs_not_validated(precision):
    """12 epochs: off, every 100 (epoch 0) and every 5 (epochs 0, 5 and 10; 10 is served by epoch 11's forward).  The
    launches a validation adds are the same for each, so every 5 costs exactly three times every 100."""
    counts = {}
    for every in (0, 100, 5):
        e, _ = _engine(precision, N=400, V=220, K=50)
        e.set_validation(every)
        n0 = e.kernel_launches()
        e.run(12, LR)
        counts[every] = e.kernel_launches() - n0
    d1, d3 = counts[100] - counts[0], counts[5] - counts[0]
    print(f"[validation] {precision}: launches {counts}")
    assert 0 < d1 <= 2 and d3 == 3 * d1, counts


_API = ("cudaMalloc", "cudaFree", "cudaMemcpy", "cudaMemset", "Synchronize", "cudaHostRegister")


def _api_counts(fn):
    """CUDA runtime calls of `fn` that allocate, free, copy, set memory or wait for the device, by name (torch.profiler)."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
    return collections.Counter(ev.name for ev in prof.events() if any(k in ev.name for k in _API))


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
def test_no_sync_or_allocation_in_the_loop(precision):
    """train(1000, val_each=1) makes exactly the allocating, copying and synchronising runtime calls of train(1000): those
    of the ten print chunks and of the final history and mapping.  The validation's scratch is allocated by
    set_validation, once per handle; here before the profiled call."""
    from tangram_b200 import Mapper
    import torch
    torch.cuda.init()
    inp = synthetic_inputs(2000, 400, 100, seed=2)
    M0 = np.random.default_rng(3).standard_normal((2000, 400)).astype(np.float32)
    kw = dict(S=inp["S"], G=inp["G"], d=inp["d"], lambda_d=1.0, device="cuda:0", M0=M0, precision=precision)
    a, b = Mapper(**kw), Mapper(**kw)
    b._engine.set_validation(1)
    b._engine.set_validation(0)
    torch.cuda.synchronize()
    with contextlib.redirect_stdout(io.StringIO()):
        plain = _api_counts(lambda: a.train(1000, print_each=100))
        val = _api_counts(lambda: b.train(1000, print_each=100, val_each=1))
    print(f"[validation] {precision}: runtime calls without validation {dict(plain)}, with {dict(val)}")
    assert sum(v for k, v in plain.items() if "Memcpy" in k) >= 11, "the profiler did not see the library's copies"
    assert val == plain
    assert len(b.history_matrix) == 1000 and np.all(np.isfinite(b.history_matrix[:, 12:16]))
