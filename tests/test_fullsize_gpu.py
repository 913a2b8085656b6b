"""BASELINE.json's full sizes (configs 2-5) against the oracle.

The CPU oracle cannot finish these sizes in seconds, but the very same closed-form restatement
(oracle/tangram_oracle.py, OracleMapper(device="cuda")) evaluated with plain torch ops on the GPU can: fp32 SGEMM
(TF32 off), no kernels of ours.  Each test runs the CUDA path and the oracle from the SAME initial mapping and compares
the loss trajectory, every logged term and the final mapping; the forward contraction is additionally checked against a
float64 evaluation on a voxel sample.  Bounds: bf16x3 (the parity-grade tensor-core mode) <= 1e-4 (north_star);
bf16 (throughput mode, BASELINE config 3 asks for it) at the bound stated next to each assert."""
import numpy as np
import pytest
import torch

from tests.helpers import traj_err

pytestmark = pytest.mark.gpu


def _workload(name):
    import bench
    from tangram_b200 import _lib
    N, V, K, T, clusters, _ = bench.WORKLOADS[name]
    inp = bench.gen_inputs(name, 0, N)
    lambdas, graphs = {}, None
    if name == "c5":
        from oracle.tangram_oracle import grid_graph, spatial_weights_from_graph
        lambdas = dict(bench.C5_LAMBDAS)
        conn, dmat = grid_graph(V)
        graphs = {_lib.GRAPH_VOXEL_WEIGHTS: spatial_weights_from_graph(conn, dmat, True, True),
                  _lib.GRAPH_NEIGHBORHOOD_FILTER: spatial_weights_from_graph(conn, dmat, False, False),
                  _lib.GRAPH_SPATIAL_WEIGHTS: spatial_weights_from_graph(conn, dmat, False, True)}
    return (N, V, K, T, clusters), inp, lambdas, graphs


def _engine(name, precision, wl=None, seed=7):
    from tangram_b200 import _lib
    from tangram_b200.engine import Engine
    (N, V, K, T, clusters), inp, lambdas, graphs = wl or _workload(name)
    eng = Engine(N, V, K, n_types=T, precision=precision,
                 density_mode=_lib.DENSITY_SOURCE if clusters else _lib.DENSITY_CELLS, **lambdas)
    eng.set_expression(inp["S"], inp["G"])
    eng.set_density(inp["d"], inp.get("d_source"))
    if graphs:
        for which, g in graphs.items():
            eng.set_graph(which, g)
        eng.set_ct_encode(inp["ct_encode"])
    eng.init_mapping_normal(seed)
    return eng


def _oracle(wl, M0, dtype=torch.float32):
    """The oracle on the GPU (plain torch ops), from the device tensor M0."""
    from oracle.tangram_oracle import OracleMapper
    (N, V, K, T, clusters), inp, lambdas, graphs = wl
    kw = dict(S=inp["S"], G=inp["G"], d=inp["d"], lambda_d=1.0, M0=M0, device="cuda", dtype=dtype, **lambdas)
    if clusters:
        kw["d_source"] = inp["d_source"]
    if graphs:
        kw.update(voxel_weights=graphs[0], neighborhood_filter=graphs[1], spatial_weights=graphs[2], ct_encode=inp["ct_encode"])
    return OracleMapper(**kw)


def _oracle_run(o, steps, lr=0.1):
    rows = []
    for _ in range(steps):
        terms, g = o.loss_and_grad()
        rows.append(terms)
        o.adam_step(g, lr)
        del g
    return rows, torch.softmax(o.M, dim=1).float()


_HIST = {"total_loss": 0, "main_loss": 1, "kl_reg": 3, "entropy_reg": 4, "l2_reg": 6, "gv_neighborhood_sim": 7,
         "ct_island_penalty": 8, "getis_ord_sim": 9}


def _rel_fro(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


@pytest.mark.parametrize("name", ["c3", "c4", "c5"])
def test_full_size_against_oracle(name):
    wl = _workload(name)
    (N, V, K, T, clusters), inp, lambdas, graphs = wl
    steps = 4
    # ---- the oracle, from the device-RNG initial mapping of the engine
    eng = _engine(name, "bf16x3", wl)
    M0 = torch.empty((N, V), dtype=torch.float32, device="cuda")
    eng.get_state(M=M0)
    P0 = torch.softmax(M0, dim=1)
    idx = torch.arange(0, V, max(1, V // 64), device="cuda")
    S = torch.from_numpy(inp["S"]).cuda()
    Y64 = (P0[:, idx].double().t() @ S.double())                      # forward contraction on a voxel sample, float64
    del P0
    o = _oracle(wl, M0)
    orows, oout = _oracle_run(o, steps)
    del o
    torch.cuda.empty_cache()
    ol = np.array([r["total_loss"] for r in orows])

    for precision in ("bf16x3", "bf16"):
        if precision == "bf16":
            eng = _engine(name, "bf16", wl)
        eng.run(1)
        Ke = int(eng.debug("shape")[0])
        Y = torch.from_numpy(eng.debug("Y").reshape(V, Ke)[:, :K]).cuda()[idx]
        yerr = _rel_fro(Y, Y64)
        eng.run(steps - 1)
        h = eng.history()
        out = torch.empty((N, V), dtype=torch.float32, device="cuda")
        eng.get_mapping(out)
        rs = out.sum(dim=1)
        assert torch.all(torch.isfinite(rs)) and float((rs - 1).abs().max()) < 2e-5 and float(out.min()) >= 0.0
        terr = traj_err(h[:, 0], ol)
        merr = _rel_fro(out, oout)
        # every logged term, relative to its own size or -- for terms that are tiny next to the loss (the KL term is ~1e-4
        # of it at a random start) -- to 1% of the total loss
        terms = {k: max(abs(float(h[t, c]) - orows[t][k]) / max(abs(orows[t][k]), 1e-2 * abs(orows[t]["total_loss"]))
                        for t in range(steps))
                 for k, c in _HIST.items() if not np.isnan(orows[0][k])}
        print(f"{name} {precision}: Y vs float64 {yerr:.2e}, loss trajectory {terr:.2e}, mapping rel-Frobenius {merr:.2e}, "
              f"per-term max rel {({k: float('%.2e' % v) for k, v in terms.items()})}")
        if precision == "bf16x3":
            assert yerr < 1e-5 and terr < 1e-4 and merr < 1e-4          # north_star's bound, at the benchmark size
            assert all(v < 1e-4 for k, v in terms.items() if k not in ("l2_reg",)), terms
        else:
            # bf16 operands (2^-9 relative rounding; SURVEY 7.3: 3.6e-5 on the loss, 2e-3 .. 1.3e-2 on the mapping at 10 .. 100 epochs)
            assert yerr < 3e-3 and terr < 1e-3 and merr < 2e-2
        # the gene-voxel score moves the way the oracle's does, step by step (rises from a random start unless the
        # oracle's own trajectory says otherwise: lr = 0.1 Adam can overshoot in the clusters regime)
        for t in range(1, steps):
            do = orows[t]["main_loss"] - orows[t - 1]["main_loss"]
            dg = float(h[t, 1] - h[t - 1, 1])
            assert abs(dg - do) < (1e-5 if precision == "bf16x3" else 5e-4) + 1e-2 * abs(do), (name, precision, t, dg, do)
        eng.close()
        del out, Y
        torch.cuda.empty_cache()

    if name == "c3":
        # project_genes' GEMM at full size on the device (cell blocks, 512-cell chains, 2304 genes): tensor-core
        # split-bf16 path vs float64 on the voxel sample
        eng = _engine(name, "bf16", wl)
        Pm = torch.empty((N, V), dtype=torch.float32, device="cuda")
        eng.get_mapping(Pm)
        X = torch.rand((N, 2304), dtype=torch.float32, device="cuda")
        outp = torch.empty((V, 2304), dtype=torch.float32, device="cuda")
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); eng.project(X, outp); e1.record(); torch.cuda.synchronize()
        ref = Pm[:, idx].double().t() @ X.double()
        err = float((outp[idx].double() - ref).norm() / ref.norm())
        print(f"project {N}x{V} mapping onto 2304 genes: {e0.elapsed_time(e1):.1f} ms, rel err vs float64 {err:.2e}")
        assert err < 1e-5
        eng.close()


@pytest.mark.parametrize("name,precision", [("c3", "bf16"), ("c4", "bf16")])
def test_full_size_determinism(name, precision):
    """Two engines on the same inputs reproduce the loss history bit for bit (no float atomics anywhere)."""
    wl = _workload(name)
    a = _engine(name, precision, wl)
    a.run(4)
    ha = a.history()
    a.close()
    b = _engine(name, precision, wl)
    b.run(4)
    assert np.array_equal(b.history()[:, :4], ha[:, :4], equal_nan=True)
    assert b.kernel_launches() > 0


def test_config2_full_horizon_with_noise_floor():
    """BASELINE config 2 as stated: 10k x 1k x 1k, 1000 epochs.  The loss trajectory holds 1e-4 over the whole run; the final
    mapping is reported next to the reference's own noise floor at that horizon -- the same oracle in fp32 vs float64
    (SURVEY 7.3 (iii): past ~100 epochs two fp32 runs that differ only in rounding disagree at the 5e-3 level)."""
    wl = _workload("c2")
    (N, V, K, T, clusters), inp, _, _ = wl
    epochs = 1000
    eng = _engine("c2", "bf16x3", wl)
    M0 = torch.empty((N, V), dtype=torch.float32, device="cuda")
    eng.get_state(M=M0)
    r32, o32 = _oracle_run(_oracle(wl, M0), epochs)
    r64, o64 = _oracle_run(_oracle(wl, M0, dtype=torch.float64), epochs)
    l32 = np.array([r["total_loss"] for r in r32])
    l64 = np.array([r["total_loss"] for r in r64])
    floor_traj, floor_map = traj_err(l32, l64), _rel_fro(o32, o64)
    for precision in ("bf16x3", "bf16"):
        if precision == "bf16":
            eng = _engine("c2", "bf16", wl)
        eng.run(epochs)
        h = eng.history()
        out = torch.empty((N, V), dtype=torch.float32, device="cuda")
        eng.get_mapping(out)
        terr, merr, merr64 = traj_err(h[:, 0], l32), _rel_fro(out, o32), _rel_fro(out, o64)
        agree = float((out.argmax(dim=1) == o32.argmax(dim=1)).float().mean())
        print(f"c2 x {epochs} epochs, {precision}: loss trajectory vs oracle fp32 {terr:.2e} (oracle fp32 vs float64: {floor_traj:.2e}); "
              f"mapping rel-Frobenius vs oracle fp32 {merr:.2e}, vs oracle float64 {merr64:.2e} (oracle fp32 vs float64: {floor_map:.2e}); "
              f"row-argmax agreement {agree:.4f}")
        if precision == "bf16x3":
            assert terr < 1e-4
            assert merr < max(1e-4, 3.0 * floor_map)       # no further from the fp32 oracle than fp32 is from exact arithmetic
        else:
            # throughput mode over the full horizon: the trajectories are chaotic in M (SURVEY 7.3), bf16 operand rounding is
            # amplified like any other perturbation -- measured 1.3e-3 on the loss, 0.24 on the mapping, 88% same arg-max
            assert terr < 3e-3 and merr < 0.4 and agree > 0.8
        eng.close()
