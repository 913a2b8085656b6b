"""The wgmma / TMA tensor-core path (precision="bf16") against the fp32 path and the oracle.
bf16 operands carry 2^-9 relative rounding, so buffers agree to ~1e-3 and the loss trajectory to
~1e-4 (SURVEY.md 7.3: bf16 operands give 3.6e-5 on the loss trajectory)."""
import numpy as np
import pytest

from oracle.tangram_oracle import OracleMapper, synthetic_inputs
from tests.helpers import max_rel, rel_fro

pytestmark = pytest.mark.gpu


def _pair(N, V, K, seed, clusters=False, **hyper):
    from tangram_b200 import Mapper
    inp = synthetic_inputs(N, V, K, seed=seed, clusters=clusters)
    kw = dict(S=inp["S"], G=inp["G"], d=inp["d"], lambda_d=1.0, **hyper)
    if clusters:
        kw["d_source"] = inp["d_source"]
    M0 = np.random.default_rng(seed).standard_normal((N, V)).astype(np.float32)
    a = Mapper(device="cuda:0", M0=M0, precision="fp32", **kw)
    b = Mapper(device="cuda:0", M0=M0, precision="bf16", **kw)
    return kw, M0, a, b


SHAPES = [
    (256, 128, 62, False),       # single tile, Ke = 64
    (1000, 257, 130, False),     # ragged everywhere
    (2048, 512, 256, False),
    (3000, 1000, 500, False),
    (48, 5000, 300, True),       # clusters regime: row-dot is split over voxels
]


@pytest.mark.parametrize("N,V,K,clusters", SHAPES)
def test_tc_buffers_match_fp32_after_one_step(N, V, K, clusters):
    kw, M0, a, b = _pair(N, V, K, seed=N + K, clusters=clusters)
    a.train(1, print_each=None)
    b.train(1, print_each=None)
    Ke = int(a._debug("shape")[0])
    Ya, Yb = a._debug("Y").reshape(V, Ke), b._debug("Y").reshape(V, Ke)
    assert rel_fro(Yb[:, :K], Ya[:, :K]) < 3e-3, "forward contraction P^T S"
    assert rel_fro(Yb[:, K:K + 2].sum(axis=1), Ya[:, K:K + 2].sum(axis=1)) < 3e-3, "density column"
    dYa, dYb = a._debug("dY").reshape(V, Ke), b._debug("dY").reshape(V, Ke)
    assert rel_fro(dYb, dYa) < 2e-2
    ra, rb = a._debug("rdot"), b._debug("rdot")
    assert np.max(np.abs(rb - ra)) < 2e-2 * np.max(np.abs(ra)) + 1e-7, "row-dot contraction"
    la, lb = a.history_matrix[0, 0], b.history_matrix[0, 0]
    assert abs(la - lb) < 2e-4 * max(1.0, abs(la))
    Ma, Mb = a.state()[0], b.state()[0]
    # first Adam step moves every element by ~lr*sign(g): the two paths may only disagree where g ~ 0
    frac_diff = np.mean(np.abs(Ma - Mb) > 0.05)
    assert frac_diff < 0.02, f"{frac_diff:.4f} of the elements stepped the other way"


def test_tc_trajectory_vs_oracle():
    N, V, K = 3000, 600, 400
    inp = synthetic_inputs(N, V, K, seed=21)
    kw = dict(S=inp["S"], G=inp["G"], d=inp["d"], lambda_d=1.0)
    o = OracleMapper(random_state=11, **kw)
    M0 = o.M.numpy().copy()
    oo, oh = o.train(30, print_each=None)
    from tangram_b200 import Mapper
    m = Mapper(device="cuda:0", M0=M0, precision="bf16", **kw)
    out, hist = m.train(30, print_each=None)
    tl = [float(x) for x in hist["total_loss"]]
    assert max_rel(tl, [float(x) for x in oh["total_loss"]]) < 1e-3
    assert rel_fro(out, oo) < 5e-2
    assert np.allclose(out.sum(axis=1), 1.0, atol=1e-5)


def test_tc_all_terms_run_and_track_fp32():
    from oracle.tangram_oracle import grid_graph, spatial_weights_from_graph
    from tangram_b200 import Mapper
    N, V, K, T = 1500, 400, 200, 8
    inp = synthetic_inputs(N, V, K, seed=2, n_types=T)
    conn, dist = grid_graph(V)
    kw = dict(
        S=inp["S"], G=inp["G"], d=inp["d"], lambda_d=1.0, lambda_g2=0.5, lambda_r=1e-3, lambda_l1=1e-7,
        lambda_l2=1e-7, lambda_neighborhood_g1=0.96, lambda_ct_islands=0.17, lambda_getis_ord=0.71,
        voxel_weights=spatial_weights_from_graph(conn, dist, True, True),
        neighborhood_filter=spatial_weights_from_graph(conn, dist, False, False),
        spatial_weights=spatial_weights_from_graph(conn, dist, False, True),
        ct_encode=inp["ct_encode"])
    M0 = np.random.default_rng(0).standard_normal((N, V)).astype(np.float32)
    a = Mapper(device="cuda:0", M0=M0, precision="fp32", **kw)
    b = Mapper(device="cuda:0", M0=M0, precision="bf16", **kw)
    _, ha = a.train(10, print_each=None)
    _, hb = b.train(10, print_each=None)
    assert max_rel([float(x) for x in hb["total_loss"]], [float(x) for x in ha["total_loss"]]) < 2e-3


def test_tc_determinism():
    from tangram_b200 import Mapper
    inp = synthetic_inputs(1200, 300, 150, seed=8)
    kw = dict(S=inp["S"], G=inp["G"], d=inp["d"], lambda_d=1.0, random_state=5, precision="bf16", device="cuda:0")
    a, _ = Mapper(**kw).train(8, print_each=None)
    b, _ = Mapper(**kw).train(8, print_each=None)
    assert np.array_equal(a, b)


def test_tc_resume_reinitialises_row_normalisation():
    """A state load drops the resident P (written by the backward epilogue) and re-runs the row pass:
    6 steps == 3 steps + checkpoint/restore + 3 steps up to bf16 rounding."""
    from tangram_b200 import Mapper
    inp = synthetic_inputs(1500, 500, 200, seed=3)
    kw = dict(S=inp["S"], G=inp["G"], d=inp["d"], lambda_d=1.0, lambda_r=1e-3, random_state=4, precision="bf16",
              device="cuda:0")
    a, ha = Mapper(**kw).train(6, print_each=None)
    m1 = Mapper(**kw)
    m1.train(3, print_each=None)
    st = m1.state()
    m2 = Mapper(**kw)
    m2.load_state(*st)
    b, hb = m2.train(3, print_each=None, resume=True)
    assert rel_fro(b, a) < 5e-3
    assert abs(float(hb["total_loss"][-1]) - float(ha["total_loss"][-1])) < 1e-4
    assert abs(hb["entropy_reg"][-1] - ha["entropy_reg"][-1]) < 1e-3 * abs(ha["entropy_reg"][-1])


@pytest.mark.parametrize("shape", [(1, 1, 1), (2, 3, 1), (5, 130, 2), (130, 65, 3), (129, 257, 65)])
@pytest.mark.parametrize("precision", ["fp32", "bf16x3", "bf16"])
def test_degenerate_and_off_tile_shapes(shape, precision):
    """One cell, one voxel, one gene, and sizes just past every tile boundary (128 rows, 64/256 columns, 64 genes)."""
    from tangram_b200 import Mapper
    N, V, K = shape
    rng = np.random.default_rng(N * 1000 + V)
    S = (rng.random((N, K)) + 0.1).astype(np.float32)
    G = (rng.random((V, K)) + 0.1).astype(np.float32)
    d = (np.ones(V) / V).astype(np.float32)
    M0 = rng.standard_normal((N, V)).astype(np.float32)
    o = OracleMapper(S, G, d=d, lambda_d=1.0, lambda_g2=0.5, M0=M0)
    oo, oh = o.train(3, print_each=None)
    m = Mapper(S, G, d=d, lambda_d=1.0, lambda_g2=0.5, M0=M0, device="cuda:0", precision=precision)
    out, hist = m.train(3, print_each=None)
    tol = 5e-2 if precision == "bf16" else 2e-5
    assert out.shape == (N, V) and np.all(np.isfinite(out))
    assert np.allclose(out.sum(axis=1), 1.0, atol=1e-5)
    assert rel_fro(out, oo) < tol
    ltol = 5e-3 if precision == "bf16" else 1e-5
    assert np.max(np.abs(np.array([float(x) for x in hist["total_loss"]]) - np.array([float(x) for x in oh["total_loss"]]))) < ltol


@pytest.mark.parametrize("precision", ["fp32", "bf16x3", "bf16"])
def test_project_multi_chunk_matches_float64(precision):
    """tgb200_project (project_genes' GEMM, tangram/utils.py:368): more than 2048 gene columns, ragged, after a few
    training steps; every mode returns fp32-grade softmax(M)^T X (split-bf16 operands on the forward kernel), and training
    continues unperturbed afterwards."""
    from tangram_b200 import Mapper
    N, V, K = 2500, 333, 90
    inp = synthetic_inputs(N, V, K, seed=17)
    M0 = np.random.default_rng(5).standard_normal((N, V)).astype(np.float32)
    kw = dict(S=inp["S"], G=inp["G"], d=inp["d"], lambda_g1=1.0, lambda_d=1.0, M0=M0, precision=precision, device="cuda:0")
    m = Mapper(**kw)
    m.train(5, print_each=None)
    Mcur = m.state()[0].astype(np.float64)
    P = np.exp(Mcur - Mcur.max(axis=1, keepdims=True)); P /= P.sum(axis=1, keepdims=True)
    X = np.random.default_rng(6).random((N, 2048 + 77)).astype(np.float32)
    got = m.project(X)
    assert got.shape == (V, X.shape[1])
    assert rel_fro(got, P.T @ X.astype(np.float64)) < 3e-6
    # projecting must not disturb the optimiser state: 5 + 5 steps == 10 steps of a fresh mapper, bit for bit
    out_a, hist_a = m.train(5, print_each=None, resume=True)     # same optimizer continues (default: a fresh Adam per train())
    m2 = Mapper(**kw)
    out_b, hist_b = m2.train(10, print_each=None)
    assert np.array_equal(out_a, out_b)


@pytest.mark.parametrize("precision,tol", [("fp32", 2e-6), ("bf16x3", 2e-6), ("bf16", 1e-4)])
def test_ragged_tiles_with_regularisers_matches_oracle(precision, tol):
    """2100 cells leave a last 128-row tile of 52 rows in the backward contraction and a ragged k-block in the forward,
    300 voxels leave a ragged 256-column tile, lambda_r takes the streaming update off its plain fast path, and
    lambda_g2 adds the voxel-wise term to dY_ext.  Loss trajectory vs the oracle (observed: 2e-7 in fp32 / bf16x3,
    1.2e-5 in bf16)."""
    from tangram_b200 import Mapper
    N, V, K = 2100, 300, 70
    inp = synthetic_inputs(N, V, K, seed=3)
    kw = dict(S=inp["S"], G=inp["G"], d=inp["d"], lambda_g1=1.0, lambda_d=1.0, lambda_g2=0.5, lambda_r=1e-3)
    M0 = np.random.default_rng(0).standard_normal((N, V)).astype(np.float32)
    _, ho = OracleMapper(M0=M0, **kw).train(3, print_each=None)
    out, hist = Mapper(M0=M0, precision=precision, device="cuda:0", **kw).train(3, print_each=None)
    assert max_rel([float(x) for x in hist["total_loss"]], [float(x) for x in ho["total_loss"]]) < tol
    assert np.allclose(out.sum(axis=1), 1.0, atol=2e-5)


@pytest.mark.parametrize("precision", ["fp32", "bf16x3", "bf16"])
def test_more_than_65535_voxels(precision):
    """Sections with more spots than gridDim.y allows (Visium HD, Slide-seq, MERFISH): the per-voxel kernels put the
    voxel index on gridDim.x.  Few cells / genes, neighbourhood + Getis-Ord terms on (CSR SpMM both ways)."""
    from oracle.tangram_oracle import grid_graph, spatial_weights_from_graph
    from tangram_b200 import Mapper
    N, V, K = 6, 66_000, 5
    rng = np.random.default_rng(4)
    S = (rng.random((N, K)) + 0.1).astype(np.float32)
    G = (rng.random((V, K)) + 0.1).astype(np.float32)
    d = (G.sum(axis=1) / G.sum()).astype(np.float32)
    conn, dist = grid_graph(V)
    kw = dict(S=S, G=G, d=d, lambda_d=1.0, lambda_neighborhood_g1=0.5, lambda_getis_ord=0.3,
              voxel_weights=spatial_weights_from_graph(conn, dist, True, True),
              spatial_weights=spatial_weights_from_graph(conn, dist, False, True))
    M0 = rng.standard_normal((N, V)).astype(np.float32)
    oo, oh = OracleMapper(M0=M0, **kw).train(3, print_each=None)
    out, hist = Mapper(M0=M0, device="cuda:0", precision=precision, **kw).train(3, print_each=None)
    assert out.shape == (N, V) and np.allclose(out.sum(axis=1), 1.0, atol=1e-5)
    assert max_rel([float(x) for x in hist["total_loss"]], [float(x) for x in oh["total_loss"]]) < (2e-3 if precision == "bf16" else 2e-5)
    assert rel_fro(out, oo) < (5e-2 if precision == "bf16" else 1e-4)


@pytest.mark.parametrize("V", [1030, 4100, 6150, 8190, 10000, 12290, 16390, 24570, 24580])
@pytest.mark.parametrize("precision", ["fp32", "bf16x3", "bf16"])
def test_row_pass_width_buckets(V, precision):
    """The exact row pass (softmax over a row of M, one CTA per row) picks threads x register slots by row width: one V in each
    bucket of launch_softmax_rows, both edges of the widest cached one, and the uncached path; entropy term on (the pass that
    recomputes) and off (the pass that keeps exp(M - max) in registers)."""
    from tangram_b200 import Mapper
    N, K = 9, 4
    rng = np.random.default_rng(V)
    S = (rng.random((N, K)) + 0.1).astype(np.float32)
    G = (rng.random((V, K)) + 0.1).astype(np.float32)
    d = (G.sum(axis=1) / G.sum()).astype(np.float32)
    M0 = (3.0 * rng.standard_normal((N, V))).astype(np.float32)
    for lam_r in (0.0, 1e-2):
        kw = dict(S=S, G=G, d=d, lambda_d=1.0, lambda_r=lam_r, lambda_l2=1e-6)
        oo, oh = OracleMapper(M0=M0, **kw).train(2, print_each=None)
        out, hist = Mapper(M0=M0, device="cuda:0", precision=precision, **kw).train(2, print_each=None)
        assert np.allclose(out.sum(axis=1), 1.0, atol=1e-5)
        assert max_rel([float(x) for x in hist["total_loss"]], [float(x) for x in oh["total_loss"]]) < (2e-3 if precision == "bf16" else 2e-5)
        assert rel_fro(out, oo) < (5e-2 if precision == "bf16" else 1e-4)


@pytest.mark.parametrize("precision", ["fp32", "bf16x3", "bf16"])
def test_manual_exchange_protocol_two_shards_on_one_gpu(precision):
    """The C-ABI's caller-driven sharded loop (tgb200_step_begin -> all-reduce of the exchange buffer -> tgb200_step_end):
    two handles hold the two halves of the cells on ONE GPU, the test plays the all-reduce by summing their exchange buffers.
    Must reproduce the unsharded handle (same arithmetic up to the order of the cell sum)."""
    import torch
    from tangram_b200.engine import Engine
    from tangram_b200.sharded import shard_rows
    N, V, K, steps = 2304, 300, 120, 5
    inp = synthetic_inputs(N, V, K, seed=23)
    M0 = np.random.default_rng(3).standard_normal((N, V)).astype(np.float32)
    kw = dict(precision=precision, lambda_r=1e-3)

    def make(r0, r1):
        e = Engine(r1 - r0, V, K, n_cells_global=N, **kw)
        e.set_expression(np.ascontiguousarray(inp["S"][r0:r1]), inp["G"])
        e.set_density(inp["d"])
        e.set_mapping(np.ascontiguousarray(M0[r0:r1]))
        return e

    whole = make(0, N)
    whole.run(steps)
    ref = np.empty((N, V), dtype=np.float32)
    whole.get_mapping(ref)
    parts = [make(*shard_rows(N, r, 2)) for r in range(2)]
    bufs = [p.exchange_tensor() for p in parts]
    for _ in range(steps):
        for p in parts:
            p.step_begin()
        torch.cuda.synchronize()
        total = bufs[0] + bufs[1]
        for b in bufs:
            b.copy_(total)
        torch.cuda.synchronize()
        for p in parts:
            p.step_end(0.1)
    got = np.concatenate([p.get_mapping(np.empty((p.cfg.n_cells, V), dtype=np.float32)) for p in parts])
    tol = 2e-2 if precision == "bf16" else 2e-5
    assert rel_fro(got, ref) < tol
    hw, hp = whole.history()[:, 0], parts[0].history()[:, 0]
    assert np.max(np.abs(hw - hp)) < (1e-3 if precision == "bf16" else 1e-5)
    assert np.array_equal(parts[0].history()[:, :5], parts[1].history()[:, :5], equal_nan=True)     # every rank logs the global loss


def test_validation_terms_bf16_with_entropy_term_off():
    """_val_loss_fn (mapping_optimizer.py:311-356) in the throughput mode with lambda_r == 0: the per-row entropy is not carried
    across iterations there, so tgb200_validation_terms re-runs the exact row pass; val_entropy must be the real value (it
    was -0.0 before), the similarity terms track the oracle at bf16 accuracy."""
    from tangram_b200 import Mapper
    inp = synthetic_inputs(900, 160, 80, seed=6)
    kw = dict(S=inp["S"], G=inp["G"], d=inp["d"], lambda_d=1.0)
    o = OracleMapper(random_state=9, **kw)
    M0 = o.M.numpy().copy()
    _, oh = o.train(6, print_each=None, val_each=2)
    m = Mapper(M0=M0, device="cuda:0", precision="bf16", **kw)
    _, hist = m.train(6, print_each=None, val_each=2)
    for k in ("val_total_loss", "val_gene_sim", "val_sp_sparsity_weighted_sim", "val_entropy"):
        assert len(hist[k]) == len(oh[k]) == 3
        assert max_rel(hist[k], oh[k]) < 5e-3, (k, hist[k], oh[k])
    assert all(v > 0.5 for v in hist["val_entropy"])                 # normalised entropy of a near-uniform mapping, not -0.0
    # the training trajectory is not disturbed by the validation passes
    _, h2 = Mapper(M0=M0, device="cuda:0", precision="bf16", **kw).train(6, print_each=None)
    assert max_rel([float(x) for x in hist["total_loss"]], [float(x) for x in h2["total_loss"]]) < 2e-4


def _fuzz_cases(n=14, seed=2024):
    rng = np.random.default_rng(seed)
    cases = []
    for i in range(n):
        N = int(rng.choice([1, 7, 130, 300, 1000, 2047, 2049, 2300, 4100, 5000]))
        V = int(rng.choice([1, 3, 63, 65, 250, 257, 640, 1000, 1500]))
        K = int(rng.choice([1, 2, 61, 62, 63, 100, 190, 300]))
        cases.append((N, V, K, bool(rng.integers(0, 2)), bool(rng.integers(0, 2)), bool(rng.integers(0, 2)), int(rng.integers(0, 1 << 30))))
    return cases


@pytest.mark.parametrize("case", _fuzz_cases(), ids=lambda c: f"{c[0]}x{c[1]}x{c[2]}-{'c' if c[3] else 'n'}{'r' if c[4] else ''}{'l' if c[5] else ''}")
@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
def test_random_shapes_against_oracle(case, precision):
    """Seeded shape fuzz over tile / pair / chunk / padding boundaries (cells around 2048, voxels around multiples of 64 and 256,
    genes around Ke = 64 boundaries), cells or clusters density, entropy and L1/L2 terms on or off: three epochs vs the oracle."""
    import os
    from tangram_b200 import Mapper
    N, V, K, clusters, ent, l12, seed = case
    rng = np.random.default_rng(seed)
    S = (rng.random((N, K)) * (rng.random((N, K)) < 0.6) + 0.05).astype(np.float32)
    G = (rng.random((V, K)) * 2 + 0.05).astype(np.float32)
    kw = dict(S=S, G=G, lambda_d=1.0)
    if clusters:
        w = rng.random(N) + 0.1
        kw.update(d=(np.ones(V) / V).astype(np.float32), d_source=(w / w.sum()).astype(np.float32))
    else:
        kw.update(d=(G.sum(axis=1) / G.sum()).astype(np.float32))
    if ent:
        kw["lambda_r"] = 1e-3
    if l12:
        kw.update(lambda_l1=1e-6, lambda_l2=1e-6)
    M0 = rng.standard_normal((N, V)).astype(np.float32)
    oo, oh = OracleMapper(M0=M0, **kw).train(3, print_each=None)
    old = os.environ.get("TGB200_CHUNKS")
    os.environ["TGB200_CHUNKS"] = "3"           # cells permitting, the three-stream chunk pipeline
    try:
        out, hist = Mapper(M0=M0, device="cuda:0", precision=precision, **kw).train(3, print_each=None)
    finally:
        if old is None:
            del os.environ["TGB200_CHUNKS"]
        else:
            os.environ["TGB200_CHUNKS"] = old
    assert np.all(np.isfinite(out)) and np.allclose(out.sum(axis=1), 1.0, atol=2e-5)
    tl, ol = np.array([float(x) for x in hist["total_loss"]]), np.array([float(x) for x in oh["total_loss"]])
    scale = max(1.0, float(np.max(np.abs(ol))))
    assert np.max(np.abs(tl - ol)) < (5e-3 if precision == "bf16" else 2e-5) * scale, (tl, ol)
    assert rel_fro(out, oo) < (6e-2 if precision == "bf16" else 5e-5)
