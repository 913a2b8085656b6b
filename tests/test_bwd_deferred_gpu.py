"""The bf16 backward contraction runs each tile's epilogue deferred, in steps between the next tile's first k-blocks
(TcEpiDpStore in gemm_tc.cuh).  What it stores must not depend on which tile follows which: dq and the row-dot are
bit-identical across the contraction's grid caps (TGB200_UPDATE_SMS 0, 16 and 126, down to three clusters), and at
every chunk count they are the centred, rounded S_ext dY_ext^T and its row-dot.  The shapes cover one tile per CTA,
many tiles per CTA, odd row-tile counts (a phantom tile in the last pair), ragged last column tiles, and tiles with
fewer k-blocks than the epilogue has steps, with more, and with as many as at C3."""
import numpy as np
import pytest

from oracle.tangram_oracle import synthetic_inputs

pytestmark = pytest.mark.gpu

SHARES = ("0", "16", "126")
CASES = [
    # N, V, K, chunk counts
    (2048, 200, 40, (1, 2)),          # 16 row tiles x 1 column tile: one tile per CTA uncapped; 1 k-block per tile
    (20000, 600, 700, (1, 2, 4)),     # 157 row tiles (odd) x 3 column tiles (the last has 2 of 4 boxes); 11 k-blocks
    (9000, 300, 2000, (1, 2)),        # 71 row tiles (odd) x 2 column tiles (the last has 1 box); 32 k-blocks
]


def _bf16(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(torch.bfloat16).to(torch.float64).numpy()


def _backward(monkeypatch, N, V, K, chunks, share):
    from tangram_b200.engine import Engine
    monkeypatch.setenv("TGB200_CHUNKS", str(chunks))
    monkeypatch.setenv("TGB200_UPDATE_SMS", share)
    inp = synthetic_inputs(N, V, K, seed=N + V)
    e = Engine(N, V, K, precision="bf16", lambda_d=1.0, lambda_r=1e-3)
    try:
        assert int(e.debug("shape")[4]) == chunks
        e.set_expression(inp["S"], inp["G"])
        e.set_density(inp["d"])
        e.set_mapping(np.random.default_rng(N).standard_normal((N, V)).astype(np.float32))
        for _ in range(2):                    # the second step leaves a Pt written by the update, not by the row pass
            e.step_begin()
            e.step_end(0.1)
        Ke, ld = (int(x) for x in e.debug("shape")[:2])
        out = {"Pt": e.debug("Pb").reshape(N, ld).copy(), "c": e.debug("rcenter").copy()}
        e.step_begin()
        e.step_end(0.1)
        out["dq"] = e.debug("dq").reshape(N, ld).copy()
        out["rdot"] = e.debug("rdot").copy()
        dY = np.zeros((ld, Ke))
        dY[:V] = e.debug("dY").reshape(V, Ke)
        out["dY"] = dY
        out["S"] = e.debug("Sx").reshape(N, Ke).copy()
        return out
    finally:
        e.close()


def _check_against_reference(o, V):
    Pt, c, dq, rdot = (o[k].astype(np.float64) for k in ("Pt", "c", "dq", "rdot"))
    S, dY = _bf16(o["S"]), o["dY"]
    ref = S @ dY.T - c[:, None]
    chain = S.shape[1] * 2.0 ** -23 * (np.abs(S) @ np.abs(dY).T)
    tol = 2.0 ** -8 * (np.abs(ref) + chain) + chain + 1e-30
    bad = np.argwhere(np.abs(dq - ref) > tol)
    assert bad.size == 0, f"{len(bad)} elements off, first at {tuple(bad[0])}"
    z = Pt[:, :V].sum(axis=1)
    r_ref = c + (Pt * dq).sum(axis=1) / z
    scale = np.abs(Pt * dq).sum(axis=1) / z
    assert np.all(np.abs(rdot - r_ref) <= 2e-3 * scale + 1e-6 * np.abs(c) + 1e-12)


@pytest.mark.parametrize("N,V,K,chunk_counts", CASES)
def test_deferred_epilogue_is_bit_identical_across_grids(monkeypatch, N, V, K, chunk_counts):
    for chunks in chunk_counts:
        ref = _backward(monkeypatch, N, V, K, chunks, SHARES[0])
        _check_against_reference(ref, V)
        for share in SHARES[1:]:
            o = _backward(monkeypatch, N, V, K, chunks, share)
            for k in ("Pt", "c", "dq", "rdot"):
                assert o[k].tobytes() == ref[k].tobytes(), (chunks, share, k)
