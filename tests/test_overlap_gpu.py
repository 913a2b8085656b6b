"""The bf16 chunk pipeline leaves TGB200_UPDATE_SMS SMs (default 16) to the streaming update beside a contraction by
giving the contraction's grid fewer clusters.  Which cluster computes a tile must not change any bit: every share, down
to a grid of one cluster, gives the same history and mapping as the uncapped grid (share 0), over run() calls and
step_begin / step_end loops, on chunks with odd row-tile counts and a ragged last column tile."""
import numpy as np
import pytest

from oracle.tangram_oracle import synthetic_inputs

pytestmark = pytest.mark.gpu

# 132 SMs hold 66 clusters: 126 leaves 3 clusters to a capped contraction, 132 leaves 1
SHARES = (None, "8", "126", "132")


def _train(monkeypatch, chunks, share, N, V, K, lam_r):
    from tangram_b200 import _lib
    from tangram_b200.engine import Engine
    monkeypatch.setenv("TGB200_CHUNKS", str(chunks))
    if share is None:
        monkeypatch.delenv("TGB200_UPDATE_SMS", raising=False)
    else:
        monkeypatch.setenv("TGB200_UPDATE_SMS", share)
    inp = synthetic_inputs(N, V, K, seed=N)
    e = Engine(N, V, K, precision="bf16", density_mode=_lib.DENSITY_CELLS, lambda_r=lam_r)
    try:
        assert int(e.debug("shape")[4]) == chunks
        e.set_expression(inp["S"], inp["G"])
        e.set_density(inp["d"])
        e.set_mapping(np.random.default_rng(N + 1).standard_normal((N, V)).astype(np.float32))
        e.run(3)
        for _ in range(2):
            e.step_begin()
            e.step_end()
        e.run(2)
        e.run(1)
        out = np.empty((N, V), dtype=np.float32)
        e.get_mapping(out)
        return e.history(), out
    finally:
        e.close()


# 4736 cells in 2 chunks: 20 and 17 row tiles; in 4 chunks: 10, 10, 8 and 9.  300 voxels: a ragged second column tile.
@pytest.mark.parametrize("chunks", [2, 4])
@pytest.mark.parametrize("N,V,K,lam_r", [(4736, 300, 70, 0.0), (4736, 300, 70, 1e-3)])
def test_update_share_is_bit_identical(monkeypatch, chunks, N, V, K, lam_r):
    ref_hist, ref_map = _train(monkeypatch, chunks, "0", N, V, K, lam_r)
    assert np.isfinite(ref_hist[:, 0]).all()
    for share in SHARES:
        hist, mp = _train(monkeypatch, chunks, share, N, V, K, lam_r)
        assert hist.tobytes() == ref_hist.tobytes(), share
        assert mp.tobytes() == ref_map.tobytes(), share
