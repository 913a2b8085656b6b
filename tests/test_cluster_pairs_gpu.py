"""The tensor-core contractions run as 2-CTA clusters: a work item is a pair of 128-row tiles that share one B tile, and
with an odd number of row tiles the last pairs have a phantom second tile that loads and multicasts its half of B but
must write nothing.  These shapes put odd row-tile counts into both contractions (one forward row tile: every pair
half phantom), ragged last column tiles, a bf16 cell chunk with an odd row-tile count, bf16x3 with the 2048-cell chain
cut, and a projection with an odd number of 512-cell chains and row tiles.  Each stage is checked against float64 by the
checkers of test_stages_gpu, which also require the pad columns of P, dP, dq and Y_ext past the live ones to stay zero."""
import numpy as np
import pytest

import tests.test_stages_gpu as st
from oracle.tangram_oracle import synthetic_inputs
from tests.helpers import rel_fro

pytestmark = pytest.mark.gpu


X3_PAIR_SHAPES = [
    (300, 100, 70, False),       # forward: one row tile (its pair partner is a phantom); backward: 3 row tiles, Ke 128 of a 256 tile
    (2049, 640, 300, False),     # two forward chains (the 2048 cut), 5 forward / 17 backward row tiles, ragged second column tile
    (4100, 1100, 130, False),    # three chains, 9 forward / 33 backward row tiles
    (1300, 390, 60, True),       # clusters mode: 4 forward row tiles, 11 backward row tiles
]


@pytest.mark.parametrize("N,V,K,clusters", X3_PAIR_SHAPES)
def test_bf16x3_stages_odd_tile_pairs(N, V, K, clusters):
    st.test_bf16x3_stages(N, V, K, clusters)


BF16_PAIR_SHAPES = [
    (8500, 520, 90, 0.0),        # two cell chunks of 34 and 33 row tiles; 5 forward row tiles per chunk
    (1100, 100, 2100, 1e-3),     # one forward row tile, 9 backward row tiles, Ke 2112: ragged ninth column tile
]


@pytest.mark.parametrize("N,V,K,lam_r", BF16_PAIR_SHAPES)
def test_bf16_stages_odd_tile_pairs(N, V, K, lam_r):
    st.test_bf16_stages(N, V, K, lam_r)


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
def test_project_odd_chains_and_row_tiles(precision):
    """tgb200_project over 1300 cells (three 512-cell chains, the last one ragged) onto 333 voxels (three 128-row tiles)
    and 300 + 77 columns: softmax(M)^T X to fp32 grade against float64."""
    from tangram_b200 import Mapper
    N, V, K = 1300, 333, 60
    inp = synthetic_inputs(N, V, K, seed=31)
    M0 = np.random.default_rng(9).standard_normal((N, V)).astype(np.float32)
    m = Mapper(S=inp["S"], G=inp["G"], d=inp["d"], lambda_d=1.0, M0=M0, precision=precision, device="cuda:0")
    m.train(2, print_each=None)
    M = m.state()[0].astype(np.float64)
    P = np.exp(M - M.max(axis=1, keepdims=True))
    P /= P.sum(axis=1, keepdims=True)
    X = np.random.default_rng(10).random((N, 377)).astype(np.float32)
    got = m.project(X)
    assert got.shape == (V, X.shape[1]) and np.all(np.isfinite(got))
    assert rel_fro(got, P.T @ X.astype(np.float64)) < 3e-6
