"""The bf16 store-only backward contraction, checked on what it stores: dq = bf16(bf16(S_ext) dY_ext^T - c) for every
column < ld (the pad columns past the last voxel included), and the row-dot r = c + sum_j Pt_ij dq_ij / sum_j Pt_ij
accumulated from those rounded values."""
import numpy as np
import pytest

from oracle.tangram_oracle import synthetic_inputs

pytestmark = pytest.mark.gpu

CASES = [
    (3000, 2000, 100),   # 192 output tiles, more than there are SMs: CTAs reuse their Pt / dq buffer and barrier phases
    (1000, 257, 130),    # ragged rows and columns, ld = 320
    (9000, 300, 70),     # two cell chunks, one launch each; the last row tile is ragged and its second half empty
    (33000, 130, 40),    # four cell chunks, one launch each; the last chunk ragged
]


def _bf16(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(torch.bfloat16).to(torch.float64).numpy()


@pytest.mark.parametrize("N,V,K", CASES)
def test_backward_stores_centred_dq_and_row_dot(N, V, K):
    from tangram_b200.engine import Engine
    inp = synthetic_inputs(N, V, K, seed=N + V)
    e = Engine(N, V, K, precision="bf16", lambda_d=1.0, lambda_r=1e-3)
    e.set_expression(inp["S"], inp["G"])
    e.set_density(inp["d"])
    e.set_mapping(np.random.default_rng(N).standard_normal((N, V)).astype(np.float32))
    for _ in range(2):                        # the second step leaves a Pt written by the update, not by the row pass
        e.step_begin()
        e.step_end(0.1)
    Ke, ld = (int(x) for x in e.debug("shape")[:2])
    Pt = e.debug("Pb").reshape(N, ld).astype(np.float64)      # what the next backward consumes
    c = e.debug("rcenter").astype(np.float64)
    e.step_begin()
    e.step_end(0.1)
    dq = e.debug("dq").reshape(N, ld).astype(np.float64)
    dY = np.zeros((ld, Ke))
    dY[:V] = e.debug("dY").reshape(V, Ke)
    rdot = e.debug("rdot").astype(np.float64)
    S = _bf16(e.debug("Sx").reshape(N, Ke))

    ref = S @ dY.T - c[:, None]
    # fp32 accumulation over Ke products, then one bf16 rounding (half an ulp: 2^-8 relative)
    chain = Ke * 2.0 ** -23 * (np.abs(S) @ np.abs(dY).T)
    err = np.abs(dq - ref)
    tol = 2.0 ** -8 * (np.abs(ref) + chain) + chain + 1e-30
    bad = np.argwhere(err > tol)
    assert bad.size == 0, f"{len(bad)} elements off, first at {tuple(bad[0])}: {dq[tuple(bad[0])]} vs {ref[tuple(bad[0])]}"

    num = (Pt * dq).sum(axis=1)
    z = Pt[:, :V].sum(axis=1)
    r_ref = c + num / z
    scale = np.abs(Pt * dq).sum(axis=1) / z
    assert np.all(np.abs(rdot - r_ref) <= 2e-3 * scale + 1e-6 * np.abs(c) + 1e-12)
