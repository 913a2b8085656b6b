"""Which stream each launch of an iteration goes to (tgb200_debug_timeline), as counts of (name, stream) so that the order
within a stream may change.  The bit-identity tests cannot see a launch that moved to another stream.

Streams: 0 the caller's, 1 the handle's contraction stream, 2 its update stream, 3 the next iteration's forward chunks
that tgb200_run issues during the backward.  Only a bf16 handle with several cell chunks has streams 1-3.
"""
import collections

import numpy as np
import pytest

from oracle.tangram_oracle import synthetic_inputs

pytestmark = pytest.mark.gpu

LR = 0.1
PIPELINE = ("tc_gemm_fwd", "row_norm", "scale_rows", "tc_gemm_bwd_dp", "rowdot_finalize", "adam_rows")


@pytest.fixture(autouse=True)
def _default_chunks(monkeypatch):
    monkeypatch.delenv("TGB200_CHUNKS", raising=False)


def _engine(precision, N, V, K, constrained=False, **lam):
    from tangram_b200 import _lib
    from tangram_b200.engine import Engine
    inp = synthetic_inputs(N, V, K, seed=N)
    if constrained:
        lam.update(lambda_count=1.0, lambda_f_reg=1.0, target_count=float(V))
    e = Engine(N, V, K, precision=precision, density_mode=_lib.DENSITY_CELLS, constrained=constrained, **lam)
    e.set_expression(inp["S"], inp["G"])
    e.set_density(inp["d"])
    rng = np.random.default_rng(N + 1)
    e.set_mapping(rng.standard_normal((N, V)).astype(np.float32))
    if constrained:
        e.set_filter(rng.standard_normal(N).astype(np.float32))
    return e, int(e.debug("shape")[4])


def _recorded(e, work):
    e.timeline(True)
    work()
    return collections.Counter((name, stream) for name, stream, _ in e.timeline(False))


@pytest.mark.parametrize("N,V,K,lam_r", [(9000, 300, 70, 1e-3), (33000, 130, 40, 0.0)])
def test_bf16_pipeline_streams(N, V, K, lam_r):
    """run(3) from a fresh mapping: the contractions and the loss stage on stream 1, the update on stream 2, and the
    second and third forwards issued ahead on stream 3.  Step by step, with a validation due, or profiled, nothing is
    issued ahead; profiling runs everything on the caller's stream."""
    e, n = _engine("bf16", N, V, K, **({"lambda_r": lam_r} if lam_r else {}))
    assert n > 1, "the pipeline needs more than one cell chunk"
    got = _recorded(e, lambda: e.run(3, LR))
    pipeline = {k: v for k, v in got.items() if k[0] in PIPELINE}
    assert pipeline == {("tc_gemm_fwd", 1): n, ("tc_gemm_fwd", 3): 2 * n,
                        ("row_norm", 1): n, ("row_norm", 3): 2 * n,
                        ("scale_rows", 1): n, ("scale_rows", 3): 2 * n,
                        ("tc_gemm_bwd_dp", 1): 3 * n,
                        ("rowdot_finalize", 2): 3 * n, ("adam_rows", 2): 3 * n}, got
    rest = {k: v for k, v in got.items() if k[0] not in PIPELINE}
    assert all(stream == 1 for _, stream in rest), got
    for name in ("loss_reduce", "loss_scalars", "dy_assemble"):
        assert rest[(name, 1)] == 3, (name, got)

    def steps():
        for _ in range(2):
            e.step_begin()
            e.step_end(LR)
    got = _recorded(e, steps)
    assert {s for _, s in got} == {1, 2}, got
    assert got[("adam_rows", 2)] == 2 * n and got[("tc_gemm_fwd", 1)] == 2 * n, got

    e.set_validation(1)
    got = _recorded(e, lambda: e.run(3, LR))
    assert {s for _, s in got} == {1, 2}, got
    assert got[("adam_rows", 2)] == 3 * n, got
    e.set_validation(0)

    got = _recorded(e, lambda: e.profile_step(LR))
    assert {s for _, s in got} == {0}, got
    assert got[("adam_rows", 0)] == n, got


@pytest.mark.parametrize("precision,N,constrained", [("bf16", 2049, False), ("bf16x3", 1500, False),
                                                     ("fp32", 1500, False), ("bf16", 2049, True)])
def test_one_chunk_handle_runs_on_the_callers_stream(precision, N, constrained):
    """A handle without streams driven on the legacy default stream (stream=None, Engine's default) labels every launch
    0: its streams are null pointers too, and a launch there is not one on the handle's contraction stream."""
    e, n = _engine(precision, N, 200, 60, constrained=constrained)
    assert n == 1

    def work():
        e.run(2, LR)
        e.step_begin()
        e.step_end(LR)
    got = _recorded(e, work)
    assert got[("loss_scalars", 0)] == 3, got
    assert {s for _, s in got} == {0}, got
