"""Validation of a cell-sharded mapping (tgb200_set_validation / tgb200_validation_terms on a shard that holds a
communicator, Mapper(process_group=).train(val_each=)), on one GPU through one-rank NCCL communicators.

A shard holds the first N_r of n_cells_global = 2 N_r cells.  Checked in fp32, bf16x3 and bf16 (one, two and four cell
chunks):

* the last validated epoch's four values against float64 _val_loss_fn from the shard's own Y_ext and rows, with the entropy
  summed over the shard's rows and divided by n_cells_global; validation_terms() equals that history row bit for bit;
* run(n) with validation every epoch (the next iteration's forward serves it, sum h in exchange tail slot [5]) against one
  run(1) per epoch with validation_terms() after each (the separate forward and its all-reduce): bit-identical;
* the entropy_reg column stays NaN with lambda_r = 0, and tail slots [5..7] are exactly 0 on iterations that carry no
  validation; with no row term the whole tail is 0 there, also right after a validated epoch (in-loop and separate
  forward) and after validation is turned off;
* set_comm(NULL) while validating is a STATE error; a sharded constrained handle refuses validation;
* a validated Mapper.train() on a one-rank NCCL group makes the allocating, copying and synchronising runtime calls of the
  same call without validation, and a gloo group refuses validation.

With one rank the all-reduce is the identity: a missing sum cannot show here.  tests/test_sharded_validation_multigpu.py,
on two GPUs, compares against the unsharded mapper.
"""
import contextlib
import io

import numpy as np
import pytest

from oracle.tangram_oracle import synthetic_inputs
from tests.test_sharded_stages_gpu import ERR_STATE, ERR_UNSUPPORTED, RUN_CASES, nccl  # noqa: F401  (nccl: fixture)
from tests.test_stages_gpu import LR, U, Run
from tests.test_validation_gpu import _api_counts, _val_float64

pytestmark = pytest.mark.gpu
LAM = dict(lambda_g2=0.3)             # lambda_r = 0: the training's entropy column must stay NaN


def _shard(nccl, precision, Nr, V, K, seed, comm, lam=LAM):
    run = nccl.track(Run(precision, 2 * Nr, V, K, seed=seed, lam=lam, rows=(0, Nr)))
    run.e.set_comm(comm, 0, 1)
    return run


@pytest.mark.parametrize("precision,Nr,V,K,chunks", RUN_CASES, ids=["fp32", "bf16x3", "bf16", "bf16-2chunks", "bf16-4chunks"])
def test_sharded_validation(nccl, precision, Nr, V, K, chunks):
    n = 4
    c = nccl.comm()
    a, twin = _shard(nccl, precision, Nr, V, K, Nr, c), _shard(nccl, precision, Nr, V, K, Nr, c)
    assert a.nchunks == chunks
    a.e.set_validation(1)
    a.e.run(n, LR)                    # epochs 0..2 served by the next forward, epoch 3 by the separate one
    h = a.e.history()
    got = h[-1, 12:16].astype(np.float64)
    Y = a.e.debug("Y").reshape(V, a.Ke)[:, :K].astype(np.float64)
    M = a.e.debug("M").reshape(Nr, a.ld)[:, :V].astype(np.float64)
    ref, _ = _val_float64(Y, a.inp["G"].astype(np.float64), M, np.ones(K, dtype=bool))
    ref[3] *= Nr / (2 * Nr)           # sum over this shard's rows / n_cells_global
    bound = 4 * np.array([V + K, V + K, V + K, V + Nr], dtype=np.float64) * U * np.maximum(1.0, np.abs(ref))
    ratio = np.abs(got - ref) / bound
    print(f"[sharded validation] {precision} {chunks} chunk(s): |err| / bound {np.array2string(ratio, precision=3)}")
    assert np.all(ratio <= 1.0), (got, ref, ratio)
    assert np.array_equal(a.e.validation_terms(), h[-1, 12:16]), "validation_terms() is not the last history row"
    assert np.all(np.isnan(h[:, 4])), "lambda_r = 0: entropy_reg must stay NaN"

    vals = []
    for _ in range(n):                # every epoch the last of its call: the separate forward and its all-reduce
        twin.e.run(1, LR)
        vals.append(twin.e.validation_terms())
    ht = twin.e.history()
    assert np.array_equal(h[:, :12], ht[:, :12], equal_nan=True), "training history differs"
    assert np.array_equal(ht[:, 12:16], np.zeros((n, 4), dtype=np.float32))
    assert np.array_equal(h[:, 12:16], np.array(vals)), (h[:, 12:16], np.array(vals))


@pytest.mark.parametrize("lam", [{}, {"lambda_r": 1e-3}], ids=["no-row-terms", "entropy"])
@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
def test_tail_slots(nccl, precision, lam):
    """The tail an iteration exchanges: [5] holds sum h only on an iteration that serves a validation; [5..7] are 0 on
    every other one, and with no row term (Mapper's defaults) the whole tail is 0 there, also right after a validated
    epoch and after validation is turned off."""
    Nr, V, K = 1000, 300, 120
    e = _shard(nccl, precision, Nr, V, K, 4, nccl.comm(), lam=lam).e

    def clean(t, what):
        assert not np.any(t[5:]), f"{what}: tail[5..7] = {t[5:]}"
        if not lam:
            assert not np.any(t), f"{what}: no row term, yet tail = {t}"

    def step_tail():
        """one epoch driven by hand; -> the tail its step_begin put in the exchange buffer (one rank: the sum)"""
        e.step_begin()
        t = e.debug("tail")
        e.step_end(LR)
        return t

    e.run(2, LR)
    clean(e.debug("tail"), "before validation")
    e.set_validation(2)
    e.run(3, LR)                      # epochs 0 and 2 validated; epoch 2 by the separate forward, whose tail stays
    t = e.debug("tail")
    assert t[5] == t[0] and t[5] != 0 and not np.any(t[6:]), t
    clean(step_tail(), "epoch 3, after the separate validation forward")
    e.run(2, LR)                      # epoch 4 validated: bf16x3 in epoch 5's forward, bf16 by a separate forward
    t = e.debug("tail")
    if precision == "bf16x3":
        assert t[5] != 0, "epoch 5's exchange must carry epoch 4's sum h"
    else:
        clean(t, "epoch 5, after the separate validation forward of epoch 4")
    clean(step_tail(), "epoch 6 (validated by step_end), after an in-loop validation")
    e.set_validation(0)
    e.run(2, LR)
    clean(e.debug("tail"), "after validation was turned off")


def test_refusals(nccl):
    """set_comm(NULL) while a shard validates is a STATE error; a shard without a communicator and a sharded constrained
    handle refuse validation."""
    from tangram_b200 import _lib
    from tangram_b200.engine import Engine
    Nr, V, K = 1000, 300, 120
    c = nccl.comm()
    e = _shard(nccl, "bf16x3", Nr, V, K, 4, c).e
    lib = e._lib
    e.set_validation(2)
    assert lib.tgb200_set_comm(e._h, None, 0, 1) == ERR_STATE, "set_comm(NULL) while validating"
    e.run(3, LR)
    assert np.isfinite(e.history()[-1, 12:16]).all()
    e.set_validation(0)
    assert lib.tgb200_set_comm(e._h, None, 0, 1) == 0
    assert lib.tgb200_set_validation(e._h, 1, None) == ERR_UNSUPPORTED           # no communicator any more

    inp = synthetic_inputs(2 * Nr, V, K, seed=1)
    f = Engine(Nr, V, K, n_cells_global=2 * Nr, precision="bf16x3", density_mode=_lib.DENSITY_CELLS, constrained=True,
               lambda_d=1.0, lambda_count=1.0, lambda_f_reg=1.0, target_count=float(V))
    nccl.engines.append(f)                                                     # closed before the communicator
    f.set_expression(np.ascontiguousarray(inp["S"][:Nr]), inp["G"])
    f.set_comm(c, 0, 1)
    assert lib.tgb200_set_validation(f._h, 1, None) == ERR_UNSUPPORTED, "sharded constrained handle"


@pytest.mark.parametrize("precision", ["bf16x3", "bf16"])
def test_mapper_validation_on_a_one_rank_group(nccl, precision):
    """train(val_each=) on a sharded Mapper with the handle's own communicator: the val_* lists are the validated history
    rows, validation_terms() equals the last one, and the validated call makes exactly the allocating, copying and
    synchronising runtime calls of the unvalidated one.  On a gloo group both are refused."""
    import torch
    import torch.distributed as dist

    from tangram_b200 import Mapper
    torch.cuda.init()
    N, V, K = 4000, 400, 100
    inp = synthetic_inputs(N, V, K, seed=2)
    M0 = np.random.default_rng(3).standard_normal((N, V)).astype(np.float32)
    kw = dict(S=inp["S"], G=inp["G"], d=inp["d"], lambda_d=1.0, device="cuda:0", M0=M0, precision=precision,
              shard=(1000, 3000))
    dist.init_process_group("nccl", store=dist.HashStore(), rank=0, world_size=1)
    try:
        a, b = Mapper(process_group=dist.group.WORLD, **kw), Mapper(process_group=dist.group.WORLD, **kw)
        try:
            assert a._sharded and a._own_comm and b._own_comm
            b._engine.set_validation(1)                  # the validation's scratch, allocated once per handle
            b._engine.set_validation(0)
            torch.cuda.synchronize()
            with contextlib.redirect_stdout(io.StringIO()):
                plain = _api_counts(lambda: a.train(300, print_each=100))
                val = _api_counts(lambda: b.train(300, print_each=100, val_each=1))
            print(f"[sharded validation] {precision}: runtime calls without validation {dict(plain)}, with {dict(val)}")
            assert sum(v for k, v in plain.items() if "Memcpy" in k) >= 4, "the profiler did not see the library's copies"
            assert val == plain
            h = b.history_matrix
            assert np.all(np.isfinite(h[:, 12:16]))
            _, hist = b.train(7, print_each=None, val_each=3)
            for c, key in enumerate(["val_total_loss", "val_gene_sim", "val_sp_sparsity_weighted_sim", "val_entropy"]):
                assert hist[key] == [float(x) for x in b.history_matrix[::3, 12 + c]], key
            b.train(1, print_each=None, val_each=1)
            vt = b.validation_terms()
            assert [vt[k] for k in ("val_total_loss", "val_gene_sim", "val_sp_sparsity_weighted_sim", "val_entropy")] == \
                [float(x) for x in b.history_matrix[-1, 12:16]]
        finally:
            a.release()
            b.release()
    finally:
        dist.destroy_process_group()
    dist.init_process_group("gloo", store=dist.HashStore(), rank=0, world_size=1)
    try:
        g = Mapper(process_group=dist.group.WORLD, **kw)
        try:
            assert g._sharded and not g._own_comm
            with pytest.raises(ValueError, match="needs an NCCL process group"):
                g.train(2, print_each=None, val_each=1)
            with pytest.raises(ValueError, match="needs an NCCL process group"):
                g.validation_terms()
        finally:
            g.release()
    finally:
        dist.destroy_process_group()
