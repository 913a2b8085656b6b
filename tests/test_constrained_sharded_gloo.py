"""Cell-sharded constrained mode on CPU: `map_cells_to_space(mode="constrained", process_group=, gather=)` with two gloo
ranks over an oracle-backed stand-in for the CUDA MapperConstrained.  What is tested is the host contract -- each rank's
rows of the reference's second M0 draw and its entries of F0, the exchange of [Y | f-weighted column sums | filter sums],
per-rank AnnData with obs['F_out'] and uns['shard_rows'], global per-gene scores, the rank-0 gather -- against the
unsharded oracle."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle.tangram_oracle import OracleMapperConstrained, synthetic_inputs
from tangram_b200.mapping_optimizer import discard_normal_rows, legacy_normal_rows
from tangram_b200.sharded import shard_rows, sharded_steps


@pytest.mark.parametrize("n_rows, n_cols, block", [(7, 5, 3), (10, 3, 4), (1, 1, 4096), (9, 11, 2)])
def test_discard_normal_rows_leaves_the_generator_where_the_full_draw_does(n_rows, n_cols, block):
    np.random.seed(11)
    np.random.normal(0, 1, (n_rows, n_cols))
    want = np.random.get_state()
    np.random.seed(11)
    discard_normal_rows(n_rows, n_cols, block_rows=block)
    got = np.random.get_state()
    assert np.array_equal(want[1], got[1]) and want[2:] == got[2:]


def test_host_constrained_draw_of_a_shard_equals_its_slice_of_the_full_draw():
    """The host path of MapperConstrained's draw for rows [r0, r1): the first N x V block discarded, rows [r0, r1) of the
    second, the rest of it discarded, then F -- same bits as the reference's three full draws, same generator state."""
    N, V = 23, 6
    np.random.seed(4)
    np.random.normal(0, 1, (N, V))
    M_full, F_full = np.random.normal(0, 1, (N, V)), np.random.normal(0, 1, N)
    want = np.random.get_state()
    for r0, r1 in (shard_rows(N, r, 3) for r in range(3)):
        np.random.seed(4)
        discard_normal_rows(N, V)
        M = legacy_normal_rows(None, N, V, r0, r1)
        discard_normal_rows(N - r1, V)
        F = np.random.normal(0, 1, N)[r0:r1]
        got = np.random.get_state()
        assert np.array_equal(M, M_full[r0:r1].astype(np.float32)) and np.array_equal(F, F_full[r0:r1])
        assert np.array_equal(want[1], got[1]) and want[2:] == got[2:]


class OracleConstrainedShardEngine:
    """step_begin / exchange_tensor / step_end over the oracle's constrained math for cells [r0, r1).  The exchange buffer
    is [Y = P^T (f o S) | f-weighted column sums of P | sum P log P, sum f, sum (f - f^2)]: everything the loss needs that
    sums over cells."""

    def __init__(self, S, G, d, M0, F0, r0, r1, lam):
        self.o = OracleMapperConstrained(S[r0:r1], G, d, M0=M0, F0=F0, **lam)
        self.lam, self.target_count = self.o.lam, self.o.target_count
        V, K = self.o.G.shape
        self.buf = torch.zeros(V * K + V + 3)
        self.history = []

    def exchange_tensor(self):
        return self.buf

    def step_begin(self):
        o = self.o
        V, K = o.G.shape
        self.P = P = torch.softmax(o.M, dim=1)
        self.f = f = torch.sigmoid(o.F)
        self.buf[: V * K] = (P.t() @ (o.S * f[:, None])).reshape(-1)
        self.buf[V * K: V * K + V] = (P * f[:, None]).sum(dim=0)
        self.buf[V * K + V] = (torch.log_softmax(o.M, dim=1) * P).sum()
        self.buf[V * K + V + 1] = f.sum()
        self.buf[V * K + V + 2] = (f - f * f).sum()

    def step_end(self, lr):
        from oracle.tangram_oracle import _cos_cols, _dcos_cols
        o, lam, P, f = self.o, self.lam, self.P, self.f
        V, K = o.G.shape
        Y = self.buf[: V * K].reshape(V, K)
        csf = self.buf[V * K: V * K + V]
        plogp, s, freg = (float(x) for x in self.buf[V * K + V:])
        c_g, nyg, ngg = _cos_cols(Y, o.G)
        c_v, nyv, ngv = _cos_cols(Y.t(), o.G.t())
        dY = -lam["g1"] * _dcos_cols(Y, o.G, c_g, nyg, ngg)
        if lam["g2"] != 0:
            dY = dY - lam["g2"] * _dcos_cols(Y.t(), o.G.t(), c_v, nyv, ngv).t()
        kl = (torch.special.xlogy(o.d, o.d) - o.d * torch.log(csf / s)).sum()
        cnt = s - self.target_count
        self.history.append(float(-lam["g1"] * c_g.mean() - lam["g2"] * c_v.mean() + lam["d"] * kl - lam["r"] * plogp
                                  + lam["c"] * abs(cnt) + lam["f"] * freg))
        g_cs = -lam["d"] * o.d / csf
        SdY = o.S @ dY.t()
        dP = f[:, None] * (SdY + g_cs[None, :])
        if lam["r"] != 0:
            dP = dP - lam["r"] * (torch.log_softmax(o.M, dim=1) + 1.0)
        dM = P * (dP - (P * dP).sum(dim=1, keepdim=True))
        df = (P * SdY).sum(dim=1) + P @ g_cs + lam["d"] * o.d.sum() / s + lam["c"] * float(np.sign(cnt)) + lam["f"] * (1 - 2 * f)
        dF = df * f * (1 - f)
        o.t += 1
        o.M, o.mM, o.vM = o._adam(o.M, dM, o.mM, o.vM, lr)
        o.F, o.mF, o.vF = o._adam(o.F, dF, o.mF, o.vF, lr)


class _FakeShardedMapperConstrained:
    """MapperConstrained's sharded surface (process_group, _rows, train, project, release) over
    OracleConstrainedShardEngine, drawing this rank's part of the reference's stream as MapperConstrained's host path does."""

    class _Cfg:
        device = 0

    def __init__(self, S, G, d, lambda_d=1, lambda_g1=1, lambda_g2=1, lambda_r=0, lambda_count=1, lambda_f_reg=1,
                 target_count=None, device=None, random_state=None, precision=None, process_group=None):
        self._cfg = self._Cfg()
        self._pg = process_group
        N, V = S.shape[0], G.shape[0]
        rank, world = dist.get_rank(process_group), dist.get_world_size(process_group)
        self._rows = r0, r1 = shard_rows(N, rank, world)
        if random_state:
            np.random.seed(seed=random_state)
        discard_normal_rows(N, V)
        M0 = legacy_normal_rows(None, N, V, r0, r1)
        discard_normal_rows(N - r1, V)
        F0 = np.random.normal(0, 1, N)[r0:r1].astype(np.float32)
        lam = dict(lambda_d=lambda_d, lambda_g1=lambda_g1, lambda_g2=lambda_g2, lambda_r=lambda_r,
                   lambda_count=lambda_count, lambda_f_reg=lambda_f_reg, target_count=target_count)
        self.eng = OracleConstrainedShardEngine(S, G, d, M0, F0, r0, r1, lam)
        self.n_cells = r1 - r0

    def train(self, num_epochs, learning_rate=0.1, print_each=None):
        sharded_steps(self.eng, num_epochs, learning_rate,
                      lambda t: dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self._pg))
        out = torch.softmax(self.eng.o.M, dim=1).numpy()
        hist = {"total_loss": ["tensor({:.4f}, grad_fn=<AddBackward0>)".format(x) for x in self.eng.history]}
        return out, torch.sigmoid(self.eng.o.F).numpy(), hist

    def project(self, X):
        return (torch.softmax(self.eng.o.M, dim=1).t() @ torch.as_tensor(X)).numpy()

    def release(self):
        pass


LAMBDAS = dict(lambda_g2=0.3, lambda_r=1e-3, lambda_count=0.5, lambda_f_reg=0.7, target_count=5)


def _api_worker(rank, world, port, inp, epochs, out):
    import pandas as pd

    import tangram_b200 as tg
    from tangram_b200 import mapping_utils as mu
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(1)
    mu.mo.MapperConstrained = _FakeShardedMapperConstrained
    N, K = inp["S"].shape
    V = inp["G"].shape[0]
    genes = [f"g{i}" for i in range(K)]
    ad_sc = tg.MiniAnnData(X=inp["S"].copy(), obs=pd.DataFrame({"i": np.arange(N)}, index=[f"c{i}" for i in range(N)]),
                           var=pd.DataFrame(index=genes))
    ad_sp = tg.MiniAnnData(X=inp["G"].copy(), obs=pd.DataFrame(index=[f"v{i}" for i in range(V)]), var=pd.DataFrame(index=genes))
    tg.pp_adatas(ad_sc, ad_sp)
    kw = dict(mode="constrained", num_epochs=epochs, random_state=9, verbose=False, process_group=dist.group.WORLD, **LAMBDAS)
    part = tg.map_cells_to_space(ad_sc, ad_sp, **kw)
    full = tg.map_cells_to_space(ad_sc, ad_sp, gather=True, **kw)
    df = part.uns["train_genes_df"].sort_index()
    out[rank] = dict(rows=part.uns["shard_rows"], X=np.asarray(part.X), obs=list(part.obs.index),
                     F_out=np.asarray(part.obs["F_out"]), scores=df["train_score"].values, genes=list(df.index),
                     loss=list(part.uns["training_history"]["total_loss"]),
                     d=np.asarray(ad_sp.obs["rna_count_based_density"], dtype=np.float32),
                     full=None if full is None else (np.asarray(full.X), list(full.obs.index), np.asarray(full.obs["F_out"]),
                                                     "shard_rows" in full.uns, len(full.uns["train_genes_df"])))
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_constrained_map_cells_to_space_two_rank_gloo():
    N, V, K, epochs = 37, 11, 9, 6                         # odd N: uneven shards
    inp = synthetic_inputs(N, V, K, seed=3)
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    out = mp.Manager().dict()
    mp.spawn(_api_worker, args=(2, port, inp, epochs, out), nprocs=2, join=True)
    assert out[0]["genes"] == out[1]["genes"]
    # the unsharded oracle from the reference's full draws (random_state=9); the result does not depend on the gene order
    lam = dict(LAMBDAS, lambda_d=1, lambda_g1=1)
    ref = OracleMapperConstrained(inp["S"], inp["G"], out[0]["d"], random_state=9, **lam)
    ro, rF, rh = ref.train(epochs, print_each=None)
    blocks = sorted((out[r]["rows"], out[r]["X"], out[r]["obs"], out[r]["F_out"]) for r in range(2))
    assert blocks[0][0] == shard_rows(N, 0, 2) and blocks[1][0] == shard_rows(N, 1, 2)
    got = np.concatenate([b[1] for b in blocks])
    got_F = np.concatenate([b[3] for b in blocks])
    assert np.linalg.norm(got - ro) / np.linalg.norm(ro) < 1e-5
    assert np.linalg.norm(got_F - rF) / np.linalg.norm(rF) < 1e-5
    assert [n for b in blocks for n in b[2]] == [f"c{i}" for i in range(N)]          # each rank: obs of ITS cells
    assert all(len(b[3]) == len(b[2]) for b in blocks)                               # obs['F_out'] of those cells
    assert out[0]["loss"] == out[1]["loss"]                                            # the history is global
    floats = [float(x.split("(")[1].split(",")[0]) for x in out[0]["loss"]]
    assert np.allclose(floats, [float(x.split("(")[1].split(",")[0]) for x in rh["total_loss"]], rtol=0, atol=2e-4)
    assert np.array_equal(out[0]["scores"], out[1]["scores"])                        # per-gene scores are global
    Gp = ro.T @ inp["S"]
    cs = (inp["G"] * Gp).sum(0) / (np.linalg.norm(inp["G"], axis=0) * np.linalg.norm(Gp, axis=0))
    assert np.allclose(np.sort(out[0]["scores"]), np.sort(cs), rtol=1e-4)
    assert out[1]["full"] is None                                                     # gather=True: rank 0 only
    fx, fobs, fF, has_rows, n_genes = out[0]["full"]
    assert fx.shape == (N, V) and fobs == [f"c{i}" for i in range(N)] and not has_rows and n_genes == K
    assert np.linalg.norm(fx - ro) / np.linalg.norm(ro) < 1e-5
    assert np.linalg.norm(fF - rF) / np.linalg.norm(rF) < 1e-5
