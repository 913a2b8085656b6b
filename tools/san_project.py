"""Dev tool: target for `compute-sanitizer --tool memcheck` over tgb200_project_map at small shapes -- one cell, a ragged
block under 2048 cells, exactly 2048, and 5000 cells in forced 2048-cell blocks (the ragged last k-block and the
two-stream staging of both slots), each with a dense and a CSR X from host and from device pointers, then a device CSR
whose column indices are past n_genes, negative or repeated within a row (the call must refuse it without writing out of
bounds) followed by a good call.

    compute-sanitizer --tool memcheck python tools/san_project.py
"""
import ctypes
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import scipy.sparse as sp  # noqa: E402
import torch  # noqa: E402

from tangram_b200 import _lib, utils  # noqa: E402


def call(M, X, K, indptr=None, indices=None, data=None, block=0):
    lib = _lib.load()
    p = lambda t: None if t is None else _lib._P(t.data_ptr())   # noqa: E731
    out = torch.empty((M.shape[1], K), dtype=torch.float32, device=M.device)
    x = (p(X), X.stride(0)) if X is not None else (None, 0)
    nnz = 0 if indices is None else indices.shape[0]
    st = lib.tgb200_project_map(p(M), M.shape[0], M.shape[1], M.stride(0), *x, p(indptr), p(indices), p(data), nnz, K,
                                p(out), block, torch.cuda.current_device(),
                                ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    return st, out


rng = np.random.default_rng(0)
for N, V, K, block in ((1, 5, 7, 0), (1000, 70, 63, 0), (2048, 333, 130, 0), (5000, 40, 2048 + 77, 2048)):
    M = rng.random((N, V), dtype=np.float32)
    X = sp.random(N, K, density=0.1, format="csr", dtype=np.float32, random_state=rng)
    ref = utils.project(M, X, _block_rows=block)
    ip, ix, dv, _ = utils._canonical_csr(X, N)
    for where in ("cpu", "cuda"):
        Mt = torch.from_numpy(M).to(where)
        st, out = call(Mt, torch.from_numpy(X.toarray()).to(where), K, block=block)
        assert st == 0 and np.array_equal(out.cpu().numpy(), ref), (N, where, "dense")
        st, out = call(Mt, None, K, *(torch.from_numpy(a).to(where) for a in (ip, ix, dv)), block=block)
        assert st == 0 and np.array_equal(out.cpu().numpy(), ref), (N, where, "csr")
    print(N, V, K, block, "ok", flush=True)

N, V, K = 2100, 40, 30
M = torch.from_numpy(rng.random((N, V), dtype=np.float32)).cuda()
X = sp.random(N, K, density=0.2, format="csr", dtype=np.float32, random_state=rng)
ip, ix, dv, _ = utils._canonical_csr(X, N)
r = int(np.argmax(np.diff(ip) >= 2))
for what, pos, val in (("past n_genes", ip[r + 1] - 1, K + 1000), ("negative", ip[r], -5), ("repeated", ip[r] + 1, ix[ip[r]])):
    bad = ix.copy()
    bad[pos] = val
    st, _ = call(M, None, K, *(torch.from_numpy(a).cuda() for a in (ip, bad, dv)))
    assert st == -1, what
    print("malformed CSR,", what, "refused", flush=True)
st, out = call(M, None, K, *(torch.from_numpy(a).cuda() for a in (ip, ix, dv)))
assert st == 0 and np.array_equal(out.cpu().numpy(), utils.project(M, X))
print("done")
