"""Dev tool: accuracy of the forward contraction in the three modes on the real C1 inputs (one step)."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np, scipy.sparse as sp
from tangram_b200 import Mapper
z = np.load(os.path.join(ROOT, "tests", "golden", "c1_reference.npz"))
S = sp.csr_matrix((z["S_data"], z["S_indices"], z["S_indptr"]), shape=tuple(z["S_shape"])).toarray().astype(np.float32)
G, d = z["G"], z["d"]
M0 = np.random.default_rng(0).standard_normal((S.shape[0], G.shape[0])).astype(np.float32)
import torch
P = torch.softmax(torch.tensor(M0, dtype=torch.float64), dim=1)
Y64 = (P.t() @ torch.tensor(S, dtype=torch.float64)).numpy()
K = S.shape[1]
for prec in ("fp32", "bf16x3", "bf16"):
    m = Mapper(S=S, G=G, d=d, lambda_d=1.0, M0=M0, precision=prec, device="cuda:0")
    m.train(1, print_each=None)
    Ke = int(m._debug("shape")[0]); splits = int(m._debug("shape")[2])
    Y = m._debug("Y").reshape(G.shape[0], Ke)[:, :K].astype(np.float64)
    rel = (Y - Y64) / np.maximum(np.abs(Y64), 1e-30)
    mask = Y64 > 1e-6
    print(f"{prec:7s} splits={splits:3d}: mean rel err {rel[mask].mean():+.3e}  rms {np.sqrt((rel[mask]**2).mean()):.3e}  loss {m.history_matrix[0,0]:.8f}")
