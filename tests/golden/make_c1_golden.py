"""BASELINE config 1 golden: the REAL reference Mapper (loaded by path) on the reference's own fixtures
(data/test_ad_sc.h5ad x data/test_ad_sp.h5ad, mode='cells', device='cpu', 100 epochs, random_state=42, lambda_g1=1,
lambda_d=1 with the rna_count_based prior = map_cells_to_space's defaults), on a fixed, seeded sample of 5000 of the
26431 cells x all 9852 voxels x 249 genes so that the stored file stays under 1 MB.
Stores the inputs (S as CSR, G, d) and the reference outputs (loss trajectory, sample rows of the mapping).

    python tests/golden/make_c1_golden.py <checkout of the original Tangram project>

Takes a couple of minutes on 8 cores."""
import contextlib
import importlib.util
import io
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from tangram_b200.h5ad import read_h5ad  # noqa: E402

REF = sys.argv[1]
spec = importlib.util.spec_from_file_location("ref_mo", os.path.join(REF, "tangram", "mapping_optimizer.py"))
ref = importlib.util.module_from_spec(spec)
spec.loader.exec_module(ref)

ad_sc = read_h5ad(os.path.join(REF, "data", "test_ad_sc.h5ad"))
ad_sp = read_h5ad(os.path.join(REF, "data", "test_ad_sp.h5ad"))
genes = ad_sc.uns["training_genes"]
CELLS = np.sort(np.random.default_rng(0).choice(ad_sc.shape[0], 5000, replace=False))
Ssp = ad_sc[:, genes].X.tocsr().astype(np.float32)[CELLS]
S = np.asarray(Ssp.toarray(), dtype=np.float32)
G = np.asarray(ad_sp[:, genes].X, dtype=np.float32)
d = np.asarray(ad_sp.obs["rna_count_based_density"], dtype=np.float32)
EPOCHS = 100
t0 = time.time()
m = ref.Mapper(S=S, G=G, d=d, lambda_g1=1, lambda_d=1, device="cpu", random_state=42)
with contextlib.redirect_stdout(io.StringIO()):
    out, hist = m.train(num_epochs=EPOCHS, learning_rate=0.1, print_each=None)
print("reference C1: %.1f s for %d epochs" % (time.time() - t0, EPOCHS))
rows = np.array([0, 1, 2500, 4999])
np.savez_compressed(
    os.path.join(HERE, "c1_reference.npz"),
    S_data=Ssp.data, S_indices=Ssp.indices.astype(np.int32), S_indptr=Ssp.indptr.astype(np.int64), S_shape=np.array(Ssp.shape),
    G=G, d=d, epochs=np.array(EPOCHS), seed=np.array(42),
    total_loss=np.array([float(x) for x in hist["total_loss"]]), main_loss=np.array(hist["main_loss"]),
    kl_reg=np.array(hist["kl_reg"]), rows=rows, out_rows=out[rows], out_colsum=out.sum(axis=0),
    out_rowmax_idx=out.argmax(axis=1).astype(np.int32), seconds=np.array(time.time() - t0))
print(os.path.getsize(os.path.join(HERE, "c1_reference.npz")) / 1e6, "MB")
