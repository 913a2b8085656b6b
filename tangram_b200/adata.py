"""Minimal AnnData stand-in used when `anndata` is not installed (it is absent from the
build image).  Only the surface that map_cells_to_space / project_genes / the reference's
plot_utils touch: X, obs, var, uns, obsm, obsp, varm, shape, obs_names / var_names,
`adata[:, genes]`, `adata[mask]`, copy().  If `anndata` is importable it is used instead."""
import numpy as np
import pandas as pd

try:  # pragma: no cover - not present in the build image
    from anndata import AnnData as _RealAnnData
except Exception:  # noqa: BLE001
    _RealAnnData = None


def _take_rows(v, idx):
    """Rows `idx` of a per-gene annotation: a DataFrame keeps its index and columns, anything else becomes an array."""
    return v.iloc[idx] if isinstance(v, (pd.DataFrame, pd.Series)) else np.asarray(v)[idx]


class MiniAnnData:
    def __init__(self, X=None, obs=None, var=None, uns=None, obsm=None, obsp=None, varm=None):
        n_obs = X.shape[0] if X is not None else (len(obs) if obs is not None else 0)
        n_var = X.shape[1] if X is not None else (len(var) if var is not None else 0)
        self.X = X
        self.obs = obs if obs is not None else pd.DataFrame(index=[str(i) for i in range(n_obs)])
        self.var = var if var is not None else pd.DataFrame(index=[str(i) for i in range(n_var)])
        self.uns = uns if uns is not None else {}
        self.obsm = obsm if obsm is not None else {}
        self.obsp = obsp if obsp is not None else {}
        self.varm = varm if varm is not None else {}
        if X is not None and (len(self.obs) != X.shape[0] or len(self.var) != X.shape[1]):
            raise ValueError("obs/var do not match X")

    @property
    def shape(self):
        return (len(self.obs), len(self.var))

    @property
    def n_obs(self):
        return len(self.obs)

    @property
    def n_vars(self):
        return len(self.var)

    @property
    def obs_names(self):
        return self.obs.index

    @property
    def var_names(self):
        return self.var.index

    def var_names_make_unique(self, join="-"):
        seen, out = {}, []
        for g in self.var.index:
            if g in seen:
                seen[g] += 1
                out.append(f"{g}{join}{seen[g]}")
            else:
                seen[g] = 0
                out.append(g)
        self.var.index = out

    def _inplace_subset_var(self, keep):
        """In-place column subset (the method scanpy's filter_genes calls on a real AnnData): X, var and the per-gene
        arrays shrink together."""
        c = self._rows(keep, self.var.index)
        if self.X is not None:
            self.X = self.X[:, c] if hasattr(self.X, "tocsr") else np.asarray(self.X)[:, c]
        self.var = self.var.iloc[c].copy()
        self.varm = {k: _take_rows(v, c) for k, v in self.varm.items()}

    def _rows(self, key, index):
        if isinstance(key, slice):
            return np.arange(len(index))[key]
        key = np.asarray(key) if not isinstance(key, (pd.Series, np.ndarray)) else np.asarray(key)
        if key.dtype == bool:
            return np.nonzero(key)[0]
        if key.dtype.kind in "iu":
            return key
        pos = index.get_indexer(list(key))
        if (pos < 0).any():
            raise KeyError("labels not found: {}".format([k for k, p in zip(key, pos) if p < 0][:5]))
        return pos

    def __getitem__(self, key):
        if not isinstance(key, tuple):
            key = (key, slice(None))
        r = self._rows(key[0], self.obs.index)
        c = self._rows(key[1], self.var.index)
        X = self.X
        if X is not None:
            X = X[r][:, c] if hasattr(X, "tocsr") else np.asarray(X)[np.ix_(r, c)]
        obsp = {k: v[r][:, r] for k, v in self.obsp.items()}
        obsm = {k: np.asarray(v)[r] for k, v in self.obsm.items()}
        varm = {k: _take_rows(v, c) for k, v in self.varm.items()}
        return MiniAnnData(X=X, obs=self.obs.iloc[r].copy(), var=self.var.iloc[c].copy(), uns=self.uns,
                           obsm=obsm, obsp=obsp, varm=varm)

    def copy(self):
        X = self.X.copy() if self.X is not None else None
        return MiniAnnData(X=X, obs=self.obs.copy(), var=self.var.copy(), uns=dict(self.uns),
                           obsm=dict(self.obsm), obsp=dict(self.obsp), varm={k: v.copy() for k, v in self.varm.items()})


def make_adata(X=None, obs=None, var=None, uns=None):
    """sc.AnnData(...) when anndata exists, MiniAnnData otherwise."""
    if _RealAnnData is not None:  # pragma: no cover
        return _RealAnnData(X=X, obs=obs, var=var, uns=uns)
    return MiniAnnData(X=X, obs=obs, var=var, uns=uns)
