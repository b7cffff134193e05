"""Gain conformance: least-squares estimates of a systematic gain along known directions of an output's error.

The element and rel-L2 rules of tests/test_conformance_cpu.py (and the partition rule of tests/block_shadow.py) ask
whether each element, or each partition, is within a rounding budget.  An error below one rounding per element with a
fixed sign passes them: a blend scale rounded to fp16 inside an epilogue, a store that rounds toward zero, a normaliser
off by one rounding.  It does not average away over a hundred residual adds per step and fifty steps.  This module asks
the other question: does the error have a consistent component along a direction the operation is made of?

Model: e = sum_j beta_j D_j (+ one intercept per nuisance group) + noise, fitted by least squares, where

  * e = out - RN(ref), the error against the correctly rounded fp64 reference (RN to the output's type).  Not
    out - ref: for out = RN16(res + a) with res on the fp16 grid and |a| small next to one ulp of res, out - ref = -a
    exactly, so an honest kernel would regress to beta_a = -1 on the branch that its store swallowed.  Against RN(ref)
    that case is zero, while a real gain still shows: a shift below one ulp flips roundings in proportion to its size;
  * D_j are fp64 tensors of out's shape: the terms the reference adds (the accumulator, a residual, the bias, a blend
    branch), or a derivative (d out / d alpha);
  * the nuisance intercepts (optional, one per (frame, channel) at the layer level) absorb constants rounded once and
    added to every token of a frame (emb_out, the single-key cross-attention rows): those are held by the element rule.

Standard errors are cluster-robust (sandwich, CR1): the remaining noise is not i.i.d., neighbouring tokens share a
tile's accumulation path and the tokens of one channel share its weight roundings.  Clusters are frames, or 128-token
tiles where there are few frames; a second clustering by channel may be given, and sigma is the larger of the two (a
launch whose rows are copies of one row, such as the embedding MLP of a constant c_noise, has as many independent
samples as channels, not as tiles).

A term fails when |beta_j| > B_j + 4 sigma_j.  B_j = U_out / 8 (2^-14 for fp16 outputs: an eighth of an fp16 rounding;
U_out is the unit roundoff of the output's type); the GEMM accumulator term also gets (K / 16) 2^-24, an allowance for
round-toward-zero in the tensor core's fp32 accumulation.  That allowance is a model of the hardware, not a
measurement; the census prints the measured beta beside it.  A direction whose (intercept-free) norm is below 1e-3 of
the output's is skipped and reported as skipped: it carries no information.

The fit accumulates its normal equations (per cluster the raw cross products of (D, e), per (cluster, group) cell the
sums of (D, e) and the count), so a reference evaluated band by band never holds its directions whole."""
import math
from typing import Dict, List, Optional, Sequence

import torch

U16 = 2.0 ** -11
U24 = 2.0 ** -24
ENERGY_MIN = 1e-3         # a direction below this fraction of the output's norm is skipped
N_SIGMA = 4.0
CHUNK = 1 << 22           # elements per accumulation slice


def unit_roundoff(dtype: torch.dtype) -> float:
    return {torch.float16: U16, torch.bfloat16: 2.0 ** -8, torch.float32: U24}[dtype]


def base_bound(dtype: torch.dtype) -> float:
    """B of every term: an eighth of the output type's rounding (2^-14 for fp16)."""
    return unit_roundoff(dtype) / 8


def accumulator_allowance(K: int) -> float:
    """The GEMM accumulator term's allowance for round-toward-zero fp32 accumulation in the tensor core: (K / 16) 2^-24
    (a model, one truncated addition of relative size 2^-24 per 16-deep MMA step)."""
    return K / 16 * U24


def rn(ref: torch.Tensor, dtype: torch.dtype) -> torch.Tensor:
    """The fp64 reference rounded to the output's type, back in fp64."""
    return ref.to(dtype).double()


def clusters(ids: torch.Tensor, size: int = 128, min_clusters: int = 8) -> torch.Tensor:
    """Cluster labels 0..G-1 of integer ids (tokens, pixels, rows): ids // size, halving size while fewer than
    ``min_clusters`` clusters come out."""
    ids = ids.reshape(-1).long()
    while True:
        lab = torch.unique(ids // size, return_inverse=True)[1]
        if size <= 1 or int(lab.max()) + 1 >= min_clusters:
            return lab
        size //= 2


class Term:
    def __init__(self, name, beta, sigma, bound, skipped):
        self.name, self.beta, self.sigma, self.bound, self.skipped = name, beta, sigma, bound, skipped

    @property
    def ratio(self) -> float:
        """|beta| / (B + 4 sigma); 0 for a skipped direction."""
        if self.skipped:
            return 0.0
        return abs(self.beta) / (self.bound + N_SIGMA * self.sigma)

    def __repr__(self):
        if self.skipped:
            return f"{self.name}: skipped (norm below {ENERGY_MIN:g} of the output's)"
        return (f"{self.name}: beta = {self.beta:.2e} (sigma {self.sigma:.1e}, B {self.bound:.1e}) = "
                f"{self.ratio:.2f}x")


class GainFit:
    """Normal equations of e = sum_j beta_j D_j (+ intercepts per group) accumulated chunk by chunk.

    ``names``: the directions; ``bounds``: B_j per name; ``n_clusters``: cluster labels run over 0..n_clusters-1;
    ``n_groups``: nuisance groups 0..n_groups-1 (None: no intercepts).  Groups need not nest in clusters."""

    def __init__(self, names: Sequence[str], bounds: Dict[str, float], n_clusters: int, n_groups: Optional[int] = None,
                 device=None, energy_min: float = ENERGY_MIN):
        self.names, self.bounds, self.energy_min = list(names), dict(bounds), energy_min
        q = len(self.names) + 1
        dd = dict(dtype=torch.float64, device=device)
        self.G = torch.zeros(q, n_clusters, q, **dd)                    # [a, cluster, b]: sum z_a z_b
        self.n_groups = n_groups
        if n_groups is not None:
            self.S = torch.zeros(n_clusters * n_groups, q, **dd)        # per (cluster, group): sum z
            self.N = torch.zeros(n_clusters * n_groups, **dd)
        self.n_clusters, self.out2, self.n = n_clusters, 0.0, 0
        self.G2 = None                                                  # the second clustering's cross products

    def add(self, e: torch.Tensor, dirs: Sequence[torch.Tensor], cluster: torch.Tensor, group=None, out=None,
            cluster2=None, n_clusters2=None):
        """One chunk: e and each direction of one shape; cluster (and group) labels broadcastable to it; ``out`` (the
        output, or its reference) for the norm the skip rule compares with; ``cluster2``: labels 0..n_clusters2-1 of
        a second clustering (channels), used for sigma only (without intercepts).  Works in slices of the leading
        dimension of about 2^22 elements, so that a large sample costs a few times its own size, not q^2 times."""
        if e.dim() >= 1 and e.numel() > CHUNK and e.shape[0] > 1:
            ex = lambda t: None if t is None else t.expand(e.shape)
            dirs_x, cl, gr, o, c2 = [ex(d) for d in dirs], ex(cluster), ex(group), ex(out), ex(cluster2)
            if e.dim() >= 2 and e[0].numel() > CHUNK:          # one leading index at a time, split further inside
                pick = lambda t, i: None if t is None else t[i]
                for i in range(e.shape[0]):
                    self.add(e[i], [d[i] for d in dirs_x], cl[i], pick(gr, i), pick(o, i), pick(c2, i), n_clusters2)
                return
            step = max(1, CHUNK // max(1, e[0].numel()))
            pick = lambda t, i: None if t is None else t[i:i + step]
            for i in range(0, e.shape[0], step):
                self.add(e[i:i + step], [d[i:i + step] for d in dirs_x], cl[i:i + step], pick(gr, i), pick(o, i),
                         pick(c2, i), n_clusters2)
            return
        shape = e.shape
        Z = torch.stack([d.expand(shape).reshape(-1).double() for d in dirs] + [e.reshape(-1).double()], 1)
        c = cluster.to(Z.device).expand(shape).reshape(-1).long()
        for a in range(Z.shape[1]):
            self.G[a].index_add_(0, c, Z[:, a:a + 1] * Z)
        if cluster2 is not None:
            if self.G2 is None:
                self.G2 = torch.zeros(Z.shape[1], n_clusters2, Z.shape[1], dtype=torch.float64, device=Z.device)
            c2 = cluster2.to(Z.device).expand(shape).reshape(-1).long()
            for a in range(Z.shape[1]):
                self.G2[a].index_add_(0, c2, Z[:, a:a + 1] * Z)
        if self.n_groups is not None:
            cell = c * self.n_groups + group.to(Z.device).expand(shape).reshape(-1).long()
            self.S.index_add_(0, cell, Z)
            self.N.index_add_(0, cell, torch.ones_like(Z[:, 0]))
        o = e if out is None else out
        self.out2 += float(o.double().pow(2).sum())
        self.n += Z.shape[0]

    def _cluster_moments(self):
        """[clusters, q, q]: per cluster the cross products of (D, e) after the intercepts are projected out."""
        M = self.G.permute(1, 0, 2)
        if self.n_groups is None:
            return M
        C, g = self.n_clusters, self.n_groups
        S = self.S.reshape(C, g, -1)
        Nc = self.N.reshape(C, g)
        zbar = S.sum(0) / Nc.sum(0).clamp_min(1)[:, None]                 # [groups, q]: group means
        corr = torch.einsum("gi,cgj->cij", zbar, S)
        return M - corr - corr.transpose(1, 2) + torch.einsum("cg,gi,gj->cij", Nc, zbar, zbar)

    @staticmethod
    def _sigma(Mc, idx, p, beta, Ainv):
        """Cluster-robust (CR1) standard errors from per-cluster cross products Mc [clusters, q, q]."""
        scores = Mc[:, idx, p] - Mc[:, idx][:, :, idx] @ beta               # [clusters, k]
        nc = int((Mc.diagonal(dim1=1, dim2=2)[:, idx].sum(1) > 0).sum())      # clusters with data
        if nc < 2:
            return torch.full_like(beta, math.inf)
        meat = scores.t() @ scores * (nc / (nc - 1))
        return (Ainv @ meat @ Ainv).diagonal().clamp_min(0).sqrt()

    def result(self) -> List[Term]:
        Mc = self._cluster_moments()
        M = Mc.sum(0)
        p = len(self.names)
        energy = M.diagonal()[:p].clamp_min(0.0)
        keep = [j for j in range(p) if math.sqrt(float(energy[j])) >= self.energy_min * math.sqrt(self.out2)
                and float(energy[j]) > 0]
        terms = {}
        if keep:
            idx = torch.tensor(keep, device=M.device)
            A = M[idx][:, idx]
            Ainv = torch.linalg.pinv(A)
            beta = Ainv @ M[idx, p]
            sig = self._sigma(Mc, idx, p, beta, Ainv)
            if self.G2 is not None and self.n_groups is None:
                sig = torch.maximum(sig, self._sigma(self.G2.permute(1, 0, 2), idx, p, beta, Ainv))
            for i, j in enumerate(keep):
                terms[j] = Term(self.names[j], float(beta[i]), float(sig[i]), self.bounds[self.names[j]], False)
        return [terms.get(j, Term(self.names[j], 0.0, 0.0, self.bounds[self.names[j]], True)) for j in range(p)]


def fit(out: torch.Tensor, ref: torch.Tensor, dirs: Dict[str, torch.Tensor], bounds: Dict[str, float],
        cluster: torch.Tensor, group=None, n_groups=None, against_rounded: bool = True,
        energy_min: float = ENERGY_MIN, cluster2=None) -> List[Term]:
    """One-shot fit: e = out - RN(ref) (``against_rounded``; else out - ref) on the directions ``dirs``; ``cluster2``:
    a second clustering (labels broadcastable to out), sigma the larger of the two."""
    names = list(dirs)
    labels = cluster.expand(out.shape).reshape(-1).long()
    n_clusters = int(labels.max()) + 1 if labels.numel() else 1
    if group is not None and n_groups is None:
        n_groups = int(group.max()) + 1
    f = GainFit(names, bounds, n_clusters, n_groups if group is not None else None, device=ref.device,
                energy_min=energy_min)
    e = out.double() - (rn(ref, out.dtype) if against_rounded else ref)
    n2 = None if cluster2 is None else int(cluster2.max()) + 1
    f.add(e, [dirs[n] for n in names], cluster, group, out=ref, cluster2=cluster2, n_clusters2=n2)
    return f.result()


def worst(terms: Sequence[Term]):
    """The term with the largest ratio (None when every direction was skipped)."""
    live = [t for t in terms if not t.skipped]
    return max(live, key=lambda t: t.ratio) if live else None


def failures(terms: Sequence[Term]) -> List[Term]:
    return [t for t in terms if t.ratio > 1.0]
