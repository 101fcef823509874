"""Float64 restatement of the latent PCA of RAVE.validation_epoch_end (rave/model.py:464-488, sklearn PCA(D).fit on the
epoch's posterior means as (B T) x D rows) that rave_b200.core.latent_analysis implements on the device:

  * moments: per chunk (one [B, D, L] tensor) the two-pass mean and centred scatter, merged in list order with Chan's
    pairwise update  d = m_b - m_a,  M2 = M2_a + M2_b + d d^T n_a n_b / n;
  * covariance M2 / (n - 1), eigendecomposition, eigenvalues descending and clipped at zero;
  * signs as sklearn >= 1.5 (svd_flip(u_based_decision=False)): each component's largest-|.| entry is positive;
  * fidelity = cumsum(ev / sum(ev)).

Pure numpy: pinned against the reference's own buffers by oracle/make_golden_validation.py.
"""
import numpy as np


def rows(mean_bdl) -> np.ndarray:
    """[B, D, L] -> [(B L), D] float64 ("b c t -> (b t) c", rave/model.py:467)."""
    a = np.asarray(mean_bdl, dtype=np.float64)
    return a.transpose(0, 2, 1).reshape(-1, a.shape[1])


def chunk_moments(x: np.ndarray):
    n = x.shape[0]
    m = x.mean(0)
    c = x - m
    return n, m, c.T @ c


def chan_merge(a, b):
    na, ma, Ma = a
    nb, mb, Mb = b
    if na == 0:
        return nb, mb.copy(), Mb.copy()
    n = na + nb
    d = mb - ma
    return n, ma + d * (nb / n), Ma + Mb + np.outer(d, d) * (na * nb / n)


def moments(means):
    """(n, mean [D], M2 [D, D]) of the rows of a list of [B, D, L] tensors, merged in list order."""
    D = np.asarray(means[0]).shape[1]
    acc = (0, np.zeros(D), np.zeros((D, D)))
    for m in means:
        acc = chan_merge(acc, chunk_moments(rows(m)))
    return acc


def pca(n, mean, M2):
    """(latent_mean, components [D, D] as rows, explained variance, fidelity) in float64."""
    cov = M2 / (n - 1)
    ev, vec = np.linalg.eigh(cov)
    ev = np.clip(ev[::-1], 0.0, None)
    comps = vec[:, ::-1].T.copy()
    piv = comps[np.arange(comps.shape[0]), np.abs(comps).argmax(1)]
    comps *= np.where(piv < 0, -1.0, 1.0)[:, None]
    return mean, comps, ev, np.cumsum(ev / ev.sum())


def latent_analysis(means):
    return pca(*moments(means))


def fidelity_logs(fidelity):
    """The four scalars validation_epoch_end logs: argmax(fidelity > p) (rave/model.py:481-486)."""
    return {f"fidelity_{p}": float(np.argmax(np.asarray(fidelity) > p)) for p in (.8, .9, .95, .99)}


def separated(ev, rel=1e-3):
    """Indices of the eigenvalues separated from both neighbours by >= rel (relative to the larger): the components that
    are determined up to sign and can be compared one by one."""
    ev = np.asarray(ev, dtype=np.float64)
    out = []
    for i in range(len(ev)):
        ok = ev[i] > 0
        for j in (i - 1, i + 1):
            if 0 <= j < len(ev):
                ok &= abs(ev[i] - ev[j]) >= rel * max(abs(ev[i]), abs(ev[j]))
        if ok:
            out.append(i)
    return out
