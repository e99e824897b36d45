"""Speaker-verification trials (DESIGN.md section 5.27) restated in numpy float64 (test infrastructure; product code
never imports it): item statistics, the same-speaker LLR of section 5.15 per trial, AS-norm, and the error rates (EER,
minDCF with its threshold, actDCF, Cllr) by np.sort / np.unique with the operation order of the specification, so that
the device's metrics can be compared bit for bit."""
import numpy as np

from oracle import link_oracle


def statistics(fea, item, M):
    """n [M] and F [M,R] float64 of the items 0 .. M-1 (link_oracle.statistics)."""
    return link_oracle.statistics(fea, item, M)


def llr_trials(n_e, F_e, n_t, F_t, Phi, c, ti, tj, chunk=1 << 16):
    """LLR [T] of every trial (enrolment item ti[t], test item tj[t]) by section 5.15's formula."""
    Phi = np.asarray(Phi, dtype=np.float64)

    def side(n, F):
        n = np.asarray(n, dtype=np.float64)
        L = 1.0 + c * n[:, None] * Phi[None, :]
        b = c * np.sqrt(Phi)[None, :] * np.asarray(F, dtype=np.float64)
        return L, b, np.sum(b * b / L - np.log(L), axis=1)
    Le, be, ee = side(n_e, F_e)
    Lt, bt, et = side(n_t, F_t)
    ti, tj = np.asarray(ti, dtype=np.int64), np.asarray(tj, dtype=np.int64)
    out = np.empty(len(ti))
    for a in range(0, len(ti), chunk):
        i, j = ti[a:a + chunk], tj[a:a + chunk]
        L = Le[i] + Lt[j] - 1.0
        x = be[i] + bt[j]
        out[a:a + chunk] = 0.5 * (np.sum(x * x / L - np.log(L), axis=1) - ee[i] - et[j])
    return out


def as_norm(llr, mean_e, std_e, mean_t, std_t, ti, tj):
    """S [T] = 1/2 [ (LLR - mu_i) / sigma_i + (LLR - mu_j) / sigma_j ]."""
    ti, tj = np.asarray(ti, dtype=np.int64), np.asarray(tj, dtype=np.int64)
    return 0.5 * ((llr - mean_e[ti]) / std_e[ti] + (llr - mean_t[tj]) / std_t[tj])


def softplus(x):
    return np.maximum(x, 0.0) + np.log1p(np.exp(-np.abs(x)))


def error_rates(scores, labels, p_targets=(0.01,), c_miss=1.0, c_fa=1.0):
    """The metrics of section 5.27 as a dict: n_target, n_nontarget, eer, cllr, and per operating point (lists in the
    order of p_targets) min_dcf, threshold, act_dcf.  Also the candidate thresholds and P_miss, P_fa at each."""
    s = np.asarray(scores, dtype=np.float64) + 0.0        # -0.0 + 0.0 = +0.0: one value
    lab = np.asarray(labels).astype(bool)
    T = len(s)
    n_tar = int(lab.sum())
    n_non = T - n_tar
    order = np.argsort(s, kind='stable')
    ss, ls = s[order], lab[order]
    cand, first = np.unique(ss, return_index=True)
    pos = np.append(first, T)
    tar_before = np.concatenate([[0], np.cumsum(ls, dtype=np.int64)])
    miss = tar_before[pos]
    fa = n_non - (pos - miss)
    pm = miss / n_tar
    pf = fa / n_non
    thresholds = np.append(cand, np.inf)
    k = int(np.nonzero(pm >= pf)[0][0])
    a = pm[k - 1] - pf[k - 1]
    b = pm[k] - pf[k]
    lam = a / (a - b)
    eer = pf[k - 1] + lam * (pf[k] - pf[k - 1])
    out = dict(n_target=n_tar, n_nontarget=n_non, eer=float(eer), min_dcf=[], threshold=[], act_dcf=[],
               candidates=thresholds, p_miss=pm, p_fa=pf)
    for p in p_targets:
        cm = c_miss * p
        cf = c_fa * (1.0 - p)
        den = min(cm, cf)
        cost = (cm * pm + cf * pf) / den
        i = int(np.argmin(cost))
        theta = np.log(cf / cm)
        m_a = int(np.sum(s[lab] < theta))
        f_a = int(np.sum(s[~lab] >= theta))
        out['min_dcf'].append(float(cost[i]))
        out['threshold'].append(float(thresholds[i]))
        out['act_dcf'].append(float((cm * (m_a / n_tar) + cf * (f_a / n_non)) / den))
    out['cllr'] = float((np.sum(softplus(-s[lab])) / n_tar + np.sum(softplus(s[~lab])) / n_non) / (2.0 * np.log(2.0)))
    return out
