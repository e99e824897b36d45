"""The calibration of a scored trial list (DESIGN.md section 5.28) restated in numpy float64 (test infrastructure;
product code never imports it): the prior-weighted logistic regression by the device's Newton state machine, PAV with
tie blocks twice (sequential pooling and the monotone-chain ROC hull), and minCllr."""
import numpy as np

MAX_PASSES = 64


def softplus(x):
    return np.maximum(x, 0.0) + np.log1p(np.exp(-np.abs(x)))


def _classes(scores, labels):
    s = np.asarray(scores, dtype=np.float64) + 0.0        # -0.0 + 0.0 = +0.0: one value
    lab = np.asarray(labels).astype(bool)
    return np.sort(s[lab]), np.sort(s[~lab])


def separable(scores, labels):
    """None when a finite minimiser exists (min_tar < max_non and min_non < max_tar), else 'above' (every target
    scores at or above every nontarget) or 'below'."""
    st, sn = _classes(scores, labels)
    if st[0] >= sn[-1]:
        return 'above'
    if st[-1] <= sn[0]:
        return 'below'
    return None


def cost(a, b, st, sn, prior):
    """C(a, b) and its gradient and Hessian (ga, gb, haa, hab, hbb)."""
    L = np.log(prior / (1.0 - prior))
    out = []
    for s, target in ((st, True), (sn, False)):
        z = a * s + b + L
        e = np.exp(-np.abs(z))
        hi, lo = 1.0 / (1.0 + e), e / (1.0 + e)
        pz, pmz = np.where(z >= 0, hi, lo), np.where(z >= 0, lo, hi)
        sp = np.maximum(-z if target else z, 0.0) + np.log1p(e)
        r = -pmz if target else pz
        h = hi * lo
        out.append(np.array([sp.sum(), (r * s).sum(), r.sum(), (h * s * s).sum(), (h * s).sum(), h.sum()]))
    f = prior / len(st) * out[0] + (1.0 - prior) / len(sn) * out[1]
    return f[0], f[1:]


def fit(scores, labels, prior=0.5, max_passes=MAX_PASSES):
    """The device's state machine: returns dict(a, b, cllr_prior, passes, status) (status 0 converged, 3 the pass
    limit).  Each pass evaluates the trial point; the first evaluation, or one whose cost did not increase, is accepted,
    d = -H^-1 g; a cost that increased halves the step.  Once -g.d / 2 <= 2^-52 C the last full step is taken without
    the test, in a pass of its own that ends the fit."""
    st, sn = _classes(scores, labels)
    ta = tb = 0.0
    have = False
    a = b = C = da = db = t = 0.0
    status = 3
    passes = 0
    polish = False
    for passes in range(1, max_passes + 1):
        Ct, (ga, gb, haa, hab, hbb) = cost(ta, tb, st, sn, prior)
        if polish:                     # the last full step, taken without the test
            a, b, C = ta, tb, Ct
            status = 0
            break
        if not have or Ct <= C:
            have, a, b, C = True, ta, tb, Ct
            det = haa * hbb - hab * hab
            da = -(hbb * ga - hab * gb) / det
            db = -(haa * gb - hab * ga) / det
            dec = -0.5 * (ga * da + gb * db)
            if not np.isfinite(dec):
                status = 3
                break
            polish = dec <= 2.0 ** -52 * C
            t = 1.0
            ta, tb = a + da, b + db
        else:
            t *= 0.5
            ta, tb = a + t * da, b + t * db
    return dict(a=float(a), b=float(b), cllr_prior=float(C / np.log(2.0)), passes=passes, status=status)


def tie_blocks(scores, labels):
    """(target count, nontarget count) per distinct score, ascending (-0.0 and +0.0 one value)."""
    s = np.asarray(scores, dtype=np.float64) + 0.0
    lab = np.asarray(labels).astype(bool)
    _, inv = np.unique(s, return_inverse=True)
    return (np.bincount(inv, weights=lab).astype(np.int64), np.bincount(inv, weights=~lab).astype(np.int64))


def pav_blocks(scores, labels):
    """PAV by sequential pooling: every tie group one initial block, ascending; a block is pooled into its predecessor
    while the predecessor's target fraction is >= its own.  Returns [(targets, nontargets)] ascending."""
    nt, nn = tie_blocks(scores, labels)
    blocks = []
    for a, b in zip(nt.tolist(), nn.tolist()):
        blocks.append([a, b])
        # prev_t / prev_n >= t / n, exactly: prev_t n >= t prev_n
        while len(blocks) > 1 and blocks[-2][0] * sum(blocks[-1]) >= blocks[-1][0] * sum(blocks[-2]):
            x = blocks.pop()
            blocks[-1][0] += x[0]
            blocks[-1][1] += x[1]
    return [tuple(b) for b in blocks]


def roc_hull(scores, labels):
    """The upper hull of the ROC points P_k = (#nontargets >= c_k, #targets >= c_k) of the candidates c_0 < .. < c_m =
    +inf, by a monotone chain over k ascending keeping strict turns only.  Returns [(x, y)] from (N_non, N_tar) to
    (0, 0)."""
    nt, nn = tie_blocks(scores, labels)
    xs = np.concatenate([np.cumsum(nn[::-1])[::-1], [0]])
    ys = np.concatenate([np.cumsum(nt[::-1])[::-1], [0]])
    h = []
    for p in zip(xs.tolist(), ys.tolist()):
        while len(h) >= 2:
            o, a = h[-2], h[-1]
            if (a[0] - o[0]) * (p[1] - o[1]) - (a[1] - o[1]) * (p[0] - o[0]) > 0:
                break
            h.pop()
        h.append(p)
    return h


def hull_segments(hull):
    """[(dy targets, dx nontargets)] of consecutive hull vertices, in hull order (highest scores last)."""
    return [(p[1] - q[1], p[0] - q[0]) for p, q in zip(hull, hull[1:])]


def min_cllr(scores, labels):
    """minCllr from the hull segments, in hull order, with the device's expression per segment."""
    lab = np.asarray(labels).astype(bool)
    n_tar, n_non = float(lab.sum()), float((~lab).sum())
    tot = 0.0
    for dy, dx in hull_segments(roc_hull(scores, labels)):
        if dx == 0 or dy == 0:
            continue
        dx, dy = float(dx), float(dy)
        u = (dx * n_tar) / (dy * n_non)
        v = (dy * n_non) / (dx * n_tar)
        tot += (dy / n_tar) * np.log1p(u) + (dx / n_non) * np.log1p(v)
    return tot / (2.0 * np.log(2.0))


def calibrate(scores, labels, prior=0.5):
    """dict(a, b, cllr_prior, min_cllr, passes, status, hull_vertices) as the device reports them (a, b, cllr_prior
    NaN for separable classes, status 1)."""
    hull = roc_hull(scores, labels)
    out = dict(min_cllr=float(min_cllr(scores, labels)), hull_vertices=len(hull))
    if separable(scores, labels) is not None:
        out.update(a=float('nan'), b=float('nan'), cllr_prior=float('nan'), passes=0, status=1)
    else:
        out.update(fit(scores, labels, prior))
    return out
