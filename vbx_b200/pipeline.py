"""The steps either side of the VB-HMM call in the reference's driver (SURVEY.md section 8f), batched:

  before:  x-vector transform  l2_norm(lda^T . l2_norm(x - mean1) - mean2)            VBx/vbhmm.py:125-129
           PLDA simultaneous diagonalisation (host, once per model)                   VBx/vbhmm.py:107-113
           projection into the PLDA space  (x - plda_mu) . plda_tr^T [:, :lda_dim]    VBx/vbhmm.py:153
           soft initialisation from hard AHC labels  softmax(onehot * smoothing)      VBx/vbhmm.py:150-152
  after:   hard labels  argsort(-q)[:, 0] (and 2nd best)                               VBx/vbhmm.py:160-162
           merge_adjacent_labels + RTTM lines                                          VBx/diarization_lib.py:113-135, vbhmm.py:48-51

The dense algebra runs on the device through torch (library GEMMs: not the hot path); the label merge is a
host-side O(T) pass exactly like the reference's.  AHC itself (VBx/vbhmm.py:131-146) is out of scope.
"""
import numpy as np
import torch

from ._lib import MAX_STATES as MAX_STATES_F32


def diagonalise_plda(plda_mu, plda_tr, plda_psi):
    """VBx/vbhmm.py:107-113: generalised eigen-problem B v = lambda W v; returns (mu, tr, psi) with psi descending."""
    from scipy.linalg import eigh
    W = np.linalg.inv(plda_tr.T.dot(plda_tr))
    B = np.linalg.inv((plda_tr.T / plda_psi).dot(plda_tr))
    acvar, wccn = eigh(B, W)
    return plda_mu, wccn.T[::-1].copy(), acvar[::-1].copy()


def l2_norm_rows(x):
    """VBx/diarization_lib.py:172-187 for a matrix of row vectors."""
    return x / torch.linalg.vector_norm(x, dim=1, keepdim=True)


def xvector_transform(x_raw, mean1, mean2, lda):
    """VBx/vbhmm.py:129 on the device.  x_raw [N,256] -> [N,128] (float64 like the reference's h5 arrays)."""
    x = l2_norm_rows(x_raw - mean1[None, :])
    x = x @ lda - mean2[None, :]
    return l2_norm_rows(x)


def plda_project(x, plda_mu, plda_tr, lda_dim):
    """VBx/vbhmm.py:153: fea = (x - plda_mu) . plda_tr^T, first lda_dim columns."""
    return ((x - plda_mu[None, :]) @ plda_tr.T)[:, :lda_dim]


def soft_init(labels, n_states, smoothing, dtype=torch.float32):
    """VBx/vbhmm.py:150-152: qinit = softmax(onehot(labels) * smoothing) (rows), float32 on labels' device."""
    q = torch.zeros((labels.shape[0], n_states), dtype=dtype, device=labels.device)
    q.scatter_(1, labels.long()[:, None], float(smoothing))
    return torch.softmax(q, dim=1)


def hard_labels(gamma, second=False):
    """VBx/vbhmm.py:160-162: most (and second most) likely speaker per frame.  Stable ordering like np.argsort(-q)."""
    order = torch.argsort(gamma, dim=1, descending=True, stable=True)
    return (order[:, 0], order[:, 1]) if second and gamma.shape[1] > 1 else order[:, 0]


def merge_adjacent_labels(starts, ends, labels):
    """Compact labelled segments: merge adjacent/overlapping segments with equal labels, split the overlap of
    differently labelled neighbours in the middle.  Same result as VBx/diarization_lib.py:113-135."""
    starts = np.asarray(starts, dtype=np.float64)
    ends = np.asarray(ends, dtype=np.float64)
    labels = np.asarray(labels)
    if len(labels) == 0:
        return starts.copy(), ends.copy(), labels.copy()
    touching = np.isclose(ends[:-1], starts[1:]) | (ends[:-1] > starts[1:])
    cut = np.nonzero(~touching | (labels[1:] != labels[:-1]))[0]        # a new segment starts at cut+1
    first = np.concatenate([[0], cut + 1])
    last = np.concatenate([cut, [len(labels) - 1]])
    s, e, l = starts[first].copy(), ends[last].copy(), labels[first].copy()
    over = np.nonzero(s[1:] < e[:-1])[0]
    mid = (e[over] + s[over + 1]) / 2.0
    e[over] = mid
    s[over + 1] = mid
    return s, e, l


def overlap_segments(seg_times, labels, labels2, overlap):
    """Overlap-aware output of one recording (DESIGN.md section 5.12) as (starts, ends, labels) in seconds: the merged
    segments of `labels` (the single-speaker output), then those of `labels2` (None: no second speaker) cut to the overlap regions
    overlap = (lo, hi) sorted disjoint ticks.  The cut is taken in seconds; seconds map to ticks monotonically, so in
    ticks it is the intersection with the regions."""
    seg = np.asarray(seg_times, dtype=np.float64).reshape(-1, 2)
    s, e, l = merge_adjacent_labels(seg[:, 0], seg[:, 1], labels)
    rows = list(zip(s.tolist(), e.tolist(), l.tolist()))
    if labels2 is not None:
        olo, ohi = (np.asarray(a, dtype=np.int64) / 1e6 for a in overlap)
        s2, e2, l2 = merge_adjacent_labels(seg[:, 0], seg[:, 1], labels2)
        for a, b, k in zip(s2.tolist(), e2.tolist(), l2.tolist()):
            i = int(np.searchsorted(ohi, a, 'right'))            # first region that ends after a
            while i < len(olo) and olo[i] < b:
                x, y = max(a, float(olo[i])), min(b, float(ohi[i]))
                if y > x:
                    rows.append((x, y, k))
                i += 1
    return (np.array([r[0] for r in rows], dtype=np.float64), np.array([r[1] for r in rows], dtype=np.float64),
            np.array([r[2] for r in rows], dtype=np.int64))


def rttm_lines(recording, starts, ends, labels):
    """VBx/vbhmm.py:48-51."""
    return [f'SPEAKER {recording} 1 {s:03f} {e - s:03f} <NA> <NA> {int(l) + 1} <NA> <NA>'
            for s, e, l in zip(starts, ends, labels)]


def diarize_recording(x_raw, seg_times, ahc_labels, transform, plda, Fa, Fb, loopP, lda_dim=128, smoothing=5.0,
                      max_iters=40, epsilon=1e-6, device=None, recording='rec', chain='tcgen05',
                      plda_is_diagonal=False, threshold=-0.015):
    """One recording end to end on the device, the AHC+VB branch of VBx/vbhmm.py:120-172.
    transform = (mean1, mean2, lda); plda = (mu, tr, psi) as read from the Kaldi model (diagonalised here as in
    VBx/vbhmm.py:136-143 unless plda_is_diagonal says it already is).
    ahc_labels=None runs the AHC initialisation on the device too (vbx_ahc, VBx/vbhmm.py:131-146, `threshold` is
    the --threshold bias); otherwise the given labels seed gamma.
    chain='tcgen05' runs the x-vector transform and the PLDA projection in the fused tensor-core kernels
    (vbx_prepare_xvectors; needs lda_dim == 128 and a raw dimension that is a multiple of 32), chain='float64'
    evaluates them with float64 torch ops on the device.  Returns (rttm lines, labels, gamma)."""
    from .batch import VbxBatch
    from . import ahc as _ahc
    dev = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
    f64 = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).to(dev)
    f32 = lambda a: f64(a).float().contiguous()
    mu, tr, psi = plda if plda_is_diagonal else diagonalise_plda(*plda)
    T = int(np.asarray(x_raw).shape[0])
    if chain not in ('tcgen05', 'float64'):
        raise ValueError("chain must be 'tcgen05' or 'float64'")
    if chain == 'tcgen05' and (lda_dim != 128 or tr.shape[0] != 128):
        raise ValueError("chain='tcgen05' needs a 128-dimensional PLDA space")
    # the front end does not depend on the number of speakers: run it on a planning-only batch first
    front = VbxBatch([T], lda_dim, 1, device=dev)
    if chain == 'tcgen05':
        mean1, mean2, lda = transform
        rho, x = front.prepare_xvectors(f32(x_raw), f32(mean1), f32(lda), f32(mean2), f32(mu), f32(tr), f32(psi))
        Phi = f32(psi)
    else:
        mean1, mean2, lda = (f64(a) for a in transform)
        x = xvector_transform(f64(x_raw), mean1, mean2, lda).contiguous()
        fea = plda_project(x, f64(mu), f64(tr), lda_dim)
        Phi = f64(psi[:lda_dim]).float()
        rho = None
    if ahc_labels is None:
        ahc_labels = _ahc.ahc_batch(front, x, threshold=threshold)[0][0]
    front.close()
    S = int(np.max(ahc_labels)) + 1
    q0 = soft_init(torch.from_numpy(np.asarray(ahc_labels)).to(dev), S, smoothing)
    vb = VbxBatch([T], lda_dim, S, device=dev)
    vb.set_option('gemm', 1)
    g = torch.zeros((T, vb.S), dtype=torch.float32, device=dev)
    g[:, :S] = q0
    p = torch.zeros((1, vb.S), dtype=torch.float32, device=dev)
    p[0, :S] = 1.0 / S
    if rho is not None:       # the speaker count was not known when the front end ran: hand its features to the new plan
        fea = rho / torch.sqrt(Phi)[None, :]
    vb.prepare_scale(fea.float().contiguous(), Phi)
    vb.run(g, p, Fa=Fa, Fb=Fb, loopProb=loopP, maxIters=max_iters, epsilon=epsilon)
    labels = vb.hard_labels(g).cpu().numpy().astype(np.int64)      # only the labels leave the device
    s, e, l = merge_adjacent_labels(seg_times[:, 0], seg_times[:, 1], labels)
    vb.close()
    return rttm_lines(recording, s, e, l), labels, g[:, :S]


def keep_labels(gamma, keep):
    """The labels of rule 2 of the speaker-count bound (DESIGN.md section 5.14) with torch ops, for the float64 tier:
    gamma [T,S] of one recording; the `keep` states of largest mass sum_t gamma[t,s] survive (ties: the lower index) and
    every frame takes its best and second best surviving state (ties: the lower index; second -1 when one survives), as
    vbx_hard_labels_keep does on the float32 tier.  Returns (first, second) int64 [T]."""
    S = int(gamma.shape[1])
    order = torch.argsort(gamma.sum(0, dtype=torch.float64), descending=True, stable=True)
    kept = torch.sort(order[:min(int(keep), S)]).values
    f, s = hard_labels(gamma[:, kept], second=True) if len(kept) > 1 else (hard_labels(gamma[:, kept]), None)
    return kept[f], (kept[s] if s is not None else torch.full_like(f, -1))


def _vb_tier(lens, ns, fea, Phi, labels, f64, smoothing, dev, make=None, hi=None, turns=None, random=None, elbo=False,
             prior=None, **run_kw):
    """The VB-HMM step (VBx/vbhmm.py:150-162) for the recordings of one state tier, packed: fea [N,R] float32, labels [N]
    AHC labels (device); turns: None, or a resegment.TurnPack of the recordings, which then start from their init
    RTTM's turns instead (vbx_init_turns, DESIGN.md section 5.20; labels is not read).  f64: the float64 kernels
    (vbx_run_f64, any state count), else one float32 batch padded to the tier, planned by `make` (default VbxBatch).  smoothing: a number or one per recording; run_kw go to run() (Fa, Fb,
    loopProb may be per-recording tensors there).  Returns [(labels, second-best labels or None, iterations, flags)] per
    recording.  hi: None, or an upper bound on the speaker count per recording: a recording whose labels hold more
    speakers takes rule 2 of DESIGN.md section 5.14 (the hi states of largest mass, one vbx_hard_labels_keep launch for
    the tier), and each tuple gains the unconstrained speaker count and 'vb' or 'mass'.  random: None, or (keys, seeds),
    one integer each per recording: the recordings then start from vbx_init_random's draws (DESIGN.md section 5.22;
    labels is not read).  elbo: every tuple also ends with the recording's final ELBO Li[b, n_iters[b] - 1] (NaN
    without iterations).  prior: None, or per recording None or its states' enrolment prior (n [ns], F [ns, R])
    (enroll.prior_states, DESIGN.md section 5.23); the batch then runs with it, zeros for the other states."""
    from .batch import VbxBatch, run_f64
    offs = np.concatenate([[0], np.cumsum(lens)])
    dt = torch.float64 if f64 else torch.float32
    vb = VbxBatch(lens, int(fea.shape[1]), ns, device=dev, f64_only=True) if f64 else \
        (make or VbxBatch)(lens, int(fea.shape[1]), ns, device=dev)
    sm = np.broadcast_to(np.asarray(smoothing, dtype=np.float64), (len(lens),))
    g = torch.zeros((vb.N, vb.S), dtype=dt, device=dev)
    p = torch.zeros((vb.B, vb.S), dtype=dt, device=dev)
    if turns is not None:              # softmax(smoothing * coverage) on the device, section 5.20
        vb.init_turns(turns, sm, g, p)
    elif random is not None:           # flat-Dirichlet rows from Philox on the device, section 5.22
        vb.init_random(random[0], random[1], g, p)
    else:
        for b in range(vb.B):          # VBx/vbhmm.py:150-152: qinit = softmax(onehot * smoothing)
            g[offs[b]:offs[b + 1], :ns[b]] = soft_init(labels[offs[b]:offs[b + 1]], int(ns[b]), float(sm[b]), dtype=dt)
            p[b, :ns[b]] = 1.0 / ns[b]
    if prior is not None and any(x is not None for x in prior):
        n_h, F_h = np.zeros((vb.B, vb.S)), np.zeros((vb.B, vb.S, vb.R))
        for b, x in enumerate(prior):
            if x is not None:
                n_h[b, :len(x[0])], F_h[b, :len(x[0])] = x
        run_kw = dict(run_kw, prior=(torch.from_numpy(n_h).to(dev), torch.from_numpy(F_h).to(dev)))
    if f64:
        res = run_f64(vb, fea.double().contiguous(), Phi.double().contiguous(), g, p, **run_kw)   # VBx/vbhmm.py:154-158
        top2 = [hard_labels(g[offs[b]:offs[b + 1], :ns[b]], second=True) for b in range(vb.B)]   # VBx/vbhmm.py:160-162
        first, second = torch.cat([t[0] for t in top2]), torch.cat([t[1] for t in top2])
    else:
        vb.prepare_scale(fea, Phi)
        res = vb.run(g, p, **run_kw)                                    # VBx/vbhmm.py:154-158
        first, second = vb.hard_labels(g, second=True)                 # VBx/vbhmm.py:160-162
    first, second = first.cpu().numpy().astype(np.int64), second.cpu().numpy().astype(np.int64)
    iters = res['n_iters'].cpu().numpy().tolist()
    flags = res['flags'].cpu().numpy().tolist()
    out = [(first[offs[b]:offs[b + 1]], second[offs[b]:offs[b + 1]] if ns[b] > 1 else None, int(iters[b]), int(flags[b]))
           for b in range(len(lens))]
    if hi is not None:
        k1 = [len(np.unique(o[0])) for o in out]
        over = [b for b in range(len(lens)) if k1[b] > hi[b]]
        if over and f64:
            for b in over:
                f, s = keep_labels(g[offs[b]:offs[b + 1], :ns[b]], hi[b])
                out[b] = (f.cpu().numpy().astype(np.int64), s.cpu().numpy().astype(np.int64) if hi[b] > 1 else None) + out[b][2:]
        elif over:
            keep = np.maximum(np.asarray(ns, dtype=np.int64), 1)
            keep[over] = np.asarray(hi, dtype=np.int64)[over]
            f, s, _ = vb.hard_labels_keep(g, keep.astype(np.int32))
            f, s = f.cpu().numpy().astype(np.int64), s.cpu().numpy().astype(np.int64)
            for b in over:
                out[b] = (f[offs[b]:offs[b + 1]], s[offs[b]:offs[b + 1]] if hi[b] > 1 else None) + out[b][2:]
        out = [o + (k1[b], 'mass' if k1[b] > hi[b] else 'vb') for b, o in enumerate(out)]
    if elbo:
        from .random_init import final_elbo
        last = final_elbo(res['Li'].cpu().numpy(), iters)
        out = [o + (float(last[b]),) for b, o in enumerate(out)]
    vb.close()
    return out


def _tier(n_states):
    """The state tier of a run whose AHC gave n_states clusters: 0 (<= 64 states, planned exactly as in an archive
    without the larger recordings) and 1 (65 .. MAX_STATES_F32, S = 128) on the float32 kernels, 2 (more) on the float64
    kernels.  VBx over-clusters in AHC and lets VB prune, so the state count varies by recording; each tier is batched on
    its own because padding every recording to the largest tier would multiply its bytes."""
    return 0 if n_states <= 64 else 1 if n_states <= MAX_STATES_F32 else 2


def _vb_stage(hyper, labels, labels_d, Zs, lens, fea, Phi, bounds, init, dev, make, split, turns=None, random=None,
              prior=None, **run_kw):
    """Everything after AHC (VBx/vbhmm.py:147-162 and the speaker-count rules of DESIGN.md section 5.14) for the entries
    (k, b): setting k of `hyper`, a list of (Fa, Fb, loopP, smoothing), on recording b.  labels[k]: setting k's AHC
    labels per recording; labels_d[k]: their concatenation on the device (used by init='AHC+VB' only).  fea [N,R] float32
    and Phi [R] as _pad_features leaves them; Zs: the AHC linkages; bounds: None or count_bounds' (lo, hi).
    init='AHC' returns the AHC labels (rule 4 under bounds, per setting).  init='AHC+VB' runs the VB-HMM with the entries
    grouped by state tier (_tier).  A float32 tier runs as batches of consecutive entries planned by `make` (VbxBatch or
    parts.make_batch) and cut by `split` (None: one batch per tier; else split(entries, ns) -> the tier's entries, in
    order, as consecutive batches, e.g. sweep.packer), with Fa, Fb and loopP as numbers when `hyper` holds one setting,
    else as per-recording float64 tensors; the float64 tier runs once per setting.  Under
    bounds the first pass applies rule 2 inside _vb_tier, and rule 3 re-runs every entry with too few speakers from its
    recording's maxclust cut (one cut per recording, shared by all settings) through the same tiers.  run_kw go to run()
    (maxIters, epsilon).  init='RTTM+VB' (DESIGN.md section 5.20) runs the first pass from turns instead, one
    (seg_times, resegment.load_init speaker list) per recording: recording b has one state per init speaker and each
    batch starts from one vbx_init_turns launch (labels and labels_d are not read; Zs only by rule 3, whose re-runs start
    from the AHC cut as above).  init='RANDOM+VB' (DESIGN.md section 5.22) runs the first pass as the entries (k, b, r),
    restart r of (k, b), with random = random_init.RandomStart: random.n_states states each, every batch started by one
    vbx_init_random launch (key random.keys[b], seed random.seed + r); each (k, b) then keeps the restart of largest
    final ELBO (random_init.best_restart) before the count rules, and its tuple ends with (restart, [final ELBO of every
    restart]).  prior: None, or per recording None or the enrolment prior of its AHC states (enroll.prior_states,
    DESIGN.md section 5.23; init='AHC+VB' without bounds only).  Returns {(k, b): (labels, labels2nd or None, iterations, flags[, n_speakers_vb, count_rule])}, the last
    two under bounds."""
    from . import ahc as _ahc
    B = len(lens)
    entries = [(k, b) for k in range(len(hyper)) for b in range(B)]
    if init == 'AHC':
        out = {(k, b): (labels[k][b].astype(np.int64), None, 0, 0) for k, b in entries}
        if bounds is not None:
            for k in range(len(hyper)):
                l1, k1, rules = _count_ahc(Zs, lens, [out[(k, b)][0] for b in range(B)], bounds)
                out.update(((k, b), (l1[b], None, 0, 0, k1[b], rules[b])) for b in range(B))
        return out
    offs = np.concatenate([[0], np.cumsum(lens)])

    def run_tiers(entries, ns, labels_d, hi, from_turns=False, from_random=False):
        """The entries e = (k, b[, r]), with ns[e] states and their labels in labels_d[k] (from_turns: their recordings'
        init turns instead; from_random: restart r's draws, and the tuples end with the final ELBO), through the state
        tiers: {e: _vb_tier tuple}."""
        tiers = [[], [], []]
        for e in entries:
            tiers[_tier(ns[e])].append(e)
        batches = [(g, False) for group in tiers[:2] for g in ([group] if split is None else split(group, ns))]
        batches += [([e for e in tiers[2] if e[0] == k], True) for k in range(len(hyper))]   # no per-recording float64 path
        out = {}
        for group, f64 in batches:
            if not group:
                continue
            recs = [e[1] for e in group]
            init_kw = {}
            if from_turns or from_random:
                if from_turns:
                    from .resegment import pack_turns
                    init_kw = dict(turns=pack_turns([turns[b] for b in recs]))
                else:
                    from .random_init import restart_seed
                    init_kw = dict(random=([random.keys[b] for b in recs], [restart_seed(random.seed, e[2]) for e in group]),
                                   elbo=True)
                g_fea = fea if recs == list(range(B)) else torch.cat([fea[offs[b]:offs[b + 1]] for b in recs])
                g_labels = None
            elif recs == list(range(B)) and all(k == group[0][0] for k, _ in group):
                g_fea, g_labels = fea, labels_d[group[0][0]]
            else:
                g_fea = torch.cat([fea[offs[b]:offs[b + 1]] for b in recs])
                g_labels = torch.cat([labels_d[k][offs[b]:offs[b + 1]] for k, b in group])
            if f64 or len(hyper) == 1:
                Fa, Fb, loopP, smoothing = hyper[group[0][0]]
            else:
                Fa, Fb, loopP = (torch.tensor([hyper[e[0]][i] for e in group], dtype=torch.float64, device=dev)
                                 for i in range(3))
                smoothing = [hyper[e[0]][3] for e in group]
            if prior is not None:
                init_kw = dict(init_kw, prior=[prior[b] for b in recs])
            sub = _vb_tier(lens[recs], np.array([ns[e] for e in group], dtype=np.int32), g_fea, Phi, g_labels, f64,
                           smoothing, dev, make=make, hi=None if hi is None else hi[recs],
                           Fa=Fa, Fb=Fb, loopProb=loopP, **init_kw, **run_kw)
            out.update(zip(group, sub))
        return out

    hi = None if bounds is None else bounds[1]
    chosen = {}
    if init == 'RANDOM+VB':
        from .random_init import best_restart
        runs = [(k, b, r) for k, b in entries for r in range(random.restarts)]     # a recording's restarts side by side
        runs = run_tiers(runs, {e: random.n_states for e in runs}, None, hi, from_random=True)
        out = {}
        for k, b in entries:
            elbos = [runs[(k, b, r)][-1] for r in range(random.restarts)]
            chosen[(k, b)] = (best_restart(elbos), elbos)
            out[(k, b)] = runs[(k, b, chosen[(k, b)][0])][:-1]
    else:
        if init == 'RTTM+VB':
            ns = {(k, b): len(turns[b][1]) for k, b in entries}
        else:
            ns = {(k, b): int(labels[k][b].max()) + 1 if lens[b] else 1 for k, b in entries}
        out = run_tiers(entries, ns, labels_d, hi, from_turns=init == 'RTTM+VB')
    if bounds is None:
        return {e: v + (chosen[e],) for e, v in out.items()} if chosen else out
    lo = bounds[0]
    low = [e for e in entries if out[e][4] < lo[e[1]]]
    recs = sorted({b for _, b in low})
    mc = dict(zip(recs, _ahc.cut_count([Zs[b] for b in recs], lens[recs], lo[recs])))
    met = [e for e in low if lens[e[1]] >= lo[e[1]]]
    again = {}
    if met:
        mc_all = np.zeros(int(offs[-1]), dtype=np.int64)
        for b in recs:
            mc_all[offs[b]:offs[b + 1]] = mc[b]
        again = run_tiers(met, {e: int(mc[e[1]].max()) + 1 for e in met},
                          [torch.from_numpy(mc_all).to(dev)] * len(hyper), None)
    for e in low:
        *r, rule = _recut_outcome(lens[e[1]], lo[e[1]], mc[e[1]], again.get(e))
        out[e] = tuple(r) + (out[e][4], rule)
    return {e: v + (chosen[e],) for e, v in out.items()} if chosen else out


def _check_init(init, overlaps, init_rttm=None, init_states=None, restarts=None, seed=None):
    """init is 'AHC', 'AHC+VB', 'RTTM+VB' or 'RANDOM+VB', an init RTTM is given with 'RTTM+VB' and only with it,
    init_states / restarts / seed only with 'RANDOM+VB' (init_states required there; random_init.check_options), and
    overlap-aware output (overlaps true) has the VB-HMM's second labels.  Returns random_init.RandomStart (without
    keys) for 'RANDOM+VB', else None."""
    from .random_init import check_options
    if init not in ('AHC', 'AHC+VB', 'RTTM+VB', 'RANDOM+VB'):
        raise ValueError('Wrong option for args.initialization.')          # VBx/vbhmm.py:163-164
    if init == 'RTTM+VB' and init_rttm is None:
        raise ValueError("init='RTTM+VB' starts from an existing diarization: it needs init_rttm")
    if init != 'RTTM+VB' and init_rttm is not None:
        raise ValueError(f"init_rttm is the starting point of init='RTTM+VB', not of init={init!r}")
    if overlaps and init == 'AHC':
        raise ValueError("overlap-aware output needs the VB-HMM's second labels: init='AHC+VB'")
    return check_options(init, init_states, restarts, seed)


def _front_end(recordings, names, lens, transform, plda, lda_dim, chain, dev, threshold, ahc=True):
    """x-vector transform + PLDA projection and AHC (VBx/vbhmm.py:125-146) for the whole archive as one batch.  Returns
    (fea [N,R] float32, Phi [R], AHC labels per recording at `threshold`, calibrated thresholds [B], linkage matrices);
    ahc=False: the projection only, and None for the last three."""
    from . import ahc as _ahc
    Dx = int(np.asarray(recordings[names[0]][0]).shape[1])
    chain = _resolve_chain(chain, transform, plda, lda_dim, Dx)
    x_all = np.concatenate([np.asarray(recordings[n][0], dtype=np.float64) for n in names])
    front, x, fea, Phi = _project(x_all, lens, transform, plda, lda_dim, chain, dev)
    ahc_labels = th = Zs = None
    if ahc:
        ahc_labels, th, Zs = _ahc.ahc_batch(front, x, threshold=threshold)      # VBx/vbhmm.py:131-146
    front.close()
    return fea, Phi, ahc_labels, th, Zs


def _resolve_chain(chain, transform, plda, lda_dim, Dx):
    """'auto' -> 'tcgen05' when the shapes allow the fused tensor-core front end, else 'float64'."""
    if chain != 'auto':
        return chain
    tr, lda = np.asarray(plda[1]), np.asarray(transform[2])
    return 'tcgen05' if (lda_dim == 128 and tr.shape[0] == 128 and lda.shape[1] == 128 and Dx % 32 == 0) else 'float64'


def _project(x_all, lens, transform, plda, lda_dim, chain, dev):
    """x-vector transform + PLDA projection (VBx/vbhmm.py:125-129, :153) of raw x-vectors x_all [N,Dx] packed as
    recordings of lens on `chain` ('tcgen05' or 'float64').  Returns (the front-end VbxBatch, for AHC and to close; the
    transformed x-vectors; fea [N,R] float32; Phi [R])."""
    from .batch import VbxBatch
    f64 = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).to(dev)
    f32 = lambda a: f64(a).float().contiguous()
    mu, tr, psi = diagonalise_plda(*plda)
    mean1, mean2, lda = transform
    front = VbxBatch(lens, 128 if chain == 'tcgen05' else 4, 1, device=dev, exact_stop=False)
    if chain == 'tcgen05':
        rho, x = front.prepare_xvectors(f32(x_all), f32(mean1), f32(lda), f32(mean2), f32(mu), f32(tr), f32(psi))
        Phi = f32(psi)
        fea = (rho / torch.sqrt(Phi)[None, :]).contiguous()
    else:
        x = xvector_transform(f64(x_all), f64(mean1), f64(mean2), f64(lda)).contiguous()
        fea = plda_project(x, f64(mu), f64(tr), lda_dim).float().contiguous()
        Phi = f64(psi[:lda_dim]).float().contiguous()
    return front, x, fea, Phi


def _pad_features(fea, Phi):
    """R up to a multiple of 4 with inert zero features (see api.VBx): labels do not depend on them."""
    pad = (-int(fea.shape[1])) % 4
    if pad:
        fea = torch.cat([fea, torch.zeros((fea.shape[0], pad), device=fea.device)], dim=1).contiguous()
        Phi = torch.cat([Phi, torch.zeros(pad, device=Phi.device)]).contiguous()
    return fea, Phi


def count_bounds(names, num_speakers=None, min_speakers=None, max_speakers=None):
    """The speaker-count constraint of every recording (DESIGN.md section 5.14), checked: None when none of the three is
    given, else (lo, hi) int64 arrays over `names`, hi = UNBOUNDED where there is no upper bound.  Each argument is an
    int for the whole archive or a {recording: int} dict holding every recording of `names`.  num_speakers = K means
    lo = hi = K; a missing bound is 1 or unbounded.  ValueError: num_speakers with a bound, a value below 1, lo > hi, a
    recording a dict lacks."""
    if num_speakers is None and min_speakers is None and max_speakers is None:
        return None
    if num_speakers is not None and (min_speakers is not None or max_speakers is not None):
        raise ValueError('give num_speakers or min_speakers / max_speakers, not both')

    def per_rec(v, what, default):
        if v is None:
            return np.full(len(names), default, dtype=np.int64)
        if isinstance(v, dict):
            missing = [n for n in names if n not in v]
            if missing:
                raise ValueError(f'{what}: no count for recordings {missing}')
            vals = [v[n] for n in names]
        else:
            vals = [v] * len(names)
        out = []
        for n, x in zip(names, vals):
            if isinstance(x, (bool, np.bool_)) or not isinstance(x, (int, np.integer)):
                raise ValueError(f'{what}: expected an integer for recording {n!r}, got {x!r}')
            if x < 1:
                raise ValueError(f'{what} must be >= 1, got {int(x)} for recording {n!r}')
            out.append(int(x))
        return np.array(out, dtype=np.int64)

    if num_speakers is not None:
        lo = per_rec(num_speakers, 'num_speakers', 1)
        return lo, lo.copy()
    lo = per_rec(min_speakers, 'min_speakers', 1)
    hi = per_rec(max_speakers, 'max_speakers', UNBOUNDED)
    bad = [n for n, a, z in zip(names, lo, hi) if a > z]
    if bad:
        raise ValueError(f'min_speakers > max_speakers for recordings {bad}')
    return lo, hi


UNBOUNDED = np.iinfo(np.int32).max     # hi of a recording without an upper bound on its speaker count


def _count_ahc(Zs, lens, labels, bounds):
    """Rule 4 of DESIGN.md section 5.14 (init='AHC'): the threshold cut's labels where their count lies in [lo, hi],
    else the maxclust cut at hi (too many) or lo (too few).  Returns (labels, unconstrained counts, rules)."""
    from . import ahc as _ahc
    lo, hi = bounds
    k1 = [len(np.unique(l)) for l in labels]
    target = [hi[b] if k1[b] > hi[b] else lo[b] if k1[b] < lo[b] else 0 for b in range(len(lens))]
    labels = list(labels)
    rules = ['vb'] * len(lens)
    for b in range(len(lens)):
        if target[b]:
            labels[b] = _ahc.cut_count([Zs[b]], [lens[b]], [target[b]])[0]
            rules[b] = 'unmet' if lens[b] < lo[b] else 'ahc'
    return labels, k1, rules


def _recut_outcome(T, lo, mc_labels, rerun):
    """Rule 3 of DESIGN.md section 5.14 for one recording: (labels, labels2nd, iterations, flags, rule) from the VB-HMM
    re-run `rerun` (its _vb_tier tuple, None when the recording has fewer than lo x-vectors) started from the maxclust
    labels mc_labels."""
    if rerun is None:
        return mc_labels, None, 0, 0, 'unmet'
    if len(np.unique(rerun[0])) >= lo:
        return tuple(rerun[:4]) + ('recut',)
    return mc_labels, None, 0, 0, 'ahc'


def _count_fields(item, k1, rule, lo, hi):
    """The reporting fields of a constrained result (DESIGN.md section 5.14)."""
    item.update(count_rule=rule, n_speakers_vb=int(k1), count=(int(lo), None if hi >= UNBOUNDED else int(hi)))
    return item


def diarize_batch(recordings, transform, plda, Fa, Fb, loopP, lda_dim=128, threshold=-0.015, smoothing=5.0, init='AHC+VB',
                  max_iters=40, epsilon=1e-6, device=None, chain='auto', output_2nd=False, overlaps=None,
                  num_speakers=None, min_speakers=None, max_speakers=None, link_threshold=None, enroll=None,
                  enroll_threshold=None, cohort=None, cohort_top=200, init_rttm=None, init_states=None, restarts=None,
                  seed=None, enroll_prior=False):
    """Every recording of an archive in one call on the device - the body of the loop VBx/vbhmm.py:120-179 for all
    recordings at once: x-vector transform + PLDA projection (vbx_prepare_xvectors) and AHC initialisation (vbx_ahc) as
    one batch, then the VB-HMM with the reference's stop rule (vbx_run) and hard labels (vbx_hard_labels) as one batch
    per state tier (<= 64 and 65 .. 128 AHC clusters in float32, more than 128 on the float64 kernels, vbx_run_f64);
    merging and RTTM lines on the host.

    recordings: {name: (x_raw [T,Dx] float array, seg_times [T,2])} in archive order.  transform = (mean1, mean2, lda),
    plda = (mu, tr, psi) as read from the Kaldi model (diagonalised here as VBx/vbhmm.py:107-113 does).
    init: 'AHC' (clustering only), 'AHC+VB' (VBx/vbhmm.py:131,147) or 'RTTM+VB' (VB resegmentation, DESIGN.md section
    5.20: the VB-HMM starts from init_rttm's speaker turns instead of AHC, one state per init speaker, gamma0 =
    softmax(smoothing * the share of each segment inside each speaker's turns) from vbx_init_turns).  init_rttm: with
    'RTTM+VB' only, an RTTM file or directory (score.read_rttm_path) or formats.read_rttm rows holding every recording
    (ValueError naming the missing ones, or those without a speaker, before any device work).  Without count bounds
    'RTTM+VB' runs no AHC; with them rule 2 applies as for 'AHC+VB' and rule 3 re-runs from the AHC linkage cut (its
    states then have no init names).  Each item then also has init_speakers (the init speaker name of each state; None
    for a rule 3 outcome) and rttm_init (its rttm lines, or rttm_overlap's with overlaps, with the speaker field set to
    that name; the rttm or rttm_overlap lines themselves for a rule 3 outcome).
    init='RANDOM+VB' (DESIGN.md section 5.22): the VB-HMM starts from random flat-Dirichlet gamma0 rows with init_states
    states (required, no default) and pi0 = 1 / init_states, drawn on the device by vbx_init_random; restarts (default
    1) runs that many starts of every recording side by side in one batch, restart r with seed (seed + r) mod 2^64
    (seed: default 0, an integer in [0, 2^64)), and each recording keeps the restart of largest final ELBO (ties: the
    lowest r).  A recording's draws depend on its name, not on the archive.  Without count bounds no AHC runs; with them
    rule 2 applies to the chosen restart and rule 3 re-runs from the AHC linkage cut.  Each item then also has restart
    (the chosen index), init_seed (seed + restart mod 2^64: restarts=1 with that seed reruns it alone), elbo (its final
    ELBO) and restart_elbos (the final ELBO of every restart; NaN where a restart ran no iteration).  chain: 'tcgen05' (fused tensor-core front end,
    needs lda_dim == 128 and a 128-dim PLDA), 'float64' (float64 torch ops), 'auto' = tcgen05 when the shapes allow.
    overlaps: None, or overlap regions {name: [(onset, offset)] seconds} (score.read_overlaps; a recording it lacks has
    none): each item then also has rttm_overlap, the overlap-aware RTTM lines (overlap_segments: the second most likely
    speaker inside the overlap regions), and overlap_seconds, the length of the recording's overlap regions.  Needs
    init='AHC+VB' (AHC alone has no second labels).
    num_speakers / min_speakers / max_speakers: a known or bounded speaker count, each an int for the whole archive or a
    {name: int} dict (count_bounds).  The rules of DESIGN.md section 5.14 then apply: a recording whose output already
    has a count inside the bounds keeps it ('vb'); too many speakers keep the hi states of largest posterior mass
    ('mass'); too few re-run the VB-HMM from the AHC linkage cut at lo clusters ('recut', or the cut itself: 'ahc';
    'unmet' when the recording has fewer than lo x-vectors).  Each item then also has count_rule, n_speakers_vb (the
    unconstrained count) and count = (lo, hi or None).
    link_threshold: None, or an LLR threshold for speaker linking across the archive (DESIGN.md section 5.15, after the
    count rules): the speakers of all recordings are scored pairwise from their VB-HMM posteriors and clustered on the
    device (link.link_speakers), and speakers whose average LLR is at least the threshold share an archive-wide id.
    Each item then also has global_speakers ({label: global id}, link.link_cut) and rttm_linked (its rttm lines, or
    rttm_overlap's with overlaps, with the speaker field set to global id + 1).
    enroll: None, or known speakers {name: raw x-vectors [n, Dx]} to name the archive's speakers by (DESIGN.md section
    5.16, after the count rules); needs enroll_threshold, an LLR threshold (there is no default).  The x-vectors go
    through the archive's front end; each recording's speakers are assigned one-to-one to enrolled speakers where their
    LLR reaches the threshold (enroll.enroll_speakers), the others are unknown-<recording>-<label + 1>, or with
    link_threshold linked among themselves across the archive and named unknown-<id + 1>.  Each item then also has
    speaker_names ({label: name}), speaker_llr ({label: the LLR that decided the name}) and rttm_named (its rttm lines,
    or rttm_overlap's with overlaps, with the speaker field set to the name).
    cohort: None, or a cohort of speakers known to be none of the archive's {name: raw x-vectors [n, Dx]} (at least 2
    speakers; DESIGN.md section 5.17).  It goes through the archive's front end, and linking and enrolment then decide
    on the normalised score S (cohort.py: every score standardised by the mean and spread of both speakers' cohort_top
    largest cohort scores), so link_threshold and enroll_threshold are on S; needs link_threshold or enroll.  Each item
    then also has score_norm = {'top_k': min(cohort_top, C), 'cohort_speakers': C}, and with enroll speaker_score
    ({label: the normalised score that decided the name}) in place of speaker_llr.
    enroll_prior: with enroll and init='AHC+VB' (no count bounds), the enrolled speakers take part in the VB-HMM
    (DESIGN.md section 5.23): each recording's AHC clusters are assigned to enrolled speakers as its final speakers
    would be (enroll.enroll_speakers at enroll_threshold, on the normalised score with a cohort), and the state of an
    assigned cluster starts from the enrolled speaker's x-vectors as its speaker prior (VbxBatch.run(prior=)).  Such a
    state is named by that speaker (also where it survives as a second label only), every other as without
    enroll_prior; speaker_llr (speaker_score) holds the cluster's value from that assignment for a prior state and the
    post-hoc value for every other.  Each item then also has prior_speakers ({state: enrolled name}).  Without any
    assignment the VB-HMM runs exactly as without enroll_prior.
    Returns {name: dict(rttm, labels, labels2nd or None, n_speakers, iterations[, rttm_overlap, overlap_seconds]
    [, count_rule, n_speakers_vb, count][, global_speakers, rttm_linked][, speaker_names, speaker_llr or speaker_score,
    rttm_named][, prior_speakers][, score_norm][, init_speakers, rttm_init])}."""
    random = _check_init(init, overlaps is not None, init_rttm, init_states, restarts, seed)
    bounds = count_bounds(list(recordings), num_speakers, min_speakers, max_speakers)
    check_enroll_prior(enroll_prior, enroll is not None, init, bounds is not None)
    if link_threshold is not None:
        from .link import check_threshold
        check_threshold(link_threshold)
    enrolled = None
    dims = {int(np.asarray(r[0]).shape[1]) for r in recordings.values()}
    if enroll is not None or enroll_threshold is not None:
        from . import enroll as _enroll
        if enroll is None:
            raise ValueError('enroll_threshold without enroll')
        _enroll.check_threshold(enroll_threshold)
        enrolled = _enroll.check_enrolment(enroll, next(iter(dims)) if len(dims) == 1 else -1)
    cohort_set = None
    if cohort is not None:
        from . import cohort as _cohort
        if link_threshold is None and enroll is None:
            raise ValueError('a cohort normalises the linking and enrolment scores: it needs link_threshold or enroll')
        _cohort.check_top_k(cohort_top)
        cohort_set = _cohort.check_cohort(cohort, next(iter(dims)) if len(dims) == 1 else -1)
    turns = None
    if init == 'RTTM+VB':
        from .resegment import load_init
        init_turns = load_init(init_rttm, list(recordings))
        turns = [(recordings[n][1], init_turns[n]) for n in recordings]
    if not torch.cuda.is_available():
        from ._lib import VbxError
        raise VbxError('diarize_batch(): no CUDA device - vbx_b200 has no CPU fallback')
    dev = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
    names = list(recordings)
    lens = np.array([np.asarray(recordings[n][0]).shape[0] for n in names], dtype=np.int64)
    if len(names) == 0:
        return {}
    # resegmentation and random starts need the AHC linkage for rule 3 of the count bounds only
    fea, Phi, ahc_labels, _, Zs = _front_end(recordings, names, lens, transform, plda, lda_dim, chain, dev, threshold,
                                             ahc=init in ('AHC', 'AHC+VB') or bounds is not None)
    offs = np.concatenate([[0], np.cumsum(lens)])
    labels_d = None
    if init != 'AHC':
        fea, Phi = _pad_features(fea, Phi)
    if init == 'AHC+VB':
        labels_d = [torch.from_numpy(np.concatenate(ahc_labels)).to(dev)]
    if random is not None:
        from .random_init import name_key
        random = random._replace(keys=[name_key(n) for n in names])
    from .batch import VbxBatch
    side = lambda sets: _side_features(sets, recordings, names, transform, plda, lda_dim, chain, dev, fea, Phi)
    enrolled_fea = cohort_fea = matched = prior = prior_speakers = None
    if enroll_prior:                   # the AHC clusters assigned to enrolled speakers, section 5.23
        from . import enroll as _enroll
        enrolled_fea = side(enrolled)
        norm_ahc = None
        if cohort_set is not None:
            cohort_fea = side(cohort_set)
            norm_ahc = _cohort_norm(cohort_fea, cohort_top, enrolled, enrolled_fea, names, fea, Phi, offs, ahc_labels,
                                    Fa, Fb, dev)
        matched = _enroll.enroll_speakers(fea, Phi, offs, ahc_labels, *enrolled_fea, Fa, Fb, enroll_threshold, dev,
                                          norm=_enroll_norm(norm_ahc))
        prior, prior_speakers = _enroll.prior_states(matched, [k for k, _ in enrolled],
                                                     [int(l.max()) + 1 if len(l) else 1 for l in ahc_labels])
        if all(x is None for x in prior):
            prior = None
    res = _vb_stage([(Fa, Fb, loopP, smoothing)], [ahc_labels], labels_d, Zs, lens, fea, Phi, bounds, init, dev,
                    VbxBatch, None, turns=turns, random=random, prior=prior, maxIters=max_iters, epsilon=epsilon)
    res = [res[(0, b)] for b in range(len(names))]
    labels1, labels2 = [r[0] for r in res], [r[1] for r in res]
    out = {}
    maps = None
    if enrolled is not None and enrolled_fea is None:
        enrolled_fea = side(enrolled)
    norm = None
    if cohort_set is not None:
        norm = _cohort_norm(side(cohort_set) if cohort_fea is None else cohort_fea, cohort_top, enrolled, enrolled_fea,
                            names, fea, Phi, offs, labels1, Fa, Fb, dev)
    if link_threshold is not None:
        from . import link as _link
        table, _, _, Z = _link.link_speakers(fea, Phi, offs, labels1, Fa, Fb, dev,
                                             norm=None if norm is None else norm['archive'][:2])
        maps = _link.link_cut(Z, table, link_threshold, labels2)
    if matched is not None:
        # prior states keep the assignment that attached the prior and its cluster-level value; every other speaker
        # reports the value post-hoc enrolment gives it
        table, assign, best = _enroll.carry_assignment(matched, labels1)
        post = _enroll.enroll_speakers(fea, Phi, offs, labels1, *enrolled_fea, Fa, Fb, enroll_threshold, dev,
                                       norm=_enroll_norm(norm))
        best = np.where(assign >= 0, best, post.best_llr)
        spk_names, spk_llr = _name_archive(table, assign, best, [k for k, _ in enrolled], link_threshold, names, dev,
                                           fea, Phi, offs, labels1, labels2, Fa, Fb, norm)
        _enroll.name_prior_states(spk_names, prior_speakers)
    elif enrolled is not None:
        spk_names, spk_llr = _enroll_archive(enrolled, enrolled_fea, enroll_threshold, link_threshold, names, dev, fea,
                                             Phi, offs, labels1, labels2, Fa, Fb, norm)
    for b, n in enumerate(names):
        ovl = None
        if overlaps is not None:
            from .score import overlap_ticks
            ovl = overlap_ticks(overlaps.get(n))
        out[n] = _result(n, recordings[n][1], labels1[b], labels2[b], res[b][2], output_2nd, ovl)
        if bounds is not None:
            _count_fields(out[n], *res[b][4:6], bounds[0][b], bounds[1][b])
        if maps is not None:
            out[n].update(global_speakers=maps[b],
                          rttm_linked=linked_lines(n, recordings[n][1], labels1[b], labels2[b], maps[b], ovl))
        if enrolled is not None:
            out[n].update(speaker_names=spk_names[b], rttm_named=named_lines(n, recordings[n][1], labels1[b], labels2[b],
                                                                             spk_names[b], ovl))
            out[n]['speaker_llr' if norm is None else 'speaker_score'] = spk_llr[b]
        if prior_speakers is not None:
            out[n]['prior_speakers'] = prior_speakers[b]
        if norm is not None:
            out[n]['score_norm'] = {'top_k': norm['K'], 'cohort_speakers': norm['C']}
        if turns is not None:
            init_fields(out[n], n, recordings[n][1], labels1[b], labels2[b], turns[b][1],
                        None if bounds is None else res[b][5], ovl)
        if random is not None:
            restart_fields(out[n], random.seed, *res[b][-1])
    return out


def restart_fields(item, seed, restart, elbos):
    """The fields of an init='RANDOM+VB' result (DESIGN.md section 5.22): the chosen restart, its seed (to rerun it
    alone), its final ELBO and every restart's.  They describe the choice also when rule 3 of the count bounds replaced
    the chosen restart's labels by a re-run from the AHC cut."""
    from .random_init import restart_seed
    item.update(restart=int(restart), init_seed=restart_seed(seed, restart), elbo=float(elbos[restart]),
                restart_elbos=[float(v) for v in elbos])
    return item


def init_fields(item, name, seg_times, labels, labels2, turns, rule=None, overlap=None):
    """The fields of an init='RTTM+VB' result (DESIGN.md section 5.20): init_speakers, the init RTTM's name of each state
    (resegment.load_init speaker list `turns`), and rttm_init, the item's lines (overlap-aware with overlap regions)
    with the speaker field set to that name.  A rule 3 outcome of the count bounds ('recut', 'ahc', 'unmet') has states
    from the AHC cut: init_speakers None, rttm_init the item's own lines."""
    if rule in ('recut', 'ahc', 'unmet'):
        item.update(init_speakers=None, rttm_init=item['rttm' if overlap is None else 'rttm_overlap'])
        return item
    from .resegment import speaker_names
    spk = speaker_names(turns)
    item.update(init_speakers=spk, rttm_init=named_lines(name, seg_times, labels, labels2, spk, overlap))
    return item


def _side_features(sets, recordings, names, transform, plda, lda_dim, chain, dev, fea, Phi):
    """Speakers outside the archive (enrolled or cohort speakers: [(name, raw x-vectors)]) through the archive's front
    end: the same chain, padded as the archive's features.  Returns (fea_s [N_s,R] float32, speaker index [N_s])."""
    Dx = int(np.asarray(recordings[names[0]][0]).shape[1])
    chain = _resolve_chain(chain, transform, plda, lda_dim, Dx)
    x_s = np.concatenate([x for _, x in sets])
    front, _, fea_s, _ = _project(x_s, [len(x_s)], transform, plda, lda_dim, chain, dev)
    front.close()
    if fea_s.shape[1] < fea.shape[1]:
        fea_s, _ = _pad_features(fea_s, Phi[:fea_s.shape[1]])
    return fea_s, np.repeat(np.arange(len(sets)), [len(x) for _, x in sets])


def _cohort_norm(cohort_fea, top_k, enrolled, enrolled_fea, names, fea, Phi, offs, labels1, Fa, Fb, dev):
    """DESIGN.md section 5.17 for diarize_batch: the cohort statistics of the archive's speakers and of the enrolled
    speakers, each checked for spread (ValueError before any linking or enrolment kernel).  Returns dict(archive,
    enrolled or None: cohort.CohortStats; table: the archive's speaker table; K; C)."""
    from . import cohort as _cohort
    from .link import speaker_table
    fea_c, spk_c = cohort_fea
    table = speaker_table(labels1)
    st = _cohort.cohort_stats(fea, Phi, offs, labels1, fea_c, spk_c, Fa, Fb, top_k, dev)
    _cohort.check_spread(st.std, [f'{names[b]} speaker {l + 1}' for b, l in zip(table.rec.tolist(), table.label.tolist())])
    se = None
    if enrolled is not None:
        se = _cohort.cohort_stats(enrolled_fea[0], Phi, None, enrolled_fea[1], fea_c, spk_c, Fa, Fb, top_k, dev)
        _cohort.check_spread(se.std, [f'enrolled {k}' for k, _ in enrolled])
    return dict(archive=st, enrolled=se, table=table, K=st.K, C=int(spk_c.max()) + 1)


def _enroll_archive(enrolled, enrolled_fea, threshold, link_threshold, names, dev, fea, Phi, offs, labels1, labels2,
                    Fa, Fb, norm=None):
    """DESIGN.md section 5.16 for diarize_batch: the device assignment of the enrolled speakers (their x-vectors through
    the archive's front end, _side_features), and the names (unknown speakers linked among themselves with
    link_threshold).  norm: None or _cohort_norm's statistics (section 5.17): both steps then run on the normalised
    scores.  Returns per recording ({label: name}, {label: llr or normalised score})."""
    from . import enroll as _enroll
    fea_e, spk_e = enrolled_fea
    res = _enroll.enroll_speakers(fea, Phi, offs, labels1, fea_e, spk_e, Fa, Fb, threshold, dev, norm=_enroll_norm(norm))
    return _name_archive(res.table, res.assign, res.best_llr, [k for k, _ in enrolled], link_threshold, names, dev, fea,
                         Phi, offs, labels1, labels2, Fa, Fb, norm)


def _enroll_norm(norm):
    """The norm= argument of enroll.enroll_speakers from _cohort_norm's statistics (None: plain LLRs)."""
    return None if norm is None else tuple(norm['archive'][:2]) + tuple(norm['enrolled'][:2])


def _name_archive(table, assign, best, enrolled_names, link_threshold, names, dev, fea, Phi, offs, labels1, labels2,
                  Fa, Fb, norm=None):
    """The names of section 5.16 from an assignment (table, assign, best) over the final first labels labels1: the
    enrolled name or an unknown one, the unknown speakers linked among themselves with link_threshold (on the
    normalised scores with _cohort_norm's statistics norm over labels1).  Returns per recording ({label: name},
    {label: llr or normalised score})."""
    from . import enroll as _enroll
    from . import link as _link
    spk_names, spk_llr = _enroll.enroll_names(table, assign, best, enrolled_names, names, labels2)
    if link_threshold is not None:
        l1 = [_enroll.mask_named(l, m) for l, m in zip(labels1, spk_names)]
        l2 = [_enroll.mask_named(l, m) for l, m in zip(labels2, spk_names)]
        sub = None
        if norm is not None:                          # the unknown speakers' rows of the archive's statistics
            t, st = norm['table'], norm['archive']
            row = {(b, l): i for i, (b, l) in enumerate(zip(t.rec.tolist(), t.label.tolist()))}
            t2 = _link.speaker_table(l1)
            idx = np.array([row[(b, l)] for b, l in zip(t2.rec.tolist(), t2.label.tolist())], dtype=np.int64)
            sub = (st.mean[idx], st.std[idx])
        lt, _, _, Z = _link.link_speakers(fea, Phi, offs, l1, Fa, Fb, dev, norm=sub)
        lk = _link.link_cut(Z, lt, link_threshold, l2)
        spk_names, spk_llr = _enroll.enroll_names(table, assign, best, enrolled_names, names, labels2, link=lk)
    return spk_names, spk_llr


def check_enroll_prior(enroll_prior, enroll, init, bounds):
    """ValueError unless enroll_prior comes with enrolled speakers (enroll true), init='AHC+VB' and no speaker-count
    bounds (bounds true): the prior is attached to AHC clusters, and rule 3 of the bounds would re-run from another
    cut."""
    if not enroll_prior:
        return
    if not enroll:
        raise ValueError('enroll_prior attaches enrolled speakers to the VB-HMM: it needs enroll')
    if init != 'AHC+VB':
        raise ValueError(f"enroll_prior attaches enrolled speakers to AHC clusters: it needs init='AHC+VB', not {init!r}")
    if bounds:
        raise ValueError('enroll_prior does not combine with num_speakers / min_speakers / max_speakers')


def rttm_name_lines(recording, starts, ends, names):
    """rttm_lines with a string speaker field: names[i] is segment i's speaker."""
    return [f'SPEAKER {recording} 1 {s:03f} {e - s:03f} <NA> <NA> {k} <NA> <NA>' for s, e, k in zip(starts, ends, names)]


def named_lines(name, seg_times, labels, labels2, names, overlap=None):
    """RTTM lines of one recording with named speakers (DESIGN.md section 5.16): the segments _result writes (the
    overlap-aware ones when overlap regions (lo, hi) ticks are given, else the merged first labels) with every label's
    speaker field set to names[label].  labels2 is used inside the overlap regions only."""
    seg = np.asarray(seg_times, dtype=np.float64)
    if overlap is not None:
        s, e, l = overlap_segments(seg, labels, labels2, overlap)
    else:
        s, e, l = merge_adjacent_labels(seg[:, 0], seg[:, 1], labels)
    return rttm_name_lines(name, s, e, [names[int(k)] for k in l])


def linked_lines(name, seg_times, labels, labels2, mapping, overlap=None):
    """RTTM lines of one recording with archive-wide speakers (DESIGN.md section 5.15): the lines _result writes (the
    overlap-aware ones when overlap regions (lo, hi) ticks are given, else the merged first labels) with every label
    replaced by mapping[label] (link.link_cut).  The map is one-to-one within a recording, so the segments are the same.
    labels2 is used inside the overlap regions only."""
    from .link import relabel
    seg = np.asarray(seg_times, dtype=np.float64)
    if overlap is not None:
        return rttm_lines(name, *overlap_segments(seg, relabel(labels, mapping), relabel(labels2, mapping), overlap))
    return rttm_lines(name, *merge_adjacent_labels(seg[:, 0], seg[:, 1], relabel(labels, mapping)))


def _result(name, seg_times, labels, labels2, iterations, output_2nd, overlap=None):
    """The per-recording result of diarize_batch: RTTM lines from merged label segments (VBx/vbhmm.py:169-179), and with
    overlap regions ((lo, hi) ticks) the overlap-aware lines and the regions' length in seconds."""
    seg = np.asarray(seg_times, dtype=np.float64)
    s, e, l = merge_adjacent_labels(seg[:, 0], seg[:, 1], labels)   # VBx/vbhmm.py:169
    item = dict(rttm=rttm_lines(name, s, e, l), labels=labels, labels2nd=labels2, iterations=int(iterations),
                n_speakers=int(len(set(labels.tolist()))), rttm2nd=None)
    if output_2nd and labels2 is not None:
        s2, e2, l2 = merge_adjacent_labels(seg[:, 0], seg[:, 1], labels2)   # VBx/vbhmm.py:174-179
        item['rttm2nd'] = rttm_lines(name, s2, e2, l2)
    if overlap is not None:
        item['rttm_overlap'] = rttm_lines(name, *overlap_segments(seg, labels, labels2, overlap))
        item['overlap_seconds'] = int(np.sum(overlap[1] - overlap[0])) * 1e-6
    return item
