"""Enrolment and cohort normalisation inside the sweep on the device (DESIGN.md section 5.19): vbx_enroll_batch through
enroll.enroll_many against enroll_speakers problem by problem and threshold by threshold (bit for bit, with and without
normalisation, one launch and several), vbx_cohort_stats_batch against cohort_stats, vbx_link_batch with mean and std
against link_speakers(norm=), and sweep_batch's names, scores and DER by name against
diarize_batch(enroll_threshold=) and score_rttm(by_name=True), with a UEM, oracle overlaps, the oracle speaker count,
AHC init, a cohort, ES2005a and the command line."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

from oracle import enroll_oracle
from test_link_gpu import SPEAKER_WIDTHS, width_phi
from vbx_b200 import _lib, cohort, enroll, formats, link, pipeline, score, sweep, synth

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), 'golden')
DEV = torch.device('cuda:0')
THETAS = [-1e6, -50.0, 0.0, 20.0, 1e6]


def _archive(seed, R, E, counts=((3, 0, 150, 1, 17, 0, 2), (0, 0, 0, 0, 0, 0, 0), (5, 2, 0, 40, 1, 1, 9), (1,) * 7)):
    """Seeded features of 7 recordings (one without x-vectors) and one problem per entry of counts (speakers per
    recording; a problem without speakers, a recording with 150), label values with gaps and x-vectors without a
    speaker; E enrolled speakers around the same centres, enrolled speakers 0 and 1 with identical x-vectors.  The last
    3 features are padded, except at the SPEAKER_WIDTHS: there every feature is live, with Phi from width_phi."""
    rng = np.random.default_rng(seed)
    R_live = R if R in SPEAKER_WIDTHS else max(R - 3, 1)
    centres = rng.standard_normal((40, R_live)) * 2.0
    lens = [max(2 * k, 6) if k else 0 for k in np.max(np.array(counts), 0)]
    lens[5] = 0
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    N = int(offs[-1])
    fea = np.zeros((N, R), np.float32)
    fea[:, :R_live] = centres[rng.integers(0, 40, N)] + rng.standard_normal((N, R_live))
    Phi = np.zeros(R, np.float32)
    Phi[:R_live] = width_phi(rng, R) if R in SPEAKER_WIDTHS else np.sort(rng.uniform(0.2, 6.0, R_live))[::-1]
    problems = []
    for ks in counts:
        labels = []
        for T, k in zip(lens, ks):
            k = min(k, T)
            if not k:
                labels.append(np.full(T, -1, np.int64))
                continue
            vals = np.sort(rng.choice(k + 4, k, replace=False))
            lab = np.concatenate([np.arange(k), rng.integers(0, k, T - k)])
            lab = vals[lab]
            lab[k:][rng.random(T - k) < 0.1] = -1
            rng.shuffle(lab)
            labels.append(lab.astype(np.int64))
        problems.append(labels)
    if E >= 2:                                        # speakers 0 and 1: one identical x-vector each
        espk = np.concatenate([[0, 1], np.arange(2, E), rng.integers(2, E, 2 * E) if E > 2 else []]).astype(np.int64)
    else:
        espk = np.zeros(3, np.int64)
    efea = np.zeros((len(espk), R), np.float32)
    efea[:, :R_live] = centres[espk % 40] + rng.standard_normal((len(espk), R_live))
    if E >= 2:
        efea[1] = efea[0]
    Fa = rng.uniform(0.1, 0.6, len(counts))
    Fb = rng.uniform(4.0, 40.0, len(counts))
    return fea, Phi, offs, problems, efea, espk, Fa, Fb


def _largest_single(kind, offs, problems, *shape):
    """One more byte than the largest workspace of a problem alone: a budget that splits the problems over several
    launches (kind 'enroll': shape = (E, N_e, n_thr); 'cohort': (C, N_c); 'link': ())."""
    lib = _lib.load()
    h = ctypes.c_void_p()
    assert lib.vbx_create(0, ctypes.byref(h)) == 0
    try:
        sizes = []
        for labels in problems:
            t = link.speaker_table(labels)
            M = np.array([len(t.rec)], dtype=np.int64)
            k = int(np.diff(np.searchsorted(t.rec, np.arange(len(labels) + 1))).max())
            need = ctypes.c_size_t()
            v = M.ctypes.data_as(ctypes.c_void_p)
            if kind == 'enroll':
                rc = lib.vbx_enroll_batch_workspace_bytes(h, 1, v, shape[0], shape[1], k, shape[2], ctypes.byref(need))
            elif kind == 'cohort':
                rc = lib.vbx_cohort_stats_batch_workspace_bytes(h, 1, v, shape[0], shape[1], ctypes.byref(need))
            else:
                rc = lib.vbx_link_batch_workspace_bytes(h, 1, v, ctypes.byref(need))
            assert rc == 0
            sizes.append(int(need.value))
        return max(sizes) + 1
    finally:
        lib.vbx_destroy(h)


def _thetas(fea, Phi, offs, problems, efea, espk, Fa, Fb, norm=None):
    """THETAS plus the tie case of section 5.16: the LLR of problem 0's first speaker against its best enrolled speaker,
    and the next double above it."""
    r = enroll.enroll_speakers(fea, Phi, offs, problems[0], efea, espk, Fa[0], Fb[0], 0.0, llr=True,
                               norm=None if norm is None else norm[0])
    top = float(r.llr[0].max())
    return THETAS + [top, float(np.nextafter(top, np.inf))]


def _norms(fea, Phi, offs, problems, efea, espk, Fa, Fb, rng):
    cfea = rng.standard_normal((30, fea.shape[1])).astype(np.float32) * 2.0
    cspk = np.arange(30) % 12
    out = []
    for g, labels in enumerate(problems):
        a = cohort.cohort_stats(fea, Phi, offs, labels, cfea, cspk, Fa[g], Fb[g], 5)
        e = cohort.cohort_stats(efea, Phi, None, espk, cfea, cspk, Fa[g], Fb[g], 5)
        out.append((a.mean, a.std, e.mean, e.std))
    return out, cfea, cspk


@pytest.mark.parametrize('R, E', [(8, 1), (16, 7), (128, 300), (16, 300), (128, 7)] + [(R, 33) for R in SPEAKER_WIDTHS])
@pytest.mark.parametrize('normalised', [False, True])
def test_enroll_many_is_enroll_speakers_problem_by_problem(R, E, normalised):
    fea, Phi, offs, problems, efea, espk, Fa, Fb = _archive(R * 1000 + E, R, E)
    norm = None
    if normalised:
        norm = _norms(fea, Phi, offs, problems, efea, espk, Fa, Fb, np.random.default_rng(R + E))[0]
    thetas = _thetas(fea, Phi, offs, problems, efea, espk, Fa, Fb, norm)
    got = enroll.enroll_many(fea, Phi, offs, problems, efea, espk, Fa, Fb, thetas, llr=True, norm=norm)
    sizes = []
    for g, labels in enumerate(problems):
        for h, t in enumerate(thetas):
            want = enroll.enroll_speakers(fea, Phi, offs, labels, efea, espk, Fa[g], Fb[g], t, llr=True,
                                          norm=None if norm is None else norm[g])
            assert np.array_equal(got[g].assign[h], want.assign), (g, t)
            assert np.array_equal(got[g].best_llr[h], want.best_llr), (g, t)
            # scipy's linear_sum_assignment on the device's scores, per problem and threshold: the same optimum (the
            # identical enrolled speakers 0 and 1 make ties, so the objective is compared, not the assignment)
            ro = np.searchsorted(got[g].table.rec, np.arange(len(labels) + 1))
            a = got[g].assign[h]
            assert len(set(zip(got[g].table.rec[a >= 0].tolist(), a[a >= 0].tolist()))) == int((a >= 0).sum())
            ref_obj = enroll_oracle.assign(got[g].llr, ro, t)[1]
            assert np.allclose(enroll_oracle.objective(got[g].llr, ro, t, a), ref_obj, rtol=1e-12, atol=1e-9), (g, t)
            if h == 0:
                for k in ('n', 'F', 'n_enroll', 'F_enroll', 'llr'):
                    x, y = getattr(got[g], k), getattr(want, k)
                    assert x.shape == y.shape and np.array_equal(x, y), (g, k)
                assert np.array_equal(got[g].table.rec, want.table.rec)
                sizes.append(len(want.table.rec))
    assert 0 in sizes and 150 <= max(sizes)
    # a budget that forces several launches: the same bits
    for mb in (_largest_single('enroll', offs, problems, int(espk.max()) + 1, len(espk), len(thetas)), None):
        again = enroll.enroll_many(fea, Phi, offs, problems, efea, espk, Fa, Fb, thetas, llr=True, norm=norm,
                                   max_bytes=mb)
        for a, b in zip(got, again):
            for k in ('assign', 'best_llr', 'n', 'F', 'n_enroll', 'F_enroll', 'llr'):
                assert np.array_equal(getattr(a, k), getattr(b, k)), k


def test_cohort_stats_many_and_link_many_with_statistics():
    fea, Phi, offs, problems, efea, espk, Fa, Fb = _archive(3, 128, 7)
    norm, cfea, cspk = _norms(fea, Phi, offs, problems, efea, espk, Fa, Fb, np.random.default_rng(3))
    for mb in (None, _largest_single('cohort', offs, problems, 12, 30)):
        st = cohort.cohort_stats_many(fea, Phi, offs, problems, cfea, cspk, Fa, Fb, 5, max_bytes=mb)
        se = cohort.cohort_stats_many(efea, Phi, None, [espk] * len(problems), cfea, cspk, Fa, Fb, 5, max_bytes=mb)
        for g in range(len(problems)):
            assert np.array_equal(st[g].mean, norm[g][0]) and np.array_equal(st[g].std, norm[g][1])
            assert np.array_equal(se[g].mean, norm[g][2]) and np.array_equal(se[g].std, norm[g][3])
            assert st[g].K == 5
    lk = [n[:2] for n in norm]
    for mb in (None, _largest_single('link', offs, problems)):
        got = link.link_many(fea, Phi, offs, problems, Fa, Fb, max_bytes=mb, dist=True, norm=lk)
        for g, labels in enumerate(problems):
            want = link.link_speakers(fea, Phi, offs, labels, Fa[g], Fb[g], dist=True, norm=lk[g])
            for x, y in zip(got[g][1:], want[1:]):
                assert x.shape == y.shape and np.array_equal(x, y), g
            D = got[g][4]
            assert np.array_equal(D, D.T)


# ---- the sweep ----------------------------------------------------------------------------------------------------------

GRID = dict(Fa=[0.3, 0.5], Fb=[17.0], loopP=[0.99], threshold=[-0.015], smoothing=[5.0])
ENROLL_T = [-10.0, 0.0, 20.0, 40.0]


@pytest.fixture(scope='module')
def model():
    z = np.load(os.path.join(GOLD, 'es2005a.npz'))
    m = np.load(os.path.join(GOLD, 'es2005a_model.npz'))
    return z, (m['mean1'], m['mean2'], m['lda']), (m['plda_mu'], m['plda_tr'], m['plda_psi'])


def _sessions(z, seed=13, n_rec=6, overlap=False, pool=10, leave_out=None):
    """synth.multi_session_archive and 20 held-out x-vectors of every pool speaker (its centre drawn as the archive
    draws it), one pool speaker left out on request."""
    recs, rows, _ = synth.multi_session_archive(z['x_raw'], n_rec=n_rec, seed=seed, pool=pool)
    x = np.asarray(z['x_raw'], dtype=np.float64)
    sd = x.std(0)
    centres = x.mean(0) + 2.0 * sd * np.random.default_rng(seed).standard_normal((pool, x.shape[1]))
    rng = np.random.default_rng(seed + 1000)
    held = {f'p{k}': centres[k] + 0.5 * sd * rng.standard_normal((20, x.shape[1])) for k in range(pool)
            if k != leave_out}
    if overlap:
        rng = np.random.default_rng(seed)
        for n, (_, seg) in recs.items():
            span = float(seg[:, 1].max())
            rows += [(n, round(float(a), 2), round(float(d), 2), f'p{int(k)}')
                     for a, d, k in zip(rng.uniform(0, span - 3, 8), rng.uniform(0.3, 3.0, 8), rng.integers(0, 10, 8))]
    return recs, rows, held


def _rows(items, key):
    return [tuple(line.split()[1:2]) + (float(line.split()[3]), float(line.split()[4]), line.split()[7])
            for it in items.values() for line in it[key]]


def _check(model, recs, rows, held, uem=None, oracle_ovl=False, oracle_count=False, init='AHC+VB', coh=None,
           links=None):
    z, transform, plda = model
    kw_s = dict(cohort=coh, cohort_top=50) if coh is not None else {}
    out = sweep.sweep_batch(recs, transform, plda, GRID, device=DEV, ref_rttm=rows, uem=uem, enroll=held,
                            enroll_thresholds=ENROLL_T, oracle_overlaps=oracle_ovl, init=init, link_thresholds=links,
                            num_speakers='oracle' if oracle_count else None, **kw_s)
    key = 'der_overlap' if oracle_ovl else 'der'
    tot, ranking = sweep.summarize_by_name(out, key)
    turns = score.reference_turns(rows)
    kw = dict(kw_s)
    if oracle_ovl:
        kw['overlaps'] = {n: [(a / 1e6, b / 1e6) for a, b in zip(*(x.tolist() for x in score.oracle_overlaps(turns[n])))]
                          for n in recs}
    if oracle_count:
        kw['num_speakers'] = score.reference_speaker_counts({n: turns[n] for n in recs}, uem)
    field = 'speaker_llr' if coh is None else 'speaker_score'
    for s in out:
        for t in ENROLL_T:
            d = pipeline.diarize_batch(recs, transform, plda, Fa=s.Fa, Fb=s.Fb, loopP=s.loopP, threshold=s.threshold,
                                       smoothing=s.smoothing, device=DEV, init=init, enroll=held, enroll_threshold=t,
                                       **kw)
            for n in recs:
                assert out[s][n]['speaker_names'][t] == d[n]['speaker_names'], (s.name, t, n)
                assert out[s][n][field][t] == d[n][field], (s.name, t, n)
                assert out[s][n]['rttm'] == d[n]['rttm']
                if coh is not None:
                    assert out[s][n]['score_norm'] == d[n]['score_norm']
            for p, c, io in score.PROTOCOLS:
                _, want = score.score_rttm(rows, _rows(d, 'rttm_named'), c, io, uem=uem, overlapping=oracle_ovl,
                                           by_name=True)
                assert tot[sweep.enroll_key(s, t)][p] == want['by_name'], (s.name, t, p)
        if links is not None:
            for t in links:
                d = pipeline.diarize_batch(recs, transform, plda, Fa=s.Fa, Fb=s.Fb, loopP=s.loopP,
                                           threshold=s.threshold, smoothing=s.smoothing, device=DEV, init=init,
                                           link_threshold=t, **kw)
                for n in recs:
                    assert out[s][n]['global_speakers'][t] == d[n]['global_speakers'], (s.name, t, n)
    assert all(sorted(ranking[p]) == sorted(tot) for p, _, _ in score.PROTOCOLS)
    return out, tot


@pytest.mark.parametrize('with_uem', [False, True])
def test_sweep_equals_diarize_batch_on_a_multi_session_archive(model, with_uem):
    recs, rows, held = _sessions(model[0], leave_out=3)
    uem = {n: [(1.0, float(seg[:, 1].max()) - 2.0)] for n, (_, seg) in recs.items()} if with_uem else None
    out, tot = _check(model, recs, rows, held, uem=uem)
    assert len(tot) == len(out) * len(ENROLL_T)


def test_sweep_with_oracle_overlaps_count_and_ahc(model):
    recs, rows, held = _sessions(model[0], seed=4, n_rec=4, overlap=True)
    _check(model, recs, rows, held, oracle_ovl=True)
    _check(model, recs, rows, held, oracle_count=True)
    _check(model, recs, rows, held, init='AHC')


def test_sweep_with_a_cohort_and_links(model):
    z = model[0]
    recs, rows, held = _sessions(z, seed=6, n_rec=4)
    coh = {f'c{k}': v for k, v in _sessions(z, seed=99, n_rec=1, pool=12)[2].items()}   # another pool
    out, _ = _check(model, recs, rows, held, coh=coh, links=[0.0, 2.0])
    for s in out:
        for it in out[s].values():
            assert 'speaker_llr' not in it and it['score_norm'] == {'top_k': 12, 'cohort_speakers': 12}


def test_a_cohort_without_spread_names_the_setting_and_speaker(model):
    z, transform, plda = model
    recs, rows, held = _sessions(z, seed=6, n_rec=3)
    x = held['p0'][:1]
    flat = {'c0': x, 'c1': x.copy(), 'c2': x.copy()}        # identical cohort speakers: every top-K score the same
    for kw in (dict(enroll=held, enroll_thresholds=[0.0]), dict(link_thresholds=[0.0])):
        with pytest.raises(ValueError, match=r'without spread .*setting Fa0\.3_Fb17_loopP0\.99_thr-0\.015_sm5: '
                                             r'ses00 speaker 1'):
            sweep.sweep_batch(recs, transform, plda, GRID, device=DEV, cohort=flat, **kw)


def test_es2005a_enrolled_with_its_own_speakers(model):
    z, transform, plda = model
    recs = {'ES2005a': (z['x_raw'], z['seg_times'])}
    rows = [('ES2005a', float(s), float(e - s), str(int(k)))
            for s, e, k in zip(z['rttm_starts'], z['rttm_ends'], z['rttm_ref_labels'])]
    plain = pipeline.diarize_batch(recs, transform, plda, Fa=0.3, Fb=17.0, loopP=0.99, device=DEV)['ES2005a']
    x = z['x_raw']
    own = {f'spk{l + 1}': x[plain['labels'] == l] for l in np.unique(plain['labels']).tolist()}
    _check(model, recs, rows, own)


def test_new_options_change_nothing_else(model):
    z, transform, plda = model
    recs, rows, held = _sessions(z, seed=6, n_rec=3)
    plain = sweep.sweep_batch(recs, transform, plda, GRID, device=DEV, ref_rttm=rows, jer=True)
    out = sweep.sweep_batch(recs, transform, plda, GRID, device=DEV, ref_rttm=rows, jer=True, enroll=held,
                            enroll_thresholds=[0.0, 0.0, 20.0])
    extra = {'speaker_names', 'speaker_llr', 'ref_speakers', 'der_blocks'}
    for s in out:
        for n in recs:
            assert list(out[s][n]['speaker_names']) == [0.0, 20.0]
            rest = {k: v for k, v in out[s][n].items() if k not in extra}
            assert rest.keys() == plain[s][n].keys()
            for k, v in rest.items():
                if isinstance(v, np.ndarray):
                    assert np.array_equal(v, plain[s][n][k])
                else:
                    assert v == plain[s][n][k], k


def _write_set(tmp_path, stem, sets):
    """{name: x [n, D]} as a Kaldi ark and utt2spk (tmp_path/<stem>.ark, .utt2spk)."""
    ekeys = [f'{k}-{i:02d}' for k, v in sets.items() for i in range(len(v))]
    formats.write_vec_flt_ark(str(tmp_path / f'{stem}.ark'), ekeys, np.concatenate(list(sets.values())))
    (tmp_path / f'{stem}.utt2spk').write_text(''.join(f'{k} {k.rsplit("-", 1)[0]}\n' for k in ekeys))


def _write_inputs(tmp_path, model, recs, rows, held):
    """The archive, segments, model, enrolment set and reference as the command line reads them; returns its argv."""
    z, transform, plda = model
    keys, seg_lines, xs = [], [], []
    for name, (x, seg) in recs.items():
        for i, (s, e) in enumerate(seg):
            k = f'{name}_{i:04d}'
            keys.append(k)
            seg_lines.append(f'{k} {name} {float(s)!r} {float(e)!r}')
        xs.append(x)
    formats.write_vec_flt_ark(str(tmp_path / 'x.ark'), keys, np.concatenate(xs))
    (tmp_path / 'x.seg').write_text('\n'.join(seg_lines) + '\n')
    _write_set(tmp_path, 'e', held)
    formats.write_kaldi_plda_text(str(tmp_path / 'plda.txt'), *plda)
    np.savez(str(tmp_path / 'transform.npz'), mean1=transform[0], mean2=transform[1], lda=transform[2])
    (tmp_path / 'ref.rttm').write_text(''.join(f'SPEAKER {r[0]} 1 {r[1]:.2f} {r[2]:.2f} <NA> <NA> {r[3]} <NA> <NA>\n'
                                               for r in rows))
    return ['--out-dir', str(tmp_path / 'out'), '--xvec-ark-file', str(tmp_path / 'x.ark'), '--segments-file',
            str(tmp_path / 'x.seg'), '--xvec-transform', str(tmp_path / 'transform.npz'), '--plda-file',
            str(tmp_path / 'plda.txt'), '--lda-dim', '128', '--Fa', '0.3,0.5', '--Fb', '17', '--loopP', '0.99',
            '--threshold=-0.015', '--enroll-ark', str(tmp_path / 'e.ark'), '--enroll-utt2spk',
            str(tmp_path / 'e.utt2spk'), '--enroll-threshold=-10,0,20,40', '--ref-rttm', str(tmp_path / 'ref.rttm')]


def test_command_line_summary(model, tmp_path):
    z, transform, plda = model
    recs, rows, held = _sessions(z, seed=6, n_rec=3)
    argv = _write_inputs(tmp_path, model, recs, rows, held)
    assert sweep.main(argv) == 0
    summary = json.loads((tmp_path / 'out' / 'summary.json').read_text())
    xv, segs = formats.read_xvectors_by_recording(str(tmp_path / 'x.ark')), formats.read_segments(str(tmp_path / 'x.seg'))
    recs2 = {n: (xv[n][1], segs[n][1]) for n in recs}
    enr = formats.read_enrolment(str(tmp_path / 'e.ark'), str(tmp_path / 'e.utt2spk'))
    plda2 = formats.read_kaldi_plda(str(tmp_path / 'plda.txt'))
    out = sweep.sweep_batch(recs2, transform, plda2, GRID, device=DEV, ref_rttm=str(tmp_path / 'ref.rttm'), enroll=enr,
                            enroll_thresholds=ENROLL_T)
    tot, ranking = sweep.summarize_by_name(out)
    rt = lambda v: json.loads(json.dumps(v))
    assert summary['ranking_by_name'] == ranking
    for s in out:
        for t in ENROLL_T:
            got = summary[s.name]['named'][f'{t:g}']
            assert got['speaker_names'] == rt({n: it['speaker_names'][t] for n, it in out[s].items()})
            assert got['der_by_name'] == rt(tot[sweep.enroll_key(s, t)])
    # the best entry's DER by name is what score --by-name gives on cli's output at that setting and threshold
    best = ranking['full'][0]
    s = next(s for s in out for t in ENROLL_T if sweep.enroll_key(s, t) == best)
    t = next(t for t in ENROLL_T if sweep.enroll_key(s, t) == best)
    d = pipeline.diarize_batch(recs2, transform, plda2, Fa=s.Fa, Fb=s.Fb, loopP=s.loopP, threshold=s.threshold,
                               smoothing=s.smoothing, device=DEV, enroll=enr, enroll_threshold=t)
    full = [p for p in score.PROTOCOLS if p[0] == 'full'][0]
    _, want = score.score_rttm(score.read_rttm_path(str(tmp_path / 'ref.rttm')), _rows(d, 'rttm_named'), full[1],
                               full[2], by_name=True)
    assert summary[s.name]['named'][f'{t:g}']['der_by_name']['full'] == rt(want['by_name'])


def test_command_line_with_a_cohort_and_links(model, tmp_path):
    z, transform, plda = model
    recs, rows, held = _sessions(z, seed=6, n_rec=3)
    coh = {f'c{k}': v for k, v in _sessions(z, seed=99, n_rec=1, pool=12)[2].items()}
    argv = _write_inputs(tmp_path, model, recs, rows, held)
    _write_set(tmp_path, 'c', coh)
    argv += ['--cohort-ark', str(tmp_path / 'c.ark'), '--cohort-utt2spk', str(tmp_path / 'c.utt2spk'), '--cohort-top',
             '5', '--link-threshold=0,2']
    assert sweep.main(argv) == 0
    summary = json.loads((tmp_path / 'out' / 'summary.json').read_text())
    xv, segs = formats.read_xvectors_by_recording(str(tmp_path / 'x.ark')), formats.read_segments(str(tmp_path / 'x.seg'))
    recs2 = {n: (xv[n][1], segs[n][1]) for n in recs}
    read = lambda stem: formats.read_enrolment(str(tmp_path / f'{stem}.ark'), str(tmp_path / f'{stem}.utt2spk'))
    out = sweep.sweep_batch(recs2, transform, formats.read_kaldi_plda(str(tmp_path / 'plda.txt')), GRID, device=DEV,
                            ref_rttm=str(tmp_path / 'ref.rttm'), enroll=read('e'), enroll_thresholds=ENROLL_T,
                            cohort=read('c'), cohort_top=5, link_thresholds=[0.0, 2.0])
    tot, ranking = sweep.summarize_by_name(out)
    tot_l, ranking_l = sweep.summarize_across_files(out)
    rt = lambda v: json.loads(json.dumps(v))
    assert summary['ranking_by_name'] == ranking and summary['ranking_across_files'] == ranking_l
    for s in out:
        assert all(it['score_norm'] == {'top_k': 5, 'cohort_speakers': 12} for it in out[s].values())
        for t in ENROLL_T:
            got = summary[s.name]['named'][f'{t:g}']
            assert got['speaker_names'] == rt({n: it['speaker_names'][t] for n, it in out[s].items()})
            assert got['der_by_name'] == rt(tot[sweep.enroll_key(s, t)])
        for t in (0.0, 2.0):
            got = summary[s.name]['linked'][f'{t:g}']
            assert got['global_speakers'] == rt({n: it['global_speakers'][t] for n, it in out[s].items()})
            assert got['der_across_files'] == rt(tot_l[sweep.link_key(s, t)])
