"""Speaker linking inside the sweep on the device (DESIGN.md section 5.18): vbx_link_batch through link.link_many against
link_speakers problem by problem (bit for bit) and scipy's partitions, its argument checks, and sweep_batch's
global_speakers and DER across files against diarize_batch(link_threshold=) and score_rttm(across_files=True) on a
multi-session archive and ES2005a, with a UEM, oracle overlaps and the oracle speaker count, and the command line."""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

from oracle import link_oracle
from test_link_gpu import SPEAKER_WIDTHS, width_phi
from vbx_b200 import _lib, formats, link, pipeline, score, sweep, synth

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), 'golden')
DEV = torch.device('cuda:0')
MS = [0, 1, 2, 33, 128, 700]


def _problems(seed, R):
    """One archive of 20 recordings and a problem per M in MS, each with its own labels (value gaps, -1 entries); Phi
    from width_phi at the SPEAKER_WIDTHS."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(40, 80, 20)
    lens[3] = 0
    centres = rng.standard_normal((60, R)) * 2.0
    fea = (centres[rng.integers(0, 60, int(lens.sum()))] + rng.standard_normal((int(lens.sum()), R))).astype(np.float32)
    Phi = (width_phi(rng, R) if R in SPEAKER_WIDTHS
           else np.sort(rng.uniform(0.2, 6.0, R))[::-1].astype(np.float32).copy())
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    problems = []
    for M in MS:
        k = np.zeros(len(lens), dtype=np.int64)
        for i in range(M):                                   # M speakers over the recordings with room for them
            b = i % len(lens)
            while k[b] >= lens[b] - 1:
                b = (b + 1) % len(lens)
            k[b] += 1
        labels = []
        for T, kb in zip(lens.tolist(), k.tolist()):
            vals = np.sort(rng.choice(kb + 5, kb, replace=False))
            lab = np.concatenate([np.arange(kb), rng.integers(0, max(kb, 1), T - kb)]) if kb else np.full(T, -1)
            lab = np.where(lab >= 0, vals[np.minimum(lab, max(kb - 1, 0))] if kb else -1, -1)
            if kb and T > kb:
                lab[kb:][rng.random(T - kb) < 0.1] = -1           # x-vectors without a speaker
            rng.shuffle(lab)
            labels.append(lab.astype(np.int64))
        assert len(link.speaker_table(labels).rec) == M
        problems.append(labels)
    Fa = rng.uniform(0.1, 0.6, len(MS))
    Fb = rng.uniform(4.0, 40.0, len(MS))
    return fea, Phi, offs, problems, Fa, Fb


def _partition(table, maps):
    g = {}
    for b, l in zip(table.rec.tolist(), table.label.tolist()):
        g.setdefault(maps[b][l], set()).add((b, l))
    return sorted(map(sorted, g.values()))


@pytest.mark.parametrize('R', [8, 16, 128] + SPEAKER_WIDTHS)
def test_link_many_is_link_speakers_problem_by_problem(R):
    fea, Phi, offs, problems, Fa, Fb = _problems(R, R)
    fea_d, Phi_d = torch.from_numpy(fea).to(DEV), torch.from_numpy(Phi).to(DEV)
    got = link.link_many(fea_d, Phi_d, offs, problems, Fa, Fb, DEV, dist=True)
    for g, labels in enumerate(problems):
        want = link.link_speakers(fea_d, Phi_d, offs, labels, Fa[g], Fb[g], DEV, dist=True)
        assert np.array_equal(got[g][0].rec, want[0].rec) and np.array_equal(got[g][0].label, want[0].label)
        for x, y in zip(got[g][1:], want[1:]):
            assert x.shape == y.shape and np.array_equal(x, y), g
        table, Z, D = got[g][0], got[g][3], got[g][4]
        if len(table.rec) < 2:
            continue
        Zs = link_oracle.link(D)
        for t in (-1e6, -200.0, -20.0, 0.0, 5.0, 50.0, 1e6):
            maps = link.link_cut(Z, table, t)
            ref = link_oracle.partition(Zs, t)
            want_p = {}
            for i, (b, l) in enumerate(zip(table.rec.tolist(), table.label.tolist())):
                want_p.setdefault(int(ref[i]), set()).add((b, l))
            assert _partition(table, maps) == sorted(map(sorted, want_p.values())), (g, t)
    # a budget that forces several launches: the same bits
    again = link.link_many(fea_d, Phi_d, offs, problems, Fa, Fb, DEV, max_bytes=_workspace_bytes(700) + 1, dist=True)
    for a, b in zip(got, again):
        for x, y in zip(a[1:], b[1:]):
            assert np.array_equal(x, y)
    with pytest.raises(ValueError, match='more than max_batch_bytes'):
        link.link_many(fea_d, Phi_d, offs, problems, Fa, Fb, DEV, max_bytes=_workspace_bytes(700) - 1)


def _handle():
    lib = _lib.load()
    h = ctypes.c_void_p()
    assert lib.vbx_create(0, ctypes.byref(h)) == 0
    return lib, h


def _workspace_bytes(*Ms):
    lib, h = _handle()
    try:
        need = ctypes.c_size_t()
        M = np.array(Ms, dtype=np.int64)
        assert lib.vbx_link_batch_workspace_bytes(h, len(Ms), M.ctypes.data_as(ctypes.c_void_p), ctypes.byref(need)) == 0
        return int(need.value)
    finally:
        lib.vbx_destroy(h)


def test_batch_workspace_bytes_and_argument_errors():
    lib, h = _handle()
    try:
        single = [_workspace_bytes(M) for M in MS]
        assert _workspace_bytes(*MS) <= sum(single)
        M = np.array([3, 2], dtype=np.int64)
        need = ctypes.c_size_t()
        lib.vbx_link_batch_workspace_bytes(h, 2, M.ctypes.data_as(ctypes.c_void_p), ctypes.byref(need))
        fea = torch.zeros((4, 8), device=DEV)
        Phi = torch.ones(8, device=DEV)
        spk = torch.zeros((2, 4), dtype=torch.int32, device=DEV)
        rec = torch.arange(5, dtype=torch.int32, device=DEV)
        ws = torch.empty(need.value, dtype=torch.uint8, device=DEV)
        Z = torch.empty((5, 4), dtype=torch.float64, device=DEV)
        stat = torch.ones(5, dtype=torch.float64, device=DEV)
        p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None
        a = lambda x: np.ascontiguousarray(x, dtype=np.float64)

        def call(R=8, Ms=M, Fa=(0.3, 0.3), Fb=(17.0, 17.0), size=need.value, mean=None, std=None):
            Ms, Fa, Fb = np.asarray(Ms, dtype=np.int64), a(Fa), a(Fb)
            v = lambda x: x.ctypes.data_as(ctypes.c_void_p)
            return lib.vbx_link_batch(h, p(fea), p(Phi), 4, R, 2, p(spk), v(Ms), p(rec), v(Fa), v(Fb), p(ws), size,
                                      None, None, None, p(Z), p(mean), p(std), None)
        assert call() == 0
        assert call(mean=stat, std=stat) == 0
        torch.cuda.synchronize()
        for bad in (dict(R=0), dict(R=129), dict(Ms=[3, _lib.LINK_MAX_SPEAKERS + 1]), dict(Ms=[3, -1]),
                    dict(Fa=(0.3, -0.3)), dict(Fa=(0.3, float('nan'))), dict(Fb=(17.0, 0.0)), dict(size=need.value - 1),
                    dict(mean=stat), dict(std=stat)):
            assert call(**bad) == -1, bad                                  # VBX_ERR_ARG
    finally:
        lib.vbx_destroy(h)


# ---- the sweep ----------------------------------------------------------------------------------------------------------

GRID = dict(Fa=[0.3, 0.5], Fb=[17.0], loopP=[0.99], threshold=[-0.015], smoothing=[5.0])
THRESHOLDS = [-10.0, 0.0, 48.0]


@pytest.fixture(scope='module')
def model():
    z = np.load(os.path.join(GOLD, 'es2005a.npz'))
    m = np.load(os.path.join(GOLD, 'es2005a_model.npz'))
    return z, (m['mean1'], m['mean2'], m['lda']), (m['plda_mu'], m['plda_tr'], m['plda_psi'])


def _sessions(z, seed=13, n_rec=6, overlap=False):
    recs, rows, _ = synth.multi_session_archive(z['x_raw'], n_rec=n_rec, seed=seed)
    if overlap:                                             # seeded second-speaker turns: the reference overlaps
        rng = np.random.default_rng(seed)
        for n, (x, seg) in recs.items():
            span = float(seg[:, 1].max())
            rows += [(n, round(float(a), 2), round(float(d), 2), f'p{int(k)}')
                     for a, d, k in zip(rng.uniform(0, span - 3, 8), rng.uniform(0.3, 3.0, 8), rng.integers(0, 10, 8))]
    return recs, rows


def _es(z):
    recs = {'ES2005a': (z['x_raw'], z['seg_times'])}
    rows = [('ES2005a', float(s), float(e - s), str(int(k)))
            for s, e, k in zip(z['rttm_starts'], z['rttm_ends'], z['rttm_ref_labels'])]
    rng = np.random.default_rng(5)
    spk = sorted({r[3] for r in rows})
    span = float(z['seg_times'][:, 1].max())
    rows += [('ES2005a', round(float(a), 2), round(float(d), 2), str(rng.choice(spk)))
             for a, d in zip(rng.uniform(0, span - 3, 40), rng.uniform(0.3, 3.0, 40))]
    return recs, rows


def _rows(items, key):
    return [tuple(line.split()[1:2]) + (float(line.split()[3]), float(line.split()[4]), line.split()[7])
            for it in items.values() for line in it[key]]


def _check(model, recs, rows, uem=None, oracle_ovl=False, oracle_count=False):
    z, transform, plda = model
    out = sweep.sweep_batch(recs, transform, plda, GRID, device=DEV, ref_rttm=rows, uem=uem, link_thresholds=THRESHOLDS,
                            oracle_overlaps=oracle_ovl, num_speakers='oracle' if oracle_count else None)
    tot, ranking = sweep.summarize_across_files(out)
    tot_o = sweep.summarize_across_files(out, 'der_overlap')[0] if oracle_ovl else None
    turns = score.reference_turns(rows)
    kw = {}
    if oracle_ovl:
        kw['overlaps'] = {n: [(a / 1e6, b / 1e6) for a, b in zip(*(x.tolist() for x in score.oracle_overlaps(turns[n])))]
                          for n in recs}
    if oracle_count:
        kw['num_speakers'] = score.reference_speaker_counts({n: turns[n] for n in recs}, uem)
    for s in out:
        for t in THRESHOLDS:
            d = pipeline.diarize_batch(recs, transform, plda, Fa=s.Fa, Fb=s.Fb, loopP=s.loopP, threshold=s.threshold,
                                       smoothing=s.smoothing, device=DEV, link_threshold=t, **kw)
            for n in recs:
                assert out[s][n]['global_speakers'][t] == d[n]['global_speakers'], (s.name, t, n)
                assert out[s][n]['rttm'] == d[n]['rttm']
            for p, c, io in score.PROTOCOLS:
                _, want = score.score_rttm(rows, _rows(d, 'rttm_linked'), c, io, uem=uem, overlapping=oracle_ovl,
                                           across_files=True)
                got = (tot_o if oracle_ovl else tot)[sweep.link_key(s, t)][p]
                assert got == want['across_files'], (s.name, t, p)
    return out, tot, ranking


@pytest.mark.parametrize('with_uem', [False, True])
def test_sweep_equals_diarize_batch_on_a_multi_session_archive(model, with_uem):
    recs, rows = _sessions(model[0])
    uem = {n: [(1.0, float(seg[:, 1].max()) - 2.0)] for n, (_, seg) in recs.items()} if with_uem else None
    out, tot, ranking = _check(model, recs, rows, uem=uem)
    assert len(tot) == len(out) * len(THRESHOLDS)
    assert all(sorted(ranking[p]) == sorted(tot) for p, _, _ in score.PROTOCOLS)


def test_sweep_with_oracle_overlaps_and_count(model):
    recs, rows = _sessions(model[0], seed=4, n_rec=4, overlap=True)
    _check(model, recs, rows, oracle_ovl=True)
    _check(model, recs, rows, oracle_count=True)


def test_sweep_on_es2005a(model):
    recs, rows = _es(model[0])
    _check(model, recs, rows)
    _check(model, recs, rows, oracle_ovl=True)


def test_sweep_linking_with_ahc_init_and_jer(model):
    z, transform, plda = model
    recs, rows = _sessions(z, seed=6, n_rec=3)
    out = sweep.sweep_batch(recs, transform, plda, GRID, device=DEV, init='AHC', ref_rttm=rows, jer=True,
                            link_thresholds=[0.0])
    plain = sweep.sweep_batch(recs, transform, plda, GRID, device=DEV, init='AHC', ref_rttm=rows, jer=True)
    for s in out:
        d = pipeline.diarize_batch(recs, transform, plda, Fa=s.Fa, Fb=s.Fb, loopP=s.loopP, threshold=s.threshold,
                                   smoothing=s.smoothing, device=DEV, init='AHC', link_threshold=0.0)
        for n in recs:
            assert out[s][n]['global_speakers'][0.0] == d[n]['global_speakers']
            extra = {'global_speakers', 'ref_speakers', 'der_blocks'}
            assert {k: v for k, v in out[s][n].items() if k not in extra}.keys() == plain[s][n].keys()
            assert out[s][n]['der'] == plain[s][n]['der'] and out[s][n]['jer'] == plain[s][n]['jer']


def test_command_line_summary(model, tmp_path):
    z, transform, plda = model
    recs, rows = _sessions(z, seed=6, n_rec=3)
    keys, seg_lines, xs = [], [], []
    for name, (x, seg) in recs.items():
        for i, (s, e) in enumerate(seg):
            k = f'{name}_{i:04d}'
            keys.append(k)
            seg_lines.append(f'{k} {name} {float(s)!r} {float(e)!r}')
        xs.append(x)
    formats.write_vec_flt_ark(str(tmp_path / 'x.ark'), keys, np.concatenate(xs))
    (tmp_path / 'x.seg').write_text('\n'.join(seg_lines) + '\n')
    formats.write_kaldi_plda_text(str(tmp_path / 'plda.txt'), *plda)
    np.savez(str(tmp_path / 'transform.npz'), mean1=transform[0], mean2=transform[1], lda=transform[2])
    (tmp_path / 'ref.rttm').write_text(''.join(f'SPEAKER {r[0]} 1 {r[1]:.2f} {r[2]:.2f} <NA> <NA> {r[3]} <NA> <NA>\n'
                                               for r in rows))
    argv = ['--out-dir', str(tmp_path / 'out'), '--xvec-ark-file', str(tmp_path / 'x.ark'), '--segments-file',
            str(tmp_path / 'x.seg'), '--xvec-transform', str(tmp_path / 'transform.npz'), '--plda-file',
            str(tmp_path / 'plda.txt'), '--lda-dim', '128', '--Fa', '0.3,0.5', '--Fb', '17', '--loopP', '0.99',
            '--threshold=-0.015', '--link-threshold=-10,0,48', '--ref-rttm', str(tmp_path / 'ref.rttm')]
    assert sweep.main(argv) == 0
    summary = json.loads((tmp_path / 'out' / 'summary.json').read_text())
    xv, segs = formats.read_xvectors_by_recording(str(tmp_path / 'x.ark')), formats.read_segments(str(tmp_path / 'x.seg'))
    out = sweep.sweep_batch({n: (xv[n][1], segs[n][1]) for n in recs}, transform, formats.read_kaldi_plda(str(tmp_path / 'plda.txt')), GRID, device=DEV,
                            ref_rttm=str(tmp_path / 'ref.rttm'), link_thresholds=THRESHOLDS)
    tot, ranking = sweep.summarize_across_files(out)
    rt = lambda v: json.loads(json.dumps(v))
    assert summary['ranking_across_files'] == ranking
    for s in out:
        for t in THRESHOLDS:
            got = summary[s.name]['linked'][f'{t:g}']
            assert got['global_speakers'] == rt({n: it['global_speakers'][t] for n, it in out[s].items()})
            assert got['der_across_files'] == rt(tot[sweep.link_key(s, t)])
    assert not (tmp_path / 'out' / 'linked').exists()
