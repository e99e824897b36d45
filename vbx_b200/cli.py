"""Self-contained command line equal to the reference driver VBx/vbhmm.py:55-179, with the same options, but every
recording of the archive is processed in ONE batch on the GPU (front end, AHC, VB-HMM, labels):

    python -m vbx_b200.cli --init AHC+VB --out-rttm-dir exp --xvec-ark-file exp/ES2005a.ark \\
        --segments-file exp/ES2005a.seg --xvec-transform VBx/models/ResNet101_16kHz/transform.h5 \\
        --plda-file VBx/models/ResNet101_16kHz/plda --threshold -0.015 --lda-dim 128 --Fa 0.3 --Fb 17 --loopP 0.99

Reads Kaldi ark / segments / PLDA (binary or text) / transform.h5 through vbx_b200.formats (no kaldi_io, h5py or
fastcluster needed) and writes one RTTM per recording, formatted as VBx/vbhmm.py:48-51.

With --overlap-rttm PATH (an overlapped-speech detector's RTTM file or directory; speakers ignored) each written RTTM is
overlap-aware (DESIGN.md section 5.12): the usual lines, plus each x-vector's second most likely speaker inside the
overlap regions.  A recording the file lacks has no overlap regions.

With --num-speakers K, or --min-speakers / --max-speakers, every recording's speaker count is held to K or to the bounds
(DESIGN.md section 5.14).  Each takes an integer for the whole archive or a file of 'recording count' lines.

With --link-threshold X the speakers of all recordings are linked across the archive (DESIGN.md section 5.15): every
written RTTM (and with --output-2nd every second-label RTTM) names its speakers by archive-wide id, so the same speaker
has the same name in every file.  Speakers are linked where their average same-speaker log-likelihood ratio is >= X.

With --enroll-ark FILE --enroll-utt2spk FILE --enroll-threshold X (all three or none) the speakers are named by the
enrolled speakers of the ark (DESIGN.md section 5.16): a speaker whose log-likelihood ratio against an enrolled speaker
reaches X takes that speaker's name, one name per speaker within a recording; the others are written as
unknown-<recording>-<label>, or with --link-threshold linked among themselves and written as unknown-<id>.  With
--output-2nd the second-label RTTMs use the same names.  With --enroll-prior as well (and --init AHC+VB, no speaker
counts) the enrolled speakers take part in the VB-HMM (DESIGN.md section 5.23): AHC clusters are assigned to them the
same way, and an assigned cluster's state starts from that speaker's x-vectors as its speaker prior.

With --cohort-ark FILE --cohort-utt2spk FILE (both or neither; needs --link-threshold or the enrolment options) the
linking and enrolment scores are normalised against the cohort speakers of the ark (DESIGN.md section 5.17), speakers
known to be none of the archive's: each score is standardised by the mean and spread of both speakers' --cohort-top
(default 200) largest cohort scores, and --link-threshold and --enroll-threshold are on that normalised score.

With --init RTTM+VB --init-rttm PATH (an RTTM file or directory holding every recording of the archive) the VB-HMM
resegments an existing diarization instead of starting from AHC (DESIGN.md section 5.20): one state per speaker of the
RTTM, each x-vector started from the speakers' shares of its segment.  The written RTTMs keep the input's speaker names
(with --output-2nd the second-label RTTMs too) unless linking or enrolment name the speakers.  --threshold is still
required, as by the reference's parser, and is used only by the AHC that the count bounds' rule 3 needs.

With --adapt [--recentre] [--adapt-within-scale W --adapt-between-scale B --adapt-mean-scale S] the PLDA is first
adapted to the archive's own x-vectors (DESIGN.md section 5.26, vbx_b200/adapt.py: the variance the archive shows
beyond the model's, added to the within- and between-speaker covariances at W (0.3) and B (0.7), the mean moved to the
archive's), with --recentre after the transform's centring means are re-estimated on the archive; everything then runs
as without, enrolled and cohort x-vectors through the adapted front end.  python -m vbx_b200.train --adapt-plda writes
the same model to files.

With --init RANDOM+VB --init-states N [--restarts R] [--seed S] the VB-HMM starts from random flat-Dirichlet
responsibilities over N states instead of AHC (DESIGN.md section 5.22), R starts per recording side by side (default 1),
restart r drawn with seed S + r (default 0); each recording keeps the restart of largest final ELBO.  No AHC runs unless
count bounds need it, so long recordings are not held up by it.  --threshold is still required, as above.
"""
import argparse
import os
import sys

import numpy as np


def speaker_count_arg(text, allow_oracle=False):
    """A speaker-count option: an integer for every recording, or the path of a two-column 'recording count' file
    (formats.read_speaker_counts) -> int or {recording: int}; with allow_oracle also the word 'oracle'."""
    from . import formats
    text = str(text)
    if allow_oracle and text == 'oracle':
        return text
    try:
        return int(text)
    except ValueError:
        pass
    if not os.path.isfile(text):
        raise argparse.ArgumentTypeError(f'expected an integer{", oracle" if allow_oracle else ""} or a count file, '
                                         f'got {text!r}')
    try:
        return formats.read_speaker_counts(text)
    except ValueError as e:
        raise argparse.ArgumentTypeError(str(e))


def add_count_options(ap, allow_oracle=False):
    """--num-speakers / --min-speakers / --max-speakers (speaker_count_arg)."""
    what = 'an integer, oracle (with --ref-rttm) or a "recording count" file' if allow_oracle else \
        'an integer or a "recording count" file'
    ap.add_argument('--num-speakers', default=None, type=lambda t: speaker_count_arg(t, allow_oracle),
                    help=f'known number of speakers: {what}')
    ap.add_argument('--min-speakers', default=None, type=speaker_count_arg, help='lower bound on the speaker count: '
                    'an integer or a "recording count" file')
    ap.add_argument('--max-speakers', default=None, type=speaker_count_arg, help='upper bound on the speaker count: '
                    'an integer or a "recording count" file')


def add_random_options(ap):
    """--init-states / --restarts / --seed of --init RANDOM+VB."""
    ap.add_argument('--init-states', default=None, type=int,
                    help='with --init RANDOM+VB: the number of HMM states the random start draws (required there)')
    ap.add_argument('--restarts', default=None, type=int,
                    help='with --init RANDOM+VB: random starts per recording; the largest final ELBO wins (default 1)')
    ap.add_argument('--seed', default=None, type=int,
                    help='with --init RANDOM+VB: seed of restart 0, an integer in [0, 2**64); restart r uses seed + r '
                         '(default 0)')


def check_random_options(ap, args):
    """Usage errors (exit 2) of the --init RANDOM+VB options."""
    random = args.init == 'RANDOM+VB'
    if random != (args.init_states is not None):
        ap.error('--init RANDOM+VB and --init-states go together')
    if not random and (args.restarts is not None or args.seed is not None):
        ap.error('--restarts and --seed are options of --init RANDOM+VB')
    if random and args.init_states < 1:
        ap.error('--init-states must be >= 1')
    if args.restarts is not None and args.restarts < 1:
        ap.error('--restarts must be >= 1')
    if args.seed is not None and not 0 <= args.seed < 1 << 64:
        ap.error('--seed must lie in [0, 2**64)')


def add_adapt_scales(ap, prefix):
    """--<prefix>within-scale / between-scale / mean-scale (adapt.SCALES; default None: not given)."""
    for k, v in (('within', 0.3), ('between', 0.7), ('mean', 1.0)):
        ap.add_argument(f'--{prefix}{k}-scale', default=None, type=float,
                        help=f'PLDA adaptation: scale of the excess variance added to the {k}-class covariance '
                             f'(default {v})' if k != 'mean' else
                             f'PLDA adaptation: weight of the mean shift in the archive\'s covariance (default {v})')


def adapt_scales(ap, args, prefix, enabled, what):
    """The given adaptation scales {within_scale, ...} of add_adapt_scales' options: usage errors (exit 2) for scales
    without `enabled` (named `what`) and for negative or non-finite ones."""
    from . import adapt
    scales = {f'{k}_scale': getattr(args, f'{prefix}{k}_scale') for k in ('within', 'between', 'mean')}
    scales = {k: v for k, v in scales.items() if v is not None}
    if scales and not enabled:
        ap.error(f'the adaptation scales need {what}')
    try:
        adapt.check_scales(**scales)
    except ValueError as e:
        ap.error(str(e))
    return scales


def add_adapt_options(ap):
    """--adapt / --recentre / --adapt-within-scale / --adapt-between-scale / --adapt-mean-scale."""
    ap.add_argument('--adapt', action='store_true',
                    help='adapt the PLDA to the archive\'s own x-vectors before diarizing it (DESIGN.md section 5.26)')
    ap.add_argument('--recentre', action='store_true',
                    help='with --adapt: re-estimate the transform\'s centring means on the archive first')
    add_adapt_scales(ap, 'adapt-')


def check_adapt_options(ap, args):
    """Usage errors (exit 2) of the --adapt options: --recentre or scales without --adapt, negative or non-finite
    scales.  Returns the given scales (adapt.adapt_backend's keywords), or None without --adapt."""
    scales = adapt_scales(ap, args, 'adapt_', args.adapt, '--adapt')
    if args.recentre and not args.adapt:
        ap.error('--recentre needs --adapt')
    return scales if args.adapt else None


def build_parser():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    # option names, types and defaults of VBx/vbhmm.py:55-102
    ap.add_argument('--init', required=True, type=str, choices=['AHC', 'AHC+VB', 'RTTM+VB', 'RANDOM+VB'])
    ap.add_argument('--out-rttm-dir', required=True, type=str)
    ap.add_argument('--xvec-ark-file', required=True, type=str)
    ap.add_argument('--segments-file', required=True, type=str)
    ap.add_argument('--xvec-transform', required=True, type=str)
    ap.add_argument('--plda-file', required=True, type=str)
    ap.add_argument('--threshold', required=True, type=float)
    ap.add_argument('--lda-dim', required=True, type=int)
    ap.add_argument('--Fa', required=True, type=float)
    ap.add_argument('--Fb', required=True, type=float)
    ap.add_argument('--loopP', required=True, type=float)
    ap.add_argument('--target-energy', required=False, type=float, default=1.0)     # unused by the cosine AHC, as in the reference
    ap.add_argument('--init-smoothing', required=False, type=float, default=5.0)
    ap.add_argument('--output-2nd', required=False, type=bool, default=False)
    # additions
    ap.add_argument('--chain', default='auto', choices=['auto', 'tcgen05', 'float64'],
                    help='front end arithmetic: fused tensor-core kernels (float32-level) or float64 torch ops')
    ap.add_argument('--device', default=None, help='CUDA device, e.g. cuda:0 (default: the current device)')
    ap.add_argument('--overlap-rttm', default=None,
                    help='overlap regions (RTTM file or directory): also write the second speaker inside them')
    add_count_options(ap)
    ap.add_argument('--link-threshold', default=None, type=float,
                    help='link speakers across the recordings: one name per speaker in every file where their average '
                         'same-speaker log-likelihood ratio is >= this')
    ap.add_argument('--enroll-ark', default=None, help='x-vectors of known speakers (Kaldi ark) to name speakers by')
    ap.add_argument('--enroll-utt2spk', default=None, help='the speaker of each x-vector of --enroll-ark (utt2spk)')
    ap.add_argument('--enroll-threshold', default=None, type=float,
                    help='least log-likelihood ratio at which a speaker takes an enrolled name')
    ap.add_argument('--enroll-prior', action='store_true',
                    help='with the enrolment options and --init AHC+VB: AHC clusters assigned to enrolled speakers start '
                         'the VB-HMM from those speakers\' x-vectors as their speaker prior')
    ap.add_argument('--cohort-ark', default=None,
                    help='x-vectors of cohort speakers (Kaldi ark), none of them in the archive, to normalise the '
                         'linking and enrolment scores by')
    ap.add_argument('--cohort-utt2spk', default=None, help='the speaker of each x-vector of --cohort-ark (utt2spk)')
    ap.add_argument('--cohort-top', default=None, type=int,
                    help='how many of each speaker\'s largest cohort scores set its mean and spread (default 200)')
    ap.add_argument('--init-rttm', default=None,
                    help='with --init RTTM+VB: the diarization (RTTM file or directory of *.rttm) the VB-HMM starts from')
    add_random_options(ap)
    add_adapt_options(ap)
    return ap


def main(argv=None):
    ap = build_parser()
    args = ap.parse_args(argv)
    assert 0 <= args.loopP <= 1, f'Expecting loopP between 0 and 1, got {args.loopP} instead.'     # VBx/vbhmm.py:103
    enr = [args.enroll_ark, args.enroll_utt2spk, args.enroll_threshold]
    if any(v is not None for v in enr) and any(v is None for v in enr):
        ap.error('--enroll-ark, --enroll-utt2spk and --enroll-threshold go together')
    coh = [args.cohort_ark, args.cohort_utt2spk]
    if any(v is not None for v in coh) and any(v is None for v in coh):
        ap.error('--cohort-ark and --cohort-utt2spk go together')
    if args.enroll_prior:
        if args.enroll_ark is None:
            ap.error('--enroll-prior needs --enroll-ark, --enroll-utt2spk and --enroll-threshold')
        if args.init != 'AHC+VB':
            ap.error('--enroll-prior needs --init AHC+VB')
        if args.num_speakers is not None or args.min_speakers is not None or args.max_speakers is not None:
            ap.error('--enroll-prior does not combine with --num-speakers / --min-speakers / --max-speakers')
    if args.cohort_top is not None and args.cohort_ark is None:
        ap.error('--cohort-top needs --cohort-ark and --cohort-utt2spk')
    if args.cohort_ark is not None and args.link_threshold is None and args.enroll_ark is None:
        ap.error('a cohort normalises the linking and enrolment scores: give --link-threshold or the enrolment options')
    if args.cohort_top is not None and args.cohort_top < 2:
        ap.error('--cohort-top must be >= 2')
    if (args.init == 'RTTM+VB') != (args.init_rttm is not None):
        ap.error('--init RTTM+VB and --init-rttm go together')
    check_random_options(ap, args)
    scales = check_adapt_options(ap, args)
    from . import formats
    from .pipeline import diarize_batch, linked_lines, named_lines
    from .score import read_overlaps
    enroll = formats.read_enrolment(args.enroll_ark, args.enroll_utt2spk) if args.enroll_ark is not None else None
    cohort = formats.read_enrolment(args.cohort_ark, args.cohort_utt2spk) if args.cohort_ark is not None else None
    norm_kw = {} if cohort is None else dict(cohort=cohort, cohort_top=200 if args.cohort_top is None else args.cohort_top)
    overlaps = read_overlaps(args.overlap_rttm) if args.overlap_rttm is not None else None
    segs = formats.read_segments(args.segments_file)                        # VBx/vbhmm.py:105
    plda = formats.read_kaldi_plda(args.plda_file)                          # VBx/vbhmm.py:107
    mean1, mean2, lda = formats.read_xvec_transform(args.xvec_transform)    # VBx/vbhmm.py:125-128
    recs = {}
    for name, (keys, x) in formats.read_xvectors_by_recording(args.xvec_ark_file).items():     # VBx/vbhmm.py:117-123
        print(name)
        seg_names, times = segs[name]
        assert np.all(np.array(seg_names) == np.array(keys))               # VBx/vbhmm.py:166
        recs[name] = (x, times)
    if scales is not None:      # section 5.26: the back end adapted to this archive, then everything as without
        from .adapt import adapt_backend
        (mean1, mean2, lda), plda, _ = adapt_backend(recs, (mean1, mean2, lda), plda, lda_dim=args.lda_dim,
                                                     chain=args.chain, device=args.device, recentre=args.recentre,
                                                     **scales)
    out = diarize_batch(recs, (mean1, mean2, lda), plda, Fa=args.Fa, Fb=args.Fb, loopP=args.loopP, lda_dim=args.lda_dim,
                        threshold=args.threshold, smoothing=args.init_smoothing, init=args.init, chain=args.chain,
                        device=args.device, output_2nd=args.output_2nd, overlaps=overlaps,
                        num_speakers=args.num_speakers, min_speakers=args.min_speakers, max_speakers=args.max_speakers,
                        link_threshold=args.link_threshold, enroll=enroll, enroll_threshold=args.enroll_threshold,
                        init_rttm=args.init_rttm, init_states=args.init_states, restarts=args.restarts, seed=args.seed,
                        enroll_prior=args.enroll_prior, **norm_kw)
    linked = args.link_threshold is not None
    named_init = args.init == 'RTTM+VB' and enroll is None and not linked
    os.makedirs(args.out_rttm_dir, exist_ok=True)                           # VBx/vbhmm.py:170
    for name, item in out.items():
        key = 'rttm_named' if enroll is not None else 'rttm_linked' if linked else 'rttm_init' if named_init else \
            'rttm' if overlaps is None else 'rttm_overlap'
        with open(os.path.join(args.out_rttm_dir, f'{name}.rttm'), 'w') as fp:
            fp.write(''.join(line + os.linesep for line in item[key]))
        if item['rttm2nd'] is not None:
            d2 = f'{args.out_rttm_dir}2nd'
            os.makedirs(d2, exist_ok=True)
            if enroll is not None:
                lines = named_lines(name, recs[name][1], item['labels2nd'], None, item['speaker_names'])
            elif named_init and item['init_speakers'] is not None:
                lines = named_lines(name, recs[name][1], item['labels2nd'], None, item['init_speakers'])
            else:
                lines = item['rttm2nd'] if not linked else \
                    linked_lines(name, recs[name][1], item['labels2nd'], None, item['global_speakers'])
            with open(os.path.join(d2, f'{name}.rttm'), 'w') as fp:
                fp.write(''.join(line + os.linesep for line in lines))
    return 0


if __name__ == '__main__':
    sys.exit(main())
