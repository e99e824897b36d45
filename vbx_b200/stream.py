"""Streaming diarization (DESIGN.md section 5.25): live streams diarized block by block on the device, each stream's
speakers carried into the VB-HMM as priors, every open stream of a push in one batch.

A push delivers a block of h >= 1 new x-vectors to any subset of the open streams.  For each of them:
  1. the block goes through the front end of diarize_batch (pipeline._project), one batch over the pushed streams;
  2. AHC of the block alone (vbx_ahc, batched), cut at `threshold`: c clusters, or the maxclust cut at S_max - K when
     K + c > S_max (c = 0 when K = S_max);
  3. the window [the stream's last min(C, count) x-vectors; the block] with K + c states: context rows start on their
     final label and block rows on K + cluster (gamma0 = softmax(smoothing * onehot), pi0 uniform), states k < K carry
     the prior (n_hist[k], F_hist[k]) of the stream's x-vectors that have left the context (vbx_stream_window);
  4. the VB-HMM with the prior over the window (VbxBatch.run(prior=)), grouped by state tier as pipeline._vb_stage
     groups it, and hard labels;
  5. only the block's rows are final: a row on a state k < K is speaker k, fresh states that hold rows become speakers
     K, K+1, ... in order of their first row, and rows that leave the context join the history (vbx_stream_commit).
The prior is exact: it is the window with the older x-vectors appended as frames held on their state (section 5.23),
so every x-vector enters once, as a frame or through the prior.  oracle/stream_oracle.py restates this in float64.

`python -m vbx_b200.stream` replays an archive as live streams (one per recording) and writes one RTTM per recording.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

from . import ahc as _ahc
from ._lib import VbxError
from .batch import StreamState, VbxBatch
from .pipeline import _pad_features, _project, _resolve_chain, _tier, merge_adjacent_labels, rttm_lines


class _Stream:
    __slots__ = ('slot', 'Dx', 'count', 'K', 'seg', 'labels')

    def __init__(self, slot, Dx):
        self.slot, self.Dx, self.count, self.K, self.seg, self.labels = slot, Dx, 0, 0, [], []


def check_settings(max_speakers, context, Fb, loopP, smoothing):
    """ValueError for settings no stream can run with: max_speakers outside 1 .. 128 (the float32 state tiers), a
    negative context, Fb = 0, loopP outside [0, 1], a non-finite smoothing."""
    if isinstance(max_speakers, bool) or not isinstance(max_speakers, (int, np.integer)) or not 1 <= max_speakers <= 128:
        raise ValueError(f'max_speakers must be an integer in [1, 128], got {max_speakers!r}')
    if isinstance(context, bool) or not isinstance(context, (int, np.integer)) or context < 0:
        raise ValueError(f'context must be an integer >= 0, got {context!r}')
    if not (np.isfinite(Fb) and Fb != 0):
        raise ValueError('Fb must be finite and non-zero')
    if not 0 <= loopP <= 1:
        raise ValueError(f'loopP must lie in [0, 1], got {loopP}')
    if not np.isfinite(smoothing):
        raise ValueError('smoothing must be finite')


def block_clusters(labels, Zs, lens, K, S_max):
    """Step 2 for every pushed stream: the threshold cut `labels` (ahc.cut) unless K + c > S_max, then the maxclust cut
    at S_max - K (ahc.cut_count), or no cluster (c = 0, labels -1) when K = S_max.  Returns (labels, c) per stream."""
    out = []
    for b, l in enumerate(labels):
        c = int(l.max()) + 1
        if K[b] + c > S_max:
            if K[b] >= S_max:
                l, c = np.full(len(l), -1, dtype=np.int64), 0
            else:
                l = _ahc.cut_count([Zs[b]], [lens[b]], [S_max - K[b]])[0]
                c = int(l.max()) + 1
        out.append((l, c))
    return out


class StreamDiarizer:
    """Live streams diarized block by block (module docstring; DESIGN.md section 5.25).  transform, plda, Fa, Fb, loopP,
    lda_dim, threshold, smoothing, max_iters, epsilon and chain as diarize_batch takes them; context = C, the look-back
    in x-vectors (default 240: 60 s at the 0.25 s shift); max_speakers = S_max, the largest speaker count of a stream
    (1 .. 128).  Speaker k of a stream is named spk<k+1> for the stream's life."""

    def __init__(self, transform, plda, Fa, Fb, loopP, lda_dim=128, threshold=-0.015, smoothing=5.0, context=240,
                 max_speakers=64, max_iters=40, epsilon=1e-6, device=None, chain='auto'):
        check_settings(max_speakers, context, Fb, loopP, smoothing)
        if chain not in ('auto', 'tcgen05', 'float64'):
            raise ValueError("chain must be 'auto', 'tcgen05' or 'float64'")
        self.transform, self.plda = transform, plda
        self.Fa, self.Fb, self.loopP = float(Fa), float(Fb), float(loopP)
        self.lda_dim, self.threshold, self.smoothing = int(lda_dim), float(threshold), float(smoothing)
        self.C, self.S_max = int(context), int(max_speakers)
        self.max_iters, self.epsilon, self.chain = int(max_iters), float(epsilon), chain
        self.Dx = int(np.asarray(transform[0]).shape[0])
        self.R = self.lda_dim + (-self.lda_dim) % 4            # the features as _pad_features leaves them
        self._device = device
        self.dev = None
        self.state = None
        self.streams = {}
        self._free = []
        self.timing = None            # None, or a list that receives one dict of stage times per push (seconds)

    def _open(self, name):
        if self.state is None:
            if not torch.cuda.is_available():
                raise VbxError('StreamDiarizer: no CUDA device - vbx_b200 has no CPU fallback')
            self.dev = torch.device('cuda', torch.cuda.current_device()) if self._device is None \
                else torch.device(self._device)
            if self.dev.index is None:
                self.dev = torch.device('cuda', torch.cuda.current_device())
            self.state = StreamState(0, self.C, self.R, self.S_max, self.dev)
        if not self._free:
            old = self.state.slots
            self.state.grow(max(16, 2 * old))
            self._free = list(range(self.state.slots - 1, old - 1, -1))
        slot = self._free.pop()
        self.state.reset(slot)
        self.streams[name] = _Stream(slot, self.Dx)
        return self.streams[name]

    def close(self, name):
        """End stream `name` and free its slot (KeyError for an unknown stream)."""
        st = self.streams.pop(name)
        self._free.append(st.slot)

    def rttm(self, name):
        """The RTTM lines of stream `name` so far, merged as diarize_batch merges an offline result."""
        st = self.streams[name]
        if not st.labels:
            return []
        seg = np.concatenate(st.seg)
        return rttm_lines(name, *merge_adjacent_labels(seg[:, 0], seg[:, 1], np.concatenate(st.labels)))

    def _check_push(self, blocks):
        if not isinstance(blocks, dict) or not blocks:
            raise ValueError('push: expected a non-empty {name: (x_raw [h, Dx], seg_times [h, 2])} dict')
        out = {}
        for name, item in blocks.items():
            x, seg = (np.asarray(a, dtype=np.float64) for a in item)
            if x.ndim != 2 or x.shape[0] < 1:
                raise ValueError(f'push: stream {name!r}: expected a block of >= 1 x-vectors [h, Dx], got {x.shape}')
            Dx = self.streams[name].Dx if name in self.streams else self.Dx
            if x.shape[1] != Dx:
                raise ValueError(f'push: stream {name!r}: x-vectors of dimension {x.shape[1]}, the stream has {Dx}')
            if seg.shape != (x.shape[0], 2):
                raise ValueError(f'push: stream {name!r}: seg_times must be [{x.shape[0]}, 2], got {seg.shape}')
            if not np.isfinite(x).all():
                raise ValueError(f'push: stream {name!r}: x-vectors must be finite')
            out[name] = (x, seg)
        return out

    def push(self, blocks):
        """One push: blocks {name: (x_raw [h, Dx], seg_times [h, 2])}; a new name opens a stream.  Streams not in
        `blocks` are untouched.  Returns {name: dict(labels int64 [h], speakers [names of labels], iterations)}.
        Everything that can refuse a block (ValueError) is checked before the first commit, and the host's copy of a
        stream's count and K follows each state tier's commit, so a push that raises leaves every stream consistent.
        With self.timing a list, each push appends its stage times in seconds: front_end and vb are CUDA-event
        intervals (they hold host work too: the PLDA diagonalisation and the block's upload; run()'s host checks of the
        prior), ahc_linkage the vbx_ahc launches and the linkage's copy to the host, ahc_host_cut a host clock around
        the cut of every block, window and commit the kernels alone, wall a host clock around the whole push; tiers
        gives each state tier's window shapes (streams, S, context, block and evicted rows, known speakers)."""
        blocks = self._check_push(blocks)
        t0 = time.perf_counter()
        streams = [self.streams[n] if n in self.streams else self._open(n) for n in blocks]
        names = list(blocks)
        dev = self.dev
        lens = np.array([len(blocks[n][0]) for n in names], dtype=np.int64)
        chain = _resolve_chain(self.chain, self.transform, self.plda, self.lda_dim, self.Dx)
        timed = self.timing is not None
        pair = (lambda: [torch.cuda.Event(enable_timing=True) for _ in range(2)]) if timed else (lambda: None)
        e_front, e_ahc = pair(), pair()
        e_front and e_front[0].record()
        front, x, fea, Phi = _project(np.concatenate([blocks[n][0] for n in names]), lens, self.transform, self.plda,
                                      self.lda_dim, chain, dev)
        e_front and e_front[1].record()
        e_ahc and e_ahc[0].record()
        th, Zs = _ahc.linkage_batch(front, x)                                     # VBx/vbhmm.py:131-143
        e_ahc and e_ahc[1].record()
        front.close()
        if not bool(torch.isfinite(fea).all()):
            raise ValueError('push: a block projects to non-finite features (an x-vector equal to the transform mean?)')
        t_cut = time.perf_counter()
        K = [st.K for st in streams]
        cl = block_clusters(_ahc.cut(Zs, th, lens, self.threshold), Zs, lens, K, self.S_max)    # VBx/vbhmm.py:144-146
        t_cut = time.perf_counter() - t_cut
        fea, Phi = _pad_features(fea, Phi)
        boff = np.concatenate([[0], np.cumsum(lens)])
        result = {}
        tiers = {}
        for b, (_, c) in enumerate(cl):
            tiers.setdefault(_tier(K[b] + c), []).append(b)
        t_win = t_vb = t_commit = 0.0
        shapes = []
        for tier in sorted(tiers):
            grp = tiers[tier]
            g_lens = lens[grp]
            g_off = np.concatenate([[0], np.cumsum(g_lens)])
            g_fea = fea if len(grp) == len(names) else torch.cat([fea[boff[b]:boff[b + 1]] for b in grp]).contiguous()
            g_lab = torch.from_numpy(np.concatenate([cl[b][0] for b in grp]).astype(np.int32)).to(dev)
            slots = [streams[b].slot for b in grp]
            ns = np.array([K[b] + cl[b][1] for b in grp], dtype=np.int32)
            vb = VbxBatch(np.minimum([streams[b].count for b in grp], self.C) + g_lens, self.R, ns, device=dev)
            e_win, e_vb, e_com = pair(), pair(), pair()
            w_fea, g, p, _, prior = vb.stream_window(self.state, slots, g_fea, g_off, g_lab, [cl[b][1] for b in grp],
                                                     self.smoothing, events=e_win)
            e_vb and e_vb[0].record()
            vb.prepare_scale(w_fea, Phi)
            res = vb.run(g, p, Fa=self.Fa, Fb=self.Fb, loopProb=self.loopP, maxIters=self.max_iters,
                         epsilon=self.epsilon, prior=prior)
            first = vb.hard_labels(g)
            e_vb and e_vb[1].record()
            final = vb.stream_commit(self.state, slots, g_fea, g_off, first, events=e_com)
            final = final.cpu().numpy().astype(np.int64)
            it = res['n_iters'].cpu().numpy()
            for j, b in enumerate(grp):                    # the host's copy follows the device state tier by tier
                n, st, l = names[b], streams[b], final[g_off[j]:g_off[j + 1]]
                st.K = max(st.K, int(l.max()) + 1)
                st.count += int(lens[b])
                st.seg.append(blocks[n][1])
                st.labels.append(l)
                result[n] = dict(labels=l, speakers=[f'spk{k + 1}' for k in l.tolist()], iterations=int(it[j]))
            if timed:
                ctx = np.minimum([streams[b].count - int(lens[b]) for b in grp], self.C)
                shapes.append(dict(streams=len(grp), S=vb.S, context_rows=int(ctx.sum()), block_rows=int(g_lens.sum()),
                                   evicted_rows=int(np.maximum(ctx + g_lens - self.C, 0).sum()),
                                   known_speakers=int(sum(K[b] for b in grp))))
                t_win += e_win[0].elapsed_time(e_win[1]) * 1e-3
                t_vb += e_vb[0].elapsed_time(e_vb[1]) * 1e-3
                t_commit += e_com[0].elapsed_time(e_com[1]) * 1e-3
            vb.close()
        result = {n: result[n] for n in names}
        if timed:
            torch.cuda.synchronize(dev)
            self.timing.append(dict(wall=time.perf_counter() - t0, front_end=e_front[0].elapsed_time(e_front[1]) * 1e-3,
                                    ahc_linkage=e_ahc[0].elapsed_time(e_ahc[1]) * 1e-3, ahc_host_cut=t_cut,
                                    window=t_win, vb=t_vb, commit=t_commit, streams=len(names),
                                    xvectors=int(lens.sum()), tiers=shapes))
        return result


def block_schedule(recordings, block_seconds):
    """The pushes that replay an archive as live streams: push k (1-based) delivers, for every recording, the x-vectors
    whose segment ends in ((k-1) B, k B] (the first push also those ending at or before 0), so a recording can skip a
    push.  recordings {name: (x, seg_times)}.  Returns [{name: row indices}] per push, pushes without rows included."""
    if not block_seconds > 0:
        raise ValueError(f'block_seconds must be > 0, got {block_seconds}')
    ends = {n: np.asarray(r[1], dtype=np.float64).reshape(-1, 2)[:, 1] for n, r in recordings.items()}
    last = max((float(e.max()) for e in ends.values() if len(e)), default=0.0)
    n_push = max(1, int(np.ceil(last / block_seconds)))
    pushes = []
    for k in range(1, n_push + 1):
        lo, hi = (k - 1) * block_seconds, k * block_seconds
        push = {}
        for n, e in ends.items():
            rows = np.nonzero(((e > lo) | (k == 1)) & (e <= hi))[0]
            if len(rows):
                push[n] = rows
        pushes.append(push)
    return pushes


def build_parser():
    from .cli import build_parser as cli_parser
    ap = argparse.ArgumentParser(description='Replay an archive as live streams: every recording is a stream, diarized '
                                             'block by block (DESIGN.md section 5.25).  One RTTM per recording.')
    base = cli_parser()
    keep = ('--out-rttm-dir', '--xvec-ark-file', '--segments-file', '--xvec-transform', '--plda-file', '--threshold',
            '--lda-dim', '--Fa', '--Fb', '--loopP', '--init-smoothing', '--chain', '--device')
    for a in base._actions:
        if a.option_strings and a.option_strings[0] in keep:
            ap._add_action(a)
    ap.add_argument('--block-seconds', type=float, default=10.0, help='push length in seconds (default 10)')
    ap.add_argument('--context', type=int, default=240, help='look-back context in x-vectors (default 240)')
    ap.add_argument('--max-speakers', type=int, default=64, help='largest speaker count of a stream, 1 .. 128')
    ap.add_argument('--timing-json', default=None, help='write the wall time of every push to this JSON file')
    return ap


def main(argv=None):
    ap = build_parser()
    args = ap.parse_args(argv)
    if not args.block_seconds > 0:
        ap.error('--block-seconds must be > 0')
    from . import formats
    segs = formats.read_segments(args.segments_file)
    plda = formats.read_kaldi_plda(args.plda_file)
    transform = formats.read_xvec_transform(args.xvec_transform)
    recs = {}
    for name, (keys, x) in formats.read_xvectors_by_recording(args.xvec_ark_file).items():
        seg_names, times = segs[name]
        assert np.all(np.array(seg_names) == np.array(keys))
        recs[name] = (x, times)
    try:
        sd = StreamDiarizer(transform, plda, args.Fa, args.Fb, args.loopP, lda_dim=args.lda_dim,
                            threshold=args.threshold, smoothing=args.init_smoothing, context=args.context,
                            max_speakers=args.max_speakers, device=args.device, chain=args.chain)
    except ValueError as e:
        ap.error(str(e))
    walls = []
    for push in block_schedule(recs, args.block_seconds):
        if not push:
            walls.append(dict(streams=0, xvectors=0, seconds=0.0))
            continue
        t0 = time.perf_counter()
        sd.push({n: (recs[n][0][rows], recs[n][1][rows]) for n, rows in push.items()})
        walls.append(dict(streams=len(push), xvectors=int(sum(len(r) for r in push.values())),
                          seconds=time.perf_counter() - t0))
    os.makedirs(args.out_rttm_dir, exist_ok=True)
    for name in recs:
        lines = sd.rttm(name) if name in sd.streams else []
        with open(os.path.join(args.out_rttm_dir, f'{name}.rttm'), 'w') as fp:
            fp.write(''.join(line + os.linesep for line in lines))
    if args.timing_json is not None:
        with open(args.timing_json, 'w') as fp:
            json.dump(dict(block_seconds=args.block_seconds, context=args.context, pushes=walls), fp)
    return 0


if __name__ == '__main__':
    sys.exit(main())
