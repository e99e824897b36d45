"""Readers/writers for the on-disk formats either side of the VB-HMM path.

The reference reads these through kaldi_io / h5py (VBx/vbhmm.py:105-128, VBx/kaldi_utils.py:25-106),
neither of which exists in this image; the byte layouts are simple enough to parse directly.
These are host-side helpers (fixture building, end-to-end checks) - not on the GPU hot path.
"""
import struct

import numpy as np


def read_vec_flt_ark(path):
    """Iterate (key, vector) over a Kaldi binary float-vector archive (what
    kaldi_io.read_vec_flt_ark yields at VBx/vbhmm.py:117; written at VBx/predict.py:193).
    Record = key + ' ' + '\\0B' + ('FV '|'DV ') + '\\x04' + int32 dim + raw little-endian data."""
    with open(path, 'rb') as f:
        buf = f.read()
    pos, n = 0, len(buf)
    while pos < n:
        sp = buf.index(b' ', pos)
        key = buf[pos:sp].decode('ascii')
        pos = sp + 1
        if buf[pos:pos + 2] != b'\0B':
            raise ValueError(f'{path}: record {key!r} is not Kaldi binary')
        tag = buf[pos + 2:pos + 5]
        if tag == b'FV ':
            dt = np.dtype('<f4')
        elif tag == b'DV ':
            dt = np.dtype('<f8')
        else:
            raise ValueError(f'{path}: unsupported vector tag {tag!r}')
        pos += 5
        if buf[pos] != 4:
            raise ValueError(f'{path}: bad size marker')
        (dim,) = struct.unpack_from('<i', buf, pos + 1)
        pos += 5
        vec = np.frombuffer(buf, dtype=dt, count=dim, offset=pos).copy()
        pos += dim * dt.itemsize
        yield key, vec


def write_vec_flt_ark(path, keys, vectors):
    """Kaldi binary float-vector archive (what VBx/predict.py:193 writes): one float32 vector per key."""
    with open(path, 'wb') as f:
        for key, v in zip(keys, vectors):
            v = np.ascontiguousarray(v, dtype='<f4')
            f.write(key.encode('ascii') + b' ' + b'\0B' + b'FV ' + b'\x04' + struct.pack('<i', v.shape[0]) + v.tobytes())


def read_xvectors_by_recording(path):
    """Group an ark by recording id = key up to the last '_' (VBx/vbhmm.py:119).
    Returns {recording: (list_of_keys, float array T x D)} preserving archive order."""
    out = {}
    for key, vec in read_vec_flt_ark(path):
        rec = key.rsplit('_', 1)[0]
        keys, vecs = out.setdefault(rec, ([], []))
        keys.append(key)
        vecs.append(vec)
    return {rec: (keys, np.array(vecs)) for rec, (keys, vecs) in out.items()}


def read_segments(path):
    """Kaldi 'segments' file -> {recording: (names array, T x 2 start/end seconds)}
    (VBx/diarization_lib.py:96-110)."""
    recs = {}
    with open(path) as f:
        for line in f:
            parts = line.split()
            if not parts:
                continue
            name, rec, start, end = parts[0], parts[1], float(parts[2]), float(parts[3])
            names, times = recs.setdefault(rec, ([], []))
            names.append(name)
            times.append((start, end))
    return {rec: (np.array(names, dtype=object), np.array(times, dtype=np.float64))
            for rec, (names, times) in recs.items()}


def _kaldi_token(buf, pos, token):
    if buf[pos:pos + len(token)] != token:
        raise ValueError(f'expected {token!r} at byte {pos}')
    return pos + len(token)


def _kaldi_vec(buf, pos):
    tag = buf[pos:pos + 3]
    dt = {b'FV ': np.dtype('<f4'), b'DV ': np.dtype('<f8')}[tag]
    pos += 3
    assert buf[pos] == 4
    (n,) = struct.unpack_from('<i', buf, pos + 1)
    pos += 5
    v = np.frombuffer(buf, dtype=dt, count=n, offset=pos).astype(np.float64)
    return v, pos + n * dt.itemsize


def _kaldi_mat(buf, pos):
    tag = buf[pos:pos + 3]
    dt = {b'FM ': np.dtype('<f4'), b'DM ': np.dtype('<f8')}[tag]
    pos += 3
    assert buf[pos] == 4
    (rows,) = struct.unpack_from('<i', buf, pos + 1)
    assert buf[pos + 5] == 4
    (cols,) = struct.unpack_from('<i', buf, pos + 6)
    pos += 10
    m = np.frombuffer(buf, dtype=dt, count=rows * cols, offset=pos).astype(np.float64)
    return m.reshape(rows, cols), pos + rows * cols * dt.itemsize


def _text_tokens(txt, pos):
    """Tokens of a Kaldi text object starting at `pos` up to and including its closing ']' -> (floats, next pos)."""
    end = txt.index(']', pos)
    body = txt[pos:end].replace('[', ' ')
    return [float(t) for t in body.split()], end + 1


def read_kaldi_plda(path):
    """Kaldi PLDA, binary or text -> (mean, transform, psi) float64 (VBx/kaldi_utils.py:25-53).
    Binary: '\\0B<Plda> ' vector matrix vector '</Plda> '.  Text: '<Plda>  [ mean ]\\n [\\n rows ]\\n [ psi ]\\n</Plda> '
    (what `ivector-copy-plda --binary=false` writes; one matrix row per line)."""
    with open(path, 'rb') as f:
        buf = f.read()
    if buf[:2] == b'\0B':
        pos = _kaldi_token(buf, 2, b'<Plda> ')
        mean, pos = _kaldi_vec(buf, pos)
        tr, pos = _kaldi_mat(buf, pos)
        psi, pos = _kaldi_vec(buf, pos)
        _kaldi_token(buf, pos, b'</Plda> ')
        return mean, tr, psi
    txt = buf.decode('ascii')
    if not txt.lstrip().startswith('<Plda>'):
        raise ValueError(f'{path}: not a Kaldi PLDA model')
    pos = txt.index('<Plda>') + len('<Plda>')
    mean, pos = _text_tokens(txt, pos)
    # the matrix: rows are separated by newlines inside one bracket pair
    lb = txt.index('[', pos)
    rb = txt.index(']', lb)
    rows = [line.split() for line in txt[lb + 1:rb].strip().splitlines() if line.strip()]
    tr = np.array([[float(v) for v in r] for r in rows], dtype=np.float64)
    psi, pos = _text_tokens(txt, rb + 1)
    if '</Plda>' not in txt[pos:]:
        raise ValueError(f'{path}: missing </Plda>')
    mean, psi = np.array(mean, dtype=np.float64), np.array(psi, dtype=np.float64)
    if tr.ndim != 2 or tr.shape[0] != tr.shape[1] or tr.shape[0] != mean.shape[0] or psi.shape[0] != mean.shape[0]:
        raise ValueError(f'{path}: inconsistent PLDA dimensions {mean.shape} {tr.shape} {psi.shape}')
    return mean, tr, psi


def write_kaldi_plda_binary(path, mean, tr, psi):
    """Binary Kaldi PLDA with float64 payloads, the layout of the shipped models (VBx/kaldi_utils.py:37-49)."""
    mean, tr, psi = (np.ascontiguousarray(a, dtype='<f8') for a in (mean, tr, psi))
    with open(path, 'wb') as f:
        f.write(b'\0B<Plda> ')
        f.write(b'DV \x04' + struct.pack('<i', mean.shape[0]) + mean.tobytes())
        f.write(b'DM \x04' + struct.pack('<i', tr.shape[0]) + b'\x04' + struct.pack('<i', tr.shape[1]) + tr.tobytes())
        f.write(b'DV \x04' + struct.pack('<i', psi.shape[0]) + psi.tobytes())
        f.write(b'</Plda> ')


def write_kaldi_plda_text(path, mean, tr, psi):
    """Text form of a Kaldi PLDA (fixtures / interchange)."""
    with open(path, 'w') as f:
        f.write('<Plda>  [ ' + ' '.join(repr(float(v)) for v in mean) + ' ]\n [\n')
        for i, row in enumerate(tr):
            f.write('  ' + ' '.join(repr(float(v)) for v in row) + (' ]\n' if i == len(tr) - 1 else '\n'))
        f.write(' [ ' + ' '.join(repr(float(v)) for v in psi) + ' ]\n</Plda> ')


def read_xvec_transform(path):
    """The reference's `transform.h5` (datasets mean1 (256,), mean2 (128,), lda (256,128), float64;
    read through h5py at VBx/vbhmm.py:125-128).  Both shipped models use an HDF5 v0 superblock with
    contiguous datasets at fixed offsets; this reader validates the signature / size / dataset names
    and slices them out (a general HDF5 parser is out of scope)."""
    if str(path).endswith('.npz'):          # the same three arrays without HDF5 (np.savez(path, mean1=, mean2=, lda=))
        z = np.load(path)
        return (np.asarray(z['mean1'], dtype=np.float64), np.asarray(z['mean2'], dtype=np.float64),
                np.asarray(z['lda'], dtype=np.float64))
    with open(path, 'rb') as f:
        buf = f.read()
    if buf[:8] != b'\x89HDF\r\n\x1a\n' or len(buf) != 267264:
        raise ValueError(f'{path}: not the expected transform.h5 layout')
    for name in (b'mean1', b'mean2', b'lda'):
        if name not in buf[:2048]:
            raise ValueError(f'{path}: dataset {name!r} missing')
    mean1 = np.frombuffer(buf, dtype='<f8', count=256, offset=2048).copy()
    mean2 = np.frombuffer(buf, dtype='<f8', count=128, offset=4096).copy()
    lda = np.frombuffer(buf, dtype='<f8', count=256 * 128, offset=5120).reshape(256, 128).copy()
    return mean1, mean2, lda


def write_rttm(fp, recording, labels, starts, ends):
    """One SPEAKER line per merged segment, formatted as VBx/vbhmm.py:48-51."""
    for label, s, e in zip(labels, starts, ends):
        fp.write(f'SPEAKER {recording} 1 {s:03f} {e - s:03f} <NA> <NA> {label + 1} <NA> <NA>\n')


def read_rttm(path):
    """-> list of (recording, start, duration, label-string)."""
    out = []
    with open(path) as f:
        for line in f:
            p = line.split()
            if p and p[0] == 'SPEAKER':
                out.append((p[1], float(p[3]), float(p[4]), p[7]))
    return out


def read_uem(path):
    """Un-partitioned evaluation map, one 'file channel onset offset' line per scored interval (seconds)
    -> {recording: [(onset, offset), ...]} in file order.  Blank lines and lines starting with ';;' are skipped."""
    out = {}
    with open(path) as f:
        for n, line in enumerate(f, 1):
            p = line.split()
            if not p or p[0].startswith(';;'):
                continue
            if len(p) != 4:
                raise ValueError(f'{path}:{n}: expected "file channel onset offset", got {line.strip()!r}')
            out.setdefault(p[0], []).append((float(p[2]), float(p[3])))
    return out


def read_utt2spk(path):
    """Kaldi utt2spk, one 'utterance speaker' line each -> {utterance: speaker} in file order.  Blank lines are skipped;
    a line without exactly two fields, or an utterance listed twice, is a ValueError."""
    out = {}
    with open(path) as f:
        for n, line in enumerate(f, 1):
            p = line.split()
            if not p:
                continue
            if len(p) != 2:
                raise ValueError(f'{path}:{n}: expected "utterance speaker", got {line.strip()!r}')
            if p[0] in out:
                raise ValueError(f'{path}:{n}: utterance {p[0]!r} listed twice')
            out[p[0]] = p[1]
    return out


def read_enrolment(ark, utt2spk):
    """Enrolment x-vectors: a Kaldi x-vector ark and its utt2spk file -> {speaker: x [n, Dx] float64}, speakers in order
    of first appearance in the ark.  ValueError: an ark key missing from utt2spk, or a speaker of utt2spk none of whose
    utterances is in the ark (utterances of utt2spk missing from the ark are otherwise ignored)."""
    spk = read_utt2spk(utt2spk)
    out = {}
    for key, vec in read_vec_flt_ark(ark):
        if key not in spk:
            raise ValueError(f'{ark}: x-vector {key!r} has no speaker in {utt2spk}')
        out.setdefault(spk[key], []).append(np.asarray(vec, dtype=np.float64))
    empty = sorted(set(spk.values()) - set(out))
    if empty:
        raise ValueError(f'{utt2spk}: speakers without x-vectors in {ark}: {empty}')
    return {k: np.stack(v) for k, v in out.items()}


def read_speaker_counts(path):
    """Two-column 'recording count' file -> {recording: int}.  Blank lines and lines starting with '#' are skipped."""
    out = {}
    with open(path) as f:
        for n, line in enumerate(f, 1):
            p = line.split()
            if not p or p[0].startswith('#'):
                continue
            if len(p) != 2:
                raise ValueError(f'{path}:{n}: expected "recording count", got {line.strip()!r}')
            try:
                out[p[0]] = int(p[1])
            except ValueError:
                raise ValueError(f'{path}:{n}: the count {p[1]!r} is not an integer')
    return out
