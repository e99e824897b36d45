"""AHC initialisation (SURVEY.md 8f.3): the oracle restatement and the host-side cut against reference-generated
goldens on the CPU; the device kernels (vbx_ahc) against both on the GPU."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, 'tests', 'golden')

from oracle import ahc_oracle                      # noqa: E402
from vbx_b200 import ahc as host_ahc               # noqa: E402

CASES = ['es2005a', 'syn_a', 'syn_b', 'syn_c']


@pytest.fixture(scope='module')
def gold():
    return np.load(os.path.join(GOLD, 'ahc_cases.npz'))


def case_x(gold, name):
    if name == 'es2005a':
        return np.load(os.path.join(GOLD, 'es2005a.npz'))['x_lda']
    return gold[name + '/x']


@pytest.mark.parametrize('name', CASES)
def test_oracle_matches_reference_goldens(gold, name):
    labels, thr, Z = ahc_oracle.ahc_labels(case_x(gold, name))
    assert abs(thr - float(gold[name + '/thr'])) <= 1e-10
    np.testing.assert_array_equal(Z[:, :2], gold[name + '/Z'][:, :2])
    np.testing.assert_allclose(Z[:, 2], gold[name + '/Z'][:, 2], rtol=0, atol=1e-12)
    np.testing.assert_array_equal(labels, gold[name + '/labels'])


@pytest.mark.parametrize('name', CASES)
def test_flat_clusters_reproduces_scipy_numbering(gold, name):
    """vbx_b200.ahc.flat_clusters == fcluster(..., 'distance') of VBx/vbhmm.py:144-146 on the golden linkages."""
    Z, thr = gold[name + '/Z'], float(gold[name + '/thr'])
    np.testing.assert_array_equal(host_ahc.flat_clusters(Z, -(thr - 0.015)) - 1, gold[name + '/labels'])
    from scipy.cluster.hierarchy import fcluster
    adjust = abs(Z[:, 2].min())
    shifted = Z.copy()
    shifted[:, 2] += adjust
    for t in np.linspace(Z[:, 2].min() - 0.01, Z[:, 2].max() + 0.01, 23):
        np.testing.assert_array_equal(host_ahc.flat_clusters(Z, t), fcluster(shifted, t + adjust, criterion='distance'))


def test_flat_clusters_edge_cases():
    assert host_ahc.flat_clusters(np.zeros((0, 4)), 0.0).tolist() == [1]
    Z = np.array([[0.0, 1.0, -0.5, 2.0]])
    assert host_ahc.flat_clusters(Z, -0.4).tolist() == [1, 1]
    assert host_ahc.flat_clusters(Z, -0.6).tolist() == [1, 2]


def _device_ahc(xs, dtype):
    from vbx_b200.batch import VbxBatch
    dev = torch.device('cuda:0')
    lens = [len(x) for x in xs]
    vb = VbxBatch(lens, 128, 2, device=dev, allocate=False)
    x = torch.from_numpy(np.concatenate(xs, axis=0)).to(dev).to(dtype).contiguous()
    out = host_ahc.ahc_batch(vb, x)
    vb.close()
    return out


@pytest.mark.gpu
def test_device_ahc_matches_reference_goldens(gold):
    """All four cases as one ragged batch, float64 x-vectors: the thresholds, every merge of the dendrograms and the
    flat-cluster labels equal the reference's."""
    labels, thr, Zs = _device_ahc([case_x(gold, n) for n in CASES], torch.float64)
    for b, name in enumerate(CASES):
        assert abs(thr[b] - float(gold[name + '/thr'])) <= 1e-9, name
        Zr = gold[name + '/Z']
        np.testing.assert_array_equal(Zs[b][:, [0, 1, 3]], Zr[:, [0, 1, 3]], err_msg=name)
        np.testing.assert_allclose(Zs[b][:, 2], Zr[:, 2], rtol=0, atol=1e-12, err_msg=name)
        np.testing.assert_array_equal(labels[b], gold[name + '/labels'], err_msg=name)


@pytest.mark.gpu
def test_device_ahc_from_float32_xvectors(gold):
    """float32 x-vectors (what the tensor-core front end hands over): same flat clusters, threshold within 1e-6."""
    labels, thr, _ = _device_ahc([case_x(gold, n) for n in CASES], torch.float32)
    for b, name in enumerate(CASES):
        assert abs(thr[b] - float(gold[name + '/thr'])) <= 1e-6, name
        np.testing.assert_array_equal(labels[b], gold[name + '/labels'], err_msg=name)


@pytest.mark.gpu
def test_device_ahc_tiny_recordings():
    """Recordings of 0, 1, 2 and 3 x-vectors next to a normal one."""
    rng = np.random.default_rng(3)
    xs = [rng.standard_normal((t, 128)) for t in (2, 1, 0, 3, 60)]
    from vbx_b200.batch import VbxBatch
    dev = torch.device('cuda:0')
    vb = VbxBatch([len(x) for x in xs], 128, 2, device=dev, allocate=False)
    x = torch.from_numpy(np.concatenate(xs, axis=0)).to(dev)
    labels, thr, Zs = host_ahc.ahc_batch(vb, x)
    assert labels[1].tolist() == [0] and labels[2].size == 0
    assert labels[0].shape == (2,) and labels[3].shape == (3,)
    ref_l, ref_t, ref_Z = ahc_oracle.ahc_labels(xs[4])
    np.testing.assert_array_equal(labels[4], ref_l)
    np.testing.assert_allclose(Zs[4], ref_Z, rtol=0, atol=1e-12)
    ref_l3, _, ref_Z3 = ahc_oracle.ahc_labels(xs[3])
    np.testing.assert_allclose(Zs[3], ref_Z3, rtol=0, atol=1e-12)
    vb.close()
