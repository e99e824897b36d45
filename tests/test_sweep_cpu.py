"""Host logic of the hyperparameter sweep (vbx_b200/sweep.py): grid parsing, setting names, the batch packer and the
error without a CUDA device.  Runs without a GPU."""
import numpy as np
import pytest

from vbx_b200 import sweep


def test_grid_is_the_product_in_key_order():
    grid = dict(Fa=[0.3, 0.4], Fb=[17], loopP=[0.99, 0.5], threshold=[-0.015], smoothing=[5, 7])
    s = sweep.grid_settings(grid)
    assert len(s) == 8
    assert s[0] == (0.3, 17.0, 0.99, -0.015, 5.0)
    assert s[1] == (0.3, 17.0, 0.99, -0.015, 7.0)
    assert s[-1] == (0.4, 17.0, 0.5, -0.015, 7.0)
    assert len(sweep.grid_settings(dict(grid, Fa=[0.3, 0.3]))) == 4        # duplicates collapse


@pytest.mark.parametrize('bad', [dict(Fb=[0.0]), dict(loopP=[1.5]), dict(loopP=[-0.1]), dict(Fa=[]), dict(Fa=[float('nan')]),
                                 dict(alpha=[1.0])])
def test_grid_rejects_bad_values(bad):
    grid = dict(Fa=[0.3], Fb=[17], loopP=[0.99], threshold=[-0.015], smoothing=[5])
    grid.update(bad)
    with pytest.raises(ValueError):
        sweep.grid_settings(grid)


def test_parse_list():
    assert sweep.parse_list('0.3,0.4, 1') == [0.3, 0.4, 1.0]
    assert sweep.parse_list('-0.015') == [-0.015]
    for bad in ('', 'a,b', ','):
        with pytest.raises(ValueError):
            sweep.parse_list(bad)


def test_setting_names_are_stable():
    s = sweep.Setting(0.3, 17.0, 0.99, -0.015, 5.0)
    assert s.name == 'Fa0.3_Fb17_loopP0.99_thr-0.015_sm5'
    assert sweep.Setting(0.4, 64, 0.65, 0.1, 2.5).name == 'Fa0.4_Fb64_loopP0.65_thr0.1_sm2.5'
    names = [x.name for x in sweep.grid_settings(dict(Fa=[0.2, 0.3], Fb=[6, 17], loopP=[0.35, 0.99], threshold=[0, 0.1],
                                                      smoothing=[5]))]
    assert len(set(names)) == len(names)


@pytest.mark.parametrize('seed', range(5))
def test_packer_places_every_entry_once_within_budget(seed):
    rng = np.random.default_rng(seed)
    sizes = rng.integers(1, 1000, size=int(rng.integers(1, 300)))      # stub sizes
    budget = int(rng.integers(sizes.max(), 5000))
    batches = sweep.pack(sizes.tolist(), budget)
    flat = [i for b in batches for i in b]
    assert sorted(flat) == list(range(len(sizes)))
    assert all(sum(sizes[i] for i in b) <= budget for b in batches)
    assert all(b for b in batches)
    # consecutive batches could not have been merged greedily: the packer does not waste batches
    for a, b in zip(batches[:-1], batches[1:]):
        assert sum(sizes[i] for i in a) + sizes[b[0]] > budget


def test_packer_refuses_an_entry_over_budget():
    with pytest.raises(ValueError, match='max_batch_bytes'):
        sweep.pack([10, 200, 10], 100)


def test_no_cuda_device_is_a_clear_error(monkeypatch):
    import torch
    from vbx_b200._lib import VbxError
    monkeypatch.setattr(torch.cuda, 'is_available', lambda: False)
    grid = dict(Fa=[0.3], Fb=[17], loopP=[0.99], threshold=[-0.015], smoothing=[5])
    with pytest.raises(VbxError, match='no CUDA device'):
        sweep.sweep_batch({'r': (np.zeros((3, 256)), np.zeros((3, 2)))}, None, None, grid)
