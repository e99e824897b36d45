"""The bench line contract, checked on the committed line of the current build (profiles/h100_bench_headline.json,
written by `python bench.py` on an H100): every key the driver reads is there and the derived numbers are consistent with each
other (value = frames / step time, roofline.frac = achieved / peak, achieved = algorithmic bytes / launch time).
CPU only - it guards the format, the numbers themselves come from the GPU run."""
import json
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LINE = os.path.join(ROOT, 'profiles', 'h100_bench_headline.json')
BASELINE = os.path.join(ROOT, 'BASELINE.json')


@pytest.fixture(scope='module')
def line():
    if not os.path.exists(LINE):
        pytest.skip('no committed bench line')
    return json.load(open(LINE))


def test_top_level_keys(line):
    for k in ('metric', 'value', 'unit', 'n_gpus', 'steps', 'warmup', 'ms_per_step', 'higher_is_better', 'scaling',
              'vs_baseline', 'dtype', 'data', 'config', 'roofline', 'cpu_baseline', 'e2e', 'clocks', 'gpu_launches'):
        assert k in line, k
    assert line['higher_is_better'] is True and line['scaling'] == 'weak' and line['n_gpus'] == 1
    assert line['warmup'] >= 3 and line['steps'] >= 1
    assert line['vs_baseline'] is None                     # BASELINE.md holds no published number for this metric
    assert line['dtype'] == 'f32' and 'synthetic' in line['data']
    assert 'workload' in line['config'] and 'model' not in line['config']
    assert line['gpu_launches'] > 0
    if os.path.exists(BASELINE):
        metric = json.load(open(BASELINE)).get('metric')
        if isinstance(metric, str):                        # "x-vectors/sec through 10 VB-HMM EM iters; achieved HBM GB/s vs 8 TB/s"
            assert metric.split(';')[0].strip().lower() == line['metric'].lower()


def test_value_is_frames_over_step_time(line):
    c = line['config']
    frames = c['recordings'] * c['frames_per_recording']
    assert abs(line['value'] - frames / (line['ms_per_step'] * 1e-3)) <= 1e-6 * line['value']
    assert line['unit'] == 'x-vectors/s'


def test_roofline_object(line):
    r = line['roofline']
    for k in ('bound', 'achieved', 'peak', 'unit', 'frac', 'traffic'):
        assert k in r, k
    assert r['bound'] == 'hbm' and r['unit'] == 'GB/s'
    assert abs(r['frac'] - r['achieved'] / r['peak']) <= 1e-9
    assert 0.0 < r['frac'] < 1.0
    assert abs(r['achieved'] - r['algorithmic_bytes_per_launch'] / (r['avg_launch_ms'] * 1e-3) / 1e9) <= 1e-6 * r['achieved']
    assert r['traffic'] is None or 0.9 * r['algorithmic_bytes_per_launch'] <= r['traffic'] <= 1.5 * r['algorithmic_bytes_per_launch']
    w = line['whole_step']
    assert abs(w['achieved_gbs'] - w['algorithmic_bytes_per_step'] / (line['ms_per_step'] * 1e-3) / 1e9) <= 1e-6 * w['achieved_gbs']
    # SURVEY 8(d): N * (4D + 4R + 4S + 2 * 4R * iters) = 11 840 B per x-vector at 10 iterations
    c = line['config']
    assert w['algorithmic_bytes_per_step'] == c['recordings'] * c['frames_per_recording'] * 11840


def test_e2e_cpu_baseline_and_clocks(line):
    e = line['e2e']
    for k in ('value', 'unit', 'h2d_bytes_per_step', 'd2h_bytes_per_step'):
        assert k in e, k
    c = line['config']
    frames = c['recordings'] * c['frames_per_recording']
    assert e['h2d_bytes_per_step'] == frames * (c['D'] + c['S']) * 4          # raw x-vectors + initial responsibilities
    assert e['d2h_bytes_per_step'] >= frames * c['S'] * 4                      # responsibilities back
    assert 0 < e['value'] < line['value']                                       # PCIe-bound: below the resident number
    b = line['cpu_baseline']
    for k in ('value', 'unit', 'cores', 'kind', 'sample'):
        assert k in b, k
    assert b['kind'] in ('reference', 'port') and b['cores'] >= 1 and b['value'] > 0
    k = line['clocks']
    # a clock below 0.8 of the maximum only counts when the card was held there by its own power limit
    capped = 'sw_power_cap' in k['reasons'] and k['power_w'] >= 0.9 * k['power_limit_w']
    assert k['sm_mhz'] > 0.8 * k['sm_max_mhz'] or capped
    assert not set(k['reasons']) & {'hw_slowdown', 'hw_thermal_slowdown', 'sw_thermal_slowdown'}
    assert line['parity']['ok'] is True
