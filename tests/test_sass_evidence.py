"""Static evidence that the shipped library is the sm_90a code DESIGN.md describes: the SASS of libvbx_b200.so holds
the Hopper warpgroup tensor-core (wgmma) / TMA / mbarrier instructions of the projection kernels, the mma.sync
contractions, and the order-pinned accesses of the forward-backward sweep.  CPU-only."""
import collections
import re
import shutil
import subprocess

import pytest

from vbx_b200 import _lib


@pytest.fixture(scope='module')
def sass():
    tool = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    try:
        out = subprocess.run([tool, '-sass', _lib.LIB_PATH], capture_output=True, text=True, timeout=300)
    except (FileNotFoundError, subprocess.TimeoutExpired):
        pytest.skip('cuobjdump not available')
    if out.returncode != 0 or 'Function :' not in out.stdout:
        pytest.skip('cuobjdump could not read the library')
    per_fn = collections.defaultdict(collections.Counter)
    fn = None
    for line in out.stdout.splitlines():
        m = re.search(r'Function : (\S+)', line)
        if m:
            fn = m.group(1)
            continue
        m = re.match(r'\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_]*)((?:\.[A-Z0-9_]+)*)', line)
        if m and fn:
            per_fn[fn][m.group(1)] += 1
            per_fn[fn][m.group(1) + m.group(2)] += 1
    assert 'sm_90a' in out.stdout or per_fn
    return per_fn


def functions(sass, needle):
    return {f: c for f, c in sass.items() if needle in f}


def test_only_sm_90a_code_is_shipped():
    tool = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    try:
        out = subprocess.run([tool, '-lelf', _lib.LIB_PATH], capture_output=True, text=True, timeout=120).stdout
    except (FileNotFoundError, subprocess.TimeoutExpired):
        pytest.skip('cuobjdump not available')
    archs = set(re.findall(r'sm_\d+a?', out))
    assert archs == {'sm_90a'}, archs


def test_projection_runs_on_wgmma_and_tma(sass):
    proj = functions(sass, 'project_wgmma_kernel')
    assert len(proj) == 3                                   # plain projection + the two passes of the x-vector front end
    for f, c in proj.items():
        assert c['HGMMA'] >= 12, (f, c['HGMMA'])            # wgmma m64n128k8 tf32, 4 k-steps x 3 split terms per block
        assert c['WARPGROUP'] >= 1, f                       # wgmma.fence / wait_group: accumulators stay in registers
        assert c['UBLKCP'] >= 1, f                          # cp.async.bulk of the pre-swizzled V images
        assert c['SYNCS'] >= 4, f                           # mbarrier pipeline


def test_in_loop_contractions_use_the_tensor_cores(sass):
    for name in ('mstep_mma_kernel', 'loglik_mma_kernel'):
        fns = functions(sass, name)
        assert fns, name
        for f, c in fns.items():
            assert c['HMMA'] >= 3, (f, c['HMMA'])           # mma.sync m16n8k8 tf32, three split-precision terms


def test_forward_backward_sweeps(sass):
    la = functions(sass, 'forward_backward_la_kernel')
    assert len(la) == 14
    for f, c in la.items():
        assert c['LDG.E.64.STRONG.SYS'] + c['LDG.E.STRONG.SYS'] + c['LDG.E.128.STRONG.SYS'] > 0, f   # order-pinned bursts
        assert c['MUFU'] > 0, f


def test_split_sweeps_and_float64_finish(sass):
    sw = functions(sass, 'fb_sweeps_kernel')
    assert len(sw) >= 5                                     # S = 4 ... 64 (+ the states-per-lane variants)
    for f, c in sw.items():
        assert c['LDG.E.64.STRONG.SYS'] + c['LDG.E.STRONG.SYS'] + c['LDG.E.128.STRONG.SYS'] > 0, f   # order-pinned bursts
        assert c['SHFL'] > 0 and c['MUFU'] > 0, f           # group reductions, off-chain reciprocals
    assert functions(sass, 'fb_combine_kernel') and functions(sass, 'fb_split_tail_kernel')
    for name in ('mstep64_kernel', 'loglik64_kernel', 'fb64_kernel', 'speaker64_kernel', 'fb_dense_kernel'):
        fns = functions(sass, name)
        assert fns, name
        for f, c in fns.items():
            assert c['DFMA'] + c['DADD'] + c['DMUL'] > 0, f  # float64 arithmetic
    assert functions(sass, 'elbo_trace_kernel') and functions(sass, 'snapshot_kernel')


def test_front_end_uses_the_three_way_split(sass):
    """The two passes of the real-data front end issue six wgmma per k-step (x3 v1, x1 v3, x2 v2, x2 v1, x1 v2, x1 v1),
    the headline projection three (lo hi, hi lo, hi hi)."""
    proj = functions(sass, 'project_wgmma_kernel')
    three = [f for f in proj if 'ILi1ELi3E' in f or 'ILi2ELi3E' in f]
    two = [f for f in proj if 'ILi0ELi2E' in f]
    assert len(three) == 2 and len(two) == 1, list(proj)
    for f in three:
        assert proj[f]['HGMMA'] >= 24, (f, proj[f]['HGMMA'])


def test_float64_ahc_kernels(sass):
    assert functions(sass, 'ahc_cosine_kernel') and functions(sass, 'ahc_linkage_kernel')
    for f, c in functions(sass, 'ahc_cosine_kernel').items():
        assert c['DFMA'] > 0, f
