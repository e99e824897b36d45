"""The S = 128 state tier without a GPU: the padding rule of the C ABI and of the Python batch API."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def lib():
    from vbx_b200 import build
    build.build_library()
    import vbx_b200._lib as L
    return L.load()


def test_padded_states_wide(lib):
    got = [lib.vbx_padded_states_wide(n) for n in (1, 3, 4, 5, 9, 17, 33, 64, 65, 100, 127, 128)]
    assert got == [4, 4, 4, 8, 16, 32, 64, 64, 128, 128, 128, 128]
    assert [lib.vbx_padded_states_wide(n) for n in (0, -1, 129, 256)] == [-1, -1, -1, -1]
    # the narrow function keeps its behaviour: 64 states at most
    assert [lib.vbx_padded_states(n) for n in (64, 65, 128)] == [64, -1, -1]


def test_python_padding_follows_the_tiers(lib):
    import vbx_b200._lib as L
    assert [L.padded_states(n) for n in (1, 31, 64, 65, 128)] == [4, 32, 64, 128, 128]
    with pytest.raises(L.VbxError, match='1..128'):
        L.padded_states(129)


def test_header_documents_the_wide_tier():
    src = open(os.path.join(ROOT, 'include', 'vbx_b200.h')).read()
    assert re.search(r'int32_t\s+vbx_padded_states_wide\s*\(\s*int32_t', src)
    flat = re.sub(r'\s*\n\s*\*\s*', ' ', src)      # comment text without its line breaks
    assert 'vbx_plan refuses S = 128 with VBX_ERR_ARG while fb_split = 2' in flat
    assert 'at S = 128 values below 4 are raised' in flat
