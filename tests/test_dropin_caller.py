"""The reference's real caller against the drop-in: `python VBx/vbhmm.py ...` unchanged (run_example.sh:23-34,
VBx/vbhmm.py:45,154-158), started through the launcher that makes `from VBx import VBx` resolve to vbx_b200.

  * the import mechanics are tested with a two-directory mock that stands in for the reference tree (no GPU needed);
  * what the drop-in computes for the reference's ES2005a call is covered on the GPU by tests/test_parity_gpu.py /
    test_pipeline.py, and the command line over the same recording by test_command_line_batch_of_recordings_to_rttm.
"""
import os
import subprocess
import sys
import textwrap

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _mock_tree(tmp_path):
    """A 'reference' directory with its own VBx.py next to the caller script, like VBx/VBx.py next to VBx/vbhmm.py."""
    d = tmp_path / 'refdir'
    d.mkdir()
    (d / 'VBx.py').write_text("def VBx(*a, **k):\n    raise SystemExit('the reference VBx.py was imported')\n")
    (d / 'helper_next_to_script.py').write_text('VALUE = 41\n')
    (d / 'caller.py').write_text(textwrap.dedent('''
        import sys
        from helper_next_to_script import VALUE          # siblings of the script must stay importable
        from VBx import VBx
        import VBx as module
        print('VBX_FROM', VBx.__module__, VALUE, sys.argv[1:], __name__, hasattr(module, 'forward_backward'), hasattr(module, 'DER'))
    '''))
    return d


def test_launcher_makes_the_shadow_module_win(tmp_path):
    d = _mock_tree(tmp_path)
    env = dict(os.environ, PYTHONPATH=ROOT)
    out = subprocess.run([sys.executable, '-m', 'vbx_b200.dropin.run', str(d / 'caller.py'), '--flag', 'x'],
                         capture_output=True, text=True, env=env, cwd=str(tmp_path), timeout=300)
    assert out.returncode == 0, out.stderr[-800:]
    assert "VBX_FROM vbx_b200.api 41 ['--flag', 'x'] __main__ True True" in out.stdout


def test_pythonpath_alone_does_not_shadow_a_sibling_module(tmp_path):
    """Why the launcher exists: the script's directory is sys.path[0], ahead of PYTHONPATH."""
    d = _mock_tree(tmp_path)
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.join(ROOT, 'vbx_b200', 'dropin'), ROOT]))
    out = subprocess.run([sys.executable, str(d / 'caller.py')], capture_output=True, text=True, env=env, timeout=300)
    assert 'VBX_FROM VBx' in out.stdout          # the sibling VBx.py won


def test_shadow_module_exports_the_reference_names():
    import importlib
    m = importlib.import_module('vbx_b200.dropin.VBx')
    assert callable(m.VBx) and callable(m.forward_backward) and callable(m.DER)
