"""CPU: the result saver imports without its optional third-party dependencies."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_result_utils_imports_without_pycocotools_and_supervision():
    code = ("import sys; sys.modules['pycocotools'] = sys.modules['pycocotools.mask'] = sys.modules['supervision'] = None\n"
            "import deva.inference.result_utils as r\n"
            "assert r.__file__.startswith(sys.argv[1]), r.__file__\n"
            "for mode in ('vipseg', 'burst', 'unsup_davis17', 'ref_davis', 'demo', 'gradio'):\n"
            "    assert r.ResultSaver('/nonexistent', 'a/b', dataset=mode, object_manager=None).dataset == mode\n"
            "try:\n"
            "    r.ResultSaver('/nonexistent', 'v', dataset='other', object_manager=None)\n"
            "except NotImplementedError:\n"
            "    pass\n"
            "else:\n"
            "    raise AssertionError('unknown dataset accepted')\n")
    pkg = os.path.join(ROOT, 'tracking-anything-with-deva_b200')
    env = dict(os.environ, PYTHONPATH=pkg)
    out = subprocess.run([sys.executable, '-c', code, pkg], env=env, capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
