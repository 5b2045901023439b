"""CPU-only: the missing-library rule of oracle_libs' fixtures, on pytest runs in a subprocess over temporary modules
that request a library that is never built.  A module whose selected tests include a gpu one fails; one without skips,
also when its gpu tests are deselected."""
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEAD = '''import oracle
import oracle_libs
import pytest

oracle.LIBS["absent"] = "libabsent.so"  # never built
absent = oracle_libs.library("absent")
'''
GPU_TEST = '''

@pytest.mark.gpu
def test_gpu(absent):
    pass
'''
CPU_TEST = '''

def test_cpu(absent):
    pass
'''


def _outcomes(tmp_path, modules, *args):
    """{test name: PASSED / FAILED / ERROR / SKIPPED} of a pytest run over `modules` ({file name: test source}), and its
    output"""
    (tmp_path / "conftest.py").write_text("def pytest_configure(config):\n    config.addinivalue_line('markers', 'gpu: GPU test')\n")
    for name, body in modules.items():
        (tmp_path / name).write_text(HEAD + body)
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    python = [sys.executable] + (["-s"] if sys.flags.no_user_site else [])
    r = subprocess.run(python + ["-m", "pytest", "-v", "-p", "no:cacheprovider", "-rA", *args, str(tmp_path)], cwd=tmp_path,
                       capture_output=True, text=True, env=env, timeout=300)
    return dict(re.findall(r"::(\w+) (PASSED|FAILED|ERROR|SKIPPED)", r.stdout)), r.stdout


def test_gpu_test_fails_and_cpu_test_skips(tmp_path):
    got, out = _outcomes(tmp_path, {"test_on_gpu.py": GPU_TEST, "test_on_cpu.py": CPU_TEST})
    assert got == {"test_gpu": "ERROR", "test_cpu": "SKIPPED"}, out
    assert "oracle/_ref/libabsent.so is missing: build it with `python __graft_entry__.py --oracle`" in out, out


def test_deselected_gpu_tests_do_not_fail_the_others(tmp_path):
    got, out = _outcomes(tmp_path, {"test_both.py": GPU_TEST + CPU_TEST}, "-m", "not gpu")
    assert got == {"test_cpu": "SKIPPED"}, out
    got, out = _outcomes(tmp_path, {"test_both.py": GPU_TEST + CPU_TEST})
    assert got == {"test_gpu": "ERROR", "test_cpu": "ERROR"}, out
