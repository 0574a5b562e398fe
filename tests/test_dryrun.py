"""GPU tests are at least dry-run here: their whole logic (fixtures, oracle side, tolerances, output keys)
and the models' Python paths execute on the CPU with the oracle-backed stand-ins in place of the CUDA modules
(tests/helpers/dryrun_gpu_tests.py).  What is left for the GPU box is the kernels, each of which has its own parity test."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_module_level_gpu_tests_pass_on_cpu_standins():
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', 'helpers', 'dryrun_gpu_tests.py')], capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stderr[-2000:]
    status = {ln.split()[0]: ln.split()[1] for ln in r.stdout.splitlines() if len(ln.split()) >= 2 and ln.split()[1] in ('PASSED', 'FAILED')}
    assert status == {'c3_parity': 'PASSED', 'c1[False]': 'PASSED', 'c4[False]': 'PASSED', 'neuralangelo': 'PASSED', 'nerf_colmap': 'PASSED', 'neus_isosurface': 'PASSED',
                      'export_colours': 'PASSED'}, r.stdout[-3000:]
