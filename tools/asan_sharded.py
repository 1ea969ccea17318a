"""Test tooling: the sharded (owner-mode) paths of the emulated library under AddressSanitizer -- report / move-list gather at
DADA2B_MOVES_EAGER = 0 / 3 / default (world 1 included), sharded re-upload with small packing blocks, the round tail's global-memory
form from mid-run (tests/test_emu_asan.py covers the unsharded kernels inside the suite; this run takes another minute).
    python tools/asan_sharded.py"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))

CHILD = """
import sys, os
sys.path.insert(0, %r); sys.path.insert(0, os.path.join(%r, 'tests', 'emu'))
import dada2_b200.api as api
api._LIBPATH = %r; api._LIB = None
import tests.test_emu_parity as T
for eager in ('0', '3', '1024'):
    os.environ['DADA2B_MOVES_EAGER'] = eager
    T._run_sharded(3, 'syn800_nogreedy')
    T._run_sharded(2, 'syn700_ragged', reupload=True)
    T._run_sharded(1, 'syn800_default')
os.environ['DADA2B_PACK_BLK'] = '7'
T._run_sharded(3, 'syn700_ragged', reupload=True)
os.environ['DADA2B_TAIL_SMEM_CLUSTERS'] = '12'
T._run_sharded(2, 'syn800_default')
print('ASAN SHARD OK')
"""

if __name__ == "__main__":
    import build_emu
    import tests.test_emu_asan as A
    lib = build_emu.build(asan=True)
    pre = A._preload()
    if pre is None:
        sys.exit("libasan not found")
    env = dict(os.environ, LD_PRELOAD=pre, ASAN_OPTIONS="detect_leaks=0:halt_on_error=1")
    out = subprocess.run([sys.executable, "-c", CHILD % (ROOT, ROOT, lib)], env=env, capture_output=True, text=True, timeout=2400)
    sys.stdout.write(out.stdout[-400:]); sys.stderr.write(out.stderr[-3000:])
    sys.exit(0 if "ASAN SHARD OK" in out.stdout and "AddressSanitizer" not in out.stderr else 1)
