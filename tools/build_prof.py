"""Build the profiling variant of the library (-DRB_TVR_PROF: clock64 stamps in the minimiser, %globaltimer marker kernels
in the pipeline) into tools/_prof/ (git-ignored).  Used by cluster_stamps.py and trace_run.py on a GPU box."""
import os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rebvo_b200 import build as B
extra = [a for a in sys.argv[1:] if a.startswith('-D')]
tag = ''.join(a for a in sys.argv[1:] if not a.startswith('-'))
out = os.path.join(os.path.dirname(os.path.abspath(__file__)), '_prof' + tag)
os.makedirs(out, exist_ok=True)
objs = []
for s in B.SOURCES:
    o = os.path.join(out, s.replace('.cu', '.o'))
    subprocess.check_call([B.NVCC] + B.FLAGS + ['-DRB_TVR_PROF'] + extra + ['-c', os.path.join(B.CSRC, s), '-o', o])
    objs.append(o)
subprocess.check_call([B.NVCC, '-shared', '-o', os.path.join(out, 'librebvo_b200_dbg.so')] + objs + ['-lcudart'])
for o in objs:
    os.remove(o)
print('ok', out)
