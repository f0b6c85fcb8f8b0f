"""TEST / BASELINE INFRASTRUCTURE — g++ builds of the host cores: oracle/_build/librda_cpu_port.so (the port, loaded by
oracle.cpu_port and bench.py) and, through build_so, the CPU twin library of tests/ (tests/shim.py)."""
import os
import subprocess
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, 'cpu_port', 'rda_cpu_port.cpp')
SO = os.path.join(HERE, '_build', 'librda_cpu_port.so')
CSRC = os.path.join(ROOT, 'rda_planner_b200', 'csrc')
HEADERS = [os.path.join(ROOT, 'include', 'rda_b200.h'), os.path.join(HERE, 'cpu_port', 'rda_cpu_port.h')]


def build_so(srcs, so, force=False):
    """Compile the C++ sources `srcs` into the shared object `so` and return its path.  An existing `so` is kept when it
    is newer than every source, the headers and every file of rda_planner_b200/csrc, or always with
    RDA_B200_NO_BUILD=1.  A tree that cannot be written gets the build in a temporary directory instead."""
    if not force and os.path.exists(so):
        if os.environ.get('RDA_B200_NO_BUILD') == '1':
            return so
        deps = list(srcs) + HEADERS + [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
        if all(os.path.getmtime(so) >= os.path.getmtime(d) for d in deps):
            return so
    if not os.access(os.path.dirname(os.path.dirname(so)), os.W_OK):
        so = os.path.join(tempfile.mkdtemp(prefix='rda_host_'), os.path.basename(so))
    os.makedirs(os.path.dirname(so), exist_ok=True)
    subprocess.check_call(['g++', '-O3', '-std=c++17', '-fopenmp', '-shared', '-fPIC', '-o', so] + list(srcs))
    return so


def build(force=False):
    return build_so([SRC], SO, force)


if __name__ == '__main__':
    print(build(force=True))
