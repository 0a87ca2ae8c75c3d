"""Build libpvraft_b200.so in-tree with nvcc for sm_90a (H100), ahead of time: the library sits next to the
package, so a tree that was built once imports and runs without nvcc.  `python -m pvraft_b200.build [--force]`."""
import os
import shlex
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIB = os.path.join(HERE, 'libpvraft_b200.so')
SOURCES = ['capi.cu', 'clusters.cu', 'flow_metrics.cu', 'corr_gemm.cu', 'corr_lookup.cu', 'fixed_point.cu', 'corr_topk.cu', 'edge_plan.cu', 'flow_consistency.cu', 'flow_propagate.cu', 'grid_index.cu', 'knn.cu', 'knn_branch.cu', 'laplacian.cu', 'pointmlp.cu', 'rigid_motion.cu', 'object_boxes.cu', 'rigid_refine.cu', 'self_supervised.cu', 'setconv_edge.cu', 'tc_linear.cu', 'tc_wgrad.cu', 'tracks.cu', 'train.cu', 'update_chain.cu']
NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '-std=c++17',
              '-Xcompiler', '-fPIC', '-Xcompiler', '-fvisibility=hidden', '--expt-relaxed-constexpr']


def _nvcc():
    for cand in (os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc', 'nvcc'):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return 'nvcc'


def stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, '..', 'include', 'pvraft_b200.h'),
                                                                os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    """Compile every CUDA source for sm_90a and link the C-ABI shared library.  Returns its path."""
    if not force and not stale():
        return LIB
    nvcc = _nvcc()
    objs = []
    procs = []
    os.makedirs(os.path.join(HERE, 'build'), exist_ok=True)
    for src in SOURCES:
        obj = os.path.join(HERE, 'build', src.replace('.cu', '.o'))
        cmd = [nvcc] + NVCC_FLAGS + shlex.split(os.environ.get('PVRAFT_NVCC_FLAGS', '')) + (['-Xptxas', '-v'] if verbose else []) + \
            ['-c', os.path.join(CSRC, src), '-o', obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    for src, p in procs:
        out, _ = p.communicate()
        if verbose and out:
            print(out)
        if p.returncode != 0:
            raise RuntimeError(f'nvcc failed on {src}:\n{out}')
    cmd = [nvcc, '-shared', '-o', LIB] + objs + ['-gencode', 'arch=compute_90a,code=sm_90a']
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError('link failed:\n' + r.stdout)
    return LIB


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
