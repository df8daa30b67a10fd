"""Guards on the machine code ptxas makes of every gemm_tc_kernel<BN> in the built library (no GPU needed).

The consumer K loop issues each ring stage as one wgmma group and waits until only that group is in flight before it releases the
stage before.  That wait keeps one stage of MMAs running only if ptxas closes each group on its last MMA.  When the commit sits
after a branch merge, ptxas closes every MMA of the stage as a group of its own and carries the commit on an extra empty MMA with
destination RZ; the wait then drains every real MMA and the producer loses one stage of lookahead, with identical results.  These
tests catch that, and any stack frame or local-memory traffic, which the consumer warpgroups would pay serially with the MMAs."""
import collections
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, 'diff-sampler_b200', 'libdiffsampler_b200.so')
KERNEL = re.compile(r'_ZN3dsb14gemm_tc_kernelILi(\d+)EEEvNS_16GemmKernelParamsE')
BNS = list(range(16, 257, 16))


@pytest.fixture(scope='module')
def tool():
    if not os.path.exists(LIB):
        pytest.skip('library not built')
    exe = shutil.which('cuobjdump') or os.path.join(os.environ.get('CUDA_HOME', '/usr/local/cuda'), 'bin', 'cuobjdump')
    if not os.path.exists(exe):
        pytest.skip('cuobjdump not found')
    return exe


@pytest.fixture(scope='module')
def sass(tool):
    """BN -> SASS instruction lines of gemm_tc_kernel<BN>."""
    out = subprocess.run([tool, '-sass', LIB], capture_output=True, text=True, check=True).stdout
    funcs = collections.defaultdict(list)
    cur = None
    for line in out.splitlines():
        if 'Function :' in line:
            m = KERNEL.search(line)
            cur = int(m.group(1)) if m else None
        elif cur is not None and re.match(r'\s*/\*[0-9a-f]{4,}\*/', line):
            funcs[cur].append(line.split('*/', 1)[1].split('/*', 1)[0].strip())
    return funcs


def test_every_tile_width_is_compiled(sass):
    assert sorted(sass) == BNS


@pytest.mark.parametrize('bn', BNS)
def test_mma_groups_close_on_their_last_mma(sass, bn):
    code = sass[bn]
    mmas = [i for i in code if re.search(r'\b[HQ]GMMA\.', i)]
    assert mmas, 'no wgmma in the kernel'
    carriers = [i for i in mmas if re.search(r'GMMA\.\S+\s+RZ,', i)]
    assert not carriers, f'empty MMA carrying a commit: {carriers[0]}'
    # Between two waits lies one group (one ring stage): exactly one MMA closes it, and it is the last one.
    group, groups = [], []
    for ins in code:
        if 'WARPGROUP.DEPBAR' in ins:
            if group:
                groups.append(group)
            group = []
        elif re.search(r'\b[HQ]GMMA\.', ins):
            group.append('gsb0' in ins)
    assert not group, 'MMAs after the last wait'
    for g in groups:
        assert g[-1] and not any(g[:-1]), f'group of {len(g)} MMAs closed at {[k for k, c in enumerate(g) if c]}'


@pytest.mark.parametrize('bn', BNS)
def test_no_local_memory(sass, bn):
    local = [i for i in sass[bn] if re.search(r'\b(STL|LDL)\b', i)]
    assert not local, f'{len(local)} local-memory accesses, first: {local[0]}'


def test_no_stack_frame(tool):
    out = subprocess.run([tool, '-res-usage', LIB], capture_output=True, text=True, check=True).stdout
    stacks = {}
    lines = out.splitlines()
    for k, line in enumerate(lines):
        m = KERNEL.search(line)
        if m and 'Function' in line:
            stacks[int(m.group(1))] = int(re.search(r'STACK:(\d+)', lines[k + 1]).group(1))
    assert sorted(stacks) == BNS
    assert all(s == 0 for s in stacks.values()), stacks
