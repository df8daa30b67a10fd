"""Guards on the machine code ptxas makes of the three fused attention kernels in the built library (no GPU needed).

Each kernel keeps its running softmax state, the score fragment, P as the register A operand and the O accumulators in registers at
one 384-thread CTA per SM: attn_kernel and attn_pair_kernel near the 168-register limit, attn_wide_kernel with two 64-column O
accumulators that live inside the wgmma across all key blocks.  A stack frame or a local-memory access would put spills between the
MMAs of every key block, and the wgmma register operands must not be spilled at all.  The MMA shapes pin the tiling: 64 x 64 x 16 for
S = Q K^T and O += P V, plus 64 x 32 x 16 for the 32-wide V^T halves of a head pair."""
import collections
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, 'diff-sampler_b200', 'libdiffsampler_b200.so')
KERNEL = re.compile(r'_ZN3dsb\d+(attn_\w*kernel)ENS_16AttnKernelParamsE')
MMA_SHAPES = {'attn_kernel': {'64x64x16'}, 'attn_pair_kernel': {'64x64x16', '64x32x16'}, 'attn_wide_kernel': {'64x64x16'}}
KERNELS = sorted(MMA_SHAPES)


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
    """kernel name -> its SASS instruction lines."""
    out = subprocess.run([tool, '-sass', LIB], capture_output=True, text=True, check=True).stdout
    funcs = collections.defaultdict(list)
    cur = None
    for line in out.splitlines():
        if 'Function :' in line:
            m = KERNEL.search(line)
            cur = m.group(1) if m else None
        elif cur is not None and re.match(r'\s*/\*[0-9a-f]{4,}\*/', line):
            funcs[cur].append(line.split('*/', 1)[1].split('/*', 1)[0].strip())
    return funcs


@pytest.fixture(scope='module')
def stacks(tool):
    """kernel name -> STACK bytes of -res-usage."""
    out = subprocess.run([tool, '-res-usage', LIB], capture_output=True, text=True, check=True).stdout
    lines, res = out.splitlines(), {}
    for k, line in enumerate(lines):
        m = KERNEL.search(line)
        if m and 'Function' in line:
            res[m.group(1)] = int(re.search(r'STACK:(\d+)', lines[k + 1]).group(1))
    return res


def test_every_attention_kernel_is_compiled(sass, stacks):
    assert sorted(sass) == KERNELS and sorted(stacks) == KERNELS


@pytest.mark.parametrize('kernel', KERNELS)
def test_no_stack_frame(stacks, kernel):
    assert stacks[kernel] == 0, stacks


@pytest.mark.parametrize('kernel', KERNELS)
def test_no_local_memory(sass, kernel):
    local = [i for i in sass[kernel] if re.search(r'\b(STL|LDL)\b', i)]
    assert not local, f'{len(local)} local-memory accesses in {kernel}, first: {local[0]}'


@pytest.mark.parametrize('kernel', KERNELS)
def test_mma_shapes(sass, kernel):
    shapes = collections.Counter(m.group(1) for i in sass[kernel] for m in [re.search(r'\bHGMMA\.(\d+x\d+x\d+)', i)] if m)
    assert set(shapes) == MMA_SHAPES[kernel], dict(shapes)
