"""GPU: on the kernel-chain path, launches_per_step() equals the number of kernels one un-graphed step() launches.

The step is built and traced in a child process: a LLaMA-65B-shaped engine run earlier in the test process (tests/test_gpu_batch_decode.py,
tests/test_gpu_large_shapes.py) left later torch.profiler sessions of that process one kernel record short, as a profiler session ahead of
the engine tests did before (tests/test_gpu_cached_attention.py test_routing)."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

TESTS = os.path.dirname(os.path.abspath(__file__))
_CHILD = """
import json, sys, time
sys.path[:0] = {paths!r}
import torch
from torch.profiler import ProfilerActivity, profile
from gptq_b200 import engine
size, bits, act, batch = {case!r}
dec = engine.synthetic_llama(size, bits=bits, groupsize=64 if size == 'tiny' else 128, act_order=act, vocab=512, seed=bits, max_seq=64, n_layers=2,
                             batch=batch, use_graph=False)
n = dec.launches_per_step()
assert n > 1, 'expected the kernel-chain path'
assert all(p is None for pm in dec.perms for p in pm.values())  # act-order layers went back to their stored form
dec.tokens.fill_(7)
dec.positions.fill_(3)
dec.step()  # warm-up: module loading and function attributes
for _ in range(3):  # a trace without any kernel record is taken again, as in gpu_util.run_kernel
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        time.sleep(0.003)
        dec.step()
        torch.cuda.synchronize()
        time.sleep(0.003)
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and not e.name.startswith(('Memcpy', 'Memset'))]
    if names:
        break
print(json.dumps([n, names]))
"""


@pytest.mark.parametrize('size,bits,act,batch', [('tiny', 4, False, 1), ('tiny', 8, False, 1), ('tiny', 3, True, 1), ('13b', 4, False, 7)])
def test_chain_launch_count(size, bits, act, batch):
    root = os.path.dirname(TESTS)
    code = _CHILD.format(paths=[root, os.path.join(root, 'gptq-for-llama_b200'), TESTS], case=(size, bits, act, batch))
    flags = ['-s'] if sys.flags.no_user_site else []
    res = subprocess.run([sys.executable, *flags, '-c', code], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-4000:]
    n, names = json.loads(res.stdout.strip().splitlines()[-1])
    if not names:
        pytest.skip('CUDA activity tracing returned no kernel events on this machine')
    assert len(names) == n, f'launches_per_step() = {n}, one step launched {len(names)}: {names}'
