"""GPU: on the kernel-chain path, launches_per_step() equals the number of kernels one un-graphed step() launches."""
import time

import pytest
import torch

pytestmark = pytest.mark.gpu


def _kernels_of(fn):
    """Number of kernel records that fn() produces under torch.profiler.  A trace without any kernel record is taken again (up to three
    times, as in gpu_util.run_kernel); a machine whose tracing returns no CUDA events at all skips the test."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            time.sleep(0.003)
            fn()
            torch.cuda.synchronize()
            time.sleep(0.003)
        names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and not e.name.startswith(('Memcpy', 'Memset'))]
        if names:
            return names
    pytest.skip('CUDA activity tracing returned no kernel events on this machine')


@pytest.mark.parametrize('size,bits,act,batch', [('tiny', 4, False, 1), ('tiny', 8, False, 1), ('tiny', 3, True, 1), ('13b', 4, False, 7)])
def test_chain_launch_count(size, bits, act, batch):
    from gptq_b200 import engine
    dec = engine.synthetic_llama(size, bits=bits, groupsize=64 if size == 'tiny' else 128, act_order=act, vocab=512, seed=bits, max_seq=64, n_layers=2,
                                 batch=batch, use_graph=False)
    n = dec.launches_per_step()
    assert n > 1, 'expected the kernel-chain path'
    assert all(p is None for pm in dec.perms for p in pm.values())  # act-order layers went back to their stored form
    dec.tokens.fill_(7)
    dec.positions.fill_(3)
    dec.step()  # warm-up: module loading and function attributes
    names = _kernels_of(dec.step)
    assert len(names) == n, f'launches_per_step() = {n}, one step launched {len(names)}: {names}'
