"""The backward pass of the quantized linears on one GPU, one JSON line:
  * kernel level, grad_in[M, K] = g[M, N] . deq(W)^T at the four LLaMA-7B linears (int4, groupsize 128), M in {2048, 8192}:
      wgmma   -- the transposed int4 GEMM on the tensor cores (csrc/qgemm_wgmma_t.cu), what ops.transpose_matmul248 routes to;
      generic -- the CUDA-core kernel, forced by passing the layer without its groupsize hint (as a stored act-order layer arrives);
      cublas  -- g @ Wdeq.T on a pre-dequantised fp16 weight: the ceiling a user reaches by spending 4x the weight memory.
    CUDA-event time per launch after warm-up, three rounds alternating the candidates in one process, median and range.  The wgmma kernel
    and cuBLAS are timed over 50 launches per round; the generic kernel over 3 (M = 2048) or 1 (M = 8192), it is that much slower.
    Rate = 2 M K N / time, also as a share of the H100 SXM data sheet's 989 TFLOP/s dense fp16 (the bound is the tensor rate).
    The outputs of the three on the timed inputs are compared in the same run.
  * module level: forward + backward of the five quantized linears of one LLaMA-7B layer (qkv, o, gate, up, down) at M = 2048 through
    QuantLinear under autograd, with the backward routed as shipped against the backward forced onto the generic kernel.
The card's name and power limit are read in the same run.  Nothing is written to disk; without a GPU the script fails."""
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'gptq-for-llama_b200'))
sys.path.insert(0, os.path.join(ROOT, 'tools'))
import quant  # noqa: E402
from gptq_b200 import ops  # noqa: E402
from microbench import rand_layer  # noqa: E402
from score_bench import gpu_identity, timed  # noqa: E402

PEAK_TFLOPS = 989.0  # H100 SXM data sheet, dense fp16, 700 W
GS = 128
SHAPES = {'qkv': (4096, 12288), 'o': (4096, 4096), 'gate/up': (4096, 11008), 'down': (11008, 4096)}  # (K, N)


def summary(ms_all, flop):
    med = statistics.median(ms_all)
    return {'ms': round(med, 4), 'ms_range': [round(min(ms_all), 4), round(max(ms_all), 4)], 'tflops': round(flop / med / 1e9, 1),
            'share_of_989': round(flop / med / 1e9 / PEAK_TFLOPS, 3)}


def kernel_level(name, K, N, M, rounds=3):
    dev = torch.device('cuda')
    w = rand_layer(K, N, 4, GS, dev)
    Wdeq = ops.dequant(*w, 4, GS)
    g = torch.randn(M, N, device=dev, generator=torch.Generator(device='cuda').manual_seed(M + N)).half()
    legs = {
        'wgmma': (lambda: ops.transpose_matmul248(g, *w, 4, 15, groupsize=GS), 50),
        'generic': (lambda: ops.transpose_matmul248(g, *w, 4, 15, groupsize=0), 3 if M <= 2048 else 1),
        'cublas': (lambda: g @ Wdeq.t(), 50),
    }
    outs = {k: fn() for k, (fn, _) in legs.items()}  # also the warm-up of every candidate at this shape
    for k in ('wgmma', 'cublas'):
        for _ in range(3):
            legs[k][0]()
    rms = outs['cublas'].float().pow(2).mean().sqrt().item()
    diff = lambda a, b: round((outs[a].float() - outs[b].float()).abs().max().item(), 6)
    times = {k: [] for k in legs}
    for _ in range(rounds):
        for k, (fn, n) in legs.items():
            times[k].append(timed(fn, n)[0])
    res = {'layer': name, 'M': M, 'K': K, 'N': N, 'bound': 'tensor', 'launches_per_round': {k: n for k, (_, n) in legs.items()}}
    res.update({k: summary(v, 2.0 * M * K * N) for k, v in times.items()})
    res['generic_over_wgmma_time'] = round(res['generic']['ms'] / res['wgmma']['ms'], 1)
    res['wgmma_over_cublas_time'] = round(res['wgmma']['ms'] / res['cublas']['ms'], 2)
    res['parity'] = {'rms_out': round(rms, 4), 'max_abs_wgmma_generic': diff('wgmma', 'generic'), 'max_abs_wgmma_cublas': diff('wgmma', 'cublas'),
                     'max_abs_generic_cublas': diff('generic', 'cublas')}
    return res


def module_level(M=2048, rounds=3):
    """Sum over the five linears of one forward + backward (input gradient only: the packed weights are frozen)."""
    dev = torch.device('cuda')
    layers = []
    for i, (K, N) in enumerate([(4096, 12288), (4096, 4096), (4096, 11008), (4096, 11008), (11008, 4096)]):
        ql = quant.QuantLinear(4, GS, K, N, False)
        ql.qweight, ql.scales, ql.qzeros, ql.g_idx = rand_layer(K, N, 4, GS, dev)
        ql = ql.to(dev)
        gen = torch.Generator(device='cuda').manual_seed(i)
        x = torch.randn(M, K, device=dev, generator=gen).half().requires_grad_(True)
        go = torch.randn(M, N, device=dev, generator=gen).half()
        layers.append((ql, x, go))
    quant.autotune_warmup_linear(torch.nn.ModuleList([q for q, _, _ in layers]))

    def step():
        for ql, x, go in layers:
            x.grad = None
            ql(x).backward(go)

    shipped = ops.transpose_matmul248
    forced = lambda *a, groupsize=0, **kw: shipped(*a, groupsize=0, **kw)  # without the hint the C entry point takes the generic kernel
    legs = {'wgmma_backward': (shipped, 10), 'generic_backward': (forced, 1)}
    times = {k: [] for k in legs}
    try:
        for k, (fn, _) in legs.items():
            ops.transpose_matmul248 = fn
            step()
        for _ in range(rounds):
            for k, (fn, n) in legs.items():
                ops.transpose_matmul248 = fn
                times[k].append(timed(step, n)[0])
    finally:
        ops.transpose_matmul248 = shipped
    res = {'M': M, 'what': 'forward + backward of qkv, o, gate, up, down (LLaMA-7B, int4 g128) through QuantLinear under autograd',
           'steps_per_round': {k: n for k, (_, n) in legs.items()}}
    for k, v in times.items():
        res[k] = {'ms': round(statistics.median(v), 3), 'ms_range': [round(min(v), 3), round(max(v), 3)]}
    res['speedup'] = round(res['generic_backward']['ms'] / res['wgmma_backward']['ms'], 1)
    return res


def main():
    assert torch.cuda.is_available(), 'backward_bench needs a CUDA device'
    torch.cuda.set_device(0)
    res = {'gpu': gpu_identity(), 'kernel': [kernel_level(name, K, N, M) for name, (K, N) in SHAPES.items() for M in (2048, 8192)]}
    res['module'] = module_level()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
