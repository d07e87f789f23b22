"""BASELINE.json config 3: LLaMA-7B int4 g128 prefill, batch 32 x seq 2048 (M = 65536), the quantized linears of one decoder
layer on the wgmma GEMM path (qkv, o, fused gate/up + SwiGLU, down), CUDA-event timed; x 32 layers = 0.849 PFLOP per forward."""
import json, os, sys, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'gptq-for-llama_b200'))
from gptq_b200 import ops
sys.path.insert(0, os.path.join(ROOT, 'tools'))
from microbench import rand_layer
dev = torch.device('cuda:0')
M, H, I = 65536, 4096, 11008
qkv, o, gate, up, down = rand_layer(H, 3 * H, 4, 128, dev), rand_layer(H, H, 4, 128, dev), rand_layer(H, I, 4, 128, dev), rand_layer(H, I, 4, 128, dev), rand_layer(I, H, 4, 128, dev)
x = torch.randn(M, H, device=dev).half()

def layer():
    a = ops.matmul248(x, *qkv, 4, None, groupsize=128)
    b = ops.matmul248(x, *o, 4, None, groupsize=128)
    h = ops.fused_mlp(x, gate, up, 4, 128)
    d = ops.matmul248(h, *down, 4, None, groupsize=128)
    return a, b, d

for _ in range(2): layer()
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(3): layer()
e1.record(); torch.cuda.synchronize()
t = e0.elapsed_time(e1) / 3 * 1e-3
flops = 2 * M * (H * 3 * H + H * H + 2 * H * I + I * H)
peak = 989.0  # TFLOP/s dense fp16, H100 SXM data sheet (700 W)
print(json.dumps({'workload': 'LLaMA-7B int4 g128 prefill batch 32 x seq 2048 (M=65536): quantized linears of one layer', 'ms_per_layer': t * 1e3,
                  'tflops': flops / t / 1e12, 'frac_of_datasheet': flops / t / 1e12 / peak, 'tokens_per_s_linears_only_32_layers': M / (t * 32)}))
