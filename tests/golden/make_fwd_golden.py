"""Generate tests/golden/fwd_ref_triton.npz: OUTPUTS OF THE REFERENCE'S OWN TRITON KERNELS, run unmodified on a GPU.

The reference (qwopqwop200/GPTQ-for-LLaMa, triton branch @ e985b70) has no CPU forward and holds no test vectors, so the
forward oracle (oracle/gptq_oracle.py) is pinned here against what the reference computes on the GPU:
    matmul248 / matmul_248_kernel          quant/quant_linear.py:263-269, :72-137   (+ bias add of QuantLinear.forward, :376)
    QuantLlamaMLP.triton_llama_mlp         quant/fused_mlp.py:206-218, :84-168
    triton_rotate_half_                    quant/fused_attn.py:61-93
    TritonLlamaRMSNorm.forward             quant/triton_norm.py:50-67
Run on a GPU (the reference sources are copied, unmodified, into the git-ignored baseline/_ref by
tools/refshim/install_ref.sh; tools/refshim/triton_compat.py adapts Triton 3.x / torch 2.11 names without touching them):

    python tests/golden/make_fwd_golden.py OUT.npz

Inputs are NOT stored: the tests regenerate them from the seeds below (torch CPU generators are platform independent) and from
the committed pack_*.npz fixtures.  While it runs, the script also compares this repo's CUDA path with the reference outputs.
"""
import glob
import os
import sys
import zlib

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))

# ---- case list (shared with the tests) -------------------------------------------------------------------------------
PACK_M = (1, 5, 16, 40)
RANDOM_CASES = [  # (name, K, N, bits, groupsize, act_order, seed, Ms)
    ('r4_512x768_g128', 512, 768, 4, 128, False, 1, (1, 8, 33)),
    ('r4_1024x256_g64_act', 1024, 256, 4, 64, True, 2, (1, 17)),
    ('r8_512x256_g128', 512, 256, 8, 128, False, 3, (1, 16)),
    ('r2_512x256_g64_act', 512, 256, 2, 64, True, 4, (2, 16)),
    ('r4_4096x512_g128', 4096, 512, 4, 128, False, 5, (1, 4)),
]
MLP_CASES = [('mlp4_512x768_g128', 512, 768, 4, 128, 6, (1, 16))]  # (name, K, N, bits, groupsize, seed, Ms)
ROPE_CASE = dict(shape=(2, 3, 3, 4, 128), positions=[[0, 5, 900], [2047, 17, 1]], seed=7)
NORM_CASES = [('norm_4x4096', 4, 4096, 8), ('norm_2x5120', 2, 5120, 9)]  # (name, M, N, seed)


def name_seed(name):
    return zlib.crc32(name.encode()) % 997  # stable across processes (hash() is not)


def x_for(seed, M, K):
    return torch.randn(M, K, generator=torch.Generator().manual_seed(1000 + seed)).half()


def rope_input():
    g = torch.Generator().manual_seed(ROPE_CASE['seed'])
    return torch.randn(*ROPE_CASE['shape'], generator=g).half(), torch.tensor(ROPE_CASE['positions'], dtype=torch.int64)


def norm_input(M, N, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(M, N, generator=g).half(), (torch.rand(N, generator=g) + 0.5).half()


def pack_fixtures():
    out = {}
    for f in sorted(glob.glob(os.path.join(HERE, 'pack_*.npz'))):
        out[os.path.basename(f)[5:-4]] = dict(np.load(f))
    return out


def main(out_path):
    sys.dont_write_bytecode = True
    for p in (ROOT, os.path.join(ROOT, 'tools', 'refshim')):
        sys.path.insert(0, p)
    import triton_compat  # noqa: F401  (before the reference is imported)
    sys.path.insert(0, os.path.join(ROOT, 'baseline', '_ref'))
    import quant as R  # the reference package
    from quant.quant_linear import matmul248 as ref_matmul248
    from quant.fused_attn import triton_rotate_half_ as ref_rope
    from oracle import gptq_oracle as O
    sys.path.insert(0, os.path.join(ROOT, 'gptq-for-llama_b200'))
    sys.modules.pop('quant', None)  # this repo's drop-in package has the same name: keep the reference under R only
    for k in [k for k in sys.modules if k.startswith('quant.')]:
        sys.modules.pop(k)
    sys.path.remove(os.path.join(ROOT, 'baseline', '_ref'))
    from gptq_b200 import ops

    dev = torch.device('cuda:0')
    out, worst = {}, {}

    def rel(a, b):
        a, b = a.float().cpu(), b.float().cpu()
        rms = b.pow(2).mean().sqrt()
        return ((a - b).abs() / torch.maximum(b.abs(), rms)).max().item()

    def note(kind, r_ours, r_oracle):
        worst[kind] = (max(worst.get(kind, (0, 0))[0], r_ours), max(worst.get(kind, (0, 0))[1], r_oracle))

    # matmul248 on the reference's own pack() fixtures
    for name, fx in pack_fixtures().items():
        bits, K, N = int(fx['bits']), int(fx['K']), int(fx['N'])
        qw, qz, sc, gi = (torch.from_numpy(fx[k]) for k in ('qweight', 'qzeros', 'scales_h', 'g_idx'))
        bias = torch.from_numpy(fx['bias_h']) if 'bias_h' in fx else None
        for M in PACK_M:
            x = x_for(name_seed(name), M, K)
            y = ref_matmul248(x.to(dev), qw.to(dev), sc.to(dev), qz.to(dev), gi.to(dev), bits, 2**bits - 1)
            if bias is not None:
                y = y + bias.to(dev)  # QuantLinear.forward, quant_linear.py:376
            out[f'pack/{name}/M{M}'] = y.cpu().numpy()
            ours = ops.matmul248(x.to(dev), qw.to(dev), sc.to(dev), qz.to(dev), gi.to(dev), bits, 2**bits - 1)  # no groupsize hint: act-order fixtures
            if bias is not None:
                ours = ours + bias.to(dev)
            note('matmul248(pack fixtures)', rel(ours, y), rel(O.qlinear_fwd(x, qw, sc, qz, gi, bits, bias), y))
    # matmul248 on seeded random packed layers
    for name, K, N, bits, gs, act, seed, Ms in RANDOM_CASES:
        qw, sc, qz, gi, _ = O.random_packed(K, N, bits, gs, seed=seed, act_order=act)
        for M in Ms:
            x = x_for(seed, M, K)
            y = ref_matmul248(x.to(dev), qw.to(dev), sc.to(dev), qz.to(dev), gi.to(dev), bits, 2**bits - 1)
            out[f'random/{name}/M{M}'] = y.cpu().numpy()
            ours = ops.matmul248(x.to(dev), qw.to(dev), sc.to(dev), qz.to(dev), gi.to(dev), bits, 2**bits - 1, groupsize=0 if act else gs)
            note('matmul248(random layers)', rel(ours, y), rel(O.qlinear_fwd(x, qw, sc, qz, gi, bits), y))
    # fused SwiGLU MLP kernel through the reference module (its buffers are the two layers' tensors)
    for name, K, N, bits, gs, seed, Ms in MLP_CASES:
        gate = O.random_packed(K, N, bits, gs, seed=seed)[:4]
        up = O.random_packed(K, N, bits, gs, seed=seed + 100)[:4]

        def ref_layer(t):
            m = R.QuantLinear(bits, gs, K, N, False)
            m.qweight, m.scales, m.qzeros, m.g_idx = t[0].clone(), t[1].clone(), t[2].clone(), t[3].clone()
            return m

        mlp = R.QuantLlamaMLP(ref_layer(gate), R.QuantLinear(bits, gs, N, K, False), ref_layer(up)).to(dev)
        for M in Ms:
            x = x_for(seed, M, K)
            y = mlp.triton_llama_mlp(x.to(dev))
            out[f'mlp/{name}/M{M}'] = y.cpu().numpy()
            ours = ops.fused_mlp(x.to(dev), tuple(t.to(dev) for t in gate), tuple(t.to(dev) for t in up), bits, gs)
            note('fused_mlp', rel(ours, y), rel(O.fused_mlp_fwd(x, gate, up, bits), y))
    # RoPE
    qk, pos = rope_input()
    y = qk.clone().to(dev)
    ref_rope(y[:, :, :2], pos.to(dev))
    out['rope/out'] = y.cpu().numpy()
    ours = qk.clone().to(dev)
    ops.rotate_half_(ours[:, :, :2], pos.to(dev))
    orc = qk.clone()
    O.rope_inplace(orc[:, :, :2], pos)
    note('rotate_half', rel(ours, y), rel(orc, y))
    # RMSNorm
    for name, M, N, seed in NORM_CASES:
        x, w = norm_input(M, N, seed)
        y = R.TritonLlamaRMSNorm(w.to(dev), 1e-6)(x.to(dev))
        out[f'norm/{name}'] = y.cpu().numpy()
        note('rmsnorm', rel(ops.rmsnorm(x.to(dev), w.to(dev), 1e-6), y), rel(O.rmsnorm_fwd(x, w, 1e-6), y))
    np.savez_compressed(out_path, **out)
    print(f'wrote {len(out)} reference outputs to {out_path} ({os.path.getsize(out_path)} bytes)')
    print('worst |err| / max(|ref|, rms(ref)) against the reference Triton outputs:   this repo (CUDA)   oracle (CPU)')
    for k, (a, b) in worst.items():
        print(f'  {k:28s} {a:.3e}   {b:.3e}')


if __name__ == '__main__':
    main(sys.argv[1])
