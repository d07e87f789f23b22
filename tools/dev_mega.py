"""Development check of the persistent decode kernel: tiny256 decode vs the oracle, printing errors instead of asserting.
GPTQ_B200_LIB=<so> python tools/dev_mega.py [bits] [act]"""
import os, sys, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'gptq-for-llama_b200'), os.path.join(ROOT, 'tests')):
    sys.path.insert(0, p)
from gptq_b200 import engine
from llama_oracle import LlamaOracle
bits = int(sys.argv[1]) if len(sys.argv) > 1 else 4
act = len(sys.argv) > 2 and sys.argv[2] == 'act'
dec = engine.synthetic_llama('tiny256', bits=bits, groupsize=64, act_order=act, vocab=512, seed=bits, max_seq=600, use_graph=False)
print('lib', os.environ.get('GPTQ_B200_LIB', 'default'), 'launches/step', dec.launches_per_step(), flush=True)
toks = torch.randint(0, 512, (40, ), generator=torch.Generator().manual_seed(0)).tolist()
ref = LlamaOracle.from_decoder(dec, eps=1e-6, base=10000.0).logits(toks)
for pos, tok in enumerate(toks):
    dec.tokens.fill_(tok); dec.positions.fill_(pos); dec.step(); torch.cuda.synchronize()
    out = dec.logits[0].float().cpu(); r = ref[pos].float()
    rms = r.pow(2).mean().sqrt().item()
    if pos < 6 or pos in (31, 32, 33, 39):
        print(f'pos {pos:3d}: max|err| {(out - r).abs().max().item():.3e}  rms(ref) {rms:.3e}  rel-to-rms {(out - r).abs().max().item() / rms:.2e}  finite {bool(torch.isfinite(out).all())}', flush=True)
