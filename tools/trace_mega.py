"""Device timeline of the persistent decode kernel (build with `make -C gptq-for-llama_b200/csrc variants`; run with
GPTQ_B200_LIB=gptq-for-llama_b200/dev/libgptq_b200_trace.so).  %globaltimer per CTA at the phase boundaries of the first layers,
plus per-operation consumer counters of layer 2 (cycles in the op, cycles waiting for ring stages, stages)."""
import ctypes, os, sys, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'gptq-for-llama_b200'))
from gptq_b200 import engine, _lib
raw = ctypes.CDLL(_lib.LIB_PATH)
size = sys.argv[1] if len(sys.argv) > 1 else '7b'
dec = engine.synthetic_llama(size, max_seq=2048, use_graph=False)
dec.k_cache.normal_(0, 0.5); dec.v_cache.normal_(0, 0.5)
dec.positions.fill_(2047); dec.tokens.fill_(1)
NCTA = torch.cuda.get_device_properties(0).multi_processor_count
buf = torch.zeros(NCTA * 64, dtype=torch.int64, device='cuda')
raw.gptq_debug_set_mega_trace.argtypes = [ctypes.c_void_p]
assert raw.gptq_debug_set_mega_trace(buf.data_ptr()) == 0
for _ in range(3):
    dec.step()
torch.cuda.synchronize()
print('logits finite:', bool(torch.isfinite(dec.logits).all()), 'rms', dec.logits.float().pow(2).mean().sqrt().item())
t = buf.cpu().view(NCTA, 64).double()
t0 = t[:, 0].min()
# no barrier between A and O: O starts when A is done, and its staging waits for the records of its heads ('O x staged': team 0)
names = ['Q start', 'Q x staged', 'Q matvec done', 'Q barrier passed', 'A done', 'O x staged', 'O done', 'O barrier passed', 'G x staged', 'G done', 'D start(after barrier)', 'D done']
for l in range(1, 3):
    print(f'layer {l}: (min / median / max over CTAs, us since kernel start)')
    for k in range(12):
        c = (t[:, l * 12 + k] - t0) / 1e3
        print(f'  {names[k]:24s} {c.min().item():8.2f} {c.median().item():8.2f} {c.max().item():8.2f}')
    early = int((t[:, l * 12 + 5] < t[:, l * 12 + 4].max()).sum())
    print(f'  CTAs whose O staging ended before the last CTA finished A: {early} / {NCTA}')
    if (l + 1) * 12 < 36:  # only ids below 36 are recorded: the next layer's start is known for layer 1 alone
        print(f'  layer total {((t[:, (l + 1) * 12] - t[:, l * 12]) / 1e3).median().item():.2f} us')
print('layer 2, team 0 of every CTA (median over CTAs): cycles in op / waiting for stages / stages / busy cycles per stage')
for i, name in enumerate(['Q', 'A', 'O', 'G', 'D']):
    tot, wait, st = t[:, 48 + 3 * i], t[:, 49 + 3 * i], t[:, 50 + 3 * i]
    busy = ((tot - wait) / st.clamp(min=1)).median().item()
    print(f'  {name}: {tot.median().item():8.0f} {wait.median().item():8.0f} ({(wait / tot.clamp(min=1)).median().item():.0%}) {st.median().item():5.0f}   {busy:7.0f}')
print(f'staging cycles inside the ops, summed over all layers / 32 (team 0): O (attention merge) {t[:, 37].median().item() / 32 / 3:.0f}, D (SwiGLU) {t[:, 38].median().item() / 32 / 3:.0f}')
print(f'producer (team 0) cycles blocked on a full ring over the whole token: median {t[:, 63].median().item():.0f} ({t[:, 63].median().item() / 1.965e3:.0f} us)')
