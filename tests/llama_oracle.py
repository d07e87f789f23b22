"""The CPU reference of a LlamaDecoder's arithmetic, which every engine test compares against.

The decisions it encodes, in one place:
  * fp16 rounding after each RMSNorm (O.rmsnorm_fwd), each quantized linear, RoPE, the attention output and each residual add;
  * RoPE through O.rope_inplace: at the RoPE base, or with the frequency table of a scaled rotation (llama3) when one is given;
  * attention as an fp32 softmax over the fp16 K / V rows, head_dim = hidden // n_heads, with n_kv_heads K / V heads (the decoder's):
    the fused qkv output is q | k | v of n_heads | n_kv_heads | n_kv_heads heads, and query head h reads K / V head h // (n_heads /
    n_kv_heads) (with n_kv_heads = n_heads, head h);
  * the RMSNorm epsilon, the RoPE base and the frequency table are the caller's, never the decoder's: a decoder built with the wrong ones
    would agree with itself.
The quantized linears take the reference's fp16 weight as matmul_248 materialises it, accumulated in fp32 (oracle.cref when it is built,
else O.dequant and an fp32 matmul: the same arithmetic, the C restatement is just faster at 7B shapes), or, with exact=True, the weight
dequantised exactly ((w - z) * s in fp32), fp32 accumulation, one fp16 rounding: the product the persistent kernel computes (it applies
scale and zero per group on the fp32 accumulator).

Tolerances of the block checks (tests/test_gpu_engine_fullsize.py): every QuantLinear output alone is held to 1e-3
(tests/test_gpu_modules.py, test_gpu_parity.py).  A block chains 3-5 such operations with an fp16 rounding after each (one fp16 ulp is
up to 9.8e-4 relative), hence the 1e-3-class block bounds."""
import torch

from attn_probe import resid_buffers
from gpu_util import assert_rel_close, report
from oracle import cref
from oracle import gptq_oracle as O

# LLaMA-1 (RoPE base 10000, RMSNorm epsilon 1e-6) and CodeLlama (base 1e6, epsilon 1e-5)
LLAMA1, CODELLAMA = (10000.0, 1e-6), (1e6, 1e-5)

ATTN_BLOCK_TOL = 4e-3     # qkv -> RoPE -> attention -> o_proj -> residual add
KV_ROW_TOL = 2.5e-3       # qkv -> RoPE (one QuantLinear + one rotation, each rounded to fp16)
MLP_HEAD_TOL = 5e-3       # gate/up -> SwiGLU -> down -> residual -> final norm -> lm_head
END_TO_END_TOL = 1.5e-2   # whole step from the embedding: sanity only (one-ulp differences early on re-roll every later rounding)

LINEARS = ('qkv', 'o', 'gate', 'up', 'down')

FAILURES = []


def check(out, ref, rel, what):
    """assert_rel_close, but every check of a test case is evaluated and reported (worst error / bound) before the case fails: the case
    ends with assert_no_failures()."""
    try:
        assert_rel_close(out, ref, rel=rel, what=what)
    except AssertionError as e:
        FAILURES.append(str(e))


def assert_no_failures():
    failed, FAILURES[:] = list(FAILURES), []
    assert not failed, '\n'.join(failed)


def scale_down_embedding_row(embed, tok, shift):
    """Multiply embedding row `tok` by 2^-shift in place, so that its mean square comes near the RMSNorm epsilon: only then does the
    epsilon move the first norm by more than an fp16 ulp, and a norm that used another epsilon shows in the output."""
    with torch.no_grad():
        embed[tok] *= 2.0**-shift


def _cpu(t):
    return t.detach().cpu()


class LlamaOracle:
    """The decoder's arithmetic on the CPU.  layers: the decoder's layer dicts ('qkv', 'o', 'gate', 'up', 'down' with qweight / scales /
    qzeros / g_idx / bits, as QLayerWeights; 'input_norm', 'post_norm'), on any device.  A layer is copied to the CPU, and its weights
    dequantised, the first time a block uses it, and kept; so is the fp32 lm_head (2 GB at a 128256-row vocabulary).  inv_freq: the fp32
    frequency table [head_dim / 2] of a scaled rotation (ops.rope_inv_freq), None for the unscaled one at `base`.  n_kv_heads: None for
    multi-head attention."""

    def __init__(self, layers, embed, final_norm, lm_head, n_heads, *, eps, base, inv_freq=None, n_kv_heads=None):
        self.layers, self.n_heads, self.eps, self.base, self.inv_freq = list(layers), n_heads, eps, base, inv_freq
        self.n_kv_heads = n_heads if n_kv_heads is None else n_kv_heads
        self.embed, self.final_norm, self.lm_head = _cpu(embed), _cpu(final_norm), _cpu(lm_head)
        self.hidden = self.embed.shape[1]
        self.head_dim = self.hidden // n_heads
        self._cpu_layers, self._weights, self._head = {}, {}, None

    @classmethod
    def from_decoder(cls, dec, *, eps, base, inv_freq=None):
        """The reference of a LlamaDecoder; its K / V head count is a shape and comes from the decoder."""
        return cls(dec.layers, dec.embed, dec.final_norm, dec.lm_head, dec.n_heads, eps=eps, base=base, inv_freq=inv_freq, n_kv_heads=dec.n_kv_heads)

    def _layer(self, li):
        if li not in self._cpu_layers:
            ly = self.layers[li]
            d = {k: (tuple(_cpu(t) for t in (ly[k].qweight, ly[k].scales, ly[k].qzeros, ly[k].g_idx)), ly[k].bits) for k in LINEARS}
            d['input_norm'], d['post_norm'] = _cpu(ly['input_norm']), _cpu(ly['post_norm'])
            self._cpu_layers[li] = d
        return self._cpu_layers[li]

    def _weight(self, li, name, exact):
        """[K, N]: the reference's fp16 weight, or with exact the fp32 (w - z) * s."""
        key = (li, name, exact)
        if key not in self._weights:
            (qweight, scales, qzeros, g_idx), bits = self._layer(li)[name]
            if exact:
                w = torch.from_numpy(O.unpack_rows(qweight.numpy(), bits))
                z = torch.from_numpy(O.unpack_cols(qzeros.numpy(), bits)) + 1
                g = g_idx.long()
                self._weights[key] = (w - z[g]).float() * scales[g].float()
            else:
                self._weights[key] = O.dequant(qweight, scales, qzeros, g_idx, bits)
        return self._weights[key]

    def _linear(self, li, name, x, exact=False):
        if not exact and cref.available():
            w, bits = self._layer(li)[name]
            return cref.qlinear_fwd(x, *w, bits)
        return (x.float() @ self._weight(li, name, exact).float()).half()

    def attention(self, li, x, pos, k_prefix=None, v_prefix=None, exact=False):
        """x [n, H] at positions pos .. pos + n - 1 entering layer li -> (x after the attention block [n, H], the new K rows [nkv, n, hd],
        the new V rows).  The rows attend to the cache prefix k_prefix / v_prefix [nkv, >= pos, hd] (rows 0 .. pos - 1 are read) and
        causally to each other.  exact: qkv and o_proj with the exactly dequantised weight."""
        n, nh, nkv, hd = x.shape[0], self.n_heads, self.n_kv_heads, self.head_dim
        qkv = self._linear(li, 'qkv', O.rmsnorm_fwd(x, self._layer(li)['input_norm'], self.eps), exact).view(1, n, nh + 2 * nkv, hd).clone()
        O.rope_inplace(qkv[:, :, None, :nh + nkv], torch.arange(pos, pos + n)[None, :], base=self.base, inv_freq=self.inv_freq)
        q, k, v = (t.transpose(0, 1) for t in qkv[0].split([nh, nkv, nkv], 1))  # [heads, n, hd]
        K = torch.cat([k_prefix[:, :pos], k], 1) if pos else k
        V = torch.cat([v_prefix[:, :pos], v], 1) if pos else v
        qg = q.float().reshape(nkv, nh // nkv, n, hd)  # query head kvh * g + j
        s = (qg @ K.float()[:, None].transpose(-1, -2)) * hd**-0.5  # [nkv, g, n, pos + n]
        s = s.masked_fill(torch.ones(n, pos + n, dtype=torch.bool).triu(pos + 1), float('-inf'))
        att = (torch.softmax(s, -1) @ V.float()[:, None]).reshape(nh, n, hd).half().transpose(0, 1).reshape(n, self.hidden)
        return x + self._linear(li, 'o', att, exact), k, v

    def mlp(self, li, x):
        """x [n, H] after the attention block of layer li -> x after the MLP block."""
        xn = O.rmsnorm_fwd(x, self._layer(li)['post_norm'], self.eps)
        (gate, bits), (up, _) = self._layer(li)['gate'], self._layer(li)['up']
        if cref.available():
            hmid = cref.fused_mlp_fwd(xn, gate, up, bits)
        else:
            a1, a2 = xn.float() @ self._weight(li, 'gate', False).float(), xn.float() @ self._weight(li, 'up', False).float()
            hmid = (a1 * torch.sigmoid(a1) * a2).half()
        return x + self._linear(li, 'down', hmid)

    def head(self, x):
        """x [n, H] after the last layer -> fp16 logits [n, vocab]."""
        if self._head is None:
            self._head = self.lm_head.float()
        return (O.rmsnorm_fwd(x, self.final_norm, self.eps).float() @ self._head.t()).half()

    def logits(self, tokens):
        """The fp16 logits at every position of one token list, from position 0 on an empty cache."""
        x = self.embed[torch.tensor(tokens)]
        for li in range(len(self.layers)):
            x = self.mlp(li, self.attention(li, x, 0)[0])
        return self.head(x)


def check_last_layer_blocks(dec, oracle, tok, pos, kc, vc, what, k_row_vs_reference=True):
    """Run one step of the persistent kernel `dec` and check its last layer block by block from the kernel's own intermediate values:
    the attention block from x entering the layer (row 0 of the residual ping-pong, attn_probe.resid_buffers), the MLP block and the head
    from x after attention.  A one-ulp difference early in a decoder re-rolls every later rounding, so only a check fed with the kernel's
    own input to the block keeps a 1e-3-class bound meaningful.  Layer li of `oracle` is layer li of dec; kc / vc are dec's cache before
    the step, on the CPU.

    The attention block is checked against the exact linears, because a softmax over 2048 keys amplifies one-ulp changes in q: at
    context 2047 of the 7B case the reference's per-weight fp16 rounding of the qkv weights alone moves the block by twice ATTN_BLOCK_TOL.
    Each QuantLinear is held to the reference's rounding within 1e-3 by tests/test_gpu_parity.py and tests/test_gpu_modules.py, and the
    appended K / V rows are held to it here (the K row only with k_row_vs_reference) as well as to the exact linears.  Returns the
    logits."""
    dec.tokens.fill_(tok)
    dec.positions.fill_(pos)
    dec.step()
    torch.cuda.synchronize()
    x_in, x_attn = (r[0].cpu() for r in resid_buffers(dec))
    li = len(dec.layers) - 1
    if li == 0:  # the input of layer 0 is the embedding row, exactly
        assert torch.equal(x_in, dec.embed[tok].cpu()), f'{what}: residual entering layer 0 is not the embedding row'
    _, k_new, v_new = oracle.attention(li, x_in[None, :], pos, kc[li, 0], vc[li, 0])
    ref_attn, k_ex, v_ex = oracle.attention(li, x_in[None, :], pos, kc[li, 0], vc[li, 0], exact=True)
    check(x_attn, ref_attn[0], rel=ATTN_BLOCK_TOL, what=f'{what}: attention block of layer {li}')
    if k_row_vs_reference:
        check(dec.k_cache[li, 0, :, pos], k_new[:, 0], rel=KV_ROW_TOL, what=f'{what}: appended K row, layer {li}')
    check(dec.v_cache[li, 0, :, pos], v_new[:, 0], rel=KV_ROW_TOL, what=f'{what}: appended V row, layer {li}')
    check(dec.k_cache[li, 0, :, pos], k_ex[:, 0], rel=KV_ROW_TOL, what=f'{what}: appended K row vs Exact, layer {li}')
    check(dec.v_cache[li, 0, :, pos], v_ex[:, 0], rel=KV_ROW_TOL, what=f'{what}: appended V row vs Exact, layer {li}')
    ref_logits = oracle.head(oracle.mlp(li, x_attn[None, :]))[0]
    check(dec.logits[0], ref_logits, rel=MLP_HEAD_TOL, what=f'{what}: MLP block of layer {li} + lm_head')
    assert int(dec.next_tokens[0]) == int(dec.logits[0].float().argmax())
    return dec.logits[0].float().cpu()


def check_scores(lps, seqs, oracle, what):
    """score() output lps of the lists seqs against float64 log-softmaxes of the oracle's fp16 logits.  The prefill and decode tests hold
    the logits to 2e-2 * max|ref logits| of the oracle; logsumexp is 1-Lipschitz in the max-norm, so the target logit and the logsumexp
    move by at most that each: 2 x 2e-2 x max|ref logits| per element.  Returns the worst |err| / bound."""
    worst = 0.0
    for s, lp in zip(seqs, lps):
        logits = oracle.logits(s)[:-1].double()
        ref = torch.log_softmax(logits, -1).gather(1, torch.tensor(s[1:])[:, None])[:, 0]
        bound = 2 * 2e-2 * logits.abs().amax(-1)
        ratio = ((lp.cpu().double() - ref).abs() / bound).max().item()
        report(ratio, f'{what} n={len(s)}')
        worst = max(worst, ratio)
    return worst


def check_blocks_on_random_cache(dec2, positions, what, *, eps, base, inv_freq=None, cache_seed, k_row_vs_reference=True, small_embedding=False,
                                 end_to_end=False):
    """The two-layer persistent-kernel decoder dec2 and its one-layer twin, built from dec2's own settings (epsilon, RoPE base, frequency
    table, K / V heads, max_seq), on one random cache (N(0, 0.25) rows drawn from cache_seed): one step at each position (token 17 i + 3),
    checked block by block (check_last_layer_blocks) against the reference built with the caller's eps, base and inv_freq.  Every position
    starts from the same cache: a step rewrites row pos, which a later, shorter context would read.
      small_embedding: the first position's token has its embedding row scaled by 2^-8 (mean square about 4e-6, near the epsilon), so that
        the one-layer checks see the epsilon;
      k_row_vs_reference=False: the appended K rows are held to the exact linears only;
      end_to_end: also the two-layer logits against the reference run from the embedding (END_TO_END_TOL).
    Returns the reference."""
    from gptq_b200 import engine
    if small_embedding:
        scale_down_embedding_row(dec2.embed, 3, 8)  # the token of the first position (17 * 0 + 3)
    dec1 = engine.LlamaDecoder(dec2.layers[:1], dec2.embed, dec2.final_norm, dec2.lm_head, dec2.n_heads, rms_eps=dec2.model.rms_eps,
                               rope_base=dec2.model.rope_base, max_seq=dec2.max_seq, n_kv_heads=dec2.n_kv_heads, rope_scaling=dec2.rope_inv_freq)
    assert dec1.launches_per_step() == 1 and dec2.launches_per_step() == 1, 'the persistent kernel must be the path under test'
    gen = torch.Generator(device=dec2.dev).manual_seed(cache_seed)
    dec2.k_cache.copy_((torch.randn(dec2.k_cache.shape, device=dec2.dev, generator=gen) * 0.5).half())
    dec2.v_cache.copy_((torch.randn(dec2.v_cache.shape, device=dec2.dev, generator=gen) * 0.5).half())
    k0, v0 = dec2.k_cache.clone(), dec2.v_cache.clone()
    kc, vc = k0.cpu(), v0.cpu()
    oracle = LlamaOracle.from_decoder(dec2, eps=eps, base=base, inv_freq=inv_freq)
    for i, pos in enumerate(positions):
        tok = (17 * i + 3) % dec2.vocab
        at = f'{what} pos={pos}'
        for dec in (dec1, dec2):
            dec.k_cache.copy_(k0[:len(dec.layers)])
            dec.v_cache.copy_(v0[:len(dec.layers)])
        check_last_layer_blocks(dec1, oracle, tok, pos, kc, vc, at + ' (1 layer)', k_row_vs_reference)
        logits2 = check_last_layer_blocks(dec2, oracle, tok, pos, kc, vc, at + ' (2 layers)', k_row_vs_reference)
        if end_to_end:
            x = dec2.embed[tok].cpu()[None, :].clone()
            for li in range(2):
                x = oracle.mlp(li, oracle.attention(li, x, pos, kc[li, 0], vc[li, 0])[0])
            check(logits2, oracle.head(x)[0], rel=END_TO_END_TOL, what=at + ': logits after 2 layers, end to end')
    assert_no_failures()
    return oracle


def check_steps(dec, oracle, seqs, label, rel=2e-2, checked=None):
    """Decode the token lists seqs, one per sequence of dec, in lock-step from position 0, each sequence at its own position: a finished
    sequence re-steps its last token at its last position, which rewrites the same row.  At every step in `checked` (default: all), each
    sequence's logits against the reference logits of that sequence alone (oracle.logits) within rel, and next_tokens the argmax.
    label(step, sequence, pos) names each check."""
    refs = [oracle.logits(s) for s in seqs]
    for k in range(max(map(len, seqs))):
        pos = [min(k, len(s) - 1) for s in seqs]
        dec.set_input([s[p] for s, p in zip(seqs, pos)], pos)
        dec.step()
        if checked is None or k in checked:
            torch.cuda.synchronize()
            for b, p in enumerate(pos):
                assert_rel_close(dec.logits[b], refs[b][p], rel=rel, what=label(k, b, p))
                assert int(dec.next_tokens[b]) == int(dec.logits[b].float().argmax()), label(k, b, p)


def step_all(dec, toks, start):
    """Decode steps of toks at positions start, start + 1, ..."""
    for i, t in enumerate(toks):
        dec.set_input(t, start + i)
        dec.step()
    torch.cuda.synchronize()


def check_extend_against_stepping(dec, toks, cached, what, prefilled=0, fill='prefill'):
    """From an empty cache: toks[:prefilled] filled by prefill() (or by extend() with fill='extend'), the positions up to `cached` stepped,
    then extend() of the next ones up to the last token and one step of the last; against stepping every token from `cached` on.  The logits
    and the extended cache rows [cached, n - 1) are held to the run-to-run spread of DESIGN.md section 2 (max 1.5e-2, rms 3e-3 of the rms);
    rows both runs step alike stay out of that window, where they would only dilute the rms bound.  Without a prefix the stepping run goes on
    from the first run's rows before `cached`.  With one, the stepping run fills and steps the prefix again, and the rows [prefilled, n) are
    held to the same bounds as well ('K rows' / 'V rows'; the extended rows alone are then 'extended K rows' / 'extended V rows')."""
    n = len(toks)
    windows = [('', cached, n - 1)] if not prefilled else [('', prefilled, n), ('extended ', cached, n - 1)]
    runs = []
    for extend in (True, False):
        if extend or prefilled:
            dec.reset()
            dec.k_cache.zero_()
            dec.v_cache.zero_()
            if prefilled and fill == 'prefill':
                assert dec.prefill(toks[:prefilled + 1]) == prefilled
            elif prefilled:
                assert dec.extend([toks[:prefilled]]) == [prefilled]
            step_all(dec, toks[prefilled:cached], prefilled)
        if extend:
            assert dec.extend([toks[cached:n - 1]]) == [n - 1]
            step_all(dec, toks[n - 1:], n - 1)
        else:
            step_all(dec, toks[cached:], cached)
        runs.append({'logits': dec.logits[0].float().clone()})
        for prefix, lo, hi in windows:
            runs[-1][f'{prefix}K rows'] = dec.k_cache[:, 0, :, lo:hi].float().clone()
            runs[-1][f'{prefix}V rows'] = dec.v_cache[:, 0, :, lo:hi].float().clone()
    got, ref = runs
    for name, r in ref.items():
        rms = r.pow(2).mean().sqrt().item()
        d = (got[name] - r).abs()
        print(f'  {what} {name}: max |diff| / rms = {d.max().item() / rms:.3g}, rms diff / rms = {d.pow(2).mean().sqrt().item() / rms:.3g}')
        assert d.max().item() <= 1.5e-2 * rms and d.pow(2).mean().sqrt().item() <= 3e-3 * rms, f'{what}: {name}'
