"""The CPU reference of a LlamaDecoder's arithmetic, which every engine test compares against.

The decisions it encodes, in one place:
  * fp16 rounding after each RMSNorm (O.rmsnorm_fwd), each quantized linear, RoPE, the attention output and each residual add;
  * RoPE through O.rope_inplace;
  * attention as an fp32 softmax over the fp16 K / V rows, head_dim = hidden // n_heads, query head h reading K / V head h;
  * the RMSNorm epsilon and the RoPE base are the caller's, never the decoder's: a decoder built with the wrong ones would agree
    with itself.
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
    dequantised, the first time a block uses it, and kept."""

    def __init__(self, layers, embed, final_norm, lm_head, n_heads, *, eps, base):
        self.layers, self.n_heads, self.eps, self.base = list(layers), n_heads, eps, base
        self.embed, self.final_norm, self.lm_head = _cpu(embed), _cpu(final_norm), _cpu(lm_head)
        self.hidden = self.embed.shape[1]
        self.head_dim = self.hidden // n_heads
        self._cpu_layers, self._weights = {}, {}

    @classmethod
    def from_decoder(cls, dec, *, eps, base):
        return cls(dec.layers, dec.embed, dec.final_norm, dec.lm_head, dec.n_heads, eps=eps, base=base)

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
        """x [n, H] at positions pos .. pos + n - 1 entering layer li -> (x after the attention block [n, H], the new K rows [nh, n, hd],
        the new V rows).  The rows attend to the cache prefix k_prefix / v_prefix [nh, >= pos, hd] (rows 0 .. pos - 1 are read) and
        causally to each other.  exact: qkv and o_proj with the exactly dequantised weight."""
        n, nh, hd = x.shape[0], self.n_heads, self.head_dim
        qkv = self._linear(li, 'qkv', O.rmsnorm_fwd(x, self._layer(li)['input_norm'], self.eps), exact).view(1, n, 3, nh, hd).clone()
        O.rope_inplace(qkv[:, :, :2], torch.arange(pos, pos + n)[None, :], base=self.base)
        q, k, v = (qkv[0, :, j].transpose(0, 1) for j in range(3))  # [nh, n, hd]
        K = torch.cat([k_prefix[:, :pos], k], 1) if pos else k
        V = torch.cat([v_prefix[:, :pos], v], 1) if pos else v
        s = (q.float() @ K.float().transpose(1, 2)) * hd**-0.5  # [nh, n, pos + n]
        s = s.masked_fill(torch.ones(n, pos + n, dtype=torch.bool).triu(pos + 1), float('-inf'))
        att = (torch.softmax(s, -1) @ V.float()).half().transpose(0, 1).reshape(n, self.hidden)
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
        return (O.rmsnorm_fwd(x, self.final_norm, self.eps).float() @ self.lm_head.float().t()).half()

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


def step_all(dec, toks, start):
    """Decode steps of toks at positions start, start + 1, ..."""
    for i, t in enumerate(toks):
        dec.set_input(t, start + i)
        dec.step()
    torch.cuda.synchronize()


def check_extend_against_stepping(dec, toks, cached, what):
    """`cached` positions stepped, extend() of the next ones up to the last token, one step of the last; against stepping all of them.
    The logits and the extended cache rows are held to the run-to-run spread of DESIGN.md section 2 (max 1.5e-2, rms 3e-3 of the rms)."""
    n = len(toks)
    step_all(dec, toks[:cached], 0)
    assert dec.extend([toks[cached:n - 1]]) == [n - 1]
    dec.set_input(toks[n - 1], n - 1)
    dec.step()
    torch.cuda.synchronize()
    got = [dec.logits[0].float().clone(), dec.k_cache[:, 0, :, cached:n - 1].float().clone(), dec.v_cache[:, 0, :, cached:n - 1].float().clone()]
    step_all(dec, toks[cached:], cached)
    ref = [dec.logits[0].float(), dec.k_cache[:, 0, :, cached:n - 1].float(), dec.v_cache[:, 0, :, cached:n - 1].float()]
    for name, g, r in zip(('logits', 'K rows', 'V rows'), got, ref):
        rms = r.pow(2).mean().sqrt().item()
        d = (g - r).abs()
        print(f'  {what} {name}: max |diff| / rms = {d.max().item() / rms:.3g}, rms diff / rms = {d.pow(2).mean().sqrt().item() / rms:.3g}')
        assert d.max().item() <= 1.5e-2 * rms and d.pow(2).mean().sqrt().item() <= 3e-3 * rms, f'{what}: {name}'
