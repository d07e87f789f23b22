"""GPU: the reference-facing modules end to end -- QuantLinear / QuantLlamaMLP / QuantLlamaAttention /
TritonLlamaRMSNorm inside a tiny HF LLaMA, i.e. what llama_inference.load_quant builds -- and
size-independent properties at BASELINE.json's full layer sizes."""
import pytest
import torch

from oracle import gptq_oracle as O
from gpu_util import assert_rel_close, cuda, fill_quant_linear, tiny_quant_llama
from llama_oracle import CODELLAMA, LLAMA1, scale_down_embedding_row

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('bits,act', [(4, False), (4, True), (3, True), (8, False), (2, False)])
def test_quantlinear_module_forward_and_backward(bits, act):
    import quant
    ql = quant.QuantLinear(bits, 64, 256, 128, True)
    fill_quant_linear(ql, bits, seed=bits, act=act)
    x = torch.randn(2, 3, 256, generator=torch.Generator().manual_seed(0)).half()
    ref = O.qlinear_fwd(x, ql.qweight, ql.scales, ql.qzeros, ql.g_idx, bits, ql.bias)
    ql = ql.cuda()
    assert ql.groupsize_hint() == (0 if act else 64)
    xd = x.cuda().requires_grad_(True)
    out = ql(xd)
    assert out.shape == (2, 3, 128) and out.dtype == torch.float16
    assert_rel_close(out, ref, what='module fwd')
    go = torch.randn(2, 3, 128, generator=torch.Generator().manual_seed(1)).half()
    out.backward(go.cuda())
    gref = O.qlinear_transpose_fwd(go, *(t.cpu() for t in (ql.qweight, ql.scales, ql.qzeros, ql.g_idx)), bits)
    assert_rel_close(xd.grad, gref, what='module bwd')


def _ref_forward(model, ids, base, eps):
    """fp32 reference forward of the (not yet fused) quantized model using the CPU oracle for every op, at the RoPE base and RMSNorm
    epsilon the caller chose (not the ones the model carries)."""
    cfg = model.config
    h = model.model.embed_tokens(ids).half()
    bsz, seq = ids.shape
    pos = torch.arange(seq)[None, :].expand(bsz, -1)
    nh, hd = cfg.num_attention_heads, cfg.hidden_size // cfg.num_attention_heads

    def lin(m, x):
        return O.qlinear_fwd(x, m.qweight, m.scales, m.qzeros, m.g_idx, m.bits, m.bias)

    for layer in model.model.layers:
        a = layer.self_attn
        x = O.rmsnorm_fwd(h, layer.input_layernorm.weight.data, eps)
        qkv = torch.stack([lin(a.q_proj, x), lin(a.k_proj, x), lin(a.v_proj, x)], dim=2).view(bsz, seq, 3, nh, hd)
        O.rope_inplace(qkv[:, :, :2], pos, base=base)
        q, k, v = (qkv[:, :, i].transpose(1, 2).float() for i in range(3))
        att = torch.nn.functional.scaled_dot_product_attention(q, k, v, is_causal=True).half()
        h = h + lin(a.o_proj, att.transpose(1, 2).reshape(bsz, seq, -1))
        x = O.rmsnorm_fwd(h, layer.post_attention_layernorm.weight.data, eps)
        m = layer.mlp
        inter = O.fused_mlp_fwd(x, (m.gate_proj.qweight, m.gate_proj.scales, m.gate_proj.qzeros, m.gate_proj.g_idx),
                                (m.up_proj.qweight, m.up_proj.scales, m.up_proj.qzeros, m.up_proj.g_idx), m.gate_proj.bits)
        h = h + lin(m.down_proj, inter)
    h = O.rmsnorm_fwd(h, model.model.norm.weight.data, eps)
    return (h.float() @ model.lm_head.weight.data.float().t())


@pytest.mark.parametrize('bits,act,rope', [pytest.param(4, False, LLAMA1, id='4-False'), pytest.param(4, True, LLAMA1, id='4-True'),
                                           pytest.param(3, True, LLAMA1, id='3-True'), pytest.param(4, False, CODELLAMA, id='4-False-codellama')])
def test_load_quant_pipeline_on_tiny_llama(bits, act, rope):
    """make_quant_linear -> (load) -> make_quant_attn / make_quant_norm / make_fused_mlp -> .to(DEV) -> forward,
    prefill then one cached decode step, against the oracle-composed reference at the RoPE base and epsilon of the config.
    At the CodeLlama settings the first token's embedding row is scaled to a mean square of about 1.6e-6 (HF's init has std 0.02),
    where epsilon 1e-5 and 1e-6 give norms a factor 2 apart."""
    import quant
    base, eps = rope
    model = tiny_quant_llama(bits=bits, act=act, rope_theta=base, rms_norm_eps=eps)
    ids = torch.randint(0, 256, (1, 9), generator=torch.Generator().manual_seed(0))
    if rope != LLAMA1:
        scale_down_embedding_row(model.model.embed_tokens.weight, int(ids[0, 0]), 4)
    ref_logits = _ref_forward(model, ids, base=base, eps=eps)
    quant.make_quant_attn(model)
    quant.make_quant_norm(model)
    quant.make_fused_mlp(model)
    model = model.cuda()
    assert quant.autotune_warmup_linear(model) > 0 and quant.autotune_warmup_fused(model) == 2
    if act or bits != 4:  # derived buffers route act-order / 3-bit layers to the tuned kernels
        assert model.model.layers[0].mlp.kernel_plan() is not None and model.model.layers[0].self_attn.qkv_proj.kernel_plan() is not None
    with torch.no_grad():
        out = model(ids[:, :8].cuda(), use_cache=True)
        what = f'bits={bits} act={act} base={base:g} eps={eps:g}'
        assert_rel_close(out.logits[0], ref_logits[0, :8], rel=2e-2, what=f'{what}: prefill logits')
        step = model(ids[:, 8:9].cuda(), past_key_values=out.past_key_values, use_cache=True)
        assert_rel_close(step.logits[0, 0], ref_logits[0, 8], rel=2e-2, what=f'{what}: decode logits')


@pytest.mark.parametrize('bits', [4, 3])
def test_engine_and_modules_derive_the_same_kernel_form(bits):
    """engine.from_hf_quant_model and the quant modules of one act-order model derive the kernel form of every layer through the same
    owner (ops.QLayerWeights, ops.mlp_kernel_form): the decoder's layers and input gathers equal the modules' kernel_plan()s.  head_dim 128
    so that the decoder takes the persistent kernel and keeps its gathers."""
    import quant
    from gptq_b200 import engine, ops
    gs = 32
    model = tiny_quant_llama(bits=bits, gs=gs, act=True, hidden=256, intermediate=768, heads=2)
    quant.make_quant_attn(model)
    quant.make_quant_norm(model)
    quant.make_fused_mlp(model)
    model = model.cuda()
    dec = engine.from_hf_quant_model(model, max_seq=16, use_graph=False)
    assert dec.launches_per_step() == 1
    for layer, kl, pm in zip(model.model.layers, dec.klayers, dec.perms):
        plans = {'qkv': layer.self_attn.qkv_proj.kernel_plan(), 'o': layer.self_attn.o_proj.kernel_plan(), 'down': layer.mlp.down_proj.kernel_plan()}
        for name, w in plans.items():
            assert kl[name].bits == w.bits == 4 and all(torch.equal(a, b) for a, b in zip(kl[name].parts(), w.parts())), name
            assert name == 'down' or torch.equal(pm[name], w.perm.int()), name
        gate, up = layer.mlp.kernel_plan()
        assert torch.equal(pm['gate'], gate.perm.int()) and torch.equal(gate.perm, up.perm)
        for name, w in (('gate', gate), ('up', up)):  # the decoder folds down_proj's gather into the column order of gate|up
            assert torch.equal(ops.dequant(*kl[name].parts(), 4, gs), ops.dequant(*w.parts(), 4, gs)[:, plans['down'].perm]), name


# ----------------------------------------------------------------------------- full BASELINE sizes: size-independent properties
FULL = [(4096, 4096), (4096, 12288), (11008, 4096)]


@pytest.mark.parametrize('K,N', FULL)
def test_full_size_matches_dequant_matmul(K, N):
    """LLaMA-7B layer sizes, M=1: CUDA matvec == fp32 matmul over the device-dequantised weight
    (the dequant kernel itself is pinned bit-exactly to the oracle above)."""
    from gptq_b200 import ops
    qw, s, qz, g, _ = cuda(*O.random_packed(K, N, 4, 128, seed=K + N))
    x = torch.randn(1, K, generator=torch.Generator().manual_seed(0)).half().cuda()
    W = ops.dequant(qw, s, qz, g, 4, 128)
    ref = (x.float() @ W.float()).half()
    out = ops.matmul248(x, qw, s, qz, g, 4, 15, groupsize=128)
    assert_rel_close(out, ref, what=f'full {K}x{N}')
    # exact homogeneity: scaling x by a power of two scales every product exactly
    out2 = ops.matmul248(x * 2, qw, s, qz, g, 4, 15, groupsize=128)
    assert torch.equal(out2, out * 2)
    # determinism
    assert torch.equal(ops.matmul248(x, qw, s, qz, g, 4, 15, groupsize=128), out)


def test_full_size_fused_mlp_matches_composition():
    from gptq_b200 import ops
    K, N = 4096, 11008
    gate = cuda(*O.random_packed(K, N, 4, 128, seed=1)[:4])
    up = cuda(*O.random_packed(K, N, 4, 128, seed=2)[:4])
    x = torch.randn(1, K, generator=torch.Generator().manual_seed(0)).half().cuda()
    a1 = x.float() @ ops.dequant(*gate, 4, 128).float()
    a2 = x.float() @ ops.dequant(*up, 4, 128).float()
    ref = (a1 * torch.sigmoid(a1) * a2).half()
    out = ops.fused_mlp(x, gate, up, 4, 128)
    assert_rel_close(out, ref, rel=2e-3, what='full fused mlp')


def test_column_slices_are_independent():
    """Sharding property used by tensor parallelism: slicing the packed tensors along N (multiples of 32)
    gives exactly the corresponding slice of the output."""
    from gptq_b200 import ops
    K, N = 1024, 512
    qw, s, qz, g, _ = cuda(*O.random_packed(K, N, 4, 128, seed=9))
    x = torch.randn(2, K, generator=torch.Generator().manual_seed(0)).half().cuda()
    full = ops.matmul248(x, qw, s, qz, g, 4, 15)
    for n0, n1 in ((0, 128), (128, 512), (256, 288)):
        part = ops.matmul248(x, qw[:, n0:n1].contiguous(), s[:, n0:n1].contiguous(), qz[:, n0 // 8:n1 // 8].contiguous(), g, 4, 15)
        assert_rel_close(part, full[:, n0:n1], what=f'cols {n0}:{n1}')


def test_act_order_kernel_plan_uses_tuned_kernels_and_matches_gather_path():
    """Act-order int4: the load-time row regrouping (derived buffer + x gather) gives the same result as the g_idx-gather kernel."""
    import quant
    from gptq_b200 import ops
    ql = quant.QuantLinear(4, 128, 1024, 512, False)
    fill_quant_linear(ql, 4, seed=11, act=True)
    x = torch.randn(3, 1024, generator=torch.Generator().manual_seed(2)).half()
    ref = O.qlinear_fwd(x, ql.qweight, ql.scales, ql.qzeros, ql.g_idx, 4)
    ql = ql.cuda()
    assert quant.autotune_warmup_linear(ql) == 1 and ql.kernel_plan() is not None
    plan = ql.kernel_plan()
    perm, qw_sorted, g_triv = plan.perm, plan.qweight, plan.g_idx
    assert plan.bits == 4 and plan.qzeros is ql.qzeros
    W_gather = ops.dequant(ql.qweight, ql.scales, ql.qzeros, ql.g_idx, 4, 0)
    W_sorted = ops.dequant(qw_sorted, ql.scales, ql.qzeros, g_triv, 4, 128)
    assert torch.equal(W_sorted, W_gather.index_select(0, perm))  # the same fp16 weights, rows regrouped
    assert_rel_close(ql(x.cuda()), ref, what='act-order fast path M=3')
    xb = torch.randn(40, 1024, generator=torch.Generator().manual_seed(3)).half()
    assert_rel_close(ql(xb.cuda()), O.qlinear_fwd(xb, *(t.cpu() for t in (ql.qweight, ql.scales, ql.qzeros, ql.g_idx)), 4), rel=2e-3, what='act-order fast path M=40')


@pytest.mark.parametrize('bits,act', [(3, False), (3, True), (2, True)])
def test_narrow_bits_are_served_by_the_int4_kernels_through_the_widened_kernel_plan(bits, act):
    """2/3-bit layers (config 4: int3 act-order): fields widened to nibbles at load time -> identical dequantised weights,
    outputs within tolerance of the oracle on the ORIGINAL packed tensors, for the matvec (M=1) and the GEMM (M=40)."""
    import quant
    from gptq_b200 import ops
    ql = quant.QuantLinear(bits, 128, 1024, 512, False)
    fill_quant_linear(ql, bits, seed=20 + bits, act=act)
    cpu = [t.clone() for t in (ql.qweight, ql.scales, ql.qzeros, ql.g_idx)]
    ql = ql.cuda()
    plan = ql.kernel_plan()
    assert plan is not None and plan.bits == 4 and (plan.perm is not None) == act
    W_orig = ops.dequant(ql.qweight, ql.scales, ql.qzeros, ql.g_idx, bits, 0)
    W_plan = ops.dequant(plan.qweight, ql.scales, plan.qzeros, plan.g_idx, 4, 128)
    assert torch.equal(W_plan, W_orig if plan.perm is None else W_orig.index_select(0, plan.perm))
    for M, rel in ((1, 1e-3), (40, 2e-3)):
        x = torch.randn(M, 1024, generator=torch.Generator().manual_seed(M)).half()
        assert_rel_close(ql(x.cuda()), O.qlinear_fwd(x, *cpu, bits), rel=rel, what=f'bits={bits} act={act} M={M}')


@pytest.mark.parametrize('bits,gs,act', [(4, 32, False), (4, 64, True), (8, 64, False)])
def test_solver_to_pack_to_kernel_on_a_bias_block(bits, gs, act):
    """The whole quantisation-side chain on the GPU for an OPT / GPT-NeoX style block (nn.Linear WITH bias, opt.py:249-285, neox.py:234-273):
    gptq.quantize_linears (Hessian, Cholesky, blocked updates on the device) -> make_quant_linear -> QuantLinear.pack (GPU packing kernels) ->
    QuantLinear.forward (CUDA kernels) reproduces the fp16 forward of the on-grid weights the solver left in the layer."""
    import copy
    import torch.nn as nn
    import gptq
    import quant

    class Block(nn.Module):
        def __init__(self):
            super().__init__()
            self.fc1, self.fc2 = nn.Linear(256, 512, bias=True), nn.Linear(512, 256, bias=True)

        def forward(self, x):
            return self.fc2(torch.relu(self.fc1(x)))

    torch.manual_seed(bits + gs)
    blk = Block().cuda()
    calib = [torch.randn(4, 32, 256, device='cuda') * (torch.rand(256, device='cuda') * 2 + 0.2) for _ in range(2)]
    res = gptq.quantize_linears(blk, calib, wbits=bits, groupsize=gs, act_order=act)
    ongrid = copy.deepcopy(blk).half()  # fp16 model carrying the solver's on-grid weights
    qblk = copy.deepcopy(blk)
    quant.make_quant_linear(qblk, {n: getattr(qblk, n) for n in res}, bits, gs)
    for n, (scale, zero, g_idx, _) in res.items():
        assert isinstance(getattr(qblk, n), quant.QuantLinear) and getattr(qblk, n).bias is not None
        getattr(qblk, n).pack(getattr(blk, n), scale, zero, g_idx)
    qblk = qblk.cuda()
    x = torch.randn(3, 256, device='cuda').half()
    for n in res:  # layer by layer: the packed layer equals the on-grid fp16 layer (dequantised weights agree to fp16 rounding of the scales)
        xin = x if n == 'fc1' else torch.relu(ongrid.fc1(x))
        assert_rel_close(getattr(qblk, n)(xin), getattr(ongrid, n)(xin), rel=4e-3, what=f'{n} bits={bits} gs={gs} act={act}')
    if act:
        assert not torch.equal(res['fc1'][2].cpu(), (torch.arange(256) // gs).int())
