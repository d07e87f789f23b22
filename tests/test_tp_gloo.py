"""CPU, world_size 2, gloo: the host logic of tensor-parallel QuantLinear (sharding + collectives).  The local matvec
is replaced by the oracle here (there is no GPU); the GPU version of this test is tests/test_gpu_tp.py."""
import os
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import gptq_oracle as O


def test_partitions():
    from gptq_b200 import tp
    assert tp.column_partition(4096, 8) == [512 * i for i in range(9)]
    b = tp.column_partition(22016, 8)  # 65B gate/up: 2752 columns per rank
    assert b[-1] == 22016 and all((b[i + 1] - b[i]) % 32 == 0 for i in range(8)) and max(b[i + 1] - b[i] for i in range(8)) == 2752
    r = tp.row_partition(22016, 128, 8)  # 65B down_proj: 172 groups -> 21 or 22 groups per rank
    sizes = [r[i + 1] - r[i] for i in range(8)]
    assert r[0] == 0 and r[-1] == 22016 and set(sizes) == {21 * 128, 22 * 128}
    with pytest.raises(ValueError):
        tp.row_partition(100, 128, 2)
    bytes_per_rank = tp.per_rank_bytes(22016, 8192, 4, 128, 8, 'row')
    assert abs(sum(bytes_per_rank) - (22016 * 8192 // 2 + 172 * 8192 * 2 + 172 * 8192 // 2)) < 1e-6


def test_shards_reassemble():
    from gptq_b200 import tp
    K, N, bits, gs = 512, 256, 4, 128
    qw, s, qz, g, b = O.random_packed(K, N, bits, gs, seed=1, bias=True)
    x = torch.randn(3, K, generator=torch.Generator().manual_seed(0)).half()
    full = O.qlinear_fwd(x, qw, s, qz, g, bits)
    cols = [O.qlinear_fwd(x, *tp.shard_columns(qw, s, qz, g, bits, r, 4)[:4], bits) for r in range(4)]
    assert torch.equal(torch.cat(cols, dim=1), full)  # column shards are exact
    acc = torch.zeros(3, N)
    for r in range(4):
        sqw, ss, sqz, sg, (k0, k1) = tp.shard_rows(qw, s, qz, g, bits, gs, r, 4)
        W = O.dequant(sqw, ss, sqz, sg, bits)
        assert torch.equal(W, O.dequant(qw, s, qz, g, bits)[k0:k1])  # a row shard dequantises to the same weights
        acc += x[:, k0:k1].float() @ W.float()
    assert torch.allclose(acc.half().float(), full.float(), rtol=1e-3, atol=1e-3)
    with pytest.raises(ValueError):
        tp.shard_rows(qw, s, qz, O.make_g_idx(K, gs, True, torch.Generator().manual_seed(0)), bits, gs, 0, 2)


@pytest.mark.parametrize('bits', [3, 2])
def test_narrow_bit_slices_reassemble(bits):
    """column_slice / row_slice of 3- and 2-bit layers (whole 32-column runs, whole packed words) dequantise exactly to the corresponding
    block: the tensor-parallel shards, scattered column runs like the decode engine's per-head qkv shards, and an uneven row shard."""
    from gptq_b200 import ops, tp
    K, N, gs = 512, 256, 128
    qw, s, qz, g, _ = O.random_packed(K, N, bits, gs, seed=bits)
    W = O.dequant(qw, s, qz, g, bits)
    b = tp.column_partition(N, 4)
    cols = [O.dequant(*tp.shard_columns(qw, s, qz, g, bits, r, 4)[:4], bits) for r in range(4)]
    assert all(torch.equal(c, W[:, b[r]:b[r + 1]]) for r, c in enumerate(cols))
    for r in range(4):
        sqw, ss, sqz, sg, (k0, k1) = tp.shard_rows(qw, s, qz, g, bits, gs, r, 4)
        assert torch.equal(O.dequant(sqw, ss, sqz, sg, bits), W[k0:k1])
    w = ops.QLayerWeights(qw, s, qz, g, bits, gs)
    c = torch.cat([torch.arange(32, 64), torch.arange(160, 256)])
    assert torch.equal(O.dequant(*w.column_slice(c).parts(), bits), W[:, c])
    rows = w.row_slice(128, 512)
    assert torch.equal(O.dequant(*rows.parts(), bits), W[128:512]) and rows.hint == gs
    for bad in (torch.arange(16, 48), torch.arange(0, 48)):
        with pytest.raises(ValueError):
            w.column_slice(bad)
    with pytest.raises(ValueError):
        w.row_slice(64, 256)


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        import quant
        from gptq_b200 import tp
        K, N, bits, gs = 512, 256, 4, 128
        qw, s, qz, g, b = O.random_packed(K, N, bits, gs, seed=1, bias=True)
        full = quant.QuantLinear(bits, gs, K, N, True)
        full.qweight, full.scales, full.qzeros, full.g_idx, full.bias = qw, s, qz, g, b
        x = torch.randn(3, K, generator=torch.Generator().manual_seed(0)).half()
        ref = O.qlinear_fwd(x, qw, s, qz, g, bits, b)

        def cpu_forward(layer):  # test-only stand-in for the CUDA kernel
            return lambda inp: O.qlinear_fwd(inp, layer.qweight, layer.scales, layer.qzeros, layer.g_idx, layer.bits, layer.bias)

        col = tp.TPQuantLinear(full, 'column', gather_output=True)
        col.local.forward = cpu_forward(col.local)
        out_c = col(x)
        row = tp.TPQuantLinear(full, 'row')
        row.local.forward = cpu_forward(row.local)
        out_r = row(x)
        ok = torch.equal(out_c, ref) and torch.allclose(out_r.float(), ref.float(), rtol=2e-3, atol=2e-3)
        ok = ok and col.local.outfeatures == N // world and row.local.infeatures == K // world
        q.put((rank, bool(ok)))
    finally:
        dist.destroy_process_group()


def test_tp_quantlinear_world2_gloo():
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = 29500 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(120)
        assert p.exitcode == 0
    res = dict(q.get(timeout=5) for _ in range(2))
    assert res == {0: True, 1: True}


def test_decoder_shards_reassemble():
    """engine.shard_for_rank (the tensor-parallel decode engine's sharding, BASELINE config 5): qkv columns go per HEAD (q | k | v of the rank's
    heads), o_proj rows follow the same heads, gate/up columns in slabs of 256 with the matching down_proj rows; every shard dequantises to exactly
    the corresponding block of the full matrix, and the shards tile it."""
    from gptq_b200 import engine
    H, I, NH, hd, bits, gs = 512, 1024, 4, 128, 4, 128
    def layer(K, N, seed):
        qw, s, qz, g, _ = O.random_packed(K, N, bits, gs, seed=seed)
        return engine.QLayerWeights(qw, s, qz, g, bits, gs)
    ly = dict(qkv=layer(H, 3 * H, 1), o=layer(H, H, 2), gate=layer(H, I, 3), up=layer(H, I, 4), down=layer(I, H, 5), input_norm=torch.ones(H).half(),
              post_norm=torch.ones(H).half())
    lm_head = torch.randn(96, H).half()
    deq = lambda w: O.dequant(w.qweight, w.scales, w.qzeros, w.g_idx, bits)
    full = {k: deq(v) for k, v in ly.items() if hasattr(v, 'qweight')}
    seen_heads, seen_cols, seen_vocab = [], [], []
    for rank in range(2):
        (sh, ), head, hl, (v0, v1) = engine.shard_for_rank([ly], lm_head, NH, hd, rank, 2)
        assert hl == 2 and torch.equal(head, lm_head[v0:v1])
        seen_vocab.append((v0, v1))
        hc = torch.arange(rank * hl * hd, (rank + 1) * hl * hd)
        assert torch.equal(deq(sh['qkv']), full['qkv'][:, torch.cat([hc, H + hc, 2 * H + hc])])
        assert torch.equal(deq(sh['o']), full['o'][hc])
        c0, c1 = rank * 2 * 256, (rank + 1) * 2 * 256
        assert torch.equal(deq(sh['gate']), full['gate'][:, c0:c1]) and torch.equal(deq(sh['up']), full['up'][:, c0:c1])
        assert torch.equal(deq(sh['down']), full['down'][c0:c1])
        assert sh['o'].hint == gs and sh['down'].hint == gs  # row shards keep the plain g_idx: the tuned kernels apply
        seen_heads.append(hc)
        seen_cols.append((c0, c1))
    assert torch.equal(torch.cat(seen_heads), torch.arange(H)) and seen_cols == [(0, 512), (512, 1024)] and seen_vocab == [(0, 48), (48, 96)]


def _decode_worker(rank, world, port, q):
    """One tensor-parallel rank of a decoder step in oracle arithmetic: what the persistent kernel computes per rank (local heads, local MLP
    slabs, local vocabulary rows), with the two per-layer reductions and the logits gather as gloo collectives."""
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        from gptq_b200 import engine
        H, I, NH, hd, bits, gs, V, T = 512, 1024, 4, 128, 4, 128, 96, 5

        def layer(K, N, seed):
            qw, s, qz, g, _ = O.random_packed(K, N, bits, gs, seed=seed)
            return engine.QLayerWeights(qw, (s.float() * 0.2).half(), qz, g, bits, gs)  # smaller scales keep the two-layer activations tame

        gen = torch.Generator().manual_seed(0)
        layers = [dict(qkv=layer(H, 3 * H, 10 * l + 1), o=layer(H, H, 10 * l + 2), gate=layer(H, I, 10 * l + 3), up=layer(H, I, 10 * l + 4), down=layer(I, H, 10 * l + 5),
                       input_norm=(torch.rand(H, generator=gen) * 0.2 + 0.9).half(), post_norm=(torch.rand(H, generator=gen) * 0.2 + 0.9).half()) for l in range(2)]
        lm_head = (torch.randn(V, H, generator=gen) * 0.05).half()
        fnorm = torch.ones(H).half()
        x0 = (torch.randn(1, H, generator=gen) * 0.5).half()
        kc = (torch.randn(2, NH, T, hd, generator=gen) * 0.5).half()  # cached rows [0, T) per layer
        vc = (torch.randn(2, NH, T, hd, generator=gen) * 0.5).half()
        w4 = lambda w: (w.qweight, w.scales, w.qzeros, w.g_idx)

        def step(lys, head, heads, reduce_):
            """heads: the global head indices this caller owns; reduce_: sums a partial [1, H] over the ranks (identity for the full model)."""
            x = x0.clone()
            nh = len(heads)
            for li, ly in enumerate(lys):
                qkv = O.qlinear_fwd(O.rmsnorm_fwd(x, ly['input_norm'], 1e-6), *w4(ly['qkv']), bits).view(1, 1, 3, nh, hd).clone()
                O.rope_inplace(qkv[:, :, :2], torch.tensor([[T]]))
                qh, kh, vh = qkv[0, 0, 0], qkv[0, 0, 1], qkv[0, 0, 2]
                K = torch.cat([kc[li, heads], kh[:, None, :]], 1).float()
                Vv = torch.cat([vc[li, heads], vh[:, None, :]], 1).float()
                att = torch.einsum('ht,htd->hd', torch.softmax(torch.einsum('hd,htd->ht', qh.float(), K) * hd**-0.5, -1), Vv).half().reshape(1, nh * hd)
                x = x + reduce_(O.qlinear_fwd(att, *w4(ly['o']), bits).float()).half()
                hmid = O.fused_mlp_fwd(O.rmsnorm_fwd(x, ly['post_norm'], 1e-6), w4(ly['gate']), w4(ly['up']), bits)
                x = x + reduce_(O.qlinear_fwd(hmid, *w4(ly['down']), bits).float()).half()
            return (O.rmsnorm_fwd(x, fnorm, 1e-6).float() @ head.float().t())[0]

        full_logits = step(layers, lm_head, list(range(NH)), lambda t: t)
        shard, head_local, hl, (v0, v1) = engine.shard_for_rank(layers, lm_head, NH, hd, rank, world)

        def allreduce(t):
            t = t.clone()
            dist.all_reduce(t)
            return t

        local = step(shard, head_local, list(range(rank * hl, (rank + 1) * hl)), allreduce)
        gathered = [torch.empty(V // world) for _ in range(world)]
        dist.all_gather(gathered, local.contiguous())
        logits = torch.cat(gathered)
        rms = full_logits.pow(2).mean().sqrt()
        err = ((logits - full_logits).abs() / torch.maximum(full_logits.abs(), rms)).max().item()
        q.put((rank, err, (v0, v1)))
    finally:
        dist.destroy_process_group()


def test_tp_decoder_step_world2_gloo():
    """The tensor-parallel decode path's host logic on CPU (gloo, world 2): sharding by heads / MLP slabs / vocabulary rows + one reduction after
    o_proj and after down_proj reproduces the unsharded decoder step (oracle arithmetic on both sides; the GPU version, where the reductions are
    peer-memory REDs inside the persistent kernel, is tests/test_gpu_tp.py)."""
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = 29650 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_decode_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(180)
        assert p.exitcode == 0
    res = sorted(q.get(timeout=5) for _ in range(2))
    assert [r[2] for r in res] == [(0, 48), (48, 96)]
    assert max(r[1] for r in res) < 5e-3, res  # fp16 rounding of the per-rank partial outputs before the sum
