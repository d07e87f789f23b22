"""GPU, 2 ranks, NCCL: tensor-parallel QuantLinear against the single-GPU result (needs >= 2 GPUs)."""
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import gptq_oracle as O

pytestmark = pytest.mark.gpu


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=torch.device('cuda', rank))
    try:
        import quant
        from gptq_b200 import tp
        K, N, bits, gs = 2048, 1024, 4, 128
        qw, s, qz, g, _ = O.random_packed(K, N, bits, gs, seed=1)
        full = quant.QuantLinear(bits, gs, K, N, False)
        full.qweight, full.scales, full.qzeros, full.g_idx = qw, s, qz, g
        full = full.cuda()
        ok = True
        for M in (1, 4, 64):
            x = torch.randn(M, K, generator=torch.Generator().manual_seed(M)).half().cuda()
            ref = full(x)
            col = tp.TPQuantLinear(full, 'column', gather_output=True)
            row = tp.TPQuantLinear(full, 'row')
            ok = ok and torch.equal(col(x), ref)
            err = (row(x).float() - ref.float()).abs()
            bound = 2e-3 * torch.maximum(ref.float().abs(), ref.float().pow(2).mean().sqrt())
            ok = ok and bool((err <= bound).all())
        q.put((rank, bool(ok)))
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs 2 GPUs')
def test_tp_quantlinear_world2_nccl():
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = 29700 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(300)
        assert p.exitcode == 0
    res = dict(q.get(timeout=5) for _ in range(2))
    assert res == {0: True, 1: True}


def _decode_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=torch.device('cuda', rank))
    try:
        from gptq_b200 import engine
        dev = f'cuda:{rank}'
        # the same full model on every rank (same seed), decoded on one GPU ...
        full = engine.synthetic_llama('tiny512', bits=4, groupsize=128, vocab=512, seed=7, max_seq=96, device=dev)
        assert full.launches_per_step() == 1
        toks = torch.randint(0, 512, (40, ), generator=torch.Generator().manual_seed(3)).tolist()
        ref = []
        for pos, tok in enumerate(toks):
            full.set_input(tok, pos)
            full.step()
            torch.cuda.synchronize()
            ref.append(full.logits[0].float().clone())
        # ... and as `world` tensor-parallel shards: o_proj / down_proj partial sums land in every rank's accumulators over NVLink
        worst = 0.0
        for mode in (1, 2):  # direct peer REDs / local reduction + slice exchange (gptq_llama_tp.reduce_mode)
            tp = engine.synthetic_llama_tp('tiny512', rank, world, full=full, max_seq=96, reduce_mode=mode)
            assert tp.launches_per_step() == 1
            for pos, tok in enumerate(toks):
                tp.set_input(tok, pos)
                tp.step()
                torch.cuda.synchronize()
                out = tp.logits[0].float()
                rms = ref[pos].pow(2).mean().sqrt()
                worst = max(worst, ((out - ref[pos]).abs() / torch.maximum(ref[pos].abs(), rms)).max().item())
                assert int(tp.next_tokens[0]) == int(out.argmax())
            dist.barrier()
        q.put((rank, worst))
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs 2 GPUs')
def test_tp_decode_world2_matches_single_gpu():
    """Tensor-parallel persistent decode kernel (peer REDs + cross-GPU barrier) against the single-GPU kernel on the same weights: every rank
    ends up with the full logits; the difference is the fp32 summation order of the shards (fp16 rounding noise, see test_gpu_engine_fullsize)."""
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = 29900 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_decode_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(300)
        assert p.exitcode == 0
    res = dict(q.get(timeout=5) for _ in range(2))
    assert set(res) == {0, 1} and max(res.values()) < 2e-2, res
