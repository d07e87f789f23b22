"""CPU: the groupsize probe (gs_probe.py) is exact under the decode kernels' arithmetic, and its anchors have teeth.

* Exactness: for every case of tests/test_gpu_decode_groupsize.py, every partial sum a kernel can form in any linear lies on its grid
  below 2^24 units (gs_probe.check_exact), every gate output is an even integer >= 20 (the sigmoid is exactly 1 in fp32), and the inputs
  stay above the fp16 subnormal grid after the 1/16 pre-scaling of the odd nibbles.
* Teeth: a kernel that read the neighbouring group's scale or zero for one stage, took another sequence's sum of x, or dropped or repeated
  one k-step would produce an observed output (K row, x after attention, x after the layer) that differs from the anchor in many
  elements, at every groupsize, the partial last group of down_proj at 1024 included, and at the 65B and 33B probe layers.
"""
from functools import lru_cache

import pytest
import torch

import gs_probe as P

CONFIGS = sorted({(s, gs, bits, act) for s, gs, bits, act, _, _ in P.CASES}, key=str)


@lru_cache(maxsize=2)
def layer(size, gs, bits, act):
    return P.layer_for(size, gs, bits, act)


@pytest.mark.parametrize('size,gs,bits,act', CONFIGS)
def test_probe_sums_are_exact_in_fp32(size, gs, bits, act):
    L = layer(size, gs, bits, act)
    r = P.check_exact(L)
    for name in ('qkv', 'o', 'gate', 'up', 'down'):
        total, stage = r[name]
        print(f'  {size} gs={gs} int{bits} act={act} {name}: largest partial sum / 2^24 units: total {total:.3f}, stage {stage:.3f}')
        assert total < 1 and stage < 1, f'{name}: a partial sum can leave fp32\'s 24 bits ({total:.3f}, {stage:.3f})'
    a = L.gate.weight().sum(0)
    assert bool((a >= 20).all() and (a < 40).all() and (a % 2 == 0).all()), 'gate outputs must be even integers in [20, 40)'
    for lin in L.linears().values():  # adjacent groups differ in zero and scale, column by column
        if lin.z.shape[0] > 1:
            assert bool((lin.z[1:] != lin.z[:-1]).all() and (lin.j[1:] != lin.j[:-1]).all())
        assert int(lin.z.min()) >= 1 and int(lin.z.max()) <= (1 << bits) - 2 and int(lin.q.max()) < (1 << bits)


@pytest.mark.parametrize('gs', [32, 128, 1024, 'full'])
def test_probe_anchors_have_teeth(gs):
    """At batch 8: each corruption moves many of the observed elements (at least a quarter of them; the sum-of-x one only sequence 1)."""
    check_teeth('7b', gs)


@pytest.mark.parametrize('size,gs', [('65b', 128), ('65b', 1024), ('33b', 1024)])
def test_probe_anchors_have_teeth_large(size, gs):
    """The same at the 65B and 33B probe layers; at 33B gs 1024 every corruption lands in a partial last group of 512."""
    check_teeth(size, gs)


def check_teeth(size, gs):
    L = layer(size, gs, 4, False)
    x_in = P.embed_rows(P.VOCAB, L.H)[torch.tensor(P.tokens(8))]
    res = P.teeth(L, x_in)
    names = {n for _, n in res}
    assert {'dropped k-step', 'repeated k-step', 'other sequence sum of x'} <= names
    if gs != 'full':
        assert {'neighbour scale', 'neighbour zero'} <= names
    for (lin, name), (diff, total) in sorted(res.items()):
        frac = diff / total
        print(f'  {size} gs={gs} {lin} {name}: {diff} / {total} observed elements differ')
        need = 0.25 / 8 if name == 'other sequence sum of x' else 0.25
        assert frac >= need, f'{size} gs={gs} {lin} {name}: only {diff} / {total} elements differ'
