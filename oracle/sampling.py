"""numpy float64 restatement of the sampling rule of gptq_sample_tokens (include/gptq_b200.h): eos suppression below the minimum length,
temperature, top-k, top-p and the Philox4x32-10 draw, or the argmax at temperature <= 0.  Test infrastructure: the GPU kernel is checked
token for token against sample_row, and the kept set against transformers' own warpers."""
import numpy as np

_M0, _M1, _W0, _W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
_MASK = 0xFFFFFFFF


def philox4x32_10(counter, key):
    """Random123's Philox4x32-10.  counter: uint32 array [..., 4], key: uint32 array [..., 2] (broadcast).  Returns uint32 [..., 4]."""
    c = np.asarray(counter, dtype=np.uint64) & _MASK
    k = np.asarray(key, dtype=np.uint64) & _MASK
    c0, c1, c2, c3 = (c[..., i].copy() for i in range(4))
    k0, k1 = k[..., 0].copy(), k[..., 1].copy()
    for r in range(10):
        if r:
            k0, k1 = (k0 + _W0) & _MASK, (k1 + _W1) & _MASK
        p0, p1 = np.uint64(_M0) * c0, np.uint64(_M1) * c2  # < 2^64: exact in uint64
        c0, c1, c2, c3 = (p1 >> 32) ^ c1 ^ k0, p1 & _MASK, (p0 >> 32) ^ c3 ^ k1, p0 & _MASK
    return np.stack([c0, c1, c2, c3], axis=-1).astype(np.uint32)


def uniform(position, seed):
    """u in [0, 1) of the draw at `position` (scalar or array) for a 64-bit seed: 53 bits of Philox(counter (p, 0, 0, 0), key (seed lo, hi))."""
    p = np.atleast_1d(np.asarray(position, dtype=np.int64)).astype(np.uint64) & _MASK
    ctr = np.stack([p, np.zeros_like(p), np.zeros_like(p), np.zeros_like(p)], axis=-1)
    s = int(seed) & 0xFFFFFFFFFFFFFFFF
    x = philox4x32_10(ctr, np.array([s & _MASK, s >> 32], dtype=np.uint64)).astype(np.float64)
    u = (np.floor(x[..., 0] / 32) * 2.0**26 + np.floor(x[..., 1] / 64)) * 2.0**-53
    return u if np.ndim(position) else float(u[0])


def _prepare(logits16, eos, min_length, position):
    l = np.asarray(logits16, dtype=np.float16).astype(np.float32).copy()
    l[np.isnan(l)] = -np.inf
    if eos is not None and 0 <= eos < l.size and position + 1 < min_length:
        l[eos] = -np.inf
    return l


def kept_weights(logits16, temperature, top_k=0, top_p=1.0, eos=-1, min_length=0, position=0):
    """(z, w) for one row at temperature > 0: z the fp32 scaled logits, w the fp64 weight of every token kept by top-k and top-p (0 elsewhere).
    Returns None when nothing is above -inf."""
    l = _prepare(logits16, eos, min_length, position)
    V = l.size
    z = (l / np.float32(temperature)).astype(np.float32)
    zmax = z.max()
    if zmax == -np.inf:
        return None
    keep = np.ones(V, dtype=bool)
    if 0 < top_k < V:
        zth = np.sort(z)[::-1][top_k - 1]
        keep = z >= zth
    if zmax == np.inf:
        w = (z == np.inf).astype(np.float64)
    else:
        w = np.exp(z.astype(np.float64) - np.float64(zmax))
    w = np.where(keep, w, 0.0)
    if top_p < 1:
        order = np.argsort(-z, kind='stable')
        zs = z[order]
        excl = np.concatenate([[0.0], np.cumsum(w[order])[:-1]])
        first = np.searchsorted(-zs, -zs, side='left')  # first position of each tie group in the descending order
        above = np.empty(V)
        above[order] = excl[first]
        keep &= (above < top_p * w.sum()) | (z == zmax)
        w = np.where(keep, w, 0.0)
    return z, w, keep


def sample_row(logits16, temperature, top_k=0, top_p=1.0, seed=0, eos=-1, min_length=0, position=0, details=False):
    """The token gptq_sample_tokens draws for one row.  With details, also a dict with the kept mask, the inclusive running weights in id
    order, W and the target u * W (for the near-boundary allowance of the GPU comparison)."""
    if not temperature > 0:
        l = _prepare(logits16, eos, min_length, position)
        tok = int(np.argmax(l))  # first maximum; -0 == +0; all -inf gives 0
        return (tok, None) if details else tok
    r = kept_weights(logits16, temperature, top_k, top_p, eos, min_length, position)
    if r is None:
        return (0, None) if details else 0
    z, w, keep = r
    run = np.cumsum(w)
    W = run[-1]
    target = uniform(position, seed) * W
    hit = np.nonzero(keep & (run > target))[0]
    tok = int(hit[0]) if hit.size else int(np.nonzero(keep)[0][-1])
    return (tok, dict(keep=keep, run=run, W=W, target=target)) if details else tok


def near_boundary(info, tok_a, tok_b, rel=2.0**-40):
    """True when tokens a and b are neighbours in the kept order and u * W lies within rel * W of the running weight between them."""
    ids = np.nonzero(info['keep'])[0]
    ia, ib = np.searchsorted(ids, tok_a), np.searchsorted(ids, tok_b)
    if abs(int(ia) - int(ib)) != 1 or ids[ia] != tok_a or ids[ib] != tok_b:
        return False
    lo = ids[min(ia, ib)]
    return abs(info['run'][lo] - info['target']) <= rel * info['W']
