"""Float64 oracle of the in-batch retrieval metrics (siglip_request_metrics) and a model of the kernels' argmax keys.

Per rank r, over the concatenated batch (global index = prefix sum of the per-rank batches + local index):
  i2t_index[i] = argmax_j <img_i, txt_j> over every text, t2i_index[j] = argmax_i <img_i, txt_j> over every image,
  ties to the lowest global index; a top-1 is a hit when it is the positional pair, or with ids a pair with the same id.
"""
import numpy as np


def retrieval_metrics(imgs, txts, ids=None):
    """imgs / txts: per-rank [B_r, D] arrays; ids: per-rank [B_r] integer arrays or None. Returns one dict per rank with
    i2t_index / t2i_index (global, int64), i2t_top1 / t2i_top1 (float) and i2t_margin / t2i_margin (best minus second
    best similarity, float64; the gap a lower-precision ranking must not cross)."""
    I = np.concatenate([np.asarray(x, np.float64) for x in imgs])
    T = np.concatenate([np.asarray(x, np.float64) for x in txts])
    S = I @ T.T
    off = np.concatenate([[0], np.cumsum([len(x) for x in imgs])]).astype(np.int64)
    gid = np.concatenate([np.asarray(x, np.int64) for x in ids]) if ids is not None else np.arange(len(I))
    i2t = np.argmax(S, axis=1)   # first occurrence = lowest index
    t2i = np.argmax(S, axis=0)

    def margin(M):
        if M.shape[1] < 2:
            return np.full(M.shape[0], np.inf)
        part = np.sort(M, axis=1)
        return part[:, -1] - part[:, -2]

    m_i2t, m_t2i = margin(S), margin(S.T)
    out = []
    for r in range(len(imgs)):
        sl = slice(off[r], off[r + 1])
        g = np.arange(off[r], off[r + 1])
        hi = gid[i2t[sl]] == gid[g]
        ht = gid[t2i[sl]] == gid[g]
        out.append(dict(i2t_index=i2t[sl].astype(np.int64), t2i_index=t2i[sl].astype(np.int64),
                        i2t_top1=float(hi.mean()), t2i_top1=float(ht.mean()),
                        i2t_margin=m_i2t[sl], t2i_margin=m_t2i[sl], S=S, off=off, gid=gid))
    return out


def hits(index, gid, first):
    """Hits of a list of global top-1 indices of the samples first, first + 1, ... (labels from gid)."""
    index = np.asarray(index, np.int64)
    return gid[index] == gid[first + np.arange(len(index))]


def metric_key(s, idx):
    """The kernels' 64-bit argmax key: (order-preserving bits of fp32 s) << 32 | (0xFFFFFFFF - idx), -0 folded to +0."""
    f = np.float32(np.float32(s) + np.float32(0.0))
    u = int(np.array(f, np.float32).view(np.uint32))
    ordered = u ^ (0xFFFFFFFF if (u >> 31) else 0x80000000)
    return (ordered << 32) | (0xFFFFFFFF - int(idx))


def key_index(k):
    return -1 if k == 0 else 0xFFFFFFFF - (k & 0xFFFFFFFF)


def key_as_int64(k):
    """A key as the int64 bit pattern a torch tensor stores."""
    return k - (1 << 64) if k >= (1 << 63) else k
