"""Float64 oracle of the top-K in-batch retrieval (siglip_request_topk) and models of its kernels.

Per rank r, over the concatenated global batch (rank r's images are [its B_r paired images; its extra images], its
texts [its B_r paired texts; its extras]; global index = prefix sum of the per-rank counts + local index):
  i2t_topk[i] = the K texts with the largest <img_i, txt_j>, best first, ties to the lower global index; t2i_topk[j]
  the same over the images; -1 past the candidates there are. recall[k - 1] = fraction of the ranked samples with a hit
  among their first k entries, where a hit is the rule of the top-1 metrics (tests/retrieval_metrics_oracle.py).
"""
import random

import numpy as np


def _ranked(S, k):
    """Per row of S (float64): the indices of its k largest entries, best first, ties to the lower index; -1 pads."""
    n, m = S.shape
    out = np.full((n, k), -1, np.int64)
    cols = np.arange(m)
    for r in range(n):
        order = np.lexsort((cols, -S[r]))[:k]
        out[r, :len(order)] = order
    return out


def topk_retrieval(imgs, txts, batches, k, img_ids=None, txt_ids=None, rank_all_images=False, rank_all_texts=False):
    """imgs / txts: per-rank [R_r, D] / [T_r, D] arrays; batches: per-rank B_r. img_ids / txt_ids: None for positional
    labels, or per-rank integer arrays: an image (text) past its rank's array carries no id and is never a hit (the
    extras without ids). rank_all_images / rank_all_texts: i2t ranks all R_r images (extra_image_ids), t2i all T_r
    texts (extra_text_ids); otherwise the B_r paired ones.
    Returns one dict per rank: i2t_topk [ni, k], t2i_topk [nt, k] (int64 global indices), i2t_recall / t2i_recall [k]
    (float64), i2t_first / t2i_first (rank of the first hit, k for none) and i2t_gap / t2i_gap (similarity of the k-th
    best minus the (k+1)-th: the separation a lower-precision ranking must not cross)."""
    I = np.concatenate([np.asarray(x, np.float64) for x in imgs])
    T = np.concatenate([np.asarray(x, np.float64) for x in txts])
    S = I @ T.T
    off = np.concatenate([[0], np.cumsum([len(x) for x in imgs])]).astype(np.int64)
    toff = np.concatenate([[0], np.cumsum([len(x) for x in txts])]).astype(np.int64)
    W = len(imgs)
    positional = img_ids is None and txt_ids is None
    # global id of every image / text; None = no id
    gi = [None] * len(I)
    gt = [None] * len(T)
    if not positional:
        for r in range(W):
            for l, v in enumerate(np.asarray(img_ids[r]).tolist()):
                gi[off[r] + l] = v
            for l, v in enumerate(np.asarray(txt_ids[r]).tolist()):
                gt[toff[r] + l] = v

    def i2t_hit(r, i, j):
        if positional:
            return j == toff[r] + i
        return gt[j] is not None and gt[j] == gi[off[r] + i]

    def t2i_hit(r, i, g):
        if positional:
            return g == off[r] + i
        return gi[g] is not None and gi[g] == gt[toff[r] + i]

    def gaps(M):
        srt = -np.sort(-M, axis=1)
        if M.shape[1] <= k:
            return np.full(M.shape[0], np.inf)
        return srt[:, k - 1] - srt[:, k]

    rows, cols = _ranked(S, k), _ranked(S.T, k)
    g_i2t, g_t2i = gaps(S), gaps(S.T)
    out = []
    for r in range(W):
        ni = len(imgs[r]) if rank_all_images else batches[r]
        nt = len(txts[r]) if rank_all_texts else batches[r]
        i2t = rows[off[r]:off[r] + ni]
        t2i = cols[toff[r]:toff[r] + nt]

        def first(lst, hit):
            f = np.full(len(lst), k, np.int64)
            for i, row in enumerate(lst):
                for s, j in enumerate(row.tolist()):
                    if j >= 0 and hit(r, i, j):
                        f[i] = s
                        break
            return f

        fi, ft = first(i2t, i2t_hit), first(t2i, t2i_hit)
        out.append(dict(i2t_topk=i2t, t2i_topk=t2i,
                        i2t_recall=np.array([(fi < q).mean() for q in range(1, k + 1)]),
                        t2i_recall=np.array([(ft < q).mean() for q in range(1, k + 1)]),
                        i2t_first=fi, t2i_first=ft,
                        i2t_gap=g_i2t[off[r]:off[r] + ni], t2i_gap=g_t2i[toff[r]:toff[r] + nt], S=S, off=off, toff=toff))
    return out


def recall_counts(first, k):
    """recall@1..k as the kernel counts it: integer counts of first-hit ranks, divided once by the sample count in fp32."""
    first = np.asarray(first)
    return np.array([np.float32(np.count_nonzero(first < q)) / np.float32(len(first)) for q in range(1, k + 1)],
                    np.float32)


# ---- models of the kernels ----

def insert_chain(k, key, stop_on_reject=False):
    """The insertion of one key as a generator of atomic steps: each next() sends (slot, key) and receives the slot's old
    value. Ends when the carried key is 0 or after slot k - 1. stop_on_reject: the broken variant that gives up as soon
    as a slot holds a larger key (it loses a displaced key's later chance)."""
    c = key
    for s in range(k):
        old = yield (s, c)
        if old < c:
            c = old
            if c == 0:
                return
        elif stop_on_reject:
            return


def run_interleaved(k, keys, seed, stop_on_reject=False, prefilter=False):
    """Runs one insertion chain per key, their atomic steps interleaved at random. Returns the final list (k slots).
    prefilter: each chain first reads slot k - 1 at a random earlier moment (a stale value) and does not start when
    its key is not above it, as the kernel's threshold does."""
    rng = random.Random(seed)
    slots = [0] * k
    history = [0]   # values slot k - 1 has held, in order
    pending = list(keys)
    rng.shuffle(pending)
    live = []
    while pending or live:
        if pending and (not live or rng.random() < 0.5):
            key = pending.pop()
            if prefilter and key <= rng.choice(history):
                continue
            gen = insert_chain(k, key, stop_on_reject)
            live.append([gen, gen.send(None)])
            continue
        idx = rng.randrange(len(live))
        gen, (s, c) = live[idx]
        old = slots[s]
        slots[s] = max(old, c)
        history.append(slots[k - 1])
        try:
            live[idx][1] = gen.send(old)
        except StopIteration:
            live.pop(idx)
        assert all(slots[i] >= slots[i + 1] for i in range(k - 1)), slots
    return slots


def merge_lists(lists, k):
    """The finalisation's merge of W sorted lists (0-padded, keys distinct across lists): the k best, best first."""
    head = [0] * len(lists)
    out = []
    for _ in range(k):
        best, bq = 0, -1
        for q, lst in enumerate(lists):
            if head[q] < k and lst[head[q]] > best:
                best, bq = lst[head[q]], q
        if bq >= 0:
            head[bq] += 1
        out.append(best)
    return out
