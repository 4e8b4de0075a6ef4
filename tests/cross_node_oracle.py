"""Float64 oracle of a group that spans nodes — test infrastructure, never the product path.

A problem is the global batch of a group of N·L ranks: rank g holds R_g = B_g + K_img images and T_g = B_g + K texts
(captions, then hard negatives or extra texts) with their per-sample data. ``global_results`` evaluates every rank's
outputs over the whole global batch with the single-feature oracles. ``node_results`` builds each node's problem with
the package's assignment plan (``cross_node.Topology``: each rank's own texts, then its counterparts' in node order,
with the owners' ids, weights, groups and label sets), evaluates it with the same oracles and folds the remote rows'
gradients and text losses back to their owners in node order, the way the exchange does."""
from __future__ import annotations

import math
from typing import Dict, List, Optional

import numpy as np

from distributed_sigmoid_loss_b200.cross_node import Topology
from exclude_groups_oracle import closed_form_groups, dtxt_of, group_labels, text_loss_of
from extra_images_oracle import label_blocks
from focal_oracle import closed_form_focal
from label_sets_oracle import set_labels

OPTIONS = ("plain", "ids", "extra_texts", "hard_negatives", "weights", "groups", "label_sets", "focal",
           "extra_images")


def make_problem(N: int, L: int, Bs: List[int], D: int, option: str, seed: int, K: int = 2) -> Dict:
    """The global batch of N·L ranks with per-rank batches Bs for one option of OPTIONS. Ids are drawn from a small
    range, so positives cross node boundaries; groups too."""
    W = N * L
    assert len(Bs) == W
    rng = np.random.default_rng(seed)
    k_txt = K if option in ("extra_texts", "hard_negatives", "label_sets") else 0
    k_img = K if option == "extra_images" else 0
    p = dict(N=N, L=L, Bs=list(Bs), D=D, option=option, K=k_txt, K_img=k_img, t_prime=math.log(6.0), bias=-2.5,
             hard_negatives=option == "hard_negatives", multi_label=2 if option == "label_sets" else 0,
             focal=(2.0, 0.25) if option == "focal" else None)
    p["img"] = [rng.standard_normal((b + k_img, D)) / math.sqrt(D) * 2 for b in Bs]
    p["txt"] = [rng.standard_normal((b + k_txt, D)) / math.sqrt(D) * 2 for b in Bs]
    if option in ("ids", "extra_texts", "extra_images"):
        p["ids"] = [rng.integers(0, 5, b) for b in Bs]
    if option == "extra_texts":
        p["extra_text_ids"] = [rng.integers(0, 7, k_txt) for _ in Bs]   # some match no image: hard negatives
    if option == "extra_images":
        p["extra_image_ids"] = [rng.integers(0, 7, k_img) for _ in Bs]
    if option in ("weights", "focal"):
        p["image_weights"] = [np.where(rng.random(b + k_img) < 0.2, 0.0, rng.random(b + k_img)) for b in Bs]
        p["text_weights"] = [np.where(rng.random(b + k_txt) < 0.2, 0.0, rng.random(b + k_txt)) for b in Bs]
    if option == "groups":
        p["image_groups"] = [rng.integers(-1, 4, b + k_img) for b in Bs]
        p["text_groups"] = [rng.integers(-1, 4, b + k_txt) for b in Bs]
    if option == "label_sets":
        p["sample_labels"] = [rng.integers(-1, 6, (b, 2)) for b in Bs]
        p["extra_text_labels"] = [rng.integers(-1, 6, (k_txt, 2)) for _ in Bs]
    return p


def _text_ids(p, g) -> Optional[np.ndarray]:
    """Ids of rank g's T_g texts (captions' sample ids, then the extra texts' ids), or None without ids."""
    if "ids" not in p:
        return None
    if "extra_text_ids" in p:
        return np.concatenate([p["ids"][g], p["extra_text_ids"][g]])
    return np.asarray(p["ids"][g])


def _text_sets(p, g) -> np.ndarray:
    return np.concatenate([p["sample_labels"][g], p["extra_text_labels"][g]])


def _image_sets(p, g) -> np.ndarray:
    return np.asarray(p["sample_labels"][g])


def _evaluate(p, imgs, txts, Bs, ids, text_ids, image_ids, image_w, text_w, image_groups, text_groups, image_sets,
              text_sets) -> List[Dict]:
    """Every rank of one problem (ranks r with images imgs[r], chunks c with texts txts[c]) through the label
    builders and closed_form_groups / closed_form_focal. text_ids[c]: the ids of chunk c's extra texts (past B_c)."""
    Rs, Ts = [len(x) for x in imgs], [len(x) for x in txts]
    if image_sets is not None:
        labels = set_labels(image_sets, text_sets, Bs)
    elif ids is not None:
        labels = label_blocks(Bs, Rs, Ts, ids, text_ids, image_ids)
    else:
        labels = label_blocks(Bs, Rs, Ts)
    if image_groups is not None:
        labels = group_labels(labels, image_groups, text_groups)
    if p["focal"] is not None:
        return closed_form_focal(imgs, txts, p["t_prime"], p["bias"], labels, *p["focal"], batches=Bs,
                                 image_weights=image_w, text_weights=text_w)
    return closed_form_groups(imgs, txts, p["t_prime"], p["bias"], labels, Bs, image_w, text_w)


def _out(res, r, dtxt, text_loss) -> Dict:
    x = res[r]
    return dict(loss=x["loss"], dimg=x["dimg"], dtxt=dtxt, dt_prime=x["dt_prime"], dbias=x["dbias"],
                image_loss=x["image_loss"], text_loss=text_loss)


def global_results(p) -> List[Dict]:
    """Per group rank: loss, dimg [R, D], dtxt [T, D], dt_prime, dbias, image_loss [R], text_loss [T] over the whole
    global batch."""
    W = p["N"] * p["L"]
    g = range(W)
    extra_ids = [np.asarray(_text_ids(p, c))[p["Bs"][c]:] for c in g] if "extra_text_ids" in p else None
    res = _evaluate(p, p["img"], p["txt"], p["Bs"], p.get("ids"), extra_ids, p.get("extra_image_ids"),
                    p.get("image_weights"), p.get("text_weights"), p.get("image_groups"), p.get("text_groups"),
                    [_image_sets(p, c) for c in g] if p["multi_label"] else None,
                    [_text_sets(p, c) for c in g] if p["multi_label"] else None)
    return [_out(res, r, dtxt_of(res, r), text_loss_of(res, r)) for r in g]


def node_chunk(p, owners, per_rank) -> np.ndarray:
    """A node chunk of per-text data: the owners' rows, in the plan's order."""
    return np.concatenate([np.asarray(per_rank[o]) for o in owners])


def node_results(p) -> List[Dict]:
    """Per group rank, the same outputs computed node by node: each node's problem from the assignment plan, the
    remote rows' gradients and text losses added to their owners' in node order."""
    N, L, Bs = p["N"], p["L"], p["Bs"]
    W = N * L
    Ts = [len(x) for x in p["txt"]]
    node_out = {}
    for n in range(N):
        ranks = [n * L + l for l in range(L)]
        owners = [Topology(g, W, L).text_owners() for g in ranks]
        txts = [node_chunk(p, o, p["txt"]) for o in owners]
        nB = [Bs[g] for g in ranks]
        ids = extra_ids = None
        if "ids" in p:
            ids = [p["ids"][g] for g in ranks]
            # the engine's extra-text ids: everything past the rank's own captions
            extra_ids = [node_chunk(p, o, [_text_ids(p, c) for c in range(W)])[Bs[g]:] for g, o in zip(ranks, owners)]
        sets = None
        if p["multi_label"]:
            tsets = [np.concatenate([p["sample_labels"][c],
                                     p["extra_text_labels"][c] if not p["hard_negatives"] else
                                     np.full((p["K"], 2), -1)]) for c in range(W)]
            sets = ([_image_sets(p, g) for g in ranks], [node_chunk(p, o, tsets) for o in owners])
        res = _evaluate(p, [p["img"][g] for g in ranks], txts, nB, ids, extra_ids,
                        [p["extra_image_ids"][g] for g in ranks] if "extra_image_ids" in p else None,
                        [p["image_weights"][g] for g in ranks] if "image_weights" in p else None,
                        [node_chunk(p, o, p["text_weights"]) for o in owners] if "text_weights" in p else None,
                        [p["image_groups"][g] for g in ranks] if "image_groups" in p else None,
                        [node_chunk(p, o, p["text_groups"]) for o in owners] if "text_groups" in p else None,
                        *(sets if sets is not None else (None, None)))
        for l, (g, o) in enumerate(zip(ranks, owners)):
            node_out[g] = (res, l, o)
    out = []
    for g in range(W):
        res, l, _ = node_out[g]
        # the owner's rows in every node's chunk: node n' holds them at rank (n', l) past the earlier owners' rows
        dtxt, tl = None, None
        for n in range(N):
            h = n * L + g % L
            res_h, l_h, o_h = node_out[h]
            start = sum(Ts[x] for x in o_h[:o_h.index(g)])
            d = dtxt_of(res_h, l_h)[start:start + Ts[g]]
            t = text_loss_of(res_h, l_h)[start:start + Ts[g]]
            dtxt = d if dtxt is None else dtxt + d
            tl = t if tl is None else tl + t
        out.append(_out(res, l, dtxt, tl))
    return out
