"""Float64 oracle of the loss with labels from sample ids (SIGLIP_OPT_SAMPLE_IDS) — test infrastructure, never the
product path. It extends ``oracle.siglip_oracle.closed_form_uneven`` (pinned on the reference's fixtures) with the id
label matrix; ``tests/test_sample_ids_cpu.py`` checks it against that function for unique ids and against float64
autograd of the reference's op sequence for duplicated ids."""
from __future__ import annotations

import math
from typing import Dict, List

import numpy as np

from oracle.siglip_oracle import _sigmoid, _softplus


def closed_form_ids(img_blocks, txt_blocks, id_blocks, t_prime: float, bias: float) -> List[Dict]:
    """`closed_form_uneven` with labels from sample ids (an extension the reference cannot run): image i of rank r and
    text j of chunk c are a positive pair iff id_blocks[r][i] == id_blocks[c][j], every other pair is a negative. Image
    i and text i of a rank share id_blocks[r][i], so the own-chunk diagonal is always positive, and unique ids give
    `closed_form_uneven`'s labels. Loss and gradients keep the formulas of distributed_sigmoid_loss.py:24-47 with these
    labels (loss divided by the rank's own batch). img_blocks[r]: [B_r, D], txt_blocks[c]: [B_c, D], id_blocks[r]:
    [B_r] integers. Returns per rank: loss, dimg [B_r, D], dt_prime, dbias and contrib[c] ([B_c, D], that rank's
    contribution to chunk c's text gradient)."""
    t = math.exp(t_prime)
    ids = [np.asarray(x, dtype=np.int64) for x in id_blocks]
    out = []
    for r, img in enumerate(img_blocks):
        img = np.asarray(img, dtype=np.float64)
        br = img.shape[0]
        res = dict(loss=0.0, dimg=np.zeros_like(img), dt_prime=0.0, dbias=0.0, contrib=[])
        for c, txt in enumerate(txt_blocks):
            txt = np.asarray(txt, dtype=np.float64)
            s = img @ txt.T
            z = t * s + bias
            y = np.where(ids[r][:, None] == ids[c][None, :], 1.0, -1.0)
            g = -y * _sigmoid(-y * z) / br
            res["loss"] += float(_softplus(-y * z).sum() / br)
            res["dimg"] += t * (g @ txt)
            res["contrib"].append(t * (g.T @ img))
            res["dt_prime"] += float(t * (g * s).sum())
            res["dbias"] += float(g.sum())
        out.append(res)
    return out
