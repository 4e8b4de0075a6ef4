"""CPU checks of process groups that span nodes: the assignment plan reproduces the global-batch loss node by node
(float64, every option the exchange carries data for), the topology derivation and its errors, every refusal, and the
exchange itself on local gloo processes against a direct computation."""
import datetime
import math
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from cross_node_oracle import OPTIONS, global_results, make_problem, node_results
from distributed_sigmoid_loss_b200 import loss as loss_mod
from distributed_sigmoid_loss_b200.cross_node import (Topology, exchange_texts, node_mean_scalars,
                                                      ranks_per_node_of_hosts, return_rows, send_rows,
                                                      validate_ranks_per_node)
from extra_text_ids_oracle import closed_form_extra_text_ids
from hard_negatives_oracle import closed_form_hard_negatives
from oracle.siglip_oracle import closed_form_uneven

SHAPES = [(2, 1, [3, 5]), (3, 1, [4, 2, 5]), (2, 2, [3, 4, 5, 2]), (2, 3, [2, 4, 3, 5, 3, 4]),
          (4, 2, [3, 2, 4, 3, 2, 5, 3, 4])]


def _close(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    np.testing.assert_allclose(a, b, rtol=1e-12, atol=1e-12 * max(1.0, float(np.abs(b).max(initial=0.0))))


@pytest.mark.parametrize("option", OPTIONS)
@pytest.mark.parametrize("N,L,Bs", SHAPES)
def test_node_problems_give_the_global_batch(N, L, Bs, option):
    p = make_problem(N, L, Bs, 6, option, seed=N * 31 + L * 7 + OPTIONS.index(option))
    want, got = global_results(p), node_results(p)
    for g in range(N * L):
        for k in ("loss", "dimg", "dtxt", "dt_prime", "dbias", "image_loss", "text_loss"):
            _close(got[g][k], want[g][k])
    if option == "ids":   # positives across node boundaries exist
        ids = p["ids"]
        assert any(set(ids[a]) & set(ids[b]) for a in range(N * L) for b in range(N * L) if a // L != b // L)


def _fold(node_res, p, key="contrib"):
    """Text gradient of every group rank from per-node closed forms whose result lists index node ranks."""
    N, L = p["N"], p["L"]
    W = N * L
    Ts = [len(x) for x in p["txt"]]
    out = [np.zeros_like(x) for x in p["txt"]]
    for n in range(N):
        for l in range(L):
            owners = Topology(n * L + l, W, L).text_owners()
            chunk = sum(x[key][l] for x in node_res[n])
            start = 0
            for o in owners:
                out[o] += chunk[start:start + Ts[o]]
                start += Ts[o]
    return out


@pytest.mark.parametrize("N,L,Bs", SHAPES)
def test_plain_and_hard_negatives_through_the_single_feature_oracles(N, L, Bs):
    """Global: closed_form_uneven (plain) / closed_form_hard_negatives; nodes: the remote rows as the hard negatives
    of closed_form_hard_negatives."""
    for option in ("plain", "hard_negatives"):
        p = make_problem(N, L, Bs, 5, option, seed=N + 10 * L)
        W = N * L
        caps = [t[:b] for t, b in zip(p["txt"], Bs)]
        exts = [t[b:] for t, b in zip(p["txt"], Bs)]
        if option == "plain":
            want = closed_form_uneven(p["img"], caps, p["t_prime"], p["bias"])
        else:
            want = closed_form_hard_negatives(p["img"], caps, exts, p["t_prime"], p["bias"])
        node_res = []
        for n in range(N):
            ranks = [n * L + l for l in range(L)]
            owned = [Topology(g, W, L).text_owners() for g in ranks]
            node_res.append(closed_form_hard_negatives(
                [p["img"][g] for g in ranks], [caps[g] for g in ranks],
                [np.concatenate([exts[o[0]]] + [p["txt"][x] for x in o[1:]]) for o in owned], p["t_prime"], p["bias"]))
        dtxt = _fold(node_res, p)
        for g in range(W):
            x = node_res[g // L][g % L]
            for k in ("loss", "dimg", "dt_prime", "dbias"):
                _close(x[k], want[g][k])
            _close(dtxt[g], sum(r["contrib"][g] for r in want))


@pytest.mark.parametrize("N,L,Bs", SHAPES)
def test_ids_and_extra_texts_through_the_extra_text_ids_oracle(N, L, Bs):
    """Remote captions carry their owners' sample ids as extra-text ids, remote extra texts their own ids."""
    p = make_problem(N, L, Bs, 5, "extra_texts", seed=3 * N + L)
    W = N * L
    caps = [t[:b] for t, b in zip(p["txt"], Bs)]
    exts = [t[b:] for t, b in zip(p["txt"], Bs)]
    tids = [np.concatenate([p["ids"][c], p["extra_text_ids"][c]]) for c in range(W)]
    want = closed_form_extra_text_ids(p["img"], caps, exts, p["ids"], p["extra_text_ids"], p["t_prime"], p["bias"])
    node_res = []
    for n in range(N):
        ranks = [n * L + l for l in range(L)]
        owned = [Topology(g, W, L).text_owners() for g in ranks]
        node_res.append(closed_form_extra_text_ids(
            [p["img"][g] for g in ranks], [caps[g] for g in ranks],
            [np.concatenate([exts[o[0]]] + [p["txt"][x] for x in o[1:]]) for o in owned], [p["ids"][g] for g in ranks],
            [np.concatenate([p["extra_text_ids"][o[0]]] + [tids[x] for x in o[1:]]) for o in owned],
            p["t_prime"], p["bias"]))
    dtxt = _fold(node_res, p)
    for g in range(W):
        x = node_res[g // L][g % L]
        for k in ("loss", "dimg", "dt_prime", "dbias"):
            _close(x[k], want[g][k])
        _close(dtxt[g], sum(r["contrib"][g] for r in want))


def test_node_mean_of_node_means_is_the_group_mean():
    p = make_problem(2, 3, [2, 4, 3, 5, 3, 4], 5, "plain", seed=1)
    want = global_results(p)
    node_means = [np.mean([want[n * 3 + l]["dt_prime"] for l in range(3)]) for n in range(2)]
    assert sum(node_means) / 2 == pytest.approx(np.mean([w["dt_prime"] for w in want]), rel=1e-13)


# -- topology --------------------------------------------------------------------------------------------------------
def test_plan_of_a_rank():
    t = Topology(5, 8, 2)
    assert (t.nodes, t.node, t.local, t.node_base) == (4, 2, 1, 4)
    assert t.counterparts() == [1, 3, 7]
    assert t.text_owners() == [5, 1, 3, 7]
    assert t.node_texts_per_rank([1, 2, 3, 4, 5, 6, 7, 8]) == [16, 20]
    # every remote text is an extra of exactly one rank of each other node
    W, L = 12, 3
    for owner in range(W):
        holders = [g for g in range(W) if owner in Topology(g, W, L).text_owners()]
        assert sorted({h // L for h in holders}) == list(range(W // L))
        assert all(h % L == owner % L for h in holders)


def test_ranks_per_node_from_hostnames():
    assert ranks_per_node_of_hosts(["a"] * 4) == 4
    assert ranks_per_node_of_hosts(["a", "a", "b", "b", "c", "c"]) == 2
    assert ranks_per_node_of_hosts(["a", "b", "c"]) == 1
    with pytest.raises(RuntimeError, match="not consecutive"):
        ranks_per_node_of_hosts(["a", "b", "a", "b"])
    with pytest.raises(RuntimeError, match="different numbers of ranks"):
        ranks_per_node_of_hosts(["a", "a", "b"])


@pytest.mark.parametrize("bad", [0, -1, 1.5, True, "2"])
def test_ranks_per_node_argument(bad):
    assert validate_ranks_per_node(None) is None and validate_ranks_per_node(3) == 3
    with pytest.raises(RuntimeError, match="ranks_per_node"):
        validate_ranks_per_node(bad)
    with pytest.raises(RuntimeError, match="ranks_per_node"):
        loss_mod.DDPSigmoidLoss(8, ranks_per_node=bad)
    with pytest.raises(RuntimeError, match="ranks_per_node"):
        loss_mod.SigLipLoss(ranks_per_node=bad)


# -- refusals --------------------------------------------------------------------------------------------------------
def _cache_across_nodes(**kw):
    cache = loss_mod.DDPSigmoidLoss(8, **kw)._cache
    cache._topology, cache._topology_known = Topology(0, 4, 2), True
    return cache


@pytest.mark.parametrize("kw,what", [(dict(distill=0.5), "distill"),
                                     (dict(multi_positive=True, hard_negatives=2), "hard_negatives with multi_positive")])
def test_options_refused_across_nodes(kw, what):
    cache = _cache_across_nodes(**kw)
    with pytest.raises(RuntimeError, match=f"{what}.*across nodes"):
        cache.get(8, 16, torch.device("cuda", 0))


def test_single_node_group_needs_no_topology():
    # without an initialised process group there is one node and no exchange
    assert loss_mod.cross_node.topology(None, None) is None
    assert loss_mod.cross_node.topology(None, 1) is None


def test_metrics_refused_across_nodes():
    loss_mod.cross_node.check_forward(False)
    with pytest.raises(RuntimeError, match="return_metrics / metrics_topk are unavailable across nodes"):
        loss_mod.cross_node.check_forward(True)


def test_host_entries_refused_across_nodes():
    eng = loss_mod.SigmoidLossEngine.__new__(loss_mod.SigmoidLossEngine)
    eng.topology = Topology(0, 2, 1)
    x = torch.zeros(4, 8, dtype=torch.bfloat16)
    for call in (lambda: eng.fwd_bwd_host(x, x, 0.0, 0.0), lambda: eng.host_submit(x, x, 0.0, 0.0)):
        with pytest.raises(RuntimeError, match="host-buffer entries are unavailable across nodes"):
            call()


# -- the exchange on local gloo processes ---------------------------------------------------------------------------
D = 3


def _rows(g, T):
    return torch.arange(T * D, dtype=torch.float64).reshape(T, D) + 1000 * g


def _weight(g, rows):
    gen = torch.Generator().manual_seed(100 + g)
    return torch.randn(rows, D, generator=gen, dtype=torch.float64)


def _worker(rank, world, L, store, Ts):
    dist.init_process_group("gloo", init_method=f"file://{store}", rank=rank, world_size=world,
                            timeout=datetime.timedelta(seconds=60))
    try:
        topo = Topology(rank, world, L)
        T = Ts[rank]
        own = _rows(rank, T).requires_grad_(True)
        tp = torch.tensor(0.5 + rank, dtype=torch.float64, requires_grad=True)
        b = torch.tensor(-1.0 - rank, requires_grad=True)
        node_text, tp2, b2 = exchange_texts(own, tp, b, topo, Ts, None, True)
        # forward rows: own, then the counterparts' rows in node order; the node context's size
        want = torch.cat([_rows(o, Ts[o]) for o in topo.text_owners()])
        assert torch.equal(node_text.detach(), want)
        assert node_text.shape[0] == topo.node_texts_per_rank(Ts)[topo.local]
        # backward: the gradient of sum over ranks of <node_text_h, W_h> for own rows, computed directly
        scal = tp2 * (rank + 1) + b2 * (2 * rank + 1)   # the exchange takes each node's value from its local rank 0
        ((node_text * _weight(rank, node_text.shape[0])).sum() + scal).backward()
        direct = torch.zeros(T, D, dtype=torch.float64)
        for h in range(world):
            owners = Topology(h, world, L).text_owners()
            if rank in owners:
                start = sum(Ts[o] for o in owners[:owners.index(rank)])
                direct += _weight(h, sum(Ts[o] for o in owners))[start:start + T]
        torch.testing.assert_close(own.grad, direct, rtol=1e-15, atol=1e-12)
        # scalars: the mean over nodes of each node's value (rank n·L's), the same on every rank
        want_tp = sum(n * L + 1 for n in range(world // L)) / (world // L)
        want_b = sum(2 * n * L + 1 for n in range(world // L)) / (world // L)
        assert float(tp.grad) == want_tp and float(b.grad) == pytest.approx(want_b)
        g_all = [torch.empty(2, dtype=torch.float64) for _ in range(world)]
        dist.all_gather(g_all, torch.stack([tp.grad, b.grad.double()]))
        assert all(torch.equal(x, g_all[0]) for x in g_all)
        # per-text values: remote rows' values back to their owners, own + others in node order
        vals = torch.cat([torch.full((Ts[o],), float(rank + 1)) for o in topo.text_owners()])
        folded = return_rows(vals[T:], vals[:T], topo, Ts, None)
        expect = sum(h + 1 for h in range(world) if rank in Topology(h, world, L).text_owners())
        assert torch.equal(folded, torch.full((T,), float(expect)))
        # int64 rows ride unchanged
        meta = torch.stack([torch.arange(T) + 100 * rank, -torch.arange(T)], dim=1)
        remote = send_rows(meta, topo, Ts, None)
        assert torch.equal(remote, torch.cat([torch.stack([torch.arange(Ts[o]) + 100 * o, -torch.arange(Ts[o])], 1)
                                              for o in topo.counterparts()]))
        assert float(node_mean_scalars(torch.tensor(1.0), torch.tensor(2.0), topo, None)[1]) == 2.0
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world,L", [(3, 1), (4, 1), (4, 2)])
def test_exchange_on_gloo_processes(tmp_path, world, L):
    Ts = [3, 5, 2, 4][:world]
    mp.spawn(_worker, args=(world, L, str(tmp_path / "store"), Ts), nprocs=world, join=True)
