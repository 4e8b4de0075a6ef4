"""Process groups that span nodes: the topology, the assignment of remote texts and their exchange.

The in-kernel exchange of a loss context reaches the GPUs of one node only (CUDA-IPC peer memory). A group of N nodes
of L ranks each (rank g = n·L + l of the group) still computes the global-batch loss: rank (n, l) appends to its own
T_(n,l) text rows (captions, then its hard negatives or extra texts) the rows of its counterparts (n', l), n' != n, in
node order, as extra texts of its node's context. Every remote text is then an extra of exactly one rank of each other
node, and the node's in-kernel exchange lets every image of that node score it once, so each image meets every text
of the global batch exactly once. The node context of local rank l holds T_l = sum_n' T_(n',l) texts, the same on every
node.

Forward, one all_to_all_single over the group sends each rank's rows to its N - 1 counterparts; backward, the reverse
one returns the remote rows' gradients, which the owner adds to its own in node order (deterministic). Rows travel as
raw bytes, so every dtype goes through NCCL and gloo alike."""
from __future__ import annotations

import socket
from typing import List, NamedTuple, Optional, Sequence

import torch
import torch.distributed as dist


class Topology(NamedTuple):
    """Rank `rank` of a group of `world` ranks in nodes of `ranks_per_node` consecutive ranks."""
    rank: int
    world: int
    ranks_per_node: int

    @property
    def nodes(self) -> int:
        return self.world // self.ranks_per_node

    @property
    def node(self) -> int:
        return self.rank // self.ranks_per_node

    @property
    def local(self) -> int:
        return self.rank % self.ranks_per_node

    @property
    def node_base(self) -> int:
        """Group rank of local rank 0 of this rank's node."""
        return self.node * self.ranks_per_node

    def counterparts(self) -> List[int]:
        """Group ranks (n', l) of the other nodes, in node order: the owners of this rank's remote text rows."""
        L = self.ranks_per_node
        return [n * L + self.local for n in range(self.nodes) if n != self.node]

    def text_owners(self) -> List[int]:
        """Owner of each block of this rank's node-context texts: itself first, then its counterparts."""
        return [self.rank] + self.counterparts()

    def node_texts_per_rank(self, texts_per_rank: Sequence[int]) -> List[int]:
        """texts_per_rank of the node context, from the group's per-rank text counts: sum over nodes per local rank."""
        L = self.ranks_per_node
        return [sum(int(texts_per_rank[n * L + l]) for n in range(self.nodes)) for l in range(L)]


def validate_ranks_per_node(ranks_per_node) -> Optional[int]:
    if ranks_per_node is None:
        return None
    if isinstance(ranks_per_node, bool) or not isinstance(ranks_per_node, int) or ranks_per_node < 1:
        raise RuntimeError(f"ranks_per_node must be None or an int >= 1, got {ranks_per_node!r}")
    return ranks_per_node


def ranks_per_node_of_hosts(hosts: Sequence[str]) -> int:
    """L from the hostname of every rank of a group: each host must hold one block of consecutive ranks, and every
    host the same number of them."""
    blocks = []   # (host, ranks)
    for h in hosts:
        if blocks and blocks[-1][0] == h:
            blocks[-1][1] += 1
        else:
            blocks.append([h, 1])
    seen = [b[0] for b in blocks]
    if len(set(seen)) != len(seen):
        host = next(h for h in seen if seen.count(h) > 1)
        raise RuntimeError(f"the ranks of host '{host}' are not consecutive in the process group (hosts by rank: "
                           f"{list(hosts)}): a node must be a block of consecutive ranks; order the ranks by host "
                           f"or pass ranks_per_node")
    sizes = {b[1] for b in blocks}
    if len(sizes) != 1:
        raise RuntimeError(f"the nodes of the process group hold different numbers of ranks "
                           f"({', '.join(f'{h}: {n}' for h, n in blocks)}): nodes of unequal size are not supported")
    return blocks[0][1]


def topology(group, ranks_per_node: Optional[int]) -> Optional[Topology]:
    """The group's topology when it spans more than one node, None when it fits one (today's path). ranks_per_node
    None gathers every rank's hostname over the group once. Collective over the group when it has more than one rank."""
    if not (dist.is_available() and dist.is_initialized()):
        return None
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    if world == 1:
        return None
    if ranks_per_node is None:
        hosts = [None] * world
        dist.all_gather_object(hosts, socket.gethostname(), group=group)
        ranks_per_node = ranks_per_node_of_hosts(hosts)
    if world % ranks_per_node:
        raise RuntimeError(f"ranks_per_node={ranks_per_node} does not divide the group's {world} ranks: nodes of "
                           f"unequal size are not supported")
    if ranks_per_node == world:
        return None
    return Topology(rank, world, ranks_per_node)


def check_options(distill, multi_positive: bool, hard_negatives: int) -> None:
    """The module options a group that spans nodes refuses."""
    if distill is not None:
        raise RuntimeError("distill is unavailable across nodes: the teacher rows would have to travel with the "
                           "texts; give each node its own group")
    if multi_positive and hard_negatives:
        raise RuntimeError("hard_negatives with multi_positive is unavailable across nodes: a remote hard negative "
                           "would need an id that matches no image (use extra_texts with such ids)")


def check_forward(return_metrics: bool) -> None:
    if return_metrics:
        raise RuntimeError("return_metrics / metrics_topk are unavailable across nodes: a text's best image over all "
                           "nodes needs the scores, and the metrics export only indices")


# -- the exchange ---------------------------------------------------------------------------------------------------
def _splits(topo: Topology, texts_per_rank: Sequence[int]):
    """(rows sent to, rows received from) every group rank: this rank's T to each counterpart, T_(n',l) from it."""
    mine = int(texts_per_rank[topo.rank])
    send, recv = [0] * topo.world, [0] * topo.world
    for g in topo.counterparts():
        send[g] = mine
        recv[g] = int(texts_per_rank[g])
    return send, recv


def _all_to_all_rows(x: torch.Tensor, send: List[int], recv: List[int], group) -> torch.Tensor:
    """all_to_all_single of the rows of x (send[g] rows to rank g, in rank order), moved as bytes."""
    x = x.contiguous()
    row_shape = tuple(x.shape[1:])
    xb = x.reshape(x.shape[0], -1).view(torch.uint8)
    out = torch.empty(sum(recv), xb.shape[1], dtype=torch.uint8, device=x.device)
    dist.all_to_all_single(out, xb, output_split_sizes=recv, input_split_sizes=send, group=group)
    return out.view(x.dtype).reshape(sum(recv), *row_shape)


def send_rows(own: torch.Tensor, topo: Topology, texts_per_rank: Sequence[int], group) -> torch.Tensor:
    """Forward exchange: this rank's own rows [T, ...] go to each counterpart; returns the counterparts' rows
    [sum T_(n',l), ...] in node order (the remote part of the node-context texts)."""
    send, recv = _splits(topo, texts_per_rank)
    return _all_to_all_rows(torch.cat([own] * (topo.nodes - 1)), send, recv, group)


def return_rows(remote: torch.Tensor, own: torch.Tensor, topo: Topology, texts_per_rank: Sequence[int],
                group) -> torch.Tensor:
    """Reverse exchange: the values of the remote rows go back to their owners, and each owner returns its own values
    plus the other nodes' values for the same rows, added in node order in fp32 (fp64 for fp64) and cast back to own's
    dtype."""
    send, recv = _splits(topo, texts_per_rank)
    back = _all_to_all_rows(remote, recv, send, group)
    parts = list(back.split(int(texts_per_rank[topo.rank])))
    parts.insert(topo.node, own)
    acc = torch.promote_types(own.dtype, torch.float32)
    total = parts[0].to(acc)
    for p in parts[1:]:
        total = total + p.to(acc)
    return total.to(own.dtype)


class _ExchangeFn(torch.autograd.Function):
    """[own; remote rows] forward, the remote rows' gradients folded back into the own rows' backward. With
    sync_scalar_grads the two scalars pass through it too, and their gradients (already the node mean) are averaged
    over the nodes, so both collectives of the backward run in one fixed order on every rank."""

    @staticmethod
    def forward(ctx, own, t_prime, bias, topo: Topology, texts_per_rank, group, sync_scalars: bool):
        ctx.topo, ctx.tpr, ctx.group, ctx.sync, ctx.rows = topo, texts_per_rank, group, sync_scalars, own.shape[0]
        remote = send_rows(own.detach(), topo, texts_per_rank, group)
        node_text = torch.cat([own.detach(), remote])
        ctx.like = torch.empty((0,) + tuple(node_text.shape[1:]), dtype=node_text.dtype, device=node_text.device)
        ctx.node_rows = node_text.shape[0]
        ctx.scalar_meta = ((t_prime.shape, t_prime.dtype, t_prime.device), (bias.shape, bias.dtype, bias.device))
        return node_text, t_prime.detach().clone(), bias.detach().clone()

    @staticmethod
    def backward(ctx, grad_text, grad_tp, grad_b):
        gt = None
        if ctx.needs_input_grad[0]:
            if grad_text is None:   # the reverse exchange is collective: every rank takes part
                grad_text = ctx.like.new_zeros((ctx.node_rows,) + tuple(ctx.like.shape[1:]))
            gt = return_rows(grad_text[ctx.rows:], grad_text[:ctx.rows], ctx.topo, ctx.tpr, ctx.group)
        if ctx.sync and (ctx.needs_input_grad[1] or ctx.needs_input_grad[2]):
            grad_tp, grad_b = (g if g is not None else torch.zeros(shape, dtype=dt, device=dev)
                               for g, (shape, dt, dev) in zip((grad_tp, grad_b), ctx.scalar_meta))
            grad_tp, grad_b = node_mean_scalars(grad_tp, grad_b, ctx.topo, ctx.group)
        return gt, grad_tp, grad_b, None, None, None, None


def node_mean_scalars(dtp: torch.Tensor, db: torch.Tensor, topo: Topology, group):
    """The mean over nodes of two scalar gradients that are already the mean over each node's ranks (bit-identical
    within a node): gathered over the group, the node values added in node order in fp64, divided by N. The result
    is the mean over every rank of the group (equal node sizes), bit-identical on all of them."""
    mine = torch.stack([dtp.detach().reshape(()).double(), db.detach().reshape(()).double()])
    vals = [torch.empty_like(mine) for _ in range(topo.world)]
    dist.all_gather(vals, mine, group=group)
    total = vals[0]
    for n in range(1, topo.nodes):
        total = total + vals[n * topo.ranks_per_node]
    total = total / topo.nodes
    return total[0].reshape(dtp.shape).to(dtp.dtype), total[1].reshape(db.shape).to(db.dtype)


def exchange_texts(own: torch.Tensor, t_prime: torch.Tensor, bias: torch.Tensor, topo: Topology,
                   texts_per_rank: Sequence[int], group, sync_scalars: bool):
    """(node-context texts [T_l, D], t_prime, bias) for a rank's own text rows [T, D] (its captions, then its extras),
    differentiable in all three: text_embeddings.grad sums the node-local and the remote contributions."""
    return _ExchangeFn.apply(own, t_prime, bias, topo, list(texts_per_rank), group, bool(sync_scalars))
