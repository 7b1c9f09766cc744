"""Cases, host references and a one-device emulator of the sequence-sharded expert-parallel prefill
(MixtralDecoder._prefill_ep_seq).  Importable without a GPU.

The EP kernels address every peer through raw device pointers, so on one GPU the N "ranks" can be N ordinary
allocations (`LocalPeers`).  `run_ep_prefill` builds N decoders over them and steps their prefill generators
(`_prefill_ep_seq_steps`, one yield after each ep_signal) round-robin, phase by phase.  A host model of the epoch
flags (`FlagModel`) follows every ep_signal and is consulted before every ep_wait / ep_reduce_norm_gather, which is
refused before it is launched if a flag it needs is not set: no wait kernel is ever launched that could spin.
"""
from __future__ import annotations

from typing import Callable, Dict, List, Sequence, Tuple

import torch

from vita_b200.parallel import token_range
from vita_b200.weights import expert_range

BF16 = torch.bfloat16
E = 8                  # Mixtral experts (tiny and full configs alike)
WHICH = (0, 2, 3)      # flag groups in use: 2 = K/V rows, 3 = routed rows, 0 = expert rows at their owner

# ------------------------------------------------------------------------------------------------ sequence cases
# (N, S): S = 37 leaves rank 3 of 4 and ranks 5-7 of 8 without tokens and 13 (odd) tokens on rank 1 of 2; S = 300 is
# the two-GPU check's case; S = 4096 at N = 8 is the serving shape of the 8-GPU prefill (chunk 512)
SEQ_CASES = [(2, 37), (2, 300), (4, 37), (4, 300), (8, 37), (8, 300), (8, 4096)]


def rank_tokens(S: int, N: int) -> List[Tuple[int, int]]:
    return [token_range(S, r, N) for r in range(N)]


def empty_ranks(S: int, N: int) -> List[int]:
    return [r for r, (t0, t1) in enumerate(rank_tokens(S, N)) if t1 == t0]


def odd_ranks(S: int, N: int) -> List[int]:
    """Ranks whose 8-byte routing records (n * 8 bytes) end in a 4-byte-word tail of the push (not a 16-byte multiple)."""
    return [r for r, (t0, t1) in enumerate(rank_tokens(S, N)) if (t1 - t0) % 2]


# ------------------------------------------------------------------------------------------------ routings
def counts_empty_and_full(S: int) -> List[int]:
    """Expert 2 receives every token, expert 5 none; the other six share the remaining S assignments."""
    c = [0] * E
    c[2] = S
    rest = [0, 1, 3, 4, 6, 7]
    for i, e in enumerate(rest):
        c[e] = S // 6 + (1 if i < S % 6 else 0)
    return c


# per-expert counts at and around multiples of 128 (empty experts included); sum = 2 S, each <= S
COUNTS_NEAR_128 = {
    300: [127, 0, 129, 1, 128, 85, 1, 129],
    4096: [1023, 1025, 0, 2047, 129, 1919, 2049, 0],
}


def routing_from_counts(counts: Sequence[int], S: int, seed: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """Top-2 routing [S, 2] int32 / weights [S, 2] fp32 in which expert e gets exactly counts[e] of the 2 S
    assignments.  The sorted multiset's elements t and t + S never coincide when every count is <= S, so each token
    gets two different experts; tokens and the order of a token's pair are then shuffled."""
    assert sum(counts) == 2 * S and max(counts) <= S
    g = torch.Generator().manual_seed(seed)
    flat = torch.repeat_interleave(torch.arange(E), torch.tensor(counts))
    ids = torch.stack([flat[:S], flat[S:]], 1)
    ids = ids[torch.randperm(S, generator=g)]
    swap = torch.rand(S, generator=g) < 0.5
    ids[swap] = ids[swap].flip(1)
    return ids.to(torch.int32).contiguous(), routing_weights(S, g)


def routing_random(S: int, seed: int) -> Tuple[torch.Tensor, torch.Tensor]:
    g = torch.Generator().manual_seed(seed)
    ids = torch.rand(S, E, generator=g).topk(2, dim=-1).indices
    return ids.to(torch.int32).contiguous(), routing_weights(S, g)


def routing_weights(S: int, g) -> torch.Tensor:
    """Renormalised top-2 weights: w0 in [0.5, 1), w1 = 1 - w0 (fp32)."""
    w0 = 0.5 + 0.5 * torch.rand(S, generator=g)
    return torch.stack([w0, 1.0 - w0], 1).float().contiguous()


def routing(kind: str, S: int, seed: int = 0):
    if kind == "empty+full":
        return routing_from_counts(counts_empty_and_full(S), S, seed)
    if kind == "near128":
        return routing_from_counts(COUNTS_NEAR_128[S], S, seed)
    assert kind == "random"
    return routing_random(S, seed)


def align_ref(ids: torch.Tensor, tw: torch.Tensor):
    """vita_moe_align on the host: stable counting sort of the assignments i = 2 t + k by expert.  Returns offsets
    [E + 1], perm_row [2S] (row of assignment i), row_token [2S], row_weight [2S], row_assign [2S] (assignment of row)."""
    flat = ids.reshape(-1).long()
    order = torch.sort(flat, stable=True).indices
    offs = torch.zeros(E + 1, dtype=torch.int64)
    offs[1:] = torch.cumsum(torch.bincount(flat, minlength=E), 0)
    perm = torch.empty_like(order)
    perm[order] = torch.arange(order.numel())
    return (offs.int(), perm.int(), (order // 2).int(), tw.reshape(-1)[order].float().contiguous(), order.int())


# ------------------------------------------------------------------------------------------------ receive slots
def recv_slot(t: int, k: int, chunk: int) -> Tuple[int, int]:
    """Where the down projection of the expert-parallel prefill stores the output row of assignment (t, k): the owner
    of token t and the row (t - owner * chunk) * 2 + k of its receive buffer."""
    owner = t // chunk
    return owner, (t - owner * chunk) * 2 + k


# ------------------------------------------------------------------------------------------------ references
def reduce_ref(h: torch.Tensor, s0: torch.Tensor, s1: torch.Tensor) -> torch.Tensor:
    """The owner's combine in the kernel's order: bf16(h + (s0 + s1)), each sum in fp32."""
    return (h.float() + (s0.float() + s1.float())).to(BF16)


def rmsnorm64(x: torch.Tensor, w: torch.Tensor, eps: float) -> torch.Tensor:
    x = x.double()
    return x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps) * w.double()


def down_ref64(act: torch.Tensor, w2: torch.Tensor, offs: Sequence[int], rw: torch.Tensor, e_lo: int, e_hi: int):
    """fp64 rows act[r] . w2[e]^T * rw[r] of the rows of experts [e_lo, e_hi) (w2 holds those experts) on act's
    device.  Returns the fp64 rows [rows, H] and their row indices."""
    rows, outs = [], []
    for e in range(e_lo, e_hi):
        r0, r1 = int(offs[e]), int(offs[e + 1])
        if r1 > r0:
            y = act[r0:r1].double() @ w2[e - e_lo].double().T
            outs.append(y * rw[r0:r1, None].double())
            rows.append(torch.arange(r0, r1))
    if not outs:
        return torch.zeros(0, w2.shape[1], dtype=torch.float64, device=act.device), torch.zeros(0, dtype=torch.int64)
    return torch.cat(outs), torch.cat(rows)


# ------------------------------------------------------------------------------------------------ flag model
class FlagNotSet(AssertionError):
    """A wait (or the reduce's built-in wait) was about to be launched on a flag nobody has set: refused before launch."""


class FlagModel:
    """Host copy of every rank's epoch flags: flags[dst][which * N + src] is the epoch rank src last signalled into
    rank dst's flags of group `which` (ep_signal stores it into every rank, itself included)."""

    def __init__(self, n_ranks: int):
        self.N = n_ranks
        self.flags = [[0] * (4 * n_ranks) for _ in range(n_ranks)]

    def signal(self, which: int, src: int, epoch: int):
        assert which in WHICH and 0 <= src < self.N, (which, src)
        for dst in range(self.N):
            self.flags[dst][which * self.N + src] = epoch

    def require(self, rank: int, which: int, epoch: int, n_wait: int):
        """Refuse unless flags[rank][which][src] >= epoch for every src < n_wait."""
        assert which in WHICH and 0 <= rank < self.N and 0 <= n_wait <= self.N, (rank, which, n_wait)
        missing = [s for s in range(n_wait) if self.flags[rank][which * self.N + s] < epoch]
        if missing:
            raise FlagNotSet(f"rank {rank} would wait for flags[{which}][{missing}] >= {epoch}, "
                             f"which hold {[self.flags[rank][which * self.N + s] for s in missing]}")

    def table(self) -> torch.Tensor:
        return torch.tensor(self.flags, dtype=torch.int32)


def guarded_ops(model: FlagModel, real, rank_of: Callable) -> Dict[str, Callable]:
    """ep_signal / ep_wait / ep_reduce_norm_gather with the signatures of vita_b200.ops: each signal is launched
    (`real`'s op) and recorded in `model`; each wait and reduce is checked against `model` first and raises FlagNotSet
    instead of launching when a flag it needs is missing.  rank_of(my_flags) names the rank whose flags are waited on."""
    N = model.N

    def ep_signal(peer_flag_ptrs, which, n_ranks, my_rank, epoch):
        assert n_ranks == N
        real.ep_signal(peer_flag_ptrs, which, n_ranks, my_rank, epoch)
        model.signal(which, my_rank, epoch)

    def ep_wait(my_flags, which, n_ranks, epoch, n_wait=None):
        assert n_ranks == N
        model.require(rank_of(my_flags), which, epoch, n_ranks if n_wait is None else n_wait)
        real.ep_wait(my_flags, which, n_ranks, epoch, n_wait=n_wait)

    def ep_reduce_norm_gather(rs_buf, my_flags, peer_h_ptrs, peer_xn_ptrs, next_norm_w, tok0, n_owned, n_ranks,
                              my_rank, epoch, H, eps, gather=True):
        assert n_ranks == N and rank_of(my_flags) == my_rank
        if n_owned:                  # the kernel waits for flags[0][src] of every rank before it reads its slots
            model.require(my_rank, 0, epoch, n_ranks)
        real.ep_reduce_norm_gather(rs_buf, my_flags, peer_h_ptrs, peer_xn_ptrs, next_norm_w, tok0, n_owned, n_ranks,
                                   my_rank, epoch, H, eps, gather=gather)

    return dict(ep_signal=ep_signal, ep_wait=ep_wait, ep_reduce_norm_gather=ep_reduce_norm_gather)


def install_guards(monkeypatch, model: FlagModel, rank_of: Callable):
    from vita_b200 import ops
    real = type("RealOps", (), {n: staticmethod(getattr(ops, n))
                                for n in ("ep_signal", "ep_wait", "ep_reduce_norm_gather")})
    for name, fn in guarded_ops(model, real, rank_of).items():
        monkeypatch.setattr(ops, name, fn)


def step_round_robin(gens: Sequence) -> list:
    """Advance the rank generators phase by phase (rank 0 .. N - 1 for each phase) until they return; every rank has
    the same number of phases.  Returns their return values."""
    out, live = [None] * len(gens), True
    while live:
        done = []
        for i, g in enumerate(gens):
            try:
                next(g)
                done.append(False)
            except StopIteration as stop:
                out[i] = stop.value
                done.append(True)
        assert all(done) or not any(done), f"ranks finished in different phases: {done}"
        live = not done[0]
    return out


# ------------------------------------------------------------------------------------------------ emulator
class LocalPeers:
    """N ranks on one device: rank r's symmetric buffer is an ordinary zeroed allocation, created with the others at
    the first request; every rank gets the base addresses of all of them (MixtralDecoder's `ep_alloc`)."""

    def __init__(self, n_ranks: int, device):
        self.N, self.device, self.bufs = n_ranks, device, None

    def alloc(self, rank: int):
        def f(nbytes: int):
            if self.bufs is None:
                self.bufs = [torch.zeros(nbytes, dtype=torch.uint8, device=self.device) for _ in range(self.N)]
            assert self.bufs[rank].numel() == nbytes
            return self.bufs[rank], [b.data_ptr() for b in self.bufs]
        return f


def rank_weights(w: dict, rank: int, N: int) -> dict:
    """Rank `rank`'s packed weights: the full ones with each layer's w13 / w2 cut to its experts (contiguous views)."""
    lo, hi = expert_range(w["layers"][0]["w13"].shape[0], rank, N)
    out = dict(w)
    out["layers"] = [dict(lw, w13=lw["w13"][lo:hi], w2=lw["w2"][lo:hi]) for lw in w["layers"]]
    out["ep"] = (rank, N)
    return out


def run_ep_prefill(cfg, weights_full: dict, N: int, emb: torch.Tensor, monkeypatch, max_seq_len: int = None) -> dict:
    """The expert-parallel prefill of `emb` [S, H] with N emulated ranks on emb's device (cfg: the LLMConfig).
    Returns per rank: own-row logits, best word, K/V pages of every layer (rows [0, S)), xn2 / ids / tw rows [0, S)
    and the device flags [4 N], plus the flag model."""
    from vita_b200.model.mixtral import MixtralDecoder
    dev, S = emb.device, emb.shape[0]
    peers = LocalPeers(N, dev)
    decs = [MixtralDecoder(cfg, rank_weights(weights_full, r, N), dev, max_seq_len=max_seq_len or S + 64,
                           max_new_tokens=8, ep_alloc=peers.alloc(r)) for r in range(N)]
    model = FlagModel(N)
    by_ptr = {d.ep_p2p["flags"].data_ptr(): r for r, d in enumerate(decs)}
    install_guards(monkeypatch, model, lambda flags: by_ptr[flags.data_ptr()])
    with torch.no_grad():
        logits = step_round_robin([d._prefill_ep_seq_steps(emb, 0, True, False) for d in decs])
    torch.cuda.synchronize()
    out = dict(model=model, logits=logits, chunk=decs[0].ep_chunk(S),
               best=[int(d.best[0]) for d in decs],
               kv=[[(d.cache.k[l][:S], d.cache.v[l][:S]) for l in range(cfg.num_hidden_layers)] for d in decs],
               xn2=[d.ep_p2p["xn2"][:S] for d in decs], ids=[d.ep_p2p["ids"][:S] for d in decs],
               tw=[d.ep_p2p["tw"][:S] for d in decs], flags=[d.ep_p2p["flags"][:4 * N].cpu() for d in decs])
    del decs
    return out
