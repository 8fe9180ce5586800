"""Particle-sharded filters: N particles partitioned over the GPUs of one box, one process
per GPU (``torch.distributed``, backend nccl), SURVEY.md section 8(e).

Per step every rank runs the fused kernels on its own shard and the ranks exchange ONE
message: an all-gather of 8 doubles per rank -- (max, sum exp, sum exp^2) of the shard's
inferential and auxiliary log-weights.  Every rank then forms the same global
log-normaliser, ESS, logLt increment and resampling decision (the prologue of the next step
kernel, csrc/smcb_step.cuh, merges the triples in rank order, so all ranks hold identical bits).
Resampling is per shard ("island" scheme): a shard resamples its own N/G particles from its
own normalised weights and restarts them at log-weight  LSE_shard(aux) - LSE_all(w) + log G,
i.e. the shard keeps its share of the total mass, which keeps the likelihood estimator
unbiased without moving particles.  This is a different (also consistent) estimator from the
reference's single global resampling; logLt parity is statistical, and G = 1 reduces to the
reference exactly.

``resampling_mode="global"`` is the exact alternative (SURVEY.md section 8e, mode 2): ONE resampling
over all N particles, as the reference does.  The shards' particles and CDFs live in peer-mapped
memory; on a resampling step every rank locates its N/G grid points in the global CDF (shard
offsets from the exchanged statistics, then the owning shard's CDF read over NVLink) and pulls
the selected ancestors from the owner's buffer -- no host round trip, no variable-size
collective; with balanced shards almost every pull is local.  Ancestors are global particle
indices, weights restart at 0, and because Philox counters follow the global particle index a
G-rank run reproduces the single-device run of the same seed up to rounding of the two-level CDF.

The helpers at the bottom restate the merge / restart algebra on the host (NumPy); the gloo
tests use them to check the scheme itself on CPU with world_size 2.
"""
import numpy as np

from . import _lib
from .collectors import default_summaries
from .core import _FusedEngine


class ShardedFilter(_FusedEngine):
    """One rank's shard of a fused filter.  ``n_local`` particles here, ``world * n_local``
    in total; Philox counters are offset by the global particle index, so the union of the
    shards draws the same numbers as one big filter would."""

    def __init__(self, spec, n_local, scheme, ESSrmin, seed, rank, world, group=None, noise=None,
                 exchange="p2p", resampling_mode="island"):
        """``exchange``: "p2p" (default, <= 8 ranks of one node) -- the kernels exchange the
        statistics themselves through NVLink peer memory, the step loop runs without the host;
        "nccl" -- one ``all_gather_into_tensor`` per step issued from Python."""
        if n_local % 2:
            raise ValueError("sharded filters need an even number of particles per rank")
        if exchange not in ("p2p", "nccl"):
            raise ValueError("exchange must be 'p2p' or 'nccl'")
        if resampling_mode not in ("island", "global"):
            raise ValueError("resampling_mode must be 'island' or 'global'")
        super().__init__(spec, n_local, scheme, ESSrmin, seed, noise=noise,
                         n_global=n_local * world, index_offset=rank * n_local,
                         world=world, rank=rank, group=group, p2p=(exchange == "p2p" and world <= 8),
                         global_rs=(resampling_mode == "global"))


class ShardedSMC:
    """Public entry point for a particle-sharded run (call it from every rank of an initialised
    ``torch.distributed`` NCCL group): ``ShardedSMC(fk=..., N=<particles on THIS rank>).run()``.
    ``N_global = world * N``.  Stock (fused) models only."""

    def __init__(self, fk=None, N=100, resampling="systematic", ESSrmin=0.5, seed=0, group=None,
                 exchange="p2p", resampling_mode="island"):
        import time
        import torch.distributed as dist
        from .state_space_models import fused_spec
        spec = fused_spec(fk)
        if spec is None or resampling not in _lib.FUSED_SCHEMES:
            raise NotImplementedError("sharded runs need a fused model and a fused resampling scheme")
        self.fk, self.N = fk, N
        self.world, self.rank = dist.get_world_size(group), dist.get_rank(group)
        self._time = time
        self._engine = ShardedFilter(spec, N, resampling, ESSrmin, seed, self.rank, self.world, group,
                                     exchange=exchange, resampling_mode=resampling_mode)
        self.t, self.logLt, self.cpu_time = 0, 0.0, None
        self.ESSs, self.logLts, self.rs_flags = [], [], []

    def run(self):
        t0 = self._time.perf_counter()
        T = self._engine.T
        self._engine.step(T - self.t)
        table = self._engine.summ.cpu().numpy()      # the one device->host read of the run
        self.ESSs, self.logLts, self.rs_flags = default_summaries(table)
        self.t, self.logLt = T, self.logLts[-1]
        self.cpu_time = self._time.perf_counter() - t0

    @property
    def X(self):
        return self._engine.X[(self.t - 1) & 1]

    @property
    def W(self):
        """This rank's slice of the GLOBALLY normalised weights (they sum to one over all ranks): exp(lw - m) / s with
        the (max, sum exp) of all N_global particles that every rank holds after the last step."""
        from .device import context, empty, ptr
        stats = self._engine.weight_stats()           # of ALL particles
        lw = self._engine.lw[(self.t - 1) & 1]
        W = empty(lw.shape[0], like=lw)
        ctx = context(lw.device)
        _lib.check(ctx.lib.smcb_weights_from_stats(ctx.handle, ptr(lw), lw.shape[0], ptr(stats), ptr(W)))
        return W

    @property
    def A(self):
        """Ancestors of the last resampling step: shard-local indices ("island"), global particle
        indices ("global")."""
        return self._engine.A


# ---------------------------------------------------------------------------
# host restatement of the exchange algebra (used by tests and by post-processing)
# ---------------------------------------------------------------------------
def merge_lse3(triples):
    """Merge per-shard (m, s, q) = (max, sum exp(v - m), sum exp(2 (v - m))) in rank order."""
    M, S, Q = -np.inf, 0.0, 0.0
    for m, s, q in triples:
        if m == -np.inf:
            continue
        if M == -np.inf:
            M, S, Q = m, s, q
            continue
        new = max(M, m)
        ea, eb = np.exp(M - new), np.exp(m - new)
        M, S, Q = new, S * ea + s * eb, Q * ea * ea + q * eb * eb
    return M, S, Q


def global_stats(triples, n_global):
    """log_mean, ESS of the union of the shards (Weights.__init__, resampling.py:217-226)."""
    M, S, Q = merge_lse3(triples)
    return M + np.log(S / n_global), S * S / Q


def island_restart(local_aux, global_w, world):
    """Log-weight a shard's particles restart from after a per-shard resampling."""
    return (np.log(local_aux[1]) + local_aux[0]) - (np.log(global_w[1]) + global_w[0]) + np.log(world)


def lse3_of(v):
    v = np.asarray(v, dtype=np.float64)
    m = v.max()
    e = np.exp(v - m)
    return m, e.sum(), (e * e).sum()


def shard_shares(aux_triples):
    """Global resampling: shard r owns [goff[r], goff[r+1]) of the global CDF, gpi[r] = its share of the
    total (auxiliary) weight mass -- what the step kernel's prologue derives from the exchanged statistics (rank order,
    sequential sums, so every rank holds the same bits)."""
    M, S, _ = merge_lse3(aux_triples)
    gpi = np.array([0.0 if m == -np.inf else s * np.exp(m - M) / S for (m, s, _q) in aux_triples])
    goff = np.zeros(len(gpi) + 1)
    for r, p in enumerate(gpi):
        goff[r + 1] = goff[r] + p
    return goff, gpi


def global_ancestors(su, goff, gpi, local_cdfs):
    """Two-level inverse CDF of the step kernel's global resampling branch: grid point ``su`` -> shard k with
    goff[k] <= su < goff[k+1] (empty shards skipped) -> position of (su - goff[k]) / gpi[k] in shard k's own
    normalised CDF.  Returns GLOBAL particle indices k * n + a."""
    su = np.asarray(su, dtype=np.float64)
    world, n = len(gpi), len(local_cdfs[0])
    k = np.zeros(su.shape, dtype=np.int64)
    for r in range(1, world):
        k += (su >= goff[r])
    for _ in range(world):                               # step off empty shards (down first, then up)
        k = np.where((k > 0) & ~(gpi[k] > 0.0), k - 1, k)
    for _ in range(world):
        k = np.where((k + 1 < world) & ~(gpi[k] > 0.0), k + 1, k)
    A = np.empty(su.shape, dtype=np.int64)
    for r in range(world):
        sel = k == r
        if not sel.any():
            continue
        v = np.minimum((su[sel] - goff[r]) / gpi[r], 1.0)
        a = np.searchsorted(local_cdfs[r], v, side="left")
        A[sel] = r * n + np.minimum(a, n - 1)
    return A
