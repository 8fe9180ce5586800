"""``SMC`` and ``FeynmanKac``: the step loop of ``particles/core.py:108-409`` on an H100.

``SMC(fk=..., N=..., resampling=..., ESSrmin=..., collect=...)`` keeps the reference's
constructor, iterator protocol and attributes (``t, X, Xp, A, wgts, aux, W, logLt,
loglt, log_mean_w, rs_flag, cpu_time, summaries``).  Two execution paths:

* FUSED (stock models recognised by ``state_space_models.fused_spec``): the whole
  step -- ESS test, scan + search + gather, propagate, log-weight, max-shifted
  normalisation, logLt recursion -- runs in libsmcb's kernels with the decision taken
  on the device; ``run()`` enqueues all T steps without a host sync and reads the
  (T, 4) summary table once.
* PLUGIN (any other ``FeynmanKac``): the reference's loop (core.py:299-383) with the
  model's ``M0 / M / logG / logeta`` called on CUDA tensors and our
  ``resampling`` / ``Weights`` kernels underneath.

There is no CPU path: without the CUDA library / device the constructor raises.
"""
import ctypes as C
import time

import numpy as np
import torch

from . import _lib
from . import collectors
from . import resampling as rs
from .device import as_device, context, empty, ptr, require_cuda, tensor_from_ptr


class FeynmanKac:
    """Abstract Feynman-Kac model -- particles/core.py:108-197."""

    def __init__(self, T):
        self.T = T

    def _error_msg(self, meth):
        return f"method/property {meth} missing in class {self.__class__.__name__}"

    def M0(self, N):
        raise NotImplementedError(self._error_msg("M0"))

    def M(self, t, xp):
        raise NotImplementedError(self._error_msg("M"))

    def logG(self, t, xp, x):
        raise NotImplementedError(self._error_msg("logG"))

    @property
    def isAPF(self):
        return "logeta" in dir(self)

    def done(self, smc):
        return smc.t >= self.T

    def time_to_resample(self, smc):
        return smc.aux.ESS < smc.N * smc.ESSrmin          # strict <, core.py:183

    def default_moments(self, W, X):
        return rs.wmean_and_var(W, X)

    def summary_format(self, smc):
        return "t=%i: resample:%s, ESS (end of iter)=%.2f" % (smc.t, smc.rs_flag, smc.wgts.ESS)


def _is_apf(fk):
    return fk.isAPF if hasattr(fk, "isAPF") else ("logeta" in dir(fk))


def _stops_at_T(fk):
    """True when ``fk`` keeps ``FeynmanKac.done`` (ours or the reference's): a run stops after T steps whatever its
    state, so it may enqueue many steps without a host read per step."""
    return getattr(getattr(type(fk), "done", None), "__qualname__", "") == "FeynmanKac.done"


def fusion_schedule(summaries, N, ESSrmin, mode, batches):
    """What each step-kernel launch of a 1-D single-device fused filter did, replayed on the host from its (T, 4)
    summary table: a list with one entry per step t >= 1, "resample", "plain" (streaming step), "fused" (streaming
    step t and step t + 1), "noop" (step t done by launch t - 1) or "mispredicted" (step t done by launch t - 1,
    then resampled after all).  ``batches`` lists the step counts of the ``step()`` calls; ``mode`` is SMCB_FUSE.
    The predictor is the kernel's: fuse when 2 ESS_{t-1} - ESS_{t-2} >= N * ESSrmin (ESS_{t-1} alone at t = 1)."""
    table = np.asarray(summaries)
    T = table.shape[0]
    ess, rs_ = table[:, 0], table[:, 2] != 0
    kinds, pre, end = [], -1, 0
    for b in batches:
        start, end = end, end + int(b)
        for t in range(max(start, 1), end):
            if pre == t:
                kinds.append("mispredicted" if rs_[t] else "noop")
            elif rs_[t]:
                kinds.append("resample")
            elif mode and t + 1 < T and t + 1 < end and (
                    mode == 2 or 2.0 * ess[t - 1] - (ess[t - 2] if t >= 2 else ess[t - 1]) >= float(N) * ESSrmin):
                kinds.append("fused")
                pre = t + 1
            else:
                kinds.append("plain")
    return kinds


class _FusedEngine:
    """Owns the device buffers of one fused filter and the smcb_filter handle."""

    def __init__(self, spec, N, scheme, ESSrmin, seed, noise=None, n_global=None, index_offset=0,
                 world=1, rank=0, group=None, p2p=False, global_rs=False, moments=False):
        self.world, self.rank, self.group = int(world), int(rank), group
        self.p2p = bool(p2p) and self.world > 1
        self.global_rs = bool(global_rs) and self.world > 1
        if self.global_rs and not self.p2p:
            raise ValueError("global resampling over shards needs the peer-memory exchange (exchange='p2p')")
        self._pool = None
        self.ctx = context()
        self.lib = self.ctx.lib
        self.N, self.T = int(N), int(spec["data"].shape[0])
        n, T = self.N, self.T
        self.dim, self.dy = int(spec.get("dim", 1)), int(spec.get("dy", 1))
        dev = self.ctx.device
        f64 = dict(dtype=torch.float64, device=dev)
        xshape = (n,) if self.dim == 1 else (self.dim, n)      # SoA: component-major
        if self.p2p:
            self._pool = _p2p_pool(self.ctx, self.world, self.rank, group)
        if self.global_rs:      # particles and CDF in peer-mapped memory: peers pull ancestors from it
            arena = self._pool.arena((2 * self.dim + 1) * n * 8)
            nd = self.dim * n
            self.X = [tensor_from_ptr(arena, xshape, owner=self._pool), tensor_from_ptr(arena + nd * 8, xshape, owner=self._pool)]
            self.cdf = tensor_from_ptr(arena + 2 * nd * 8, (n,), owner=self._pool)
        else:
            self.X = [torch.empty(xshape, **f64), torch.empty(xshape, **f64)]
            self.cdf = torch.empty(n, **f64)
        self.lw = [torch.empty(n, **f64), torch.empty(n, **f64)]
        self.A = torch.empty(n, dtype=torch.int64, device=dev)
        self.summ = torch.zeros((T, _lib.SUMMARY_STRIDE), **f64)
        # collectors.Moments on the device: per step the weighted mean / variance of every component
        self.mom = torch.zeros((T, 8), **f64) if moments else None
        # the observations are the only per-run host input of this path: pinned -> device
        self.data_host = torch.from_numpy(spec["data"].reshape(-1)).pin_memory()
        self.data = self.data_host.to(dev, non_blocking=True)
        self.sc = None
        if spec.get("step_consts") is not None:
            self.sc = as_device(spec["step_consts"])
        self.scratch = torch.empty(n + 2, **f64) if scheme == "multinomial" else None
        self.z_in = self.u_in = None
        if noise is not None:
            z, u = noise
            self.z_in = None if z is None else as_device(z)
            self.u_in = None if u is None else as_device(u)
        d = _lib.FilterDesc()
        d.model, d.fk, d.scheme, d.dim = spec["model"], spec["fk"], _lib.RS_CODES[scheme], self.dim
        d.dy, d.n_params = self.dy, len(spec["params"])
        d.n, d.n_global = n, int(n_global or n)
        d.index_offset, d.T = int(index_offset), T
        d.essrmin, d.seed = float(ESSrmin), int(seed) & (2 ** 64 - 1)
        for i, v in enumerate(spec["params"]):
            d.params[i] = float(v)
        d.X[0], d.X[1] = self.X[0].data_ptr(), self.X[1].data_ptr()
        d.lw[0], d.lw[1] = self.lw[0].data_ptr(), self.lw[1].data_ptr()
        d.A, d.cdf = self.A.data_ptr(), self.cdf.data_ptr()
        d.data, d.summaries = self.data.data_ptr(), self.summ.data_ptr()
        d.z_in = self.z_in.data_ptr() if self.z_in is not None else None
        d.u_in = self.u_in.data_ptr() if self.u_in is not None else None
        d.scratch = self.scratch.data_ptr() if self.scratch is not None else None
        d.step_consts = self.sc.data_ptr() if self.sc is not None else None
        d.moments = self.mom.data_ptr() if self.mom is not None else None
        d.world, d.rank = self.world, self.rank
        if self.world > 1:      # per-step exchange buffers of the sharded filter (16 doubles / rank)
            self.local_stats = torch.zeros(16, **f64)
            self.gathered = torch.zeros(16 * self.world, **f64)
            d.local_stats, d.gathered = self.local_stats.data_ptr(), self.gathered.data_ptr()
            if self.p2p:
                mail = self._pool.mailbox()
                d.mail_local = mail[self.rank]
                for r in range(self.world):
                    d.mail_peer[r] = mail[r]
            if self.global_rs:
                nd = self.dim * n * 8
                d.rs_global = 1
                for r in range(self.world):
                    base = self._pool.arena_of(r)
                    d.peer_X0[r], d.peer_X1[r], d.peer_cdf[r] = base, base + nd, base + 2 * nd
        self.desc = d
        h = C.c_void_p()
        _lib.check(self.lib.smcb_filter_create(self.ctx.handle, C.byref(d), C.byref(h)))
        self.handle = h

    def step(self, nsteps=1):
        self.ctx.bind_stream()
        if self.world == 1 or self.p2p:      # the whole loop is enqueued by the C side
            _lib.check(self.lib.smcb_filter_step(self.handle, int(nsteps)))
            return
        import torch.distributed as dist
        for _ in range(int(nsteps)):    # kernels -> one tiny all-gather (NCCL, stream-ordered) -> finish
            _lib.check(self.lib.smcb_filter_step_local(self.handle))
            dist.all_gather_into_tensor(self.gathered, self.local_stats, group=self.group)
            _lib.check(self.lib.smcb_filter_step_finish(self.handle))

    def step_timed(self, nsteps):
        """smcb_filter_step_timed: per-kernel device milliseconds (CUDA events)."""
        self.ctx.bind_stream()
        out = (C.c_double * 8)()
        _lib.check(self.lib.smcb_filter_step_timed(self.handle, int(nsteps), out))
        ms = dict(zip(("init", "step_rs", "tail", "step"), out[0:4]))
        cnt = dict(zip(("init", "step_rs", "tail", "step"), (int(v) for v in out[4:8])))
        return ms, cnt

    def state(self):
        out = (C.c_double * 8)()
        _lib.check(self.lib.smcb_filter_state(self.handle, out))
        return list(out)

    def weight_stats(self):
        """(max, log_mean, ESS, sum exp) of the last step's log-weights, over every shard of a sharded filter: the
        filter state [.., 4: ESS, 5: log_mean, 6: max, 7: sum exp] as a device tensor laid out as ``Weights._stats``."""
        st = self.state()
        return torch.tensor([st[6], st[5], st[4], st[7]], dtype=torch.float64, device=self.lw[0].device)

    def fusion_stats(self):
        """Counts of the fused pairs of streaming steps (SMCB_FUSE): launches that ran two steps, launches that
        found their step done, and launches whose pre-computed step resampled after all."""
        out = (C.c_int64 * 3)()
        _lib.check(self.lib.smcb_filter_fusion_stats(self.handle, out))
        return dict(zip(("fused", "noop", "mispredicted"), (int(v) for v in out)))

    def close(self):
        """Free the filter handle.  Peer-mapped memory (mailboxes, arenas) belongs to the per-(process, group)
        pool and stays mapped for the next sharded filter, so closing needs no collective call."""
        if getattr(self, "handle", None):
            self.lib.smcb_filter_destroy(self.handle)      # synchronises this rank's stream
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class _SqmcEngine(_FusedEngine):
    """A fused filter stepped by SQMC (csrc/smcb_sqmc.cu): the buffers, summary table and attributes of
    ``_FusedEngine``; every step resamples through the Hilbert order of the particles (core.py:339-349).
    ``points``: None (Sobol' points of key (seed, t)) or, per step t, the (N, du + 1) points to use ((N, du) at t = 0),
    as the reference's ``rqmc.sobol`` would return them."""

    def __init__(self, spec, N, seed, points=None):
        u_in = None
        if points is not None:
            dim = int(spec.get("dim", 1))
            T = int(spec["data"].shape[0])
            if len(points) < T:
                raise ValueError(f"SQMC points: need one point set per step ({T}), got {len(points)}")
            u_in = np.zeros((T, dim + 1, N))
            for t in range(T):
                p = np.asarray(points[t], dtype=np.float64).reshape(N, -1)
                rows = dim if t == 0 else dim + 1
                if p.shape[1] < rows:
                    raise ValueError(f"SQMC points of step {t}: need {rows} columns, got {p.shape[1]}")
                u_in[t, :rows] = p[:, :rows].T
        super().__init__(spec, N, "systematic", 0.5, seed, noise=None if u_in is None else (None, u_in))
        nb = int(self.lib.smcb_sqmc_scratch_bytes(self.N, self.dim))
        if nb < 0:
            raise ValueError(f"SQMC: bad sizes (N={self.N}, dim={self.dim})")
        self._scratch = torch.empty(nb + 256, dtype=torch.uint8, device=self.ctx.device)
        base = self._scratch.data_ptr()
        self._scratch_ptr = base + (-base) % 256
        self._t = 0

    def step(self, nsteps=1):
        self.ctx.bind_stream()
        _lib.check(self.lib.smcb_sqmc_step(self.handle, int(nsteps), self._scratch_ptr))
        self._t += int(nsteps)

    def step_timed(self, nsteps):
        raise NotImplementedError("step_timed runs the SMC step kernel; time SQMC with CUDA events around step()")

    def fusion_stats(self):
        raise NotImplementedError("an SQMC filter fuses no streaming steps")

    def weight_stats(self):
        lw = self.lw[(self._t - 1) & 1].clone()
        st = torch.empty(4, dtype=torch.float64, device=lw.device)
        _lib.check(self.lib.smcb_normalise(self.ctx.handle, ptr(lw), self.N, None, ptr(st)))
        return st


class _P2PPool:
    """Peer-mapped memory of one (process, process group): ONE mailbox and one (growing) arena per rank, allocated
    and exchanged once -- a single tensor all-gather of the 64-byte CUDA IPC handles -- and then reused by every
    sharded filter of the group: constructing the second ``ShardedSMC`` costs no collective, no
    ``cudaIpcOpenMemHandle`` and no barrier.

    Reuse is made safe by generations.  The mailbox has four slabs; filter number g of the group (all ranks make
    their filters in the same order) uses slab g % 4 and zeroes -- locally, stream-ordered -- slab (g + 2) % 4.
    Epochs inside a slab are step indices.  Nobody can still be writing into the slab being zeroed: it last served
    generation g - 2, and this rank could only finish generation g - 1 after every peer had sent the statistics of
    that filter's last step, i.e. after all their kernels of generation g - 2 had retired.  The arena (particles and
    CDF of the exact global resampling) needs no tag: peers read it only inside a resampling step of the current
    filter, and a rank finishes a filter only after every peer's reads of its last step are done."""

    def __init__(self, ctx, world, rank, group):
        self.ctx, self.lib, self.world, self.rank, self.group = ctx, ctx.lib, world, rank, group
        self._mail = None          # [ptr per rank]
        self._arena = None         # [ptr per rank]
        self._arena_bytes = 0
        self._gen = 0

    def _exchange(self, nbytes):
        """Allocate nbytes here (zeroed, synchronously), hand the IPC handle to every rank, map theirs."""
        import torch.distributed as dist
        ptr_ = C.c_void_p()
        hbuf = C.create_string_buffer(64)
        _lib.check(self.lib.smcb_p2p_alloc(self.ctx.handle, int(nbytes), C.byref(ptr_), hbuf))
        mine = torch.frombuffer(bytearray(hbuf.raw), dtype=torch.uint8).to(self.ctx.device)
        allh = torch.empty(64 * self.world, dtype=torch.uint8, device=self.ctx.device)
        dist.all_gather_into_tensor(allh, mine, group=self.group)
        allh = allh.cpu().numpy().tobytes()
        out = []
        for r in range(self.world):
            if r == self.rank:
                out.append(ptr_.value)
                continue
            pp = C.c_void_p()
            _lib.check(self.lib.smcb_p2p_open(self.ctx.handle, allh[64 * r:64 * (r + 1)], C.byref(pp)))
            out.append(pp.value)
        return out

    def mailbox(self):
        """[mailbox of rank r as mapped here] for the next filter of this group."""
        nslab, slab = 4, 2 * self.world * 32 * 8
        if self._mail is None:
            self._mail = self._exchange(nslab * slab)
        g = self._gen
        self._gen += 1
        tensor_from_ptr(self._mail[self.rank] + ((g + 2) % nslab) * slab, (slab // 8,), owner=self).zero_()
        return [p + (g % nslab) * slab for p in self._mail]

    def arena(self, nbytes):
        if self._arena is None or nbytes > self._arena_bytes:
            self._arena = self._exchange(nbytes)      # a smaller, earlier arena stays mapped until process exit
            self._arena_bytes = nbytes
        return self._arena[self.rank]

    def arena_of(self, r):
        return self._arena[r]


_pools = {}


def _p2p_pool(ctx, world, rank, group):
    key = (ctx.device.index, id(group) if group is not None else None, world, rank)
    if key not in _pools:
        _pools[key] = _P2PPool(ctx, world, rank, group)
    return _pools[key]


def _aos(x):
    """(N, d) view of a component-major (d, N) particle buffer; (N,) buffers as they are."""
    return x if x.ndim == 1 else x.t()


class _Results:
    """The reference's ``rs_flag, logLt, log_mean_w, loglt, X, Xp, A`` of a device-run filter after ``t`` steps, from
    ``row(s)``, row s of its (T, 4) summary table (ESS, logLt, rs_flag, log_mean_w) on the host; ``gen(s)``, the (N,)
    or (d, N) particle buffer step s wrote (steps alternate between two buffers); and ``anc()``, the ancestor buffer,
    which holds the last step's ancestors when that step resampled."""

    def __init__(self, t, N, row, gen, anc):
        self.t, self.N = t, N
        self._row, self._gen, self._anc = row, gen, anc

    @property
    def rs_flag(self):
        return False if self.t == 0 else bool(self._row(self.t - 1)[2])

    @property
    def logLt(self):
        return 0.0 if self.t == 0 else float(self._row(self.t - 1)[1])

    @property
    def log_mean_w(self):
        return float(self._row(self.t - 1)[3])

    @property
    def loglt(self):
        if self.t == 1 or self.rs_flag:
            return self.log_mean_w
        return self.log_mean_w - float(self._row(self.t - 2)[3])

    @property
    def X(self):
        return None if self.t == 0 else _aos(self._gen(self.t - 1))

    @property
    def A(self):
        if self.t <= 1:
            return None
        A = self._anc()
        return A if self.rs_flag else torch.arange(self.N, device=A.device)      # core.py:335

    @property
    def Xp(self):
        if self.t <= 1:
            return None
        prev = self._gen(self.t - 2)
        if not self.rs_flag:
            return _aos(prev)
        out = torch.empty_like(prev)
        ctx = context(prev.device)
        _lib.check(ctx.lib.smcb_gather(ctx.handle, ptr(prev), self.N, ptr(self._anc()), self.N,
                                       1 if prev.ndim == 1 else prev.shape[0], ptr(out)))
        return _aos(out)


class SMC:
    """Drop-in for ``particles.SMC`` (particles/core.py:200-409).

    Extra keyword arguments (all optional, defaults keep the reference's behaviour):
    ``seed`` re-keys the device generator for this run; ``fused=False`` forces the
    plugin path; ``noise=(z, u)`` injects standard normals / uniforms (parity tests).
    """

    def __init__(self, fk=None, N=100, qmc=False, resampling="systematic", ESSrmin=0.5,
                 store_history=False, verbose=False, collect=None, seed=None, fused=None,
                 noise=None):
        require_cuda()
        _lib.load()
        from .smc_samplers import from_reference_smc2
        fk = from_reference_smc2(fk) or fk          # the reference's SMC2 of a stock 1-D model: the filter bank
        if resampling not in rs.rs_funcs:
            raise ValueError(f"{resampling} is not a valid resampling scheme")
        self.fk, self.N, self.qmc = fk, N, qmc
        self.resampling, self.ESSrmin, self.verbose = resampling, ESSrmin, verbose
        self.t = 0
        self._done = 0        # completed steps (== t outside of a step; collectors see t = index)
        self.cpu_time = None
        self.summaries = None if collect == "off" else collectors.Summaries(collect)
        self._seed = np.random.randint(0, 2 ** 31 - 1) if seed is None else int(seed)
        self._engine = None
        self._dev_moments = False
        self._noise = noise
        spec = None
        if fused is not False:
            from .state_space_models import fused_spec
            # a model that only adds the smoothing hooks to a stock class runs fused when it is smoothed on-line
            spec = fused_spec(fk, smoothing_hooks=self.summaries is not None and bool(self.summaries.online))
            if spec is not None and resampling not in _lib.FUSED_SCHEMES:
                spec = None                      # residual, ssp, killing, ...: plugin path (stand-alone kernels)
            if spec is None and fused is True:
                raise NotImplementedError("this Feynman-Kac model has no fused kernel")
            if qmc:
                spec = fused_spec(fk)            # SQMC ignores the resampling scheme, as the reference does
        if qmc:
            self._qmc_points = None if noise is None else [np.asarray(p.cpu() if torch.is_tensor(p) else p,
                                                                      dtype=np.float64) for p in noise]
        if spec is not None and qmc:
            self._engine = _SqmcEngine(spec, N, self._seed, self._qmc_points)
            self._row_cache = {}
        elif spec is not None:
            # collect=[Moments()] with the default mom_func: the step kernel accumulates sum w x / sum w x^2 next
            # to its log-sum-exp triple and writes a (T, 8) table -- run() keeps its sync-free fast path
            self._dev_moments = self.summaries is not None and self.summaries.device_moments(fk)
            self._engine = _FusedEngine(spec, N, resampling, ESSrmin, self._seed, noise,
                                        moments=self._dev_moments)
            self._row_cache = {}
        else:
            context().seed(self._seed)
            self._p = {"rs_flag": False, "logLt": 0.0, "wgts": rs.Weights(), "aux": None,
                       "X": None, "Xp": None, "A": None}
        from . import smoothing
        self.hist = smoothing.generate_hist_obj(store_history, self)   # smoothing.py:151-161

    # ------------------------------------------------------------------ fused
    @property
    def fused(self):
        return self._engine is not None

    def _row(self, t):
        """(ESS, logLt, rs_flag, log_mean_w) of step t, read from the device table on first use.  The row read before
        stays cached as well, so that ``loglt`` (rows t - 1 and t) and ``rs_flag`` (row t) do not evict each other."""
        if t not in self._row_cache:
            self._row_cache = dict(list(self._row_cache.items())[-1:])
            self._row_cache[t] = self._engine.summ[t].cpu().numpy()
        return self._row_cache[t]

    def _results(self):
        e = self._engine
        return _Results(self._done, self.N, self._row, lambda s: e.X[s & 1], lambda: e.A)

    def _engine_gen(self, t):
        """Generation t of the fused filter as the on-line smoothers read it, after step t and before step t + 2
        (step s writes buffers [s & 1]): views of the device buffers, and the ancestors chosen on the device from
        the step's resampling flag -- no host sync."""
        e = self._engine
        A = None
        if t > 0:
            A = torch.where(e.summ[t, 2] != 0, e.A, torch.arange(self.N, device=e.A.device))
        return collectors._Gen(t, _aos(e.X[t & 1]), e.lw[t & 1], A)

    def _cur(self):
        return (self._done - 1) & 1      # step s writes buffers [s & 1]

    # ------------------------------------------------------------- attributes
    @property
    def X(self):
        return self._results().X if self.fused else self._p["X"]

    @X.setter
    def X(self, v):
        self._p["X"] = v

    @property
    def h_order(self):
        """SQMC: the Hilbert order of the particles the last step resampled from (core.py:344).  On the plugin path it
        exists from inside step 1 on, as in the reference, so that ``hist.save`` records it for t = 1."""
        if not self.fused:
            if not self.qmc or self._p.get("h_order") is None:
                raise AttributeError("h_order exists after a resampling step of SQMC (qmc=True)")
            return self._p["h_order"]
        if not self.qmc or self._done < 2:
            raise AttributeError("h_order exists after a resampling step of SQMC (qmc=True)")
        from .hilbert import hilbert_order
        return hilbert_order(self._engine.X[self._done & 1])     # generation t - 1 (step s writes X[s & 1])

    @property
    def rs_flag(self):
        return self._results().rs_flag if self.fused else self._p["rs_flag"]

    @property
    def logLt(self):
        return self._results().logLt if self.fused else self._p["logLt"]

    @property
    def log_mean_w(self):
        return self._results().log_mean_w if self.fused else self._p["log_mean_w"]

    @property
    def loglt(self):
        return self._results().loglt if self.fused else self._p["loglt"]

    @property
    def A(self):
        return self._results().A if self.fused else self._p["A"]

    @property
    def Xp(self):
        return self._results().Xp if self.fused else self._p["Xp"]

    @property
    def wgts(self):
        if not self.fused:
            return self._p["wgts"]
        if self._done == 0:
            return rs.Weights()
        return rs.Weights._from_device_stats(self._engine.lw[self._cur()], self._engine.weight_stats())

    @property
    def aux(self):
        if not self.fused:
            return self._p["aux"]
        return self.wgts

    @property
    def W(self):
        return self.wgts.W

    def __str__(self):
        return self.fk.summary_format(self)

    # ----------------------------------------------------------- plugin path
    def reset_weights(self):                                  # core.py:299-305
        p = self._p
        if _is_apf(self.fk):
            lw = rs.log_mean_exp(self.logetat, W=p["wgts"].W) - self._gather(self.logetat, p["A"])
            p["wgts"] = rs.Weights(lw=lw)
        else:
            p["wgts"] = rs.Weights()

    def setup_auxiliary_weights(self):                        # core.py:307-313
        p = self._p
        if _is_apf(self.fk):
            self.logetat = as_device(self.fk.logeta(self.t - 1, p["X"]))
            p["aux"] = p["wgts"].add(self.logetat)
        else:
            p["aux"] = p["wgts"]

    def _gather(self, X, A):
        if not isinstance(X, (torch.Tensor, np.ndarray)):
            return X[A]          # particle containers (smc_samplers.ThetaParticles) index themselves
        ctx = context()
        X = as_device(X)
        d = 1 if X.ndim == 1 else X.shape[1]
        out = torch.empty((A.shape[0],) + tuple(X.shape[1:]), dtype=X.dtype, device=X.device)
        _lib.check(ctx.lib.smcb_gather_rows(ctx.handle, ptr(X), X.shape[0], ptr(A), A.shape[0], d,
                                            ptr(out)))
        return out

    def generate_particles(self):                             # core.py:315-321
        if self.qmc:
            u = self._points(self.fk.du)
            self._p["X"] = self.fk.Gamma0(u[:, 0].contiguous() if u.shape[1] == 1 else u)
        else:
            self._p["X"] = self.fk.M0(self.N)

    def _points(self, d):
        """(N, d) points of step t on the plugin path: the injected ones, or the Sobol' points of key (seed, t) that
        the fused SQMC engine draws."""
        if self._qmc_points is not None:
            return as_device(np.ascontiguousarray(self._qmc_points[self.t].reshape(self.N, -1)[:, :d]))
        from .rqmc import sobol_points
        return sobol_points(self.N, d, self._seed, self.t).t().contiguous()

    def resample_move_qmc(self):                              # core.py:339-349
        from .hilbert import hilbert_order, hilbert_sort
        p = self._p
        p["rs_flag"] = True
        du = self.fk.du
        u = self._points(du + 1)
        tau = hilbert_order(u[:, 0].contiguous())            # argsort of one coordinate
        h = hilbert_sort(p["X"])
        p["h_order"] = h
        su = self._gather(u[:, 0].contiguous(), tau)
        idx = rs.inverse_cdf(su, self._gather(p["aux"].W, h))
        p["A"] = self._gather(h.view(torch.float64), idx).view(torch.int64)     # h[idx]: an 8-byte copy
        p["Xp"] = self._gather(p["X"], p["A"])
        v = self._gather(u[:, 1:].contiguous(), tau)
        self.reset_weights()
        p["X"] = self.fk.Gamma(self.t, p["Xp"], v[:, 0].contiguous() if du == 1 else v)

    def reweight_particles(self):                             # core.py:323-324
        p = self._p
        p["wgts"] = p["wgts"].add(self.fk.logG(self.t, p["Xp"], p["X"]))

    def resample_move(self):                                  # core.py:326-337
        p = self._p
        p["rs_flag"] = bool(self.fk.time_to_resample(self))
        if p["rs_flag"]:
            p["A"] = rs.resampling(self.resampling, p["aux"].W, M=self.N)
            p["Xp"] = self._gather(p["X"], p["A"])
            self.reset_weights()
        else:
            p["A"] = torch.arange(self.N, device="cuda")
            p["Xp"] = p["X"]
        p["X"] = self.fk.M(self.t, p["Xp"])

    def compute_summaries(self):                              # core.py:351-367
        p = self._p
        if self.t > 0:
            prec = p["log_mean_w"]
        p["log_mean_w"] = p["wgts"].log_mean
        if self.t == 0 or p["rs_flag"]:
            p["loglt"] = p["log_mean_w"]
        else:
            p["loglt"] = p["log_mean_w"] - prec
        p["logLt"] += p["loglt"]
        if self.verbose:
            print(self)
        if self.hist:
            self.hist.save(self)
        if self.summaries:
            self.summaries.collect(self)

    # -------------------------------------------------------------- iterator
    def __next__(self):
        """One step of a particle filter (core.py:369-383)."""
        if self.fk.done(self):
            raise StopIteration
        if self.fused:
            self._engine.step(1)
            self._done += 1
            if self.verbose:
                print(self)
            if self.hist:
                self.hist.save(self)              # core.py:362-363 (before the collectors)
            if self.summaries:
                self.summaries.collect(self)      # smc.t is still the index of this step
            self.t += 1
            return
        if self.t == 0:
            self.generate_particles()
        else:
            self.setup_auxiliary_weights()
            if self.qmc:
                self.resample_move_qmc()
            else:
                self.resample_move()
        self.reweight_particles()
        self.compute_summaries()
        self.t += 1
        self._done = self.t

    def next(self):
        return self.__next__()

    def __iter__(self):
        return self

    def run(self):
        """Run until completion (core.py:391-409); ``cpu_time`` is the wall time of this
        call, device work included (utils.timer semantics, utils.py:81-89)."""
        t0 = time.perf_counter()
        online = [] if self.summaries is None else self.summaries.device_rows
        if self.fused and not self.verbose and not self.hist \
                and (self.summaries is None or self.summaries.only_defaults or self._dev_moments
                     or len(online) == len(self.summaries._collectors) - self.summaries._n_default) \
                and _stops_at_T(self.fk):
            T = self._engine.T
            first = self.t
            if online:
                # one-step batches: generation t - 1 stays intact in buffers (t - 1) & 1 while the smoothers read
                # it after step t (a batch of one step never fuses two steps)
                for t in range(first, T):
                    self._engine.step(1)
                    self.t, self._done = t, t + 1
                    for col in online:
                        col._step(self, t)
                self.t = self._done = T
            elif first < T:
                self._engine.step(T - first)
                self.t = self._done = T
            table = self._engine.summ.cpu().numpy()       # the one device->host read of the run
            self._row_cache = {T - 1: table[T - 1]}
            if self.summaries is not None:
                self.summaries._extend_defaults(*collectors.default_summaries(table[first:T]))
                if self._dev_moments:
                    self.summaries._extend_moments(self._engine.mom.cpu().numpy()[first:T], self._engine.dim)
                for col in online:
                    col._flush()
        elif self._ibis_stretches():
            self._run_ibis()
        else:
            for _ in self:
                pass
            if self.fused:
                torch.cuda.synchronize()
        self.cpu_time = time.perf_counter() - t0

    # ------------------------------------------------------- IBIS stretches
    def _ibis_stretches(self):
        """True for an IBIS run over a model with a device likelihood, without verbose output, history or
        collectors beyond the defaults, whose resampling rule is FKSMCsampler's: ``run()`` may then add the data
        rows of a stretch of non-resampling steps with one host read."""
        from .smc_samplers import IBIS, FKSMCsampler
        fk = self.fk
        return (isinstance(fk, IBIS) and hasattr(fk.model, "logpyt_rows") and not self.verbose and not self.hist
                and (self.summaries is None or self.summaries.only_defaults)
                and type(fk).time_to_resample is FKSMCsampler.time_to_resample
                and _stops_at_T(fk) and not _is_apf(fk))

    def _run_ibis(self):
        """The per-step loop, with every run of non-resampling steps done as stretches (DESIGN.md section 5.10).
        From the state after step t - 1 whose ESS stays above the threshold, the rows t .. t + K - 1 are scanned
        into a (K, n) scratch buffer of cumulative log-weights, each scratch row is normalised into a (K, 4) table
        (smcb_normalise: the bits the per-step path computes), the table is read once, and the rows up to the first
        one whose ESS falls below ESSrmin * X.N are committed.  The resampling step that follows, and the steps
        whose predecessor is below the threshold, run through the iterator.  Same bits as ``for _ in pf: pass``."""
        fk, p, ctx = self.fk, self._p, context()
        st = self._ibis_stats = {"stretches": 0, "rows": 0, "reads": 0, "scanned": 0, "last": 0}
        K = IBIS_K0
        while not fk.done(self):
            X = p["X"]
            if self.t == 0 or p["wgts"].ESS < X.N * self.ESSrmin:      # step t resamples (time_to_resample)
                next(self)
                K = IBIS_K0
                continue
            n, t = X.N, self.t
            k = max(1, min(K, IBIS_SCRATCH_BYTES // (8 * n), fk.T - t))
            scratch, table = empty((k, n)), empty((k, 4))
            lw = p["wgts"].lw
            fk.model.logpyt_rows(X.theta, t, k, lw, scratch=scratch)
            for r in range(k):
                _lib.check(ctx.lib.smcb_normalise(ctx.handle, ptr(scratch[r]), n, None, ptr(table[r])))
            tab = table.cpu().numpy()                     # the one device->host read of the stretch
            below = np.flatnonzero(tab[:, 2] < n * self.ESSrmin)
            m = int(below[0]) + 1 if below.size else k
            fk.model.logpyt_rows(X.theta, t, m, lw, X.lpost, X.llik)
            st["stretches"] += 1
            st["reads"] += 1
            st["rows"] += m
            st["scanned"] += k
            st["last"] = t + m
            wgts = rs.Weights._from_device_stats(lw, table[m - 1])
            wgts._host = tab[m - 1]
            ess, logLts = [], []
            for r in range(m):                            # compute_summaries, step by step
                prec, p["log_mean_w"] = p["log_mean_w"], float(tab[r, 1])
                p["loglt"] = p["log_mean_w"] - prec
                p["logLt"] += p["loglt"]
                ess.append(float(tab[r, 2]))
                logLts.append(p["logLt"])
            p["wgts"] = p["aux"] = wgts
            p["rs_flag"] = X.shared["rs_flag"] = False
            p["A"] = torch.arange(self.N, device="cuda")
            p["Xp"] = X
            if self.summaries:
                self.summaries._extend_defaults(ess, logLts, [False] * m)
            self.t += m
            self._done = self.t
            K = K if below.size else K * IBIS_K_GROWTH


# IBIS stretches (SMC._run_ibis): the first stretch after a resampling scans IBIS_K0 rows, each stretch that ends
# without an ESS crossing multiplies the next one's rows by IBIS_K_GROWTH, and the (K, n) fp64 scratch buffer stays
# within IBIS_SCRATCH_BYTES.  Chosen by measurement with tools/bench_ibis.py (DESIGN.md section 5.10).
IBIS_K0, IBIS_K_GROWTH, IBIS_SCRATCH_BYTES = 8, 2, 64 << 20


# ---------------------------------------------------------------------------------------------------- multiSMC
# Cost model of the routing rule, in seconds per filter step, measured with tools/bench_multismc.py on an NVIDIA H100
# 80GB HBM3 at a 400 W power limit (DESIGN.md section 5.7):
#   * one run of the single engine, end to end (construction, T steps, summary read) over T: LOOP_STEP, interpolated
#     in log N between the measured points and clamped at both ends;
#   * one wave of the batched kernel (every CTA runs one filter): BATCH_STEP_S + N * BATCH_PARTICLE_S in the resident
#     tier; N * STREAM_PARTICLE_S in the streaming tier with one CTA per SM, times 1 + STREAM_SHARE for every further
#     CTA that shares an SM (they split its memory bandwidth).
LOOP_STEP = ((256, 11.9e-6), (4096, 12.6e-6), (16384, 13.0e-6), (65536, 15.1e-6), (131072, 19.0e-6),
             (262144, 18.0e-6), (1048576, 119e-6), (10_000_000, 165e-6))
BATCH_STEP_S, BATCH_PARTICLE_S = 3.6e-6, 1.6e-9
STREAM_PARTICLE_S, STREAM_SHARE = 3.8e-9, 0.45


def loop_step_s(N):
    """Measured end-to-end cost of one single-engine step at N particles (LOOP_STEP, log-log interpolation)."""
    xs = np.log([n for n, _ in LOOP_STEP])
    ys = np.log([v for _, v in LOOP_STEP])
    return float(np.exp(np.interp(np.log(max(N, 1)), xs, ys)))


def batch_pays(N, R, tier, grid, n_sm=132):
    """True when R filters of N particles finish sooner in batched launches -- ceil(R / grid) waves, one filter per
    CTA -- than one after another through ``SMC``, by the measured cost model above."""
    grid = max(int(grid), 1)
    waves = -(-R // grid)
    if tier == _lib.BATCH_RESIDENT:
        wave = BATCH_STEP_S + N * BATCH_PARTICLE_S
    else:
        per_sm = -(-min(R, grid) // n_sm)
        wave = N * STREAM_PARTICLE_S * (1 + STREAM_SHARE * (per_sm - 1))
    return waves * wave < R * loop_step_s(N)


_SMC_ARGS = {"fk", "N", "qmc", "resampling", "ESSrmin", "store_history", "verbose", "collect"}


def batch_key(kw, _specs=None):
    """(group key, fused spec) of a run that ``multiSMC`` can run in a batched launch, or (None, None) for a run
    that takes the per-run path (``SMC(**kw, seed=seed).run()``).  ``kw`` are the run's ``SMC`` arguments.
    The key holds what selects the kernel and the shapes; model constants, data and ``ESSrmin`` are per run."""
    if set(kw) - _SMC_ARGS or kw.get("qmc") or kw.get("store_history") or kw.get("verbose"):
        return None, None
    fk, N = kw.get("fk"), int(kw.get("N", 100))
    scheme = kw.get("resampling", "systematic")
    if fk is None or scheme not in _lib.FUSED_SCHEMES or N < 1:
        return None, None
    if not _stops_at_T(fk):
        return None, None
    from .state_space_models import fused_spec
    if _specs is None:
        spec = fused_spec(fk)
    else:                                   # one spec per distinct Feynman-Kac object (its runs share it)
        if id(fk) not in _specs:
            _specs[id(fk)] = (fk, fused_spec(fk))
        spec = _specs[id(fk)][1]
    if spec is None or int(spec.get("dim", 1)) != 1 or int(spec.get("dy", 1)) != 1:
        return None, None
    collect = kw.get("collect")
    moments = False
    if collect != "off":
        summ = collectors.Summaries(collect)
        if not summ.only_defaults:
            if summ.device_rows or not summ.device_moments(fk):
                return None, None
            moments = True
    key = (spec["model"], spec["fk"], scheme, N, int(spec["data"].shape[0]), moments, collect == "off")
    return key, spec


class BatchRun(_Results):
    """One filter of a batched ``multiSMC`` group, after its run: the attributes of ``SMC`` after ``run()``
    (``t, N, fk, logLt, rs_flag, log_mean_w, loglt, X, Xp, A, wgts, W, summaries, cpu_time``) as views of the group's
    device buffers of its chunk.  ``cpu_time`` is the wall time of the chunk (upload, launch, device work and the one
    read of its summary table) divided by its number of runs: the cost per run of the batched launch.  ``summaries``
    is built from the chunk's table on first access."""

    def __init__(self, buf, i, fk, N, resampling, ESSrmin, seed, table, mom, collect, cpu_time):
        super().__init__(table.shape[0], N, table.__getitem__, lambda s: buf["X"][i, s & 1, :N],
                         lambda: buf["A"][i, :N])
        self._buf, self._i = buf, i
        self.fk, self.resampling, self.ESSrmin = fk, resampling, ESSrmin
        self.qmc, self.verbose, self.hist, self.seed = False, False, None, seed
        self.T = self.t
        self._table, self._mom, self._collect = table, mom, collect
        self._summaries = None
        self.cpu_time = cpu_time

    @property
    def summaries(self):
        if self._summaries is None and self._collect != "off":
            sm = collectors.Summaries(self._collect)
            sm._extend_defaults(*collectors.default_summaries(self._table))
            if self._mom is not None:
                sm._extend_moments(self._mom, 1)
            self._summaries = sm
        return self._summaries

    @property
    def wgts(self):
        return rs.Weights(lw=self._buf["lw"][self._i, :self.N])

    @property
    def aux(self):
        return self.wgts

    @property
    def W(self):
        return self.wgts.W

    def __str__(self):
        return self.fk.summary_format(self)


def _batch_desc(key, R, tier):
    """The header of the ``BatchDesc`` of R runs of the group ``key``: kernel selection, tier and shapes."""
    model, fkind, scheme, N, T = key[:5]
    d = _lib.BatchDesc()
    d.model, d.fk, d.scheme, d.dim, d.dy = model, fkind, _lib.RS_CODES[scheme], 1, 1
    d.tier = _lib.BATCH_TIERS[tier]
    d.N, d.T, d.R = N, T, R
    return d


def plan_group(key, R, tier="auto"):
    """(tier, grid) that ``smcb_batch_plan`` chooses for R runs of the group ``key``."""
    plan = (C.c_int64 * 2)()
    ctx = context()
    _lib.check(ctx.lib.smcb_batch_plan(ctx.handle, C.byref(_batch_desc(key, R, tier)), plan))
    return int(plan[0]), int(plan[1])


def run_batch(kws, seeds, noise=None, tier="auto", timer=None, out_func=None, _planned=None):
    """Run the filters ``SMC(**kws[i], seed=seeds[i])`` -- which must share one ``batch_key`` -- in batched launches
    and return, per run, its ``BatchRun`` or, with ``out_func``, ``out_func(run)``.

    Memory: the group is cut into chunks that fit half of the free device memory, one launch each.  The streaming
    tier's CDF and spacings are one scratch set, reused by every chunk and released on return.  With ``out_func`` a
    chunk's buffers are released as soon as its runs are reduced, so the device holds one chunk at a time; without
    it every run's outputs stay alive, and each chunk is sized from the memory left after the previous ones.
    ``noise``: None or one ``(z, u)`` per run with the layout of ``SMC(noise=...)``; ``tier``: "auto", "resident" or
    "streaming"; ``timer``: None, or a list that receives the pair of CUDA events recorded before the first and
    after the last launch."""
    key, specs = _planned or (None, [])
    if _planned is None:
        keyed = [batch_key(kw) for kw in kws]
        keys = {k for k, _ in keyed}
        if len(keys) != 1 or None in keys:
            raise ValueError("run_batch: the runs do not form one batchable group")
        key, specs = keys.pop(), [s for _, s in keyed]
    scheme, N, T, moments = key[2:6]
    R, ld = len(kws), N + (N & 1)
    ctx = context()
    ctx.bind_stream()
    dev = ctx.device
    f64 = dict(dtype=torch.float64, device=dev)
    n_params = len(specs[0]["params"])
    streaming = plan_group(key, R, tier)[0] == _lib.BATCH_STREAMING
    d = _batch_desc(key, R, tier)
    d.n_params = n_params
    multi = scheme == "multinomial"
    # bytes per run: outputs (X ping-pong, lw, A, summary and moment rows) and inputs (data, step constants, params,
    # seed, ESSrmin, injected noise); the streaming tier's scratch (CDF, spacings) separately
    noise_b = 0 if noise is None else 8 * T * (N + N + 1)
    out_b = 8 * (4 * ld + T * (_lib.SUMMARY_STRIDE + (8 if moments else 0) + 2) + n_params + 2) + noise_b
    scr_b = 8 * (ld + (ld + 2 if multi else 0)) if streaming else 0
    chunk = max(1, min(R, int(0.5 * torch.cuda.mem_get_info(dev)[0]) // (out_b + scr_b)))
    scr = None
    if streaming:
        scr = {"cdf": torch.empty((chunk, ld), **f64)}
        if multi:
            scr["scratch"] = torch.empty((chunk, ld + 2), **f64)
    ev = None
    if timer is not None:
        ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
    out = []
    r0 = 0
    while r0 < R:
        if r0 > 0 and out_func is None:       # earlier chunks stay alive: size this one from what they left
            chunk = max(1, min(chunk, int(0.5 * torch.cuda.mem_get_info(dev)[0]) // out_b))
        rc = min(chunk, R - r0)
        t0 = time.perf_counter()
        sl = slice(r0, r0 + rc)
        up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)    # noqa: E731
        params = up(np.array([np.asarray(s["params"], dtype=np.float64) for s in specs[sl]]))
        data = up(np.stack([s["data"].reshape(-1) for s in specs[sl]]).astype(np.float64))
        sc = None
        if specs[0].get("step_consts") is not None:
            sc = up(np.stack([np.asarray(s["step_consts"], dtype=np.float64) for s in specs[sl]]))
        seed_t = up(np.asarray([int(s) & (2 ** 64 - 1) for s in seeds[sl]], dtype=np.uint64).view(np.int64))
        ess_t = up(np.asarray([float(kw.get("ESSrmin", 0.5)) for kw in kws[sl]], dtype=np.float64))
        z_t = u_t = None
        if noise is not None:
            z_t = as_device(np.stack([np.asarray(z, dtype=np.float64).reshape(T, -1, N) for z, _ in noise[sl]]))
            u_t = as_device(np.stack([np.asarray(u, dtype=np.float64).reshape(T, N + 1) for _, u in noise[sl]]))
        b = {"X": torch.empty((rc, 2, ld), **f64), "lw": torch.empty((rc, ld), **f64),
             "A": torch.empty((rc, ld), dtype=torch.int64, device=dev)}
        summ = torch.zeros((rc, T, _lib.SUMMARY_STRIDE), **f64)
        mom = torch.zeros((rc, T, 8), **f64) if moments else None
        d.R = rc
        d.seed, d.essrmin, d.params, d.data = seed_t.data_ptr(), ess_t.data_ptr(), params.data_ptr(), data.data_ptr()
        d.step_consts = None if sc is None else sc.data_ptr()
        d.X, d.lw, d.A = b["X"].data_ptr(), b["lw"].data_ptr(), b["A"].data_ptr()
        d.cdf = scr["cdf"].data_ptr() if streaming else None
        d.scratch = scr["scratch"].data_ptr() if streaming and multi else None
        d.summaries = summ.data_ptr()
        d.moments = None if mom is None else mom.data_ptr()
        d.z_in = None if z_t is None else z_t.data_ptr()
        d.u_in = None if u_t is None else u_t.data_ptr()
        if ev is not None and r0 == 0:
            ev[0].record()
        _lib.check(ctx.lib.smcb_batch_run(ctx.handle, C.byref(d)))
        if ev is not None and r0 + rc == R:
            ev[1].record()
        table = summ.cpu().numpy()            # the one device->host read of the chunk (+ the moments table)
        mtab = None if mom is None else mom.cpu().numpy()
        cpu = (time.perf_counter() - t0) / rc
        for j in range(rc):
            kw = kws[r0 + j]
            run = BatchRun(b, j, kw["fk"], N, scheme, float(kw.get("ESSrmin", 0.5)), seeds[r0 + j], table[j],
                           None if mtab is None else mtab[j], kw.get("collect"), cpu)
            out.append(run if out_func is None else out_func(run))
        del b, run                            # with out_func, nothing refers to this chunk's buffers any more
        r0 += rc
    if ev is not None:
        timer.append(ev)
    return out


def multiSMC(nruns=10, nprocs=0, out_func=None, collect=None, **args):
    """Run many SMC filters -- ``nruns`` per combination of the list- and dict-valued arguments -- as
    ``particles.multiSMC`` does (particles/core.py:431-518): same cartesian product, same output dicts (``'run'``,
    the varied arguments, ``'seed'``, ``'output'``), same seeds after ``np.random.seed``; ``collect`` is never part
    of the product.  ``'output'`` is ``out_func(run)``, or the run itself (merged into the dict when ``out_func``
    returns a dict).  As in the reference, ``out_func`` reduces each run as soon as it is done, so only what it
    returns is kept.

    On the device, a run's seed is its Philox key: output i is the run ``SMC(**args_i, seed=seed_i).run()``, up to
    the order of floating-point reductions.  Runs that share a model, Feynman-Kac kind, scheme, N, T and collectors
    form a group (``batch_key``); a group for which ``batch_pays`` holds goes through batched launches
    (csrc/smcb_batch.cu, one CTA per filter) and its runs are ``BatchRun`` objects.  Every other run goes one by one
    through ``SMC``.  ``nprocs`` is accepted and has no effect: the device is the parallelism."""
    from . import utils
    inputs, outputs = utils.expand(nruns=nruns, seeding=True, protected_args={"collect": collect}, **args)
    results = [None] * len(inputs)
    groups, single, specs = {}, [], {}
    for i, ip in enumerate(inputs):
        kw = {k: v for k, v in ip.items() if k != "seed"}
        key, spec = batch_key(kw, specs)
        if key is None:
            single.append(i)
        else:
            groups.setdefault(key, []).append((i, kw, spec))
    for key, members in groups.items():
        n_sm = torch.cuda.get_device_properties(context().device).multi_processor_count
        if not batch_pays(key[3], len(members), *plan_group(key, len(members)), n_sm=n_sm):
            single.extend(i for i, _, _ in members)
            continue
        outs = run_batch([kw for _, kw, _ in members], [inputs[i]["seed"] for i, _, _ in members],
                         out_func=out_func, _planned=(key, [spec for _, _, spec in members]))
        for (i, _, _), o in zip(members, outs):
            results[i] = o
    for i in sorted(single):
        kw = dict(inputs[i])
        seed = kw.pop("seed")
        if seed:
            np.random.seed(seed)                # what the reference's seeder does before each run
        pf = SMC(seed=int(seed), **kw)
        pf.run()
        results[i] = pf if out_func is None else out_func(pf)
        del pf
    return [utils.add_to_dict(op, res) for op, res in zip(outputs, results)]
