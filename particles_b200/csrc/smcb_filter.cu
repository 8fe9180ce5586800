// smcb_filter.cu -- host side of the fused filter (C-ABI entry points) + the 1-D model family.
// The kernels live in smcb_step.cuh; the d-dimensional models are instantiated in
// smcb_filter_nd.cu so that the two translation units compile in parallel.
#include <stdlib.h>

#include "smcb_step.cuh"

int smcb_bind_nd(smcb_filter *f);      // smcb_filter_nd.cu
int smcb_bind_1d_more(smcb_filter *f); // smcb_filter_1d.cu

static int smcb_bind_1d(smcb_filter *f) {
    const smcb_filter_desc *d = &f->desc;
    switch (d->model) {
        case SMCB_MODEL_STOCHVOL: return bind_fk<StochVolM>(f);
        case SMCB_MODEL_LINGAUSS: return bind_fk<LinGaussM>(f);
        case SMCB_MODEL_GORDON:
        case SMCB_MODEL_THETALOGISTIC:
        case SMCB_MODEL_DISCRETECOX:
        case SMCB_MODEL_STOCHVOLLEV: return smcb_bind_1d_more(f);
        default:
            set_error("fused filter: model id %d is not available in the fused 1-D family", d->model);
            return SMCB_ENOSYS;
    }
}

static int filter_setup(smcb_filter *f, smcb_ctx *c, const smcb_filter_desc *d);

extern "C" int smcb_filter_create(smcb_ctx *c, const smcb_filter_desc *d, smcb_filter **out) {
    SMCB_REQUIRE(c && d && out, "smcb_filter_create: NULL argument");
    SMCB_REQUIRE(d->n >= 1 && d->T >= 1, "smcb_filter_create: need n >= 1 and T >= 1");
    SMCB_REQUIRE(d->X[0] && d->X[1] && d->lw[0] && d->lw[1] && d->A && d->cdf && d->data && d->summaries,
                 "smcb_filter_create: NULL device buffer");
    SMCB_REQUIRE((d->index_offset & 1) == 0, "smcb_filter_create: index_offset must be even");
    SMCB_REQUIRE(d->dim >= 1 && d->dim <= 4, "smcb_filter_create: fused kernels exist for state dimension 1..4 (dim=%d)", d->dim);
    SMCB_REQUIRE(d->dy >= 1 && d->dy <= kMaxDy, "smcb_filter_create: observation dimension must be 1..%d", kMaxDy);
    SMCB_REQUIRE(d->essrmin >= 0.0 && d->essrmin <= 1.0, "smcb_filter_create: ESSrmin must be in [0, 1]");
    smcb_filter *f = new (std::nothrow) smcb_filter();
    SMCB_REQUIRE(f != nullptr, "smcb_filter_create: out of host memory");
    f->ctx = c;
    f->desc = *d;
    f->t_host = 0;
    f->timed = false;
    f->mem = nullptr;
    const int rc = filter_setup(f, c, d);
    if (rc) {                       // nothing of a half-built filter survives an error
        if (f->mem) cudaFree(f->mem);
        delete f;
        return rc;
    }
    *out = f;
    return SMCB_OK;
}

static bool env_flag(const char *name, bool dflt) {
    const char *v = getenv(name);
    if (!v || !*v) return dflt;
    return v[0] != '0';
}

static int filter_setup(smcb_filter *f, smcb_ctx *c, const smcb_filter_desc *d) {
    int rc = (d->dim == 1) ? smcb_bind_1d(f) : smcb_bind_nd(f);
    if (rc) return rc;

    const int64_t n = d->n;
    FilterArgs &a = f->args;
    memset(&a, 0, sizeof(a));
    a.math_tab = c->math_tab;
    a.X[0] = d->X[0]; a.X[1] = d->X[1]; a.lw[0] = d->lw[0]; a.lw[1] = d->lw[1];
    a.A = reinterpret_cast<long long *>(d->A);
    a.cdf = d->cdf;
    a.su = (d->scheme == SMCB_RS_MULTINOMIAL) ? d->scratch : nullptr;
    SMCB_REQUIRE(d->scheme != SMCB_RS_MULTINOMIAL || d->scratch != nullptr,
                 "smcb_filter_create: multinomial needs desc.scratch of n + 2 doubles");
    a.data = d->data;
    a.sc = d->step_consts;
    a.summaries = d->summaries;
    a.moments = d->moments;
    a.z_in = d->z_in; a.u_in = d->u_in;
    a.dy = d->dy;
    a.n = n; a.n_global = d->n_global > 0 ? d->n_global : n;
    a.index_offset = d->index_offset; a.T = d->T;
    a.essrmin = d->essrmin;
    a.key = key_of(d->seed);
    {   // one CTA per SM, each owning a contiguous range of pairs; at least one pair per thread and CTA
        int dev = 0, sms = kSMs;
        SMCB_CUDA(cudaGetDevice(&dev));
        SMCB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
        const int64_t npairs = (n + 1) / 2;
        int64_t g = sms < kMaxStepGrid ? sms : kMaxStepGrid;
        const int64_t gmax = (npairs + f->block_size - 1) / f->block_size;
        if (g > gmax) g = gmax;
        if (g < 1) g = 1;
        int64_t chunk = (npairs + g - 1) / g;
        g = (npairs + chunk - 1) / chunk;
        a.chunk = chunk;
        f->grid_move = (int)g;
        a.grid = f->grid_move;
        // slabs of the streaming branch (smcb_step.cuh): records in the (otherwise idle) CDF staging buffers
        const bool apf = d->fk == SMCB_FK_APF || d->fk == SMCB_FK_AUXBOOT;
        const bool mom = d->moments != nullptr;
        a.slab_lane = (!apf && !mom) ? 1 : 0;
        a.slab_stride = a.slab_lane ? 96 : 4 + (apf ? 4 : 0) + (mom ? 2 * d->dim : 0);
        const int64_t cap = f->slab_doubles / a.slab_stride;
        const int64_t n_iter = (chunk + f->pairs_per_iteration - 1) / f->pairs_per_iteration;
        // smallest slab (>= 2 iterations) whose records fit next to a tail of at least ~one single-iteration slab
        // per warp: n_big + n_small <= cap with n_big = ceil((n_iter - n_small) / slab_it)
        int64_t slab_it = 2, n_small = 0;
        for (;; slab_it++) {
            const int64_t ns = (cap * slab_it - n_iter) / (slab_it - 1) - 1;
            const int64_t want = n_iter < 32 ? n_iter : 32;
            if (ns >= want) { n_small = ns < 0 ? 0 : (ns > n_iter / 8 ? n_iter / 8 : ns); break; }
        }
        if (n_small > n_iter) n_small = n_iter;
        a.slab_it = (int)slab_it;
        a.slab_small = (int)n_small;
    }
    a.world = d->world > 1 ? d->world : 1;
    a.rank = d->world > 1 ? d->rank : 0;
    // fused pairs of streaming steps (smcb_step.cuh): 1-D, single device; SMCB_FUSE=0 off, 1 on (default),
    // 2 fuse whenever allowed (no predictor: every resampling step after a streaming one is a misprediction)
    {
        const char *v = getenv("SMCB_FUSE");
        const int mode = (!v || !*v) ? 1 : (v[0] == '0' ? 0 : (v[0] == '2' ? 2 : 1));
        a.fuse_mode = (d->dim == 1 && a.world == 1) ? mode : 0;
    }
    // device memory: header (StepState[2] | fusion words | grid-barrier counter | timeout flag) + partials + block
    // aggregates [+ the second step's slab records of a fused pair]
    constexpr size_t kHdr = 512;
    static_assert(2 * sizeof(StepState) <= 256, "StepState outgrew its header slot");
    const size_t part = (size_t)kPartSlots * kMaxStepGrid * kPartStride * sizeof(double);
    const size_t agg = (size_t)(kMaxStepGrid + 8) * sizeof(double);
    const size_t slab = a.fuse_mode ? (size_t)f->grid_move * f->slab_doubles * sizeof(double) : 0;
    SMCB_CUDA(cudaMalloc(&f->mem, kHdr + part + agg + slab));
    SMCB_CUDA(cudaMemsetAsync(f->mem, 0, kHdr + part + agg, c->stream));
    a.st = reinterpret_cast<StepState *>(f->mem);
    a.fuse = reinterpret_cast<long long *>(f->mem + 256);
    a.bar = reinterpret_cast<unsigned long long *>(f->mem + 384);
    a.sync_timeout = reinterpret_cast<int *>(f->mem + 392);
    a.partials = reinterpret_cast<double *>(f->mem + kHdr);
    a.blk_agg = reinterpret_cast<double *>(f->mem + kHdr + part);
    a.fuse_slab = a.fuse_mode ? reinterpret_cast<double *>(f->mem + kHdr + part + agg) : nullptr;
    a.local_stats = d->local_stats;
    a.gathered = d->gathered;
    a.mail_local = (a.world > 1) ? d->mail_local : nullptr;
    for (int r = 0; r < 8; r++) a.mail_peer[r] = (a.world > 1 && r < a.world) ? d->mail_peer[r] : nullptr;
    SMCB_REQUIRE(a.world == 1 || (a.rank >= 0 && a.rank < a.world), "smcb_filter_create: bad rank");
    SMCB_REQUIRE(a.world == 1 || a.mail_local || (d->local_stats && d->gathered),
                 "smcb_filter_create: world > 1 needs either a peer mailbox or local_stats / gathered");
    SMCB_REQUIRE(a.world <= 8, "smcb_filter_create: at most 8 ranks");
    if (a.mail_local) {
        for (int r = 0; r < a.world; r++)
            SMCB_REQUIRE(a.mail_peer[r] != nullptr, "smcb_filter_create: mail_peer[%d] is NULL", r);
    }
    a.rs_global = (a.world > 1 && d->rs_global) ? 1 : 0;
    if (a.rs_global) {
        SMCB_REQUIRE(a.mail_local != nullptr, "smcb_filter_create: global resampling needs the peer mailbox");
        SMCB_REQUIRE((n & 1) == 0, "smcb_filter_create: global resampling needs an even shard size");
        if (d->scheme != SMCB_RS_SYSTEMATIC && d->scheme != SMCB_RS_STRATIFIED) {
            set_error("fused filter: global resampling over shards supports systematic and stratified");
            return SMCB_ENOSYS;
        }
        for (int r = 0; r < a.world; r++) {
            SMCB_REQUIRE(d->peer_X0[r] && d->peer_X1[r] && d->peer_cdf[r],
                         "smcb_filter_create: peer_X0 / peer_X1 / peer_cdf[%d] is NULL", r);
            a.pX[r][0] = d->peer_X0[r]; a.pX[r][1] = d->peer_X1[r]; a.pcdf[r] = d->peer_cdf[r];
        }
    }
    // launch attributes: programmatic dependent launch hides the launch latency of step t+1 behind step t;
    // a cooperative launch guarantees the co-residency the grid barrier of a resampling step relies on
    // (the grid is one CTA per SM, so it is co-resident anyway unless another kernel occupies the device).
    f->pdl = env_flag("SMCB_PDL", true);
    f->coop = env_flag("SMCB_COOP", false);
    return SMCB_OK;
}

extern "C" int smcb_filter_destroy(smcb_filter *f) {
    if (!f) return SMCB_OK;
    cudaStreamSynchronize(f->ctx->stream);
    cudaFree(f->mem);
    delete f;
    return SMCB_OK;
}

static int launch_one(smcb_filter *f) {
    if (f->t_host >= f->desc.T) {
        set_error("smcb_filter_step: all %lld steps already done (StopIteration)", (long long)f->desc.T);
        return SMCB_EINVAL;
    }
    int rc = (f->t_host == 0) ? f->launch_init(f) : f->launch_step(f);
    if (rc && f->t_host > 0 && (f->pdl || f->coop)) {     // a launch attribute this driver rejects: plain launches
        cudaGetLastError();
        f->pdl = false; f->coop = false;
        rc = f->launch_step(f);
    }
    if (rc) return rc;
    f->t_host++;
    return SMCB_OK;
}

// sharded filters with the host-driven exchange: one step = step_local (this rank's step kernel, then its
// statistics in desc.local_stats), an all-gather of 16 doubles per rank done by the host layer (NCCL, same
// stream), then step_finish (summaries of the step: global log-normaliser, ESS, logLt, next decision)
extern "C" int smcb_filter_step_local(smcb_filter *f) {
    SMCB_REQUIRE(f != nullptr && f->args.world > 1 && f->args.mail_local == nullptr,
                 "smcb_filter_step_local: not a sharded filter with the host-driven exchange");
    f->args.batch_end = f->t_host + 1;
    int rc = launch_one(f);
    if (rc) return rc;
    return f->launch_publish(f);
}

extern "C" int smcb_filter_step_finish(smcb_filter *f) {
    SMCB_REQUIRE(f != nullptr && f->args.world > 1, "smcb_filter_step_finish: not a sharded filter");
    return f->launch_tail(f);
}

extern "C" int smcb_filter_step(smcb_filter *f, int64_t nsteps) {
    SMCB_REQUIRE(f != nullptr, "smcb_filter_step: NULL filter");
    SMCB_REQUIRE(f->args.world == 1 || f->args.mail_local != nullptr,
                 "smcb_filter_step: sharded filters without a peer mailbox use step_local / step_finish");
    if (nsteps <= 0) return SMCB_OK;
    f->args.batch_end = f->t_host + nsteps;       // a fused pair never reaches past the steps asked for
    // the device needs no host decision between steps: enqueue them all, then the tail that finalises the last
    for (int64_t i = 0; i < nsteps; i++) {
        int rc = launch_one(f);
        if (rc) return rc;
    }
    return f->launch_tail(f);
}

// Same as smcb_filter_step, with a CUDA-event pair around every kernel launch (on the launching stream, plain
// serialised launches).  out[0..3] = summed device milliseconds of {init, step kernels of resampling steps,
// tail, step kernels of non-resampling steps}, out[4..7] = number of launches of each.  Synchronises once.
extern "C" int smcb_filter_step_timed(smcb_filter *f, int64_t nsteps, double *out8) {
    SMCB_REQUIRE(f && out8, "smcb_filter_step_timed: NULL argument");
    SMCB_REQUIRE(nsteps >= 1 && nsteps <= 100000, "smcb_filter_step_timed: nsteps out of range");
    SMCB_REQUIRE(f->t_host + nsteps <= f->desc.T, "smcb_filter_step_timed: past the last step");
    SMCB_REQUIRE(f->args.world == 1, "smcb_filter_step_timed: single-device filters only");
    cudaStream_t s = f->ctx->stream;
    const size_t nev = (size_t)(nsteps + 1) * 2;
    cudaEvent_t *ev = new (std::nothrow) cudaEvent_t[nev];
    double *rows = new (std::nothrow) double[(size_t)nsteps * SMCB_SUMMARY_STRIDE];
    size_t made = 0;
    int rc = SMCB_OK;
    const int64_t t_first = f->t_host;
    auto fail = [&](cudaError_t e, const char *what) {
        set_error("smcb_filter_step_timed: %s -> %s", what, cudaGetErrorString(e));
        rc = SMCB_ECUDA;
    };
    if (!ev || !rows) { set_error("smcb_filter_step_timed: out of host memory"); rc = SMCB_EINVAL; }
    for (; rc == SMCB_OK && made < nev; made++) {
        cudaError_t e = cudaEventCreate(&ev[made]);
        if (e != cudaSuccess) { fail(e, "cudaEventCreate"); break; }
    }
    f->timed = true;
    f->args.batch_end = t_first + nsteps;
    for (int64_t i = 0; rc == SMCB_OK && i <= nsteps; i++) {
        cudaEventRecord(ev[2 * i], s);
        rc = (i < nsteps) ? launch_one(f) : f->launch_tail(f);
        cudaEventRecord(ev[2 * i + 1], s);
    }
    f->timed = false;
    if (rc == SMCB_OK) {
        cudaError_t e = cudaStreamSynchronize(s);
        if (e != cudaSuccess) fail(e, "cudaStreamSynchronize");
    }
    if (rc == SMCB_OK) {
        cudaError_t e = cudaMemcpy(rows, f->args.summaries + (size_t)t_first * SMCB_SUMMARY_STRIDE,
                                   sizeof(double) * nsteps * SMCB_SUMMARY_STRIDE, cudaMemcpyDeviceToHost);
        if (e != cudaSuccess) fail(e, "cudaMemcpy(summaries)");
    }
    if (rc == SMCB_OK) {
        for (int j = 0; j < 8; j++) out8[j] = 0.0;
        for (int64_t i = 0; i <= nsteps; i++) {
            float ms = 0.f;
            cudaEventElapsedTime(&ms, ev[2 * i], ev[2 * i + 1]);
            int kind = 2;                                            // tail
            if (i < nsteps) {
                const int64_t t = t_first + i;
                kind = (t == 0) ? 0 : (rows[(size_t)i * SMCB_SUMMARY_STRIDE + 2] != 0.0 ? 1 : 3);
            }
            out8[kind] += ms;
            out8[4 + kind] += 1.0;
        }
    }
    for (size_t i = 0; i < made; i++) cudaEventDestroy(ev[i]);
    delete[] ev;
    delete[] rows;
    return rc;
}

extern "C" int smcb_filter_state(smcb_filter *f, double *out8) {
    SMCB_REQUIRE(f && out8, "smcb_filter_state: NULL argument");
    SMCB_REQUIRE(f->t_host >= 1, "smcb_filter_state: no step has run yet");
    struct { StepState st[2]; char pad[384 - 2 * sizeof(StepState)]; unsigned long long bar; int timeout; int pad2; } h;
    static_assert(sizeof(h) == 400, "header snapshot layout");
    SMCB_CUDA(cudaMemcpyAsync(&h, f->mem, sizeof(h), cudaMemcpyDeviceToHost, f->ctx->stream));
    SMCB_CUDA(cudaStreamSynchronize(f->ctx->stream));
    const StepState &s = h.st[(f->t_host - 1) & 1];
    out8[0] = (double)(s.t + 1); out8[1] = (double)((f->t_host - 1) & 1); out8[2] = (double)s.rs; out8[3] = s.logLt;
    out8[4] = s.ess; out8[5] = s.log_mean_w; out8[6] = s.wm; out8[7] = s.ws;
    if (h.timeout) {
        set_error(h.timeout == 2 ? "fused filter: the grid barrier of a resampling step timed out (the step kernel was "
                                   "not co-resident: another kernel occupies the device)"
                                 : "sharded filter: a wait on a peer GPU's flag timed out (a rank died or fell out of step)");
        return SMCB_ECUDA;
    }
    if (s.t != f->t_host - 1) {
        set_error("smcb_filter_state: the last step is not finalised (internal error: t=%lld, expected %lld)",
                  (long long)s.t, (long long)(f->t_host - 1));
        return SMCB_ECUDA;
    }
    return SMCB_OK;
}

extern "C" int smcb_filter_fusion_stats(smcb_filter *f, int64_t *out3) {
    SMCB_REQUIRE(f && out3, "smcb_filter_fusion_stats: NULL argument");
    long long h[4];
    SMCB_CUDA(cudaMemcpyAsync(h, f->args.fuse, sizeof(h), cudaMemcpyDeviceToHost, f->ctx->stream));
    SMCB_CUDA(cudaStreamSynchronize(f->ctx->stream));
    for (int i = 0; i < 3; i++) out3[i] = h[1 + i];
    return SMCB_OK;
}

// ---------------------------------------------------------------------------
// peer memory for the fused statistics exchange (one process per GPU, same node)
// ---------------------------------------------------------------------------
extern "C" int smcb_p2p_alloc(smcb_ctx *c, int64_t bytes, void **dev_ptr, unsigned char *handle64) {
    SMCB_REQUIRE(c && dev_ptr && handle64 && bytes > 0, "smcb_p2p_alloc: bad argument");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    void *p = nullptr;
    SMCB_CUDA(cudaMalloc(&p, (size_t)bytes));
    SMCB_CUDA(cudaMemset(p, 0, (size_t)bytes));
    cudaIpcMemHandle_t h;
    SMCB_CUDA(cudaIpcGetMemHandle(&h, p));
    memcpy(handle64, &h, 64);
    *dev_ptr = p;
    return SMCB_OK;
}

extern "C" int smcb_p2p_open(smcb_ctx *c, const unsigned char *handle64, void **dev_ptr) {
    SMCB_REQUIRE(c && dev_ptr && handle64, "smcb_p2p_open: bad argument");
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, 64);
    SMCB_CUDA(cudaIpcOpenMemHandle(dev_ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return SMCB_OK;
}

extern "C" int smcb_p2p_close(void *peer_ptr) {
    if (peer_ptr) SMCB_CUDA(cudaIpcCloseMemHandle(peer_ptr));
    return SMCB_OK;
}

extern "C" int smcb_p2p_free(void *dev_ptr) {
    if (dev_ptr) SMCB_CUDA(cudaFree(dev_ptr));
    return SMCB_OK;
}
