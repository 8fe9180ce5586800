"""ctypes binding of libsmcb.so (the C-ABI declared in include/smcb.h).

The product path has NO CPU fallback: if the library is missing or no CUDA device
is visible, the calls below raise instead of computing somewhere else.
"""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.environ.get("SMCB_LIB") or os.path.join(HERE, "libsmcb.so")   # SMCB_LIB: kernel-variant experiments

SMCB_MAX_PARAMS = 256
SUMMARY_STRIDE = 4

OK, EINVAL, ECUDA, ENOSYS = 0, -1, -2, -3   # return codes of every entry point

RS_CODES = {"multinomial": 0, "stratified": 1, "systematic": 2, "residual": 3, "ssp": 4}
FUSED_SCHEMES = ("multinomial", "stratified", "systematic")     # schemes built into the fused step kernel
FK_BOOTSTRAP, FK_GUIDED, FK_APF, FK_AUXBOOT = 0, 1, 2, 3
MODEL_STOCHVOL, MODEL_LINGAUSS, MODEL_GORDON, MODEL_THETALOGISTIC = 0, 1, 2, 3
MODEL_BEARINGS, MODEL_MVLINGAUSS, MODEL_DISCRETECOX, MODEL_STOCHVOLLEV = 4, 5, 6, 7
LSE_SUM, LSE_MEAN, LSE_ESSL = 0, 1, 2
# law codes of smcb_dist_logpdf / smcb_dist_rvs
LAW_INVGAMMA, LAW_LOGNORMAL, LAW_TRUNCNORMAL, LAW_BINOMIAL, LAW_GEOMETRIC = 0, 1, 2, 3, 4
LAW_NEGBINOMIAL, LAW_DISCRETEUNIFORM, LAW_GAMMA, LAW_NORMAL, LAW_STUDENT = 5, 6, 7, 8, 9
LAW_LAPLACE, LAW_LOGISTIC = 10, 11
# bits of smcb_dirichlet_logpdf's *bad: the tests of scipy.stats.dirichlet's input check
DIRICHLET_RANGE, DIRICHLET_ZERO, DIRICHLET_SUM, DIRICHLET_NAN = 1, 2, 4, 8

c_dp = C.c_void_p  # device pointers travel as integers


# Every descriptor has __slots__ = (): a misspelt field name raises AttributeError instead of creating a Python
# attribute that the library never reads.
class FilterDesc(C.Structure):
    __slots__ = ()
    _fields_ = [
        ("model", C.c_int32), ("fk", C.c_int32), ("scheme", C.c_int32), ("dim", C.c_int32),
        ("dy", C.c_int32), ("n_params", C.c_int32), ("world", C.c_int32), ("rank", C.c_int32),
        ("n", C.c_int64), ("n_global", C.c_int64), ("index_offset", C.c_int64), ("T", C.c_int64),
        ("essrmin", C.c_double), ("seed", C.c_uint64),
        ("params", C.c_double * SMCB_MAX_PARAMS),
        ("X", c_dp * 2), ("lw", c_dp * 2), ("A", c_dp), ("cdf", c_dp), ("data", c_dp),
        ("summaries", c_dp), ("z_in", c_dp), ("u_in", c_dp), ("scratch", c_dp),
        ("step_consts", c_dp), ("local_stats", c_dp), ("gathered", c_dp),
        ("mail_local", c_dp), ("mail_peer", c_dp * 8),
        ("rs_global", C.c_int32), ("reserved0", C.c_int32), ("moments", c_dp), ("reserved1", c_dp),
        ("peer_X0", c_dp * 8), ("peer_X1", c_dp * 8), ("peer_cdf", c_dp * 8),
    ]


SMOOTH_ON2, SMOOTH_MCMC, SMOOTH_REJECT, SMOOTH_GATHER = 0, 1, 2, 3


class SmoothDesc(C.Structure):
    __slots__ = ()
    _fields_ = [
        ("method", C.c_int32), ("model", C.c_int32), ("dim", C.c_int32), ("n_params", C.c_int32),
        ("T", C.c_int64), ("N", C.c_int64), ("M", C.c_int64), ("nsteps", C.c_int64), ("max_trials", C.c_int64),
        ("params", C.c_double * SMCB_MAX_PARAMS), ("step_consts", c_dp),
        ("X", c_dp), ("lw", c_dp), ("A", c_dp), ("x_stride_n", C.c_int64), ("x_stride_c", C.c_int64),
        ("log_bound", c_dp), ("cdf", c_dp), ("cdf_ld", C.c_int64), ("idx_T", c_dp),
        ("u", c_dp), ("prop", c_dp), ("lu", c_dp), ("u_exact", c_dp),
        ("idx", c_dp), ("paths", c_dp), ("counts", c_dp), ("order", c_dp),
    ]


ONLINE_PARIS, ONLINE_ON2_W, ONLINE_PHI_PARIS, ONLINE_PHI_ON2 = 0, 1, 2, 3


class OnlineDesc(C.Structure):
    __slots__ = ()
    _fields_ = [
        ("method", C.c_int32), ("model", C.c_int32), ("dim", C.c_int32), ("n_params", C.c_int32),
        ("t", C.c_int64), ("N", C.c_int64), ("Np", C.c_int64), ("max_trials", C.c_int64),
        ("row0", C.c_int64), ("rows", C.c_int64), ("k", C.c_int64), ("seed", C.c_uint64),
        ("log_bound", C.c_double), ("step_const", C.c_double), ("params", C.c_double * SMCB_MAX_PARAMS),
        ("X_prev", c_dp), ("X", c_dp), ("x_stride_n", C.c_int64), ("x_stride_c", C.c_int64),
        ("lw_prev", c_dp), ("cdf", c_dp), ("prop", c_dp), ("lu", c_dp), ("u_exact", c_dp),
        ("B", c_dp), ("counts", c_dp), ("omega", c_dp), ("phi_prev", c_dp), ("psi", c_dp), ("phi", c_dp),
    ]


TF_ON2_ROWS, TF_ON_LOGW = 0, 1


class TwoFilterDesc(C.Structure):
    __slots__ = ()
    _fields_ = [
        ("method", C.c_int32), ("model", C.c_int32), ("dim", C.c_int32), ("n_params", C.c_int32),
        ("t", C.c_int64), ("N", C.c_int64), ("Ninfo", C.c_int64), ("row0", C.c_int64), ("rows", C.c_int64),
        ("M", C.c_int64), ("step_const", C.c_double), ("params", C.c_double * SMCB_MAX_PARAMS),
        ("X", c_dp), ("Xinfo", c_dp), ("x_stride", C.c_int64), ("xi_stride", C.c_int64),
        ("lw", c_dp), ("psi", c_dp), ("L", c_dp), ("S", c_dp), ("I", c_dp), ("J", c_dp), ("mf", c_dp), ("mi", c_dp),
        ("log_omega", c_dp), ("xf", c_dp), ("xi", c_dp),
    ]


VAR_EVE, VAR_SUMS = 0, 1
VAR_CENTRED, VAR_WEIGHTS = 0, 1


class VarDesc(C.Structure):
    __slots__ = ()
    _fields_ = [
        ("method", C.c_int32), ("mode", C.c_int32), ("lin_w", C.c_int32), ("rs_host", C.c_int32),
        ("N", C.c_int64), ("k", C.c_int64), ("L", C.c_int64),
        ("rs_flag", c_dp), ("parity", c_dp), ("B", c_dp * 2), ("A", c_dp), ("lw", c_dp), ("phi", c_dp),
        ("lw_rows", c_dp), ("phi_rows", c_dp), ("row_ld", C.c_int64), ("zero", c_dp), ("unsorted", c_dp),
        ("scratch", c_dp), ("out", c_dp),
    ]


BATCH_AUTO, BATCH_RESIDENT, BATCH_STREAMING = 0, 1, 2
BATCH_TIERS = {"auto": BATCH_AUTO, "resident": BATCH_RESIDENT, "streaming": BATCH_STREAMING}


class BatchDesc(C.Structure):
    __slots__ = ()
    _fields_ = [
        ("model", C.c_int32), ("fk", C.c_int32), ("scheme", C.c_int32), ("dim", C.c_int32),
        ("dy", C.c_int32), ("n_params", C.c_int32), ("tier", C.c_int32), ("reserved0", C.c_int32),
        ("N", C.c_int64), ("T", C.c_int64), ("R", C.c_int64),
        ("seed", c_dp), ("essrmin", c_dp), ("params", c_dp), ("data", c_dp), ("step_consts", c_dp),
        ("X", c_dp), ("lw", c_dp), ("A", c_dp), ("cdf", c_dp), ("scratch", c_dp),
        ("summaries", c_dp), ("moments", c_dp), ("z_in", c_dp), ("u_in", c_dp),
    ]


BANK_STATE = 8


class BankDesc(C.Structure):
    __slots__ = ()
    _fields_ = [
        ("model", C.c_int32), ("fk", C.c_int32), ("scheme", C.c_int32), ("tier", C.c_int32),
        ("n_params", C.c_int32), ("restart", C.c_int32),
        ("N", C.c_int64), ("T", C.c_int64), ("R", C.c_int64), ("t1", C.c_int64),
        ("idx", c_dp), ("n_idx", C.c_int64), ("essrmin", C.c_double),
        ("key", c_dp), ("params", c_dp), ("data", c_dp), ("step_consts", c_dp), ("sc_ld", C.c_int64),
        ("X", c_dp), ("lw", c_dp), ("state", c_dp), ("A", c_dp), ("summaries", c_dp),
        ("cdf", c_dp), ("scratch", c_dp), ("scratch_rows", C.c_int64),
    ]


CSMC_GENEALOGY, CSMC_BACKWARD = 0, 1


class CsmcDesc(C.Structure):
    __slots__ = ()
    _fields_ = [
        ("model", C.c_int32), ("fk", C.c_int32), ("n_params", C.c_int32), ("draw", C.c_int32),
        ("pin", C.c_int32), ("reserved0", C.c_int32),
        ("N", C.c_int64), ("T", C.c_int64), ("R", C.c_int64), ("essrmin", C.c_double),
        ("key", c_dp), ("params", c_dp), ("data", c_dp), ("data_ld", C.c_int64),
        ("step_consts", c_dp), ("sc_ld", C.c_int64), ("xstar", c_dp),
        ("X", c_dp), ("lw", c_dp), ("A", c_dp), ("traj", c_dp), ("logLt", c_dp), ("summaries", c_dp),
        ("z_in", c_dp), ("u_in", c_dp), ("ud_in", c_dp),
    ]


HMM_FORWARD, HMM_BACKWARD, HMM_SAMPLE = 0, 1, 2
HMM_MAX_K = 128


class HmmDesc(C.Structure):
    __slots__ = ()
    _fields_ = [
        ("method", C.c_int32), ("K", C.c_int32), ("B", C.c_int64), ("ld", C.c_int64),
        ("t0", C.c_int64), ("t1", C.c_int64), ("N", C.c_int64), ("seed", C.c_uint64),
        ("trans", c_dp), ("trans_stride", C.c_int64), ("init", c_dp), ("init_stride", C.c_int64),
        ("logft", c_dp), ("pred", c_dp), ("filt", c_dp), ("logpyt", c_dp), ("smth", c_dp),
        ("U", c_dp), ("paths", c_dp),
    ]


KALMAN_FILTER, KALMAN_SMOOTH = 0, 1
KALMAN_MAX_D = 32


class KalmanDesc(C.Structure):
    __slots__ = ()
    _fields_ = [
        ("method", C.c_int32), ("dx", C.c_int32), ("dy", C.c_int32), ("pad_", C.c_int32),
        ("B", C.c_int64), ("ld", C.c_int64), ("t0", C.c_int64), ("t1", C.c_int64),
        ("F", c_dp), ("G", c_dp), ("covX", c_dp), ("covY", c_dp), ("mu0", c_dp), ("cov0", c_dp),
        ("F_stride", C.c_int64), ("G_stride", C.c_int64), ("covX_stride", C.c_int64), ("covY_stride", C.c_int64),
        ("mu0_stride", C.c_int64), ("cov0_stride", C.c_int64), ("y", c_dp), ("y_stride", C.c_int64),
        ("pred_mean", c_dp), ("pred_cov", c_dp), ("filt_mean", c_dp), ("filt_cov", c_dp), ("logpyt", c_dp),
        ("smth_mean", c_dp), ("smth_cov", c_dp),
    ]


class VsDesc(C.Structure):
    __slots__ = ()
    _fields_ = [
        ("p", C.c_int32), ("use_ldet", C.c_int32), ("xtx", c_dp), ("xty", c_dp), ("vm2", C.c_double),
        ("coef_len", C.c_double), ("coef_log", C.c_double), ("coef_in_log", C.c_double), ("gw", C.c_double),
        ("lq", C.c_double), ("l1q", C.c_double),
    ]


# name -> (restype, argtypes): every symbol include/smcb.h declares
PROTOTYPES = {
    "smcb_last_error": (C.c_char_p, []),
    "smcb_version": (C.c_int, []),
    "smcb_create": (C.c_int, [C.POINTER(C.c_void_p), C.c_int, C.c_uint64]),
    "smcb_destroy": (C.c_int, [C.c_void_p]),
    "smcb_set_stream": (C.c_int, [C.c_void_p, C.c_void_p]),
    "smcb_seed": (C.c_int, [C.c_void_p, C.c_uint64]),
    "smcb_launch_count": (C.c_int64, [C.c_void_p]),
    "smcb_normalise": (C.c_int, [C.c_void_p, c_dp, C.c_int64, c_dp, c_dp]),
    "smcb_weights_from_stats": (C.c_int, [C.c_void_p, c_dp, C.c_int64, c_dp, c_dp]),
    "smcb_lse": (C.c_int, [C.c_void_p, C.c_int, c_dp, c_dp, C.c_int64, c_dp]),
    "smcb_exp_and_normalise": (C.c_int, [C.c_void_p, c_dp, C.c_int64, c_dp]),
    "smcb_wmean_and_var": (C.c_int, [C.c_void_p, c_dp, c_dp, C.c_int64, C.c_int, c_dp]),
    "smcb_cumsum": (C.c_int, [C.c_void_p, c_dp, C.c_int64, c_dp]),
    "smcb_searchsorted": (C.c_int, [C.c_void_p, c_dp, C.c_int64, c_dp, C.c_int64, c_dp]),
    "smcb_resample_scratch_doubles": (C.c_int64, [C.c_int64, C.c_int64]),
    "smcb_resample": (C.c_int, [C.c_void_p, C.c_int, c_dp, C.c_int64, C.c_int64, c_dp, c_dp, c_dp]),
    "smcb_gather": (C.c_int, [C.c_void_p, c_dp, C.c_int64, c_dp, C.c_int64, C.c_int, c_dp]),
    "smcb_gather_rows": (C.c_int, [C.c_void_p, c_dp, C.c_int64, c_dp, C.c_int64, C.c_int, c_dp]),
    "smcb_normal_rvs": (C.c_int, [C.c_void_p, c_dp, C.c_double, c_dp, C.c_double, c_dp, c_dp, C.c_int64]),
    "smcb_mvnormal_rvs": (C.c_int, [C.c_void_p, c_dp, c_dp, c_dp, c_dp, c_dp, C.c_int, c_dp, c_dp, C.c_int64]),
    "smcb_mvnormal_logpdf": (C.c_int, [C.c_void_p, c_dp, c_dp, c_dp, c_dp, c_dp, c_dp, C.c_int, c_dp,
                                       C.c_int64]),
    "smcb_standard_normal": (C.c_int, [C.c_void_p, c_dp, C.c_int64]),
    "smcb_uniform": (C.c_int, [C.c_void_p, c_dp, C.c_int64]),
    "smcb_dist_logpdf": (C.c_int, [C.c_void_p, C.c_int, c_dp, C.c_double, c_dp, c_dp, c_dp, c_dp, c_dp, c_dp,
                                   C.c_int64]),
    "smcb_dist_rvs": (C.c_int, [C.c_void_p, C.c_int, c_dp, c_dp, c_dp, c_dp, c_dp, c_dp, C.c_int64]),
    "smcb_dirichlet_logpdf": (C.c_int, [C.c_void_p, c_dp, C.c_int64, c_dp, C.c_int, C.c_double, c_dp, c_dp,
                                        C.c_int64]),
    "smcb_dirichlet_rvs": (C.c_int, [C.c_void_p, c_dp, C.c_int, c_dp, C.c_int64]),
    "smcb_vcn_chol": (C.c_int, [C.c_void_p, c_dp, C.c_int, c_dp, c_dp, C.c_int64]),
    "smcb_vcn_rvs": (C.c_int, [C.c_void_p, c_dp, C.c_int64, c_dp, C.c_int, c_dp, C.c_int64]),
    "smcb_vcn_logpdf": (C.c_int, [C.c_void_p, c_dp, C.c_int64, c_dp, C.c_int64, c_dp, C.c_int, c_dp, C.c_int64]),
    "smcb_mixture_logpdf": (C.c_int, [C.c_void_p, c_dp, c_dp, C.c_int64, C.c_int, c_dp, C.c_int64]),
    "smcb_logistic_target": (C.c_int, [C.c_void_p, c_dp, C.c_int64, C.c_int, c_dp, C.c_int64, C.c_double,
                                       C.c_double, c_dp, c_dp, c_dp]),
    "smcb_logistic_wf_move": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_int, c_dp, c_dp, c_dp, c_dp, c_dp,
                                        C.c_int64, C.c_double, C.c_double, c_dp, c_dp, c_dp, c_dp, c_dp, c_dp,
                                        c_dp, c_dp]),
    "smcb_logistic_logpyt": (C.c_int, [C.c_void_p, c_dp, C.c_int64, C.c_int, c_dp, C.c_int64, C.c_int64, C.c_int64,
                                       C.c_int, c_dp, c_dp, c_dp, c_dp]),
    "smcb_logistic_ns_target": (C.c_int, [C.c_void_p, c_dp, C.c_int64, C.c_int, c_dp, C.c_int64, C.c_double,
                                          C.c_double, c_dp, c_dp, c_dp]),
    "smcb_logistic_ns_move": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, C.c_int, c_dp, c_dp, c_dp, c_dp, c_dp,
                                        C.c_int64, C.c_double, C.c_double, c_dp, c_dp, c_dp, c_dp, c_dp, c_dp,
                                        c_dp, c_dp]),
    "smcb_ns_threshold": (C.c_int, [C.c_void_p, c_dp, C.c_int64, C.c_int64, C.c_int64, C.c_double, C.c_int,
                                    C.c_double, C.c_double, C.c_double, c_dp, c_dp]),
    "smcb_vs_loglik": (C.c_int, [C.c_void_p, C.POINTER(VsDesc), c_dp, C.c_int64, C.c_int, C.c_double, C.c_double,
                                 c_dp, c_dp, c_dp, c_dp, c_dp, c_dp, c_dp]),
    "smcb_nested_logistic": (C.c_int, [C.c_void_p, C.c_int, c_dp, c_dp, C.c_int64, C.c_int, c_dp, c_dp, c_dp]),
    "smcb_binary_wf_move": (C.c_int, [C.c_void_p, C.POINTER(VsDesc), c_dp, c_dp, C.c_int64, C.c_int, C.c_double,
                                      c_dp, c_dp, c_dp, c_dp, c_dp, c_dp, c_dp, c_dp, c_dp, c_dp, c_dp, c_dp]),
    "smcb_rw_propose": (C.c_int, [C.c_void_p, c_dp, C.c_int64, C.c_int, c_dp, c_dp, c_dp]),
    "smcb_mh_accept": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, c_dp, c_dp, c_dp, c_dp, c_dp, c_dp, c_dp, c_dp,
                                 c_dp, c_dp]),
    "smcb_next_annealing_epn": (C.c_int, [C.c_void_p, c_dp, C.c_int64, C.c_double, C.c_double, c_dp]),
    "smcb_rw_calibrate": (C.c_int, [C.c_void_p, c_dp, c_dp, C.c_int64, C.c_int, C.c_double, c_dp]),
    "smcb_essl_grid": (C.c_int, [C.c_void_p, c_dp, C.c_int64, C.c_double, C.c_double, c_dp, c_dp]),
    "smcb_wcov_sums": (C.c_int, [C.c_void_p, c_dp, c_dp, C.c_int64, C.c_int, c_dp, c_dp]),
    "smcb_chol_from_sums": (C.c_int, [C.c_void_p, c_dp, c_dp, C.c_int, C.c_double, c_dp]),
    "smcb_device_math": (C.c_int, [C.c_void_p, C.c_int, c_dp, c_dp, C.c_int64]),
    "smcb_filter_create": (C.c_int, [C.c_void_p, C.POINTER(FilterDesc), C.POINTER(C.c_void_p)]),
    "smcb_filter_destroy": (C.c_int, [C.c_void_p]),
    "smcb_filter_step": (C.c_int, [C.c_void_p, C.c_int64]),
    "smcb_filter_step_local": (C.c_int, [C.c_void_p]),
    "smcb_filter_step_finish": (C.c_int, [C.c_void_p]),
    "smcb_p2p_alloc": (C.c_int, [C.c_void_p, C.c_int64, C.POINTER(C.c_void_p), C.c_char_p]),
    "smcb_p2p_open": (C.c_int, [C.c_void_p, C.c_char_p, C.POINTER(C.c_void_p)]),
    "smcb_p2p_close": (C.c_int, [C.c_void_p]),
    "smcb_p2p_free": (C.c_int, [C.c_void_p]),
    "smcb_filter_step_timed": (C.c_int, [C.c_void_p, C.c_int64, C.POINTER(C.c_double)]),
    "smcb_filter_state": (C.c_int, [C.c_void_p, C.POINTER(C.c_double)]),
    "smcb_filter_fusion_stats": (C.c_int, [C.c_void_p, C.POINTER(C.c_int64)]),
    "smcb_sobol": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_int, C.c_uint64, C.c_uint64, c_dp, c_dp]),
    "smcb_hilbert_scratch_bytes": (C.c_int64, [C.c_int64, C.c_int]),
    "smcb_hilbert_sort": (C.c_int, [C.c_void_p, c_dp, C.c_int64, C.c_int, c_dp, c_dp, c_dp]),
    "smcb_sqmc_scratch_bytes": (C.c_int64, [C.c_int64, C.c_int]),
    "smcb_sqmc_step": (C.c_int, [C.c_void_p, C.c_int64, c_dp]),
    "smcb_ndtri": (C.c_int, [C.c_void_p, c_dp, c_dp, C.c_int64]),
    "smcb_backward_sample": (C.c_int, [C.c_void_p, C.POINTER(SmoothDesc)]),
    "smcb_online_smooth": (C.c_int, [C.c_void_p, C.POINTER(OnlineDesc)]),
    "smcb_two_filter": (C.c_int, [C.c_void_p, C.POINTER(TwoFilterDesc)]),
    "smcb_variance": (C.c_int, [C.c_void_p, C.POINTER(VarDesc)]),
    "smcb_variance_scratch_doubles": (C.c_int64, [C.c_int64, C.c_int64, C.c_int64]),
    "smcb_batch_plan": (C.c_int, [C.c_void_p, C.POINTER(BatchDesc), C.POINTER(C.c_int64)]),
    "smcb_batch_run": (C.c_int, [C.c_void_p, C.POINTER(BatchDesc)]),
    "smcb_bank_plan": (C.c_int, [C.c_void_p, C.POINTER(BankDesc), C.POINTER(C.c_int64)]),
    "smcb_bank_advance": (C.c_int, [C.c_void_p, C.POINTER(BankDesc)]),
    "smcb_bank_gather": (C.c_int, [C.c_void_p, C.POINTER(BankDesc), c_dp, C.c_int64, C.POINTER(BankDesc),
                                   C.c_uint64, C.c_uint64, c_dp]),
    "smcb_bank_merge": (C.c_int, [C.c_void_p, C.POINTER(BankDesc), C.POINTER(BankDesc), c_dp]),
    "smcb_bank_keys": (C.c_int, [C.c_void_p, c_dp, C.c_int64, C.c_uint64, C.c_uint64]),
    "smcb_mh_accept_flags": (C.c_int, [C.c_void_p, C.c_int64, C.c_int, c_dp, c_dp, c_dp, c_dp, c_dp, c_dp, c_dp,
                                       c_dp, c_dp, c_dp, c_dp]),
    "smcb_csmc_plan": (C.c_int, [C.c_void_p, C.POINTER(CsmcDesc), C.POINTER(C.c_int64)]),
    "smcb_csmc_run": (C.c_int, [C.c_void_p, C.POINTER(CsmcDesc)]),
    "smcb_hmm": (C.c_int, [C.c_void_p, C.POINTER(HmmDesc)]),
    "smcb_kalman": (C.c_int, [C.c_void_p, C.POINTER(KalmanDesc)]),
}

_lib = None


class SmcbError(RuntimeError):
    pass


def load():
    """Load libsmcb.so and bind every prototype (no GPU needed for this)."""
    global _lib
    if _lib is None:
        if not os.path.exists(SO_PATH):
            raise SmcbError(
                f"{SO_PATH} is missing: build it with `python -m particles_b200.build` "
                "(there is no CPU fallback for this path)")
        lib = C.CDLL(SO_PATH)
        for name, (res, args) in PROTOTYPES.items():
            fn = getattr(lib, name)   # AttributeError if the symbol is not exported
            fn.restype, fn.argtypes = res, args
        _lib = lib
    return _lib


def check(rc):
    if rc == OK:
        return
    msg = load().smcb_last_error().decode()
    if rc == EINVAL:
        raise ValueError(msg)
    if rc == ENOSYS:
        raise NotImplementedError(msg)
    raise SmcbError(msg)
