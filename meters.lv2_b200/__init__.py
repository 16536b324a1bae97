"""meters.lv2_b200 — host-side mirror (Python/ctypes) of the b200meters C ABI (include/b200meters.h).

The product is the CUDA library `libb200meters.so` built in-tree from csrc/ by build.py; this module
only binds its C entry points for tests and bench.py.  Class and method names follow the reference's
DSP classes (Ebu_r128_proc, TruePeakdsp, Kmeterdsp, Stcorrdsp, the spectr30 plugin, the phasewheel
FFT analysis), each batched over N instances.  There is no CPU path: constructing a bank without the
built library or without a CUDA device raises.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200meters.so")
HIST_LEN = 751
MIX_WORDS = 1508
MAX_GROUPS = 65536          # B200M_MAX_GROUPS: albums per group_reduce / group_finish call
NO_GROUP = 0xFFFFFFFF       # B200M_NO_GROUP: an instance counted in no album (-1 in the Python interface)
MAX_BLOCK = 8192
_v = C.c_void_p
_lib = None


class B200MError(RuntimeError):
    pass


class EbuResult(C.Structure):
    _fields_ = [(n, C.c_float) for n in ("loudness_M", "maxloudn_M", "loudness_S", "maxloudn_S", "integrated",
                                          "integ_thr", "range_min", "range_max", "range_thr")] + \
               [("hist_M_count", C.c_int32), ("hist_S_count", C.c_int32), ("frag_power", C.c_float)]


EBU_RESULT_DTYPE = np.dtype([(n, "<f4") for n in ("loudness_M", "maxloudn_M", "loudness_S", "maxloudn_S", "integrated",
                                                    "integ_thr", "range_min", "range_max", "range_thr")] +
                            [("hist_M_count", "<i4"), ("hist_S_count", "<i4"), ("frag_power", "<f4")])
# one point of the loudness log (b200m_ebu_point): the values after one completed 50 ms fragment of an instance
EBU_POINT_DTYPE = np.dtype([(n, "<f4") for n in ("loudness_M", "loudness_S", "integrated", "range_min", "range_max")])
R128_POINT_DTYPE = np.dtype([(n, "<f4") for n in ("loudness_M", "loudness_S", "integrated", "range_min", "range_max", "dbtp")])
TPK_RESULT_DTYPE = np.dtype([("tp_m", "<f4"), ("tp_p", "<f4"), ("km_rms", "<f4"), ("km_peak", "<f4")])

_PROTOS = {
    "b200m_abi_version": (C.c_int, []),
    "b200m_last_error": (C.c_char_p, []),
    "b200m_device_count": (C.c_int, []),
    "b200m_host_alloc": (C.c_int, [C.POINTER(_v), C.c_size_t]),
    "b200m_host_free": (C.c_int, [_v]),
    "b200m_launch_count": (C.c_uint64, []),
    "b200m_peak_probe": (C.c_int, [C.c_int, C.c_int, C.POINTER(C.c_double)]),
    "b200m_design_ebu": (C.c_int, [C.c_float, _v]),
    "b200m_design_tpk": (C.c_int, [C.c_float, _v, _v, _v]),
    "b200m_design_cor": (C.c_int, [C.c_int, C.c_float, C.c_float, _v]),
    "b200m_design_spec": (C.c_int, [C.c_double, _v]),
    # EBU
    "b200m_ebu_create": (C.c_int, [C.POINTER(_v), C.c_int, C.c_uint32, C.c_uint32, C.c_float]),
    "b200m_ebu_create_weighted": (C.c_int, [C.POINTER(_v), C.c_int, C.c_uint32, C.c_uint32, _v, C.c_float]),
    "b200m_bs1770_weights": (C.c_int, [C.c_uint32, _v, _v, _v]),
    "b200m_ebu_destroy": (C.c_int, [_v]),
    "b200m_ebu_reset": (C.c_int, [_v, C.c_int32, _v]),
    "b200m_ebu_integr_start": (C.c_int, [_v, C.c_int32, _v]),
    "b200m_ebu_integr_pause": (C.c_int, [_v, C.c_int32, _v]),
    "b200m_ebu_integr_reset": (C.c_int, [_v, C.c_int32, _v]),
    "b200m_ebu_process_device": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32, _v]),
    "b200m_ebu_process_host": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32]),
    "b200m_ebu_process_ragged_device": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32, _v, _v]),
    "b200m_ebu_process_ragged_host": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32, _v]),
    "b200m_ebu_results": (C.c_int, [_v, _v, _v]),
    "b200m_ebu_histogram": (C.c_int, [_v, C.c_uint32, _v, _v, _v]),
    "b200m_ebu_log_enable": (C.c_int, [_v, C.c_uint32, _v]),
    "b200m_ebu_log_drain": (C.c_int, [_v, _v, _v, _v, _v]),
    "b200m_ebu_log_capacity": (C.c_uint32, [_v]),
    "b200m_ebu_coeffs": (C.c_int, [_v, _v]),
    "b200m_ebu_state": (C.c_int, [_v, C.c_uint32, _v, _v, _v, _v, _v]),
    "b200m_ebu_mix_reduce": (C.c_int, [_v, _v, _v]),
    "b200m_ebu_mix_finish": (C.c_int, [_v, _v, _v, _v]),
    "b200m_ebu_group_reduce": (C.c_int, [_v, _v, C.c_uint32, _v, _v]),
    "b200m_ebu_group_finish": (C.c_int, [_v, _v, C.c_uint32, _v, _v]),
    # True peak + K-meter
    "b200m_tpk_create": (C.c_int, [C.POINTER(_v), C.c_int, C.c_uint32, C.c_float, C.c_uint32]),
    "b200m_tpk_destroy": (C.c_int, [_v]),
    "b200m_tpk_process_device": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32, C.c_uint32, _v]),
    "b200m_tpk_process_host": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32, C.c_uint32]),
    "b200m_tpk_read_device": (C.c_int, [_v, _v]),
    "b200m_tpk_process_ragged_device": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32, _v, _v]),
    "b200m_tpk_process_ragged_host": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32, _v]),
    "b200m_selftest_log10f": (C.c_int, [C.c_int, C.c_uint32, C.c_uint32, _v, _v]),
    "b200m_lv2_gon_layout": (C.c_int, [_v, C.c_int]),
    "b200m_ebu_clear": (C.c_int, [_v, C.c_int32, _v]),
    "b200m_tpk_clear": (C.c_int, [_v, C.c_int32, _v]),
    "b200m_spec_set_precision": (C.c_int, [_v, C.c_int]),
    "b200m_cor_set_precision": (C.c_int, [_v, C.c_int]),
    "b200m_pw_debug_capture": (C.c_int, [_v, C.c_int]),
    "b200m_pw_attach_cor": (C.c_int, [_v, _v]),
    "b200m_tpk_set_precision": (C.c_int, [_v, C.c_int]),
    "b200m_tpk_precision": (C.c_int, [_v]),
    "b200m_tpk_results": (C.c_int, [_v, _v, _v]),
    "b200m_tpk_reset": (C.c_int, [_v, C.c_int32, _v]),
    "b200m_tpk_reset_kmeter": (C.c_int, [_v, _v]),
    "b200m_tpk_coeffs": (C.c_int, [_v, _v, _v, _v]),
    "b200m_tpk_state": (C.c_int, [_v, _v, _v, _v, _v, _v, _v, _v]),
    "b200m_tpk_debug_capture": (C.c_int, [_v, C.c_int]),
    "b200m_tpk_debug_timeline": (C.c_int, [_v, _v, C.c_int]),
    "b200m_tpk_debug_upsampled": (C.c_int, [_v, C.c_uint32, _v, C.c_uint32, _v]),
    "b200m_tpk_hist_enable": (C.c_int, [_v, C.c_int, C.c_float, C.c_float, _v]),
    "b200m_tpk_hist_read": (C.c_int, [_v, _v, _v, _v, _v, _v]),
    # EBUr128 plugin cycle
    "b200m_r128_create": (C.c_int, [C.POINTER(_v), C.c_int, C.c_uint32, C.c_float, C.c_int]),
    "b200m_r128_create_nch": (C.c_int, [C.POINTER(_v), C.c_int, C.c_uint32, C.c_uint32, C.c_float, C.c_int]),
    "b200m_r128_create_weighted": (C.c_int, [C.POINTER(_v), C.c_int, C.c_uint32, C.c_uint32, _v, C.c_float, C.c_int]),
    "b200m_r128_destroy": (C.c_int, [_v]),
    "b200m_r128_control": (C.c_int, [_v, C.c_int32, C.c_int, _v]),
    "b200m_r128_run_device": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32, _v]),
    "b200m_r128_run_host": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32]),
    "b200m_r128_run_ragged_device": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32, _v, _v]),
    "b200m_r128_run_ragged_host": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32, _v]),
    "b200m_r128_results": (C.c_int, [_v, _v, _v, _v]),
    "b200m_r128_set_dbtp": (C.c_int, [_v, C.c_int]),
    "b200m_r128_set_dbtp_inst": (C.c_int, [_v, C.c_int32, C.c_int]),
    "b200m_r128_set_precision": (C.c_int, [_v, C.c_int]),
    "b200m_r128_histogram": (C.c_int, [_v, C.c_uint32, _v, _v, _v]),
    "b200m_r128_snapshot_size": (C.c_size_t, [_v]),
    "b200m_r128_snapshot": (C.c_int, [_v, _v, C.c_size_t, _v]),
    "b200m_r128_restore": (C.c_int, [_v, _v, C.c_size_t, _v]),
    "b200m_ebu_snapshot_size": (C.c_size_t, [_v]),
    "b200m_ebu_snapshot": (C.c_int, [_v, _v, C.c_size_t, _v]),
    "b200m_ebu_restore": (C.c_int, [_v, _v, C.c_size_t, _v]),
    "b200m_tpk_snapshot_size": (C.c_size_t, [_v]),
    "b200m_tpk_snapshot": (C.c_int, [_v, _v, C.c_size_t, _v]),
    "b200m_tpk_restore": (C.c_int, [_v, _v, C.c_size_t, _v]),
    "b200m_r128_log_enable": (C.c_int, [_v, C.c_uint32, _v]),
    "b200m_r128_log_drain": (C.c_int, [_v, _v, _v, _v, _v]),
    "b200m_r128_ebu": (_v, [_v]),
    "b200m_r128_tpk": (_v, [_v]),
    # Stcorr
    "b200m_dr14_create": (C.c_int, [C.POINTER(_v), C.c_int, C.c_uint32, C.c_uint32, C.c_double, C.c_int]),
    "b200m_dr14_destroy": (C.c_int, [_v]),
    "b200m_dr14_run_device": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32, _v]),
    "b200m_dr14_run_host": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32]),
    "b200m_dr14_run_ragged_device": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32, _v, _v]),
    "b200m_dr14_run_ragged_host": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32, _v]),
    "b200m_dr14_reset": (C.c_int, [_v, _v]),
    "b200m_dr14_control": (C.c_int, [_v, _v, C.c_uint32, C.c_int, _v]),
    "b200m_dr14_results": (C.c_int, [_v, _v, _v]),
    "b200m_dr14_histogram": (C.c_int, [_v, C.c_uint32, C.c_uint32, _v, _v]),
    "b200m_dr14_log_enable": (C.c_int, [_v, C.c_uint32, _v]),
    "b200m_dr14_log_drain": (C.c_int, [_v, _v, _v, _v, _v]),
    "b200m_dr14_log_capacity": (C.c_uint32, [_v]),
    "b200m_dr14_group_reduce": (C.c_int, [_v, _v, C.c_uint32, _v, _v, _v]),
    "b200m_dr14_group_finish": (C.c_int, [_v, _v, _v, C.c_uint32, C.c_uint32, _v, _v]),
    "b200m_cor_create": (C.c_int, [C.POINTER(_v), C.c_int, C.c_uint32, C.c_int, C.c_float, C.c_float]),
    "b200m_cor_destroy": (C.c_int, [_v]),
    "b200m_cor_process_device": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32, _v]),
    "b200m_cor_process_host": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32]),
    "b200m_cor_process_ctl_device": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32, _v, _v]),
    "b200m_cor_process_ctl_host": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32, _v]),
    "b200m_cor_process_ragged_device": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32, _v, _v]),
    "b200m_cor_process_ragged_host": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32, _v]),
    "b200m_cor_results": (C.c_int, [_v, _v, _v]),
    "b200m_cor_state": (C.c_int, [_v, _v, _v]),
    "b200m_cor_coeffs": (C.c_int, [_v, _v]),
    "b200m_cor_clear": (C.c_int, [_v, C.c_int32, _v]),
    "b200m_cor_hist_enable": (C.c_int, [_v, C.c_int, C.c_float, _v]),
    "b200m_cor_hist_read": (C.c_int, [_v, _v, _v, _v]),
    # needle-meter ballistics
    "b200m_ppm_create": (C.c_int, [C.POINTER(_v), C.c_int, C.c_uint32, C.c_float, C.c_int]),
    "b200m_ppm_destroy": (C.c_int, [_v]),
    "b200m_ppm_set_gain": (C.c_int, [_v, C.c_float, C.c_float]),
    "b200m_ppm_set_gain_inst": (C.c_int, [_v, C.c_int32, C.c_float, C.c_float]),
    "b200m_ppm_clear": (C.c_int, [_v, C.c_int32, _v]),
    "b200m_ppm_process_device": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32, _v]),
    "b200m_ppm_process_host": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32]),
    "b200m_ppm_process_ragged_device": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32, _v, _v]),
    "b200m_ppm_process_ragged_host": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32, _v]),
    "b200m_ppm_read_device": (C.c_int, [_v, _v]),
    "b200m_ppm_results": (C.c_int, [_v, _v, _v]),
    "b200m_ppm_state": (C.c_int, [_v, _v, _v]),
    "b200m_ppm_hist_enable": (C.c_int, [_v, C.c_int, C.c_float, _v]),
    "b200m_ppm_hist_read": (C.c_int, [_v, _v, _v, _v]),
    "b200m_ppm_hist_edges": (C.c_int, [_v]),
    "b200m_design_ppm": (C.c_int, [C.c_int, C.c_float, _v]),
    # bit-meter, signal distribution histogram
    "b200m_bim_create": (C.c_int, [C.POINTER(_v), C.c_int, C.c_uint32, C.c_double]),
    "b200m_bim_destroy": (C.c_int, [_v]),
    "b200m_bim_control": (C.c_int, [_v, C.c_int, _v]),
    "b200m_bim_control_inst": (C.c_int, [_v, C.c_int32, C.c_int, _v]),
    "b200m_bim_run_device": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32, _v]),
    "b200m_bim_run_host": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32]),
    "b200m_bim_run_ragged_device": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32, _v, _v]),
    "b200m_bim_run_ragged_host": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32, _v]),
    "b200m_bim_results": (C.c_int, [_v, C.c_uint32, _v, _v, _v, _v, _v]),
    "b200m_bim_window_closed": (C.c_int, [_v]),
    "b200m_bim_published": (C.c_int, [_v, C.c_uint32, _v, _v, _v, _v, _v]),
    "b200m_bim_results_all": (C.c_int, [_v, _v, _v, _v, _v, _v, _v, _v, _v, _v, _v]),
    "b200m_sdh_create": (C.c_int, [C.POINTER(_v), C.c_int, C.c_uint32, C.c_double]),
    "b200m_sdh_destroy": (C.c_int, [_v]),
    "b200m_sdh_control": (C.c_int, [_v, C.c_int, _v]),
    "b200m_sdh_control_inst": (C.c_int, [_v, C.c_int32, C.c_int, _v]),
    "b200m_sdh_run_device": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32, _v]),
    "b200m_sdh_run_host": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32]),
    "b200m_sdh_run_ragged_device": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32, _v, _v]),
    "b200m_sdh_run_ragged_host": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32, _v]),
    "b200m_sdh_results": (C.c_int, [_v, C.c_uint32, _v, _v, _v, _v, _v]),
    "b200m_sdh_results_all": (C.c_int, [_v, _v, _v, _v, _v, _v]),
    # spectr30
    "b200m_spec_create": (C.c_int, [C.POINTER(_v), C.c_int, C.c_uint32, C.c_uint32, C.c_double]),
    "b200m_spec_destroy": (C.c_int, [_v]),
    "b200m_spec_process_device": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32, C.c_float, C.c_float, _v]),
    "b200m_spec_process_host": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32, C.c_float, C.c_float]),
    "b200m_spec_process_ctl_device": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32, _v, _v]),
    "b200m_spec_process_ctl_host": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32, _v]),
    "b200m_spec_process_ragged_device": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32, _v, _v, _v]),
    "b200m_spec_process_ragged_host": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32, _v, _v]),
    "b200m_spec_clear": (C.c_int, [_v, C.c_int32, _v]),
    "b200m_spec_results": (C.c_int, [_v, _v, _v]),
    "b200m_spec_state": (C.c_int, [_v, C.c_uint32, _v, _v, _v, _v]),
    "b200m_spec_coeffs": (C.c_int, [_v, _v]),
    "b200m_spec_ltas_enable": (C.c_int, [_v, C.c_int, _v]),
    "b200m_spec_ltas_read": (C.c_int, [_v, _v, _v, _v]),
    # phasewheel
    "b200m_pw_create": (C.c_int, [C.POINTER(_v), C.c_int, C.c_uint32, C.c_uint32, C.c_double]),
    "b200m_pw_set_mode": (C.c_int, [_v, C.c_int]),
    "b200m_pw_destroy": (C.c_int, [_v]),
    "b200m_pw_process_device": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32, C.c_float, C.POINTER(C.c_int), _v]),
    "b200m_pw_process_host": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32, C.c_float, C.POINTER(C.c_int)]),
    "b200m_pw_process_ragged_device": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32, _v, C.c_float, C.POINTER(C.c_int), _v]),
    "b200m_pw_process_ragged_host": (C.c_int, [_v, _v, C.c_size_t, C.c_uint32, _v, C.c_float, C.POINTER(C.c_int)]),
    "b200m_pw_results": (C.c_int, [_v, _v, _v, _v, _v]),
    "b200m_pw_raw": (C.c_int, [_v, C.c_uint32, _v, _v, _v, _v, _v]),
    "b200m_pw_device_results": (C.c_int, [_v, C.POINTER(_v), C.POINTER(_v), C.POINTER(_v)]),
    "b200m_pw_xspec_enable": (C.c_int, [_v, C.c_int, _v]),
    "b200m_pw_xspec_read": (C.c_int, [_v, _v, _v, _v]),
    # PCM input
    "b200m_pcm_planar_device": (C.c_int, [C.c_int, _v, C.c_int, C.c_uint32, C.c_uint32, C.c_uint32, C.c_size_t, _v, C.c_size_t, _v]),
}
EXPORTS = tuple(_PROTOS)


def load_lib(path):
    """Load a build of libb200meters.so, this tree's or another (to compare two builds), with the prototypes of _PROTOS."""
    L = C.CDLL(os.path.abspath(path))
    for name, (res, args) in _PROTOS.items():
        try:
            fn = getattr(L, name)
        except AttributeError:      # an export this build lacks: missing_exports() reports it, calling it raises AttributeError
            continue
        fn.restype, fn.argtypes = res, args
    return L


def lib():
    """Load this tree's libb200meters.so (fails loudly if it has not been built: there is no fallback)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise B200MError("%s is missing: run `python meters.lv2_b200/build.py` "
                             "(or __graft_entry__.build()); there is no CPU fallback" % LIB_PATH)
        _lib = load_lib(LIB_PATH)
    return _lib


def missing_exports():
    """Names declared in include/b200meters.h that the built library does not export."""
    L = lib()
    return [n for n in _PROTOS if not hasattr(L, n)]


def _ck(rc):
    if rc != 0:
        raise B200MError("b200meters error %d: %s" % (rc, lib().b200m_last_error().decode()))


def _np_ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def _dev_ptr(x):
    """torch CUDA tensor | int device pointer -> (pointer, row stride in floats, rows, cols)."""
    if isinstance(x, int):
        raise TypeError("pass (ptr, stride, nfram) explicitly via process_ptr()")
    assert x.is_cuda and x.dim() == 2 and x.stride(1) == 1, "need a [channels, nfram] float32 CUDA tensor"
    stride = x.stride(0) if x.shape[0] > 1 else max(x.stride(0), x.shape[1])   # 1-row tensors may report stride 0/1
    return C.c_void_p(x.data_ptr()), stride, x.shape[0], x.shape[1]


def _stream_ptr(stream):
    if stream is None:
        try:
            import torch
            if torch.cuda.is_available():
                return C.c_void_p(torch.cuda.current_stream().cuda_stream)
        except ImportError:
            pass
        return C.c_void_p(0)
    if isinstance(stream, int):
        return C.c_void_p(stream)
    return C.c_void_p(stream.cuda_stream)


def _host_planar(x):
    """numpy [channels, nfram] float32 (row-contiguous) or a pinned torch CPU tensor."""
    if isinstance(x, np.ndarray):
        assert x.dtype == np.float32 and x.ndim == 2 and x.strides[1] == 4
        stride = x.strides[0] // 4 if x.shape[0] > 1 else max(x.strides[0] // 4, x.shape[1])
        return _np_ptr(x), stride, x.shape[0], x.shape[1]
    assert (not x.is_cuda) and x.dim() == 2 and x.stride(1) == 1
    return C.c_void_p(x.data_ptr()), x.stride(0), x.shape[0], x.shape[1]


def design_ebu(fsamp):
    o = np.empty(7, np.float32)
    _ck(lib().b200m_design_ebu(fsamp, _np_ptr(o)))
    return o


def design_tpk(fsamp):
    w = np.empty(4, np.float32); t = np.empty(120, np.float32); k = np.empty(2, np.float32)
    _ck(lib().b200m_design_tpk(fsamp, _np_ptr(w), _np_ptr(t), _np_ptr(k)))
    return w, t, k


def design_cor(fsamp, flp=2e3, tcf=0.3):
    w = np.empty(2, np.float32)
    _ck(lib().b200m_design_cor(int(fsamp), flp, tcf, _np_ptr(w)))
    return w


def design_spec(rate):
    W = np.empty((30, 6, 6), np.float64)
    _ck(lib().b200m_design_spec(rate, _np_ptr(W)))
    return W


def bs1770_weights(azimuth, elevation):
    """ITU-R BS.1770-4 channel weights of a layout from its loudspeaker positions in degrees (b200m_bs1770_weights): 1.41 where
    |elevation| < 30 and 60 <= |azimuth| <= 120, else 1.0.  Needs no GPU."""
    az = np.ascontiguousarray(azimuth, np.float32).ravel(); el = np.ascontiguousarray(elevation, np.float32).ravel()
    assert az.shape == el.shape, "one elevation per azimuth"
    g = np.empty(az.size, np.float32)
    _ck(lib().b200m_bs1770_weights(az.size, _np_ptr(az), _np_ptr(el), _np_ptr(g)))
    return g


def _gains(gains, nchan):
    """caller weights as a float32 array of nchan entries (the C side validates their values)"""
    g = np.ascontiguousarray(gains, np.float32).ravel()
    if g.size != nchan:
        raise B200MError("%d gains for %d channels" % (g.size, nchan))
    return g


def _lengths(lengths, n_inst):
    """per-instance frame counts as a uint32 array of n_inst entries (the C side checks them against nfram)"""
    a = np.asarray(lengths).ravel()
    if a.size != n_inst:
        raise B200MError("%d lengths for %d instances" % (a.size, n_inst))
    if a.size and (a.min() < 0 or a.max() > 0xffffffff):
        raise B200MError("lengths must be frame counts >= 0")
    return np.ascontiguousarray(a, np.uint32)


def _groups(groups, n):
    """album ids (>= 0, or -1 for no album) of n instances or clips as an int64 array (the C side checks them against n_groups)"""
    a = np.asarray(groups).ravel()
    if a.size != n:
        raise B200MError("%d album ids for %d instances" % (a.size, n))
    if a.size and (not np.issubdtype(a.dtype, np.integer) or a.min() < -1 or a.max() >= NO_GROUP):
        raise B200MError("album ids must be integers >= 0, or -1 for no album")
    return a.astype(np.int64)


def _group_rows(d, what, words=MIX_WORDS):
    """(pointer, G) of an int32 CUDA tensor [G, words]"""
    import torch
    if not (d.is_cuda and d.dtype == torch.int32 and d.dim() == 2 and d.shape[1] == words and d.is_contiguous()):
        raise B200MError("%s must be a contiguous int32 CUDA tensor [G, %d]" % (what, words))
    return C.c_void_p(d.data_ptr()), d.shape[0]


def host_alloc(rows, cols):
    """[rows, cols] float32 numpy array in pinned host memory from b200m_host_alloc (placed on the GPU-local NUMA node);
    freed with b200m_host_free when the array is garbage-collected."""
    import weakref
    p = _v()
    nbytes = int(rows) * int(cols) * 4
    _ck(lib().b200m_host_alloc(C.byref(p), nbytes))
    buf = (C.c_float * (int(rows) * int(cols))).from_address(p.value)
    a = np.frombuffer(buf, dtype=np.float32).reshape(int(rows), int(cols))
    weakref.finalize(buf, lib().b200m_host_free, _v(p.value))
    return a


def peak_probe(kind, device=0):
    """kind 0: fp32 unfused mul+add, kind 1: fp64; returns 1e9 lane-ops/s measured on the device."""
    v = C.c_double(0)
    _ck(lib().b200m_peak_probe(device, kind, C.byref(v)))
    return v.value


def launch_count():
    return int(lib().b200m_launch_count())


class _Bank:
    _pfx = None         # the bank's C prefix: its entry points are b200m_<pfx>_*
    _owns = True        # close() destroys the handle (False: a view of a bank another object owns)

    def __init__(self):
        self.h = _v()

    def _fn(self, name):
        return getattr(lib(), "b200m_%s_%s" % (self._pfx, name))

    def close(self):
        if getattr(self, "h", None) and self.h.value:
            if self._owns:
                self._fn("destroy")(self.h)
            self.h = _v()

    def _block(self, verb, x, rows, *args, stream=None):
        """one block over x of `rows` rows: b200m_<pfx>_<verb>_host(h, x, stride, nfram, *args) for a numpy array or CPU tensor,
        b200m_<pfx>_<verb>_device(h, x, stride, nfram, *args, stream) for a CUDA tensor; numpy arrays in args go by pointer (args
        keeps them alive until the call returns)"""
        host = isinstance(x, np.ndarray) or not x.is_cuda
        p, s, r, n = _host_planar(x) if host else _dev_ptr(x)
        assert r == rows
        cargs = [_np_ptr(a) if isinstance(a, np.ndarray) else a for a in args]
        if host:
            _ck(self._fn(verb + "_host")(self.h, p, s, n, *cargs))
        else:
            _ck(self._fn(verb + "_device")(self.h, p, s, n, *cargs, _stream_ptr(stream)))

    def _drain(self, drain, cap, dtype, stream):
        """drain(h, points, count, lost, stream), a b200m_*_log_drain, of a log of `cap` points per instance: (points [n_inst, cap]
        dtype, oldest first, NaN past count; count uint32 [n_inst]; lost uint64 [n_inst], older points overwritten before they
        were drained)"""
        pts = np.empty((self.n_inst, max(int(cap), 1)), dtype)
        cnt = np.empty(self.n_inst, np.uint32); lost = np.empty(self.n_inst, np.uint64)
        _ck(drain(self.h, _np_ptr(pts), _np_ptr(cnt), _np_ptr(lost), _stream_ptr(stream)))
        return pts, cnt, lost

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Ebu_r128_proc(_Bank):
    """N x LV2M::Ebu_r128_proc (ebumeter/ebu_r128_proc.h:66-125)."""
    _pfx = "ebu"

    def __init__(self, n_inst, nchan=2, fsamp=48000.0, device=0, gains=None):
        """gains: None for the reference's weights (nchan 1..5), or nchan per-channel weights (nchan 1..32, b200m_ebu_create_weighted)"""
        super().__init__()
        self.n_inst, self.nchan = n_inst, nchan
        if gains is None:
            _ck(lib().b200m_ebu_create(C.byref(self.h), device, n_inst, nchan, fsamp))
        else:
            self.gains = _gains(gains, nchan)
            _ck(lib().b200m_ebu_create_weighted(C.byref(self.h), device, n_inst, nchan, _np_ptr(self.gains), fsamp))

    def reset(self, inst=-1, stream=None):
        """Ebu_r128_proc::reset of one instance (its 50 ms fragment clock restarts with the next block), or of all with inst=-1"""
        _ck(lib().b200m_ebu_reset(self.h, inst, _stream_ptr(stream)))

    def clear(self, inst, stream=None):
        """reset() of one instance without restarting its fragment clock"""
        _ck(lib().b200m_ebu_clear(self.h, inst, _stream_ptr(stream)))

    def integr_start(self, inst=-1, stream=None):
        _ck(lib().b200m_ebu_integr_start(self.h, inst, _stream_ptr(stream)))

    def integr_pause(self, inst=-1, stream=None):
        _ck(lib().b200m_ebu_integr_pause(self.h, inst, _stream_ptr(stream)))

    def integr_reset(self, inst=-1, stream=None):
        _ck(lib().b200m_ebu_integr_reset(self.h, inst, _stream_ptr(stream)))

    def process(self, x, stream=None, lengths=None):
        """x: [n_inst*nchan, nfram] float32 CUDA tensor (device path) or numpy/pinned CPU (host path).
        lengths: None, or n_inst frame counts <= nfram: instance i processes only the first lengths[i] frames of its rows (0: it is
        not called at all), as a private Ebu_r128_proc fed just those frames (b200m_ebu_process_ragged_*)."""
        if lengths is None:
            self._block("process", x, self.n_inst * self.nchan, stream=stream)
        else:
            self._block("process_ragged", x, self.n_inst * self.nchan, _lengths(lengths, self.n_inst), stream=stream)

    def process_ptr(self, ptr, stride, nfram, stream=None):
        _ck(lib().b200m_ebu_process_device(self.h, C.c_void_p(ptr), stride, nfram, _stream_ptr(stream)))

    def results(self, stream=None):
        out = np.empty(self.n_inst, EBU_RESULT_DTYPE)
        _ck(lib().b200m_ebu_results(self.h, _np_ptr(out), _stream_ptr(stream)))
        return out

    def log_enable(self, capacity, stream=None):
        """keep the last `capacity` loudness points of every instance on the device, one per completed 50 ms fragment
        (b200m_ebu_log_enable); 0 turns the log off, (re)enabling empties it"""
        _ck(lib().b200m_ebu_log_enable(self.h, int(capacity), _stream_ptr(stream)))

    def log_drain(self, stream=None):
        """the points logged since the last drain (b200m_ebu_log_drain): (points [n_inst, capacity] EBU_POINT_DTYPE, oldest first,
        NaN past count; count uint32 [n_inst]; lost uint64 [n_inst], older points overwritten before they were drained)"""
        # the bank's capacity, whoever enabled the log
        return self._drain(lib().b200m_ebu_log_drain, lib().b200m_ebu_log_capacity(self.h), EBU_POINT_DTYPE, stream)

    def histogram(self, inst, stream=None):
        hm = np.empty(HIST_LEN, np.int32); hs = np.empty(HIST_LEN, np.int32)
        _ck(lib().b200m_ebu_histogram(self.h, inst, _np_ptr(hm), _np_ptr(hs), _stream_ptr(stream)))
        return hm, hs

    def coeffs(self):
        o = np.empty(7, np.float32)
        _ck(lib().b200m_ebu_coeffs(self.h, _np_ptr(o)))
        return o

    def state(self, inst, stream=None):
        z = np.empty((self.nchan, 4), np.float32); pw = np.empty(64, np.float32)
        fr = np.empty(1, np.float32); c = np.empty(4, np.int32)
        _ck(lib().b200m_ebu_state(self.h, inst, _np_ptr(z), _np_ptr(pw), _np_ptr(fr), _np_ptr(c), _stream_ptr(stream)))
        return z, pw, fr[0], c

    def mix_reduce(self, d_out, stream=None):
        """d_out: int32 CUDA tensor of MIX_WORDS elements."""
        _ck(lib().b200m_ebu_mix_reduce(self.h, C.c_void_p(d_out.data_ptr()), _stream_ptr(stream)))

    def mix_finish(self, d_mix, stream=None):
        out = np.empty(5, np.float32)
        _ck(lib().b200m_ebu_mix_finish(self.h, C.c_void_p(d_mix.data_ptr()), _np_ptr(out), _stream_ptr(stream)))
        return out

    def group_reduce(self, groups, d_out, stream=None):
        """album histogram sums (b200m_ebu_group_reduce): groups holds n_inst album ids, 0 .. G - 1 or -1 (no album); d_out, an
        int32 CUDA tensor [G, MIX_WORDS], receives each album's mix_reduce vector.  Ordered like the getters: after a host-path
        call it runs on the bank's own stream, which group_finish synchronises."""
        p, n_groups = _group_rows(d_out, "d_out")
        g = np.ascontiguousarray(_groups(groups, self.n_inst).astype(np.uint32))     # -1 wraps to B200M_NO_GROUP
        _ck(lib().b200m_ebu_group_reduce(self.h, _np_ptr(g), n_groups, p, _stream_ptr(stream)))

    def group_finish(self, d_groups, stream=None):
        """mix_finish of every row of d_groups (int32 CUDA tensor [G, MIX_WORDS], b200m_ebu_group_finish): float32 [G, 5] of
        integrated, integ_thr, range_min, range_max, range_thr"""
        p, n_groups = _group_rows(d_groups, "d_groups")
        out = np.empty((n_groups, 5), np.float32)
        _ck(lib().b200m_ebu_group_finish(self.h, p, n_groups, _np_ptr(out), _stream_ptr(stream)))
        return out


TPK_TRUEPEAK, TPK_KMETER = 1, 2
TP_MODE_PROCESS, TP_MODE_MAX = 0, 1
PREC_EXACT, PREC_FMA = 0, 1


class TruePeakKmeter(_Bank):
    """N x (LV2M::TruePeakdsp + LV2M::Kmeterdsp), one mono meter of each per channel
    (jmeters/truepeakdsp.h:28-61, jmeters/kmeterdsp.h:27-62; combined as in src/dr14.c:391-394)."""
    _pfx = "tpk"

    def __init__(self, n_chan, fsamp=48000.0, flags=TPK_TRUEPEAK | TPK_KMETER, device=0):
        super().__init__()
        self.n_chan, self.flags = n_chan, flags
        _ck(lib().b200m_tpk_create(C.byref(self.h), device, n_chan, fsamp, flags))

    def process(self, x, tp_mode=TP_MODE_PROCESS, stream=None, lengths=None):
        """lengths: None, or n_chan frame counts <= nfram (tp_mode process() only): channel i runs over the first lengths[i] frames of
        its row only (0: it is not called, and the next read() leaves it alone), b200m_tpk_process_ragged_*"""
        if lengths is not None and tp_mode != TP_MODE_PROCESS:
            raise B200MError("ragged blocks are process() blocks; ragged process_max runs in EBUr128.run(lengths=)")
        if lengths is None:
            self._block("process", x, self.n_chan, tp_mode, stream=stream)
        else:
            self._block("process_ragged", x, self.n_chan, _lengths(lengths, self.n_chan), stream=stream)

    def process_ptr(self, ptr, stride, nfram, tp_mode=TP_MODE_PROCESS, stream=None):
        _ck(lib().b200m_tpk_process_device(self.h, C.c_void_p(ptr), stride, nfram, tp_mode, _stream_ptr(stream)))

    def process_max(self, x, stream=None):
        self.process(x, TP_MODE_MAX, stream)

    def set_precision(self, mode):
        """PREC_EXACT (bit-identical floats, default) or PREC_FMA (fused FIR, readings within +-1e-4 dB)"""
        _ck(lib().b200m_tpk_set_precision(self.h, int(mode)))

    def read_device(self, stream=None):
        _ck(lib().b200m_tpk_read_device(self.h, _stream_ptr(stream)))

    def results(self, stream=None):
        out = np.empty(self.n_chan, TPK_RESULT_DTYPE)
        _ck(lib().b200m_tpk_results(self.h, _np_ptr(out), _stream_ptr(stream)))
        return out

    def read(self, stream=None):
        """read() of every meter + fetch: the per-run() sequence of dr14_run (src/dr14.c:425-430)."""
        self.read_device(stream)
        return self.results(stream)

    def reset(self, chan=-1, stream=None):
        _ck(lib().b200m_tpk_reset(self.h, chan, _stream_ptr(stream)))

    def clear(self, chan=-1, stream=None):
        """chan (-1: all) back to a newly constructed meter (b200m_tpk_clear), its histogram rows too while the plane is on"""
        _ck(lib().b200m_tpk_clear(self.h, chan, _stream_ptr(stream)))

    def hist_enable(self, on=True, tp_limit_db=-1.0, km_limit_db=-10.0, stream=None):
        """the histogram plane (b200m_tpk_hist_enable): on, every channel counts each process() frame's true-peak reading (the
        largest of its four |out|) and each group of 4 frames' K-meter reading sqrtf(2 z2) in the 242 bins of PPM_HIST_EDGES, with
        PPM_HIST_STATS_DTYPE's statistics, overs against 10^(tp_limit_db / 20) and 10^(km_limit_db / 20); (re)enabling zeroes every
        row and sets the limits; off, the bank stops counting and runs its plain kernels.  process_max raises while it is on."""
        _ck(lib().b200m_tpk_hist_enable(self.h, int(bool(on)), float(tp_limit_db), float(km_limit_db), _stream_ptr(stream)))

    def hist(self, stream=None):
        """(tp_counts, tp_stats, km_counts, km_stats) of the histogram plane (b200m_tpk_hist_read): counts int64 [n_chan, 242] and
        stats PPM_HIST_STATS_DTYPE [n_chan] of each meter, None for a meter the bank lacks; raises while the plane is off"""
        rows = []
        for flag in (TPK_TRUEPEAK, TPK_KMETER):
            if self.flags & flag:
                rows.append((np.empty((self.n_chan, PPM_HIST_BINS), np.uint64), np.empty(self.n_chan, PPM_HIST_STATS_DTYPE)))
            else:
                rows.append((None, None))
        ptrs = [_np_ptr(a) if a is not None else None for r in rows for a in r]
        _ck(lib().b200m_tpk_hist_read(self.h, *ptrs, _stream_ptr(stream)))
        (tc, ts), (kc, ks) = rows
        return (None if tc is None else tc.astype(np.int64), ts, None if kc is None else kc.astype(np.int64), ks)

    def coeffs(self):
        w = np.empty(4, np.float32); t = np.empty(120, np.float32); k = np.empty(2, np.float32)
        _ck(lib().b200m_tpk_coeffs(self.h, _np_ptr(w), _np_ptr(t), _np_ptr(k)))
        return w, t, k

    def state(self, stream=None):
        n = self.n_chan
        m, p, z1, z2 = (np.empty(n, np.float32) for _ in range(4))
        res = np.empty(n, np.int32); km = np.empty((n, 8), np.float32)
        _ck(lib().b200m_tpk_state(self.h, _np_ptr(m), _np_ptr(p), _np_ptr(z1), _np_ptr(z2), _np_ptr(res), _np_ptr(km), _stream_ptr(stream)))
        return dict(m=m, p=p, z1=z1, z2=z2, res=res, km=km)

    def debug_capture(self, enable=True):
        _ck(lib().b200m_tpk_debug_capture(self.h, int(enable)))

    def debug_upsampled(self, chan, n_out, stream=None):
        out = np.empty(n_out, np.float32)
        _ck(lib().b200m_tpk_debug_upsampled(self.h, chan, _np_ptr(out), n_out, _stream_ptr(stream)))
        return out


COR_HIST_BINS = 200           # B200M_COR_HIST_BINS
# the correlation histogram's 201 bin edges, -1 .. 1 in steps of 0.01: bin k holds readings r with floorf ((r + 1) * 100) == k
# (fp32), readings past +-1 clamped to bins 0 and 199
COR_HIST_EDGES = (np.arange(COR_HIST_BINS + 1) - 100) / 100.0


class Stcorrdsp(_Bank):
    """N x LV2M::Stcorrdsp (jmeters/stcorrdsp.h:27-55); channels 2i, 2i+1 = L, R of pair i."""
    _pfx = "cor"

    def __init__(self, n_inst, fsamp=48000, flp=2e3, tcf=0.3, device=0):
        super().__init__()
        self.n_inst = n_inst
        _ck(lib().b200m_cor_create(C.byref(self.h), device, n_inst, int(fsamp), flp, tcf))

    def process(self, x, run=None, stream=None, lengths=None):
        """run: None (every pair) or n_inst flags; a pair whose flag is 0 is held, its state and reading left as they are.
        lengths: None, or n_inst frame counts <= nfram: pair i runs over the first lengths[i] frames of its rows only (0: held),
        b200m_cor_process_ragged_*; not together with run"""
        if run is not None and lengths is not None:
            raise B200MError("pass run or lengths, not both")
        mask = None if run is None else np.ascontiguousarray(run, np.uint8)
        assert mask is None or mask.shape == (self.n_inst,)
        if lengths is not None:
            self._block("process_ragged", x, 2 * self.n_inst, _lengths(lengths, self.n_inst), stream=stream)
        elif mask is None:
            self._block("process", x, 2 * self.n_inst, stream=stream)
        else:
            self._block("process_ctl", x, 2 * self.n_inst, mask, stream=stream)

    def set_precision(self, mode):
        """PREC_EXACT: serial, bit-identical; PREC_FMA: time-parallel warp scan, correlation within 1e-5"""
        _ck(lib().b200m_cor_set_precision(self.h, int(mode)))

    def process_ptr(self, ptr, stride, nfram, stream=None):
        _ck(lib().b200m_cor_process_device(self.h, C.c_void_p(ptr), stride, nfram, _stream_ptr(stream)))

    def read(self, stream=None):
        out = np.empty(self.n_inst, np.float32)
        _ck(lib().b200m_cor_results(self.h, _np_ptr(out), _stream_ptr(stream)))
        return out

    def state(self, stream=None):
        s = np.empty((self.n_inst, 5), np.float32)
        _ck(lib().b200m_cor_state(self.h, _np_ptr(s), _stream_ptr(stream)))
        return s

    def coeffs(self):
        w = np.empty(2, np.float32)
        _ck(lib().b200m_cor_coeffs(self.h, _np_ptr(w)))
        return w

    def clear(self, inst=-1, stream=None):
        """pair inst (-1: all) back to a newly constructed Stcorrdsp, its histogram row too while the plane is on; an attached
        phasewheel ring is not touched"""
        _ck(lib().b200m_cor_clear(self.h, inst, _stream_ptr(stream)))

    def hist_enable(self, on=True, gate_db=-70.0, stream=None):
        """the correlation histogram plane (b200m_cor_hist_enable): on, every pair counts each frame's reading r in
        COR_HIST_EDGES's 200 bins and adds it to a float64 sum, if zll + zrr >= 2 * 10^(gate_db / 10) and r is finite; (re)enabling
        zeroes every pair's row and sets the gate (-inf: no gate); off, the bank stops counting and runs its plain kernels"""
        _ck(lib().b200m_cor_hist_enable(self.h, int(bool(on)), float(gate_db), _stream_ptr(stream)))

    def hist(self, stream=None):
        """(counts int64 [n_inst, 200], sums float64 [n_inst]) of the histogram plane (b200m_cor_hist_read); raises while it is off"""
        c = np.empty((self.n_inst, COR_HIST_BINS), np.uint64); s = np.empty(self.n_inst, np.float64)
        _ck(lib().b200m_cor_hist_read(self.h, _np_ptr(c), _np_ptr(s), _stream_ptr(stream)))
        return c.astype(np.int64), s


PPM_VU, PPM_IEC1, PPM_IEC2, PPM_MS = 0, 1, 2, 3


def design_ppm(kind, fsamp):
    w = np.empty(4, np.float32)
    _ck(lib().b200m_design_ppm(kind, fsamp, _np_ptr(w)))
    return w


PPM_HIST_BINS = 242           # B200M_PPM_HIST_BINS
# b200m_ppm_hist_stats
PPM_HIST_STATS_DTYPE = np.dtype([("nonfinite", "<u8"), ("over_groups", "<u8"), ("overs", "<u8"), ("longest_over", "<u8"),
                                 ("run", "<u8"), ("peak", "<f4"), ("pad", "<u4")])
# the dB value of each of the needle histogram's 241 edges: bin 0 lies below -80 dB, bin k (1..240) from edge k - 1 up to edge k,
# bin 241 at +40 dB and above
PPM_HIST_EDGES_DB = -80.0 + 0.5 * np.arange(PPM_HIST_BINS - 1)
_ppm_edges = None


def __getattr__(name):
    # PPM_HIST_EDGES, the library's float32 edges (b200m_ppm_hist_edges), is read from the library on first use, so that importing
    # the package does not need it
    global _ppm_edges
    if name == "PPM_HIST_EDGES":
        if _ppm_edges is None:
            e = np.empty(PPM_HIST_BINS - 1, np.float32)
            _ck(lib().b200m_ppm_hist_edges(_np_ptr(e)))
            e.flags.writeable = False
            _ppm_edges = e
        return _ppm_edges
    raise AttributeError("module %r has no attribute %r" % (__name__, name))


class NeedleMeters(_Bank):
    """N x Vumeterdsp / Iec1ppmdsp / Iec2ppmdsp, or N stereo pairs x (Msppmdsp M, Msppmdsp S) (jmeters/*.cc)."""
    _pfx = "ppm"

    def __init__(self, n_units, kind, fsamp=48000.0, device=0):
        super().__init__()
        self.n_units, self.kind = n_units, kind
        self.rows = 2 * n_units if kind == PPM_MS else n_units
        self.n_meters = self.rows
        _ck(lib().b200m_ppm_create(C.byref(self.h), device, n_units, fsamp, kind))

    def set_gain(self, db_m, db_s, unit=-1):
        """Msppmdsp::set_gain of pair `unit`'s M and S meters (-1: every pair); applied with the next process()"""
        _ck(lib().b200m_ppm_set_gain_inst(self.h, unit, db_m, db_s))

    def clear(self, unit=-1, stream=None):
        """unit (-1: all) back to newly constructed meters (M/S: gains -6 / -6 dB), its histogram rows too while the plane is on"""
        _ck(lib().b200m_ppm_clear(self.h, unit, _stream_ptr(stream)))

    def hist_enable(self, on=True, limit_db=0.0, stream=None):
        """the needle histogram plane (b200m_ppm_hist_enable): on, every meter counts each group of 4 frames' reading v = g * s in
        the 242 bins of PPM_HIST_EDGES and keeps PPM_HIST_STATS_DTYPE's statistics, overs against 10^(limit_db / 20); (re)enabling
        zeroes every row and sets the limit; off, the bank stops counting and runs its plain kernels"""
        _ck(lib().b200m_ppm_hist_enable(self.h, int(bool(on)), float(limit_db), _stream_ptr(stream)))

    def hist(self, stream=None):
        """(counts int64 [n_meters, 242], stats PPM_HIST_STATS_DTYPE [n_meters]) of the histogram plane (b200m_ppm_hist_read);
        raises while it is off"""
        c = np.empty((self.n_meters, PPM_HIST_BINS), np.uint64); st = np.empty(self.n_meters, PPM_HIST_STATS_DTYPE)
        _ck(lib().b200m_ppm_hist_read(self.h, _np_ptr(c), _np_ptr(st), _stream_ptr(stream)))
        return c.astype(np.int64), st

    def process(self, x, stream=None, lengths=None):
        """lengths: None, or n_units frame counts <= nfram: unit u (a meter, or an M/S pair) runs over the first lengths[u] frames
        of its rows only (0: it is not called, and the next read() leaves it alone), b200m_ppm_process_ragged_*"""
        if lengths is None:
            self._block("process", x, self.rows, stream=stream)
        else:
            self._block("process_ragged", x, self.rows, _lengths(lengths, self.n_units), stream=stream)

    def read(self, stream=None):
        _ck(lib().b200m_ppm_read_device(self.h, _stream_ptr(stream)))
        out = np.empty(self.n_meters, np.float32)
        _ck(lib().b200m_ppm_results(self.h, _np_ptr(out), _stream_ptr(stream)))
        return out

    def state(self, stream=None):
        s = np.empty((self.n_meters, 4), np.float32)
        _ck(lib().b200m_ppm_state(self.h, _np_ptr(s), _stream_ptr(stream)))
        return s


CTL_START, CTL_PAUSE, CTL_RESET, CTL_AVERAGE, CTL_WINDOWED, CTL_CLEAR = 1, 2, 3, 4, 5, 6


class _StatBank(_Bank):
    def __init__(self, n_inst, rate=48000.0, device=0):
        super().__init__()
        self.n_inst = n_inst
        _ck(self._fn("create")(C.byref(self.h), device, n_inst, rate))

    def control(self, cmd, stream=None, inst=-1):
        """CTL_* on one instance, or on every instance with inst = -1"""
        _ck(self._fn("control_inst")(self.h, inst, cmd, _stream_ptr(stream)))

    def run(self, x, stream=None, lengths=None):
        """one run of every instance over x [n_inst, nfram] (CUDA tensor: device path; numpy / CPU tensor: host path).
        lengths: None, or n_inst frame counts <= nfram: instance i runs over its first lengths[i] frames only (0: it is not run,
        its window clock stands still), b200m_*_run_ragged_*."""
        if lengths is None:
            self._block("run", x, self.n_inst, stream=stream)
        else:
            self._block("run_ragged", x, self.n_inst, _lengths(lengths, self.n_inst), stream=stream)

    def run_ptr(self, ptr, stride, nfram, stream=None):
        _ck(self._fn("run_device")(self.h, C.c_void_p(ptr), stride, nfram, _stream_ptr(stream)))


class Bitmeter(_StatBank):
    """N x the bit-meter plugin's statistics (src/bitmeter.c:63-105,248-327)."""
    _pfx = "bim"

    def results(self, inst, stream=None):
        h = np.empty(584, np.int32); c = np.empty(5, np.int32); mm = np.empty(2, np.float32); it = C.c_int64(0)
        _ck(lib().b200m_bim_results(self.h, inst, _np_ptr(h), _np_ptr(c), _np_ptr(mm), C.byref(it), _stream_ptr(stream)))
        return h, c, mm, it.value

    def results_all(self, stream=None):
        """every instance in one synchronisation: dict of hist [n, 584], cnt [n, 5], minmax [n, 2], itime [n], closed [n] (the
        last run closed that instance's window) and pub_hist, pub_cnt, pub_minmax, pub_itime (its last published snapshot)"""
        n = self.n_inst
        r = dict(hist=np.empty((n, 584), np.int32), cnt=np.empty((n, 5), np.int32), minmax=np.empty((n, 2), np.float32),
                 itime=np.empty(n, np.int64), closed=np.empty(n, np.int32), pub_hist=np.empty((n, 584), np.int32),
                 pub_cnt=np.empty((n, 5), np.int32), pub_minmax=np.empty((n, 2), np.float32), pub_itime=np.empty(n, np.int64))
        _ck(lib().b200m_bim_results_all(self.h, *(_np_ptr(r[k]) for k in ("hist", "cnt", "minmax", "itime", "closed", "pub_hist", "pub_cnt",
                                                                            "pub_minmax", "pub_itime")), _stream_ptr(stream)))
        return r


class SigDistHist(_StatBank):
    """N x the signal-distribution-histogram plugin's statistics (src/sigdistlv2.c:287-327)."""
    _pfx = "sdh"

    def results(self, inst, stream=None):
        h = np.empty(361, np.int32); mp = np.empty(2, np.int32); av = np.empty(3, np.float64); it = C.c_int64(0)
        _ck(lib().b200m_sdh_results(self.h, inst, _np_ptr(h), _np_ptr(mp), _np_ptr(av), C.byref(it), _stream_ptr(stream)))
        return h, mp, av, it.value

    def results_all(self, stream=None):
        """every instance in one synchronisation: (hist [n, 361], max_peak [n, 2], avg_tmp_var [n, 3] fp64, itime [n])"""
        n = self.n_inst
        h = np.empty((n, 361), np.int32); mp = np.empty((n, 2), np.int32); av = np.empty((n, 3), np.float64); it = np.empty(n, np.int64)
        _ck(lib().b200m_sdh_results_all(self.h, _np_ptr(h), _np_ptr(mp), _np_ptr(av), _np_ptr(it), _stream_ptr(stream)))
        return h, mp, av, it


DR14_RESULT_DTYPE = np.dtype([("v_rms", "<f4", 2), ("v_peak", "<f4", 2), ("m_peak", "<f4", 2), ("m_rms", "<f4", 2), ("dr", "<f4", 2),
                              ("dr_total", "<f4"), ("block_count", "<f4")])
# one point of the DR-14 window log (b200m_dr14_point): one completed 3 s window of an instance and the readings after it
DR14_POINT_DTYPE = np.dtype([("window", "<f4"), ("silent", "<f4"), ("rms", "<f4", 2), ("peak", "<f4", 2), ("m_rms", "<f4", 2),
                             ("peak2", "<f4", 2), ("dr", "<f4", 2), ("dr_total", "<f4"), ("block_count", "<f4")])


DR14_RESET, DR14_CLEAR = 1, 2
DR14_MAX_GROUPS = 16384     # B200M_DR14_MAX_GROUPS: albums per DR14.group_reduce / group_finish call
# one album's DR (b200m_dr14_album): m_rms, dr, dr_total, block_count as in DR14_RESULT_DTYPE, peak2 as in DR14_POINT_DTYPE, m_peak
# the largest member true-peak hold (dB); channel 1 and dr_total NaN in a mono bank
DR14_ALBUM_DTYPE = np.dtype([("m_rms", "<f4", 2), ("peak2", "<f4", 2), ("dr", "<f4", 2), ("dr_total", "<f4"), ("block_count", "<f4"),
                             ("m_peak", "<f4", 2), ("windows", "<f4"), ("members", "<f4")])


def dr14_group_words(n_channels):
    """B200M_DR14_GROUP_WORDS: int32 words of one album row of DR14.group_reduce (histograms, window count, member count)"""
    return n_channels * 8000 + 2


class DR14(_Bank):
    """N x dr14_run (src/dr14.c:354-482): DR-14 mode (dr_mode=True) or TPnRMS (False); results = the plugin's output ports."""
    _pfx = "dr14"

    def __init__(self, n_inst, n_channels=2, rate=48000.0, dr_mode=True, device=0):
        super().__init__()
        self.n_inst, self.nchan = n_inst, n_channels
        _ck(lib().b200m_dr14_create(C.byref(self.h), device, n_inst, n_channels, rate, int(bool(dr_mode))))

    def run(self, x, stream=None, lengths=None):
        """one dr14_run of every instance over x [n_inst*nchan, nfram] (CUDA tensor: device path; numpy / CPU tensor: host path).
        lengths: None, or n_inst frame counts <= nfram: instance i runs over its first lengths[i] frames only (0: the plugin did not
        run: no process, no read, its window clock stands still), b200m_dr14_run_ragged_*."""
        if lengths is None:
            self._block("run", x, self.n_inst * self.nchan, stream=stream)
        else:
            self._block("run_ragged", x, self.n_inst * self.nchan, _lengths(lengths, self.n_inst), stream=stream)

    def run_ptr(self, ptr, stride, nfram, stream=None):
        _ck(lib().b200m_dr14_run_device(self.h, C.c_void_p(ptr), stride, nfram, _stream_ptr(stream)))

    def reset(self, stream=None):
        _ck(lib().b200m_dr14_reset(self.h, _stream_ptr(stream)))

    def control(self, cmd, inst=None, stream=None):
        """DR14_RESET / DR14_CLEAR of the listed instances (a sequence of indices), or of every instance with inst=None"""
        if inst is None:
            _ck(lib().b200m_dr14_control(self.h, None, 0, cmd, _stream_ptr(stream)))
        else:
            sel = np.ascontiguousarray(inst, np.uint32)
            _ck(lib().b200m_dr14_control(self.h, _np_ptr(sel), sel.size, cmd, _stream_ptr(stream)))

    def results(self, stream=None):
        out = np.empty(self.n_inst, DR14_RESULT_DTYPE)
        _ck(lib().b200m_dr14_results(self.h, _np_ptr(out), _stream_ptr(stream)))
        return out

    def histogram(self, inst, chan, stream=None):
        h = np.empty(8000, np.uint32)
        _ck(lib().b200m_dr14_histogram(self.h, inst, chan, _np_ptr(h), _stream_ptr(stream)))
        return h

    def log_enable(self, capacity, stream=None):
        """keep the last `capacity` window points of every instance on the device, one per completed 3 s window, silent ones
        included (b200m_dr14_log_enable, DR mode only); 0 turns the log off, (re)enabling empties it"""
        _ck(lib().b200m_dr14_log_enable(self.h, int(capacity), _stream_ptr(stream)))

    def log_drain(self, stream=None):
        """the points logged since the last drain (b200m_dr14_log_drain): (points [n_inst, capacity] DR14_POINT_DTYPE, oldest first,
        NaN past count; count uint32 [n_inst]; lost uint64 [n_inst], older points overwritten before they were drained)"""
        return self._drain(lib().b200m_dr14_log_drain, lib().b200m_dr14_log_capacity(self.h), DR14_POINT_DTYPE, stream)

    def _peaks(self, d, n_groups, parts):
        """(pointer, n_parts) of a float32 CUDA tensor [G, nchan, 3], or with parts also [P, G, nchan, 3]"""
        import torch
        shape = tuple(d.shape)
        ok = d.is_cuda and d.dtype == torch.float32 and d.is_contiguous() and shape[-3:] == (n_groups, self.nchan, 3)
        if not (ok and (d.dim() == 3 or (parts and d.dim() == 4))):
            raise B200MError("d_peaks must be a contiguous float32 CUDA tensor [%s%d, %d, 3]" % ("P, " if parts else "", n_groups, self.nchan))
        return C.c_void_p(d.data_ptr()), (shape[0] if d.dim() == 4 else 1)

    def group_reduce(self, groups, d_rows, d_peaks, stream=None):
        """album DR state (b200m_dr14_group_reduce, DR mode): groups holds n_inst album ids, 0 .. G - 1 or -1 (no album); d_rows, an
        int32 CUDA tensor [G, dr14_group_words(nchan)], receives each album's summed histograms, window count and member count;
        d_peaks, a float32 CUDA tensor [G, nchan, 3], its top two window peaks and true-peak hold (linear).  Ordered like the getters:
        after a host-path call it runs on the bank's own stream, which group_finish synchronises."""
        p, n_groups = _group_rows(d_rows, "d_rows", dr14_group_words(self.nchan))
        q, _ = self._peaks(d_peaks, n_groups, False)
        g = np.ascontiguousarray(_groups(groups, self.n_inst).astype(np.uint32))     # -1 wraps to B200M_NO_GROUP
        _ck(lib().b200m_dr14_group_reduce(self.h, _np_ptr(g), n_groups, p, q, _stream_ptr(stream)))

    def group_finish(self, d_rows, d_peaks, stream=None):
        """the DR of every album (b200m_dr14_group_finish): d_rows as group_reduce fills it (summed over shards), d_peaks [G, nchan, 3]
        or the [P, G, nchan, 3] parts of P shards (shard.allreduce_dr14_groups); a DR14_ALBUM_DTYPE array of G"""
        p, n_groups = _group_rows(d_rows, "d_rows", dr14_group_words(self.nchan))
        q, n_parts = self._peaks(d_peaks, n_groups, True)
        out = np.empty(n_groups, DR14_ALBUM_DTYPE)
        _ck(lib().b200m_dr14_group_finish(self.h, p, q, n_parts, n_groups, _np_ptr(out), _stream_ptr(stream)))
        return out


# the 30 bands' nominal centre frequencies in Hz, 1000 * 2^((i - 16) / 3) (src/spectrumlv2.c:100-118): 24.8 Hz .. 20.2 kHz
SPEC_BAND_HZ = 1000.0 * 2.0 ** ((np.arange(30) - 16) / 3.0)


class Spectr30(_Bank):
    """N x the spectr30 plugin (src/spectrumlv2.c:73-257): ports 0..59 per instance."""
    _pfx = "spec"

    def __init__(self, n_inst, nchan=2, rate=48000.0, device=0):
        super().__init__()
        self.n_inst, self.nchan = n_inst, nchan
        _ck(lib().b200m_spec_create(C.byref(self.h), device, n_inst, nchan, rate))

    def process(self, x, speed=1.0, reset=-4.0, stream=None, lengths=None):
        """speed / reset: ports 60 / 61, one value for every instance or an array of n_inst (each instance its own).
        lengths: None, or n_inst frame counts <= nfram: instance i runs over the first lengths[i] frames of its rows only (0: it is
        not run and its controls are ignored), b200m_spec_process_ragged_*"""
        rows = self.n_inst * self.nchan
        ln = None if lengths is None else _lengths(lengths, self.n_inst)
        if ln is None and not (np.ndim(speed) or np.ndim(reset)):
            self._block("process", x, rows, speed, reset, stream=stream)
            return
        ctl = np.empty((self.n_inst, 2), np.float32)
        ctl[:, 0] = speed; ctl[:, 1] = reset
        if ln is None:
            self._block("process_ctl", x, rows, ctl, stream=stream)
        else:
            self._block("process_ragged", x, rows, ctl, ln, stream=stream)

    def clear(self, inst=-1, stream=None):
        """instance inst (-1: all) back to a freshly created spectr30"""
        _ck(lib().b200m_spec_clear(self.h, inst, _stream_ptr(stream)))

    def set_precision(self, mode):
        """PREC_EXACT: ports bit-identical to the reference; PREC_FMA: fused multiply-adds, band levels within +-1e-4 dB"""
        _ck(lib().b200m_spec_set_precision(self.h, int(mode)))

    def process_ptr(self, ptr, stride, nfram, speed=1.0, reset=-4.0, stream=None):
        _ck(lib().b200m_spec_process_device(self.h, C.c_void_p(ptr), stride, nfram, speed, reset, _stream_ptr(stream)))

    def read(self, stream=None):
        out = np.empty((self.n_inst, 60), np.float32)
        _ck(lib().b200m_spec_results(self.h, _np_ptr(out), _stream_ptr(stream)))
        return out

    def state(self, inst, stream=None):
        z = np.empty((30, 6, 2), np.float64); v = np.empty(30, np.float32); m = np.empty(30, np.float32)
        _ck(lib().b200m_spec_state(self.h, inst, _np_ptr(z), _np_ptr(v), _np_ptr(m), _stream_ptr(stream)))
        return z, v, m

    def coeffs(self):
        W = np.empty((30, 6, 6), np.float64)
        _ck(lib().b200m_spec_coeffs(self.h, _np_ptr(W)))
        return W

    def ltas_enable(self, on=True, stream=None):
        """the long-term average spectrum plane (b200m_spec_ltas_enable): on, every band of every instance adds up its per-frame
        power v * v and counts the finite frames it added; (re)enabling zeroes every instance's sums and counts"""
        _ck(lib().b200m_spec_ltas_enable(self.h, int(bool(on)), _stream_ptr(stream)))

    def ltas(self, stream=None):
        """(sums float64 [n_inst, 30], counts int64 [n_inst, 30]) of the LTAS plane (b200m_spec_ltas_read): the band's average power
        is sums / counts; raises while the plane is off"""
        s = np.empty((self.n_inst, 30), np.float64); c = np.empty((self.n_inst, 30), np.uint64)
        _ck(lib().b200m_spec_ltas_read(self.h, _np_ptr(s), _np_ptr(c), _stream_ptr(stream)))
        return s, c.astype(np.int64)


# the terms of a cross-spectrum plane row, in order (B200M_PW_XSPEC_LL .. RL_IM): |L_k|^2, |R_k|^2, Re and Im (R_k conj L_k)
PW_XSPEC_TERMS = ("ll", "rr", "rl_re", "rl_im")


class Phasewheel(_Bank):
    """N x (2 x FFTAnalysis + phasewheel process_audio) (gui/fft.c:208-361, gui/phasewheel.c:1307-1342)."""
    _pfx = "pw"

    def __init__(self, n_inst, fft_bins=1024, rate=48000.0, device=0):
        super().__init__()
        self.n_inst, self.bins = n_inst, fft_bins
        _ck(lib().b200m_pw_create(C.byref(self.h), device, n_inst, fft_bins, rate))

    def process(self, x, db_thresh=1e-6, stream=None, lengths=None):
        """one block of every instance over x [2 n_inst, nfram]; returns 1 if an analysis completed.
        lengths: None, or n_inst frame counts <= nfram: instance i runs over the first lengths[i] frames of its rows only, with its own
        ring offset and analysis clock (0: it is not called), b200m_pw_process_ragged_*"""
        fired = C.c_int(0)
        if lengths is None:
            self._block("process", x, 2 * self.n_inst, db_thresh, C.byref(fired), stream=stream)
        else:
            self._block("process_ragged", x, 2 * self.n_inst, _lengths(lengths, self.n_inst), db_thresh, C.byref(fired), stream=stream)
        return fired.value

    def process_ptr(self, ptr, stride, nfram, db_thresh=1e-6, stream=None):
        fired = C.c_int(0)
        _ck(lib().b200m_pw_process_device(self.h, C.c_void_p(ptr), stride, nfram, db_thresh, C.byref(fired), _stream_ptr(stream)))
        return fired.value

    def debug_capture(self, enable=True):
        """keep ft->power / ft->phase of both channels of every analysis (needed by raw())"""
        _ck(lib().b200m_pw_debug_capture(self.h, int(enable)))

    def attach_cor(self, cor):
        """fused feed: process*() also runs `cor` (a Stcorrdsp bank of n_inst pairs) on the same block, reading the input once"""
        _ck(lib().b200m_pw_attach_cor(self.h, cor.h if cor is not None else None))
        self._cor = cor

    def set_mode(self, mode):
        """0: phasewheel process_audio; 1: stereoscope process_audio (read() then returns lr[] as `phase`)"""
        _ck(lib().b200m_pw_set_mode(self.h, int(mode)))

    def read(self, stream=None):
        ph = np.empty((self.n_inst, self.bins), np.float32); lv = np.empty((self.n_inst, self.bins), np.float32)
        pk = np.empty(self.n_inst, np.float32)
        _ck(lib().b200m_pw_results(self.h, _np_ptr(ph), _np_ptr(lv), _np_ptr(pk), _stream_ptr(stream)))
        return ph, lv, pk

    def raw(self, inst, stream=None):
        a = [np.empty(self.bins, np.float32) for _ in range(4)]
        _ck(lib().b200m_pw_raw(self.h, inst, *[_np_ptr(v) for v in a], _stream_ptr(stream)))
        return a

    def xspec_enable(self, on=True, stream=None):
        """the cross-spectrum plane (b200m_pw_xspec_enable): on, every analysis of every instance adds the PW_XSPEC_TERMS of each bin
        to the instance's row, or counts itself skipped when a spectrum is not finite; (re)enabling zeroes every row and count, off
        stops adding and keeps them"""
        _ck(lib().b200m_pw_xspec_enable(self.h, int(bool(on)), _stream_ptr(stream)))

    def xspec(self, stream=None):
        """(sums float64 [n_inst, 4, fft_bins] in PW_XSPEC_TERMS order, analyses int64 [n_inst], skipped int64 [n_inst]) of the
        cross-spectrum plane (b200m_pw_xspec_read); raises before the plane was first enabled"""
        s = np.empty((self.n_inst, 4, self.bins), np.float64); c = np.empty((self.n_inst, 2), np.uint64)
        _ck(lib().b200m_pw_xspec_read(self.h, _np_ptr(s), _np_ptr(c), _stream_ptr(stream)))
        c = c.astype(np.int64)
        return s, c[:, 0].copy(), c[:, 1].copy()


class EBUr128(_Bank):
    """N x the EBUr128 plugin's audio cycle (ebur128_run, src/ebulv2.cc:341-367): EBU R128 + optional dBTP.
    nchan 1..5 channels per instance (rows inst * nchan + c, order L R C Ls Rs, no LFE); the plugin itself is stereo.
    gains: nchan per-channel loudness weights for any layout of 1..32 channels (b200m_r128_create_weighted; bs1770_weights gives
    the BS.1770-4 ones); a zero weight keeps a row (an LFE) out of the loudness but in the dBTP hold."""
    _pfx = "r128"
    START, PAUSE, RESET, CLEAR_TPMAX, CLEAR, NEW = 1, 2, 3, 4, 5, 6

    def __init__(self, n_inst, fsamp=48000.0, dbtp_enable=True, device=0, nchan=2, gains=None):
        super().__init__()
        self.n_inst, self.nchan = n_inst, nchan
        if gains is None:
            _ck(lib().b200m_r128_create_nch(C.byref(self.h), device, n_inst, nchan, fsamp, int(dbtp_enable)))
        else:
            self.gains = _gains(gains, nchan)
            _ck(lib().b200m_r128_create_weighted(C.byref(self.h), device, n_inst, nchan, _np_ptr(self.gains), fsamp, int(dbtp_enable)))
        self.ebu = Ebu_r128_proc.__new__(Ebu_r128_proc)
        self.ebu.h = _v(lib().b200m_r128_ebu(self.h)); self.ebu.n_inst = n_inst; self.ebu.nchan = nchan
        self.ebu._owns = False

    def close(self):
        if getattr(self, "ebu", None) is not None:
            self.ebu.h = _v()
        super().close()

    def control(self, cmd, inst=-1, stream=None):
        _ck(lib().b200m_r128_control(self.h, inst, cmd, _stream_ptr(stream)))

    def run(self, x, stream=None, lengths=None):
        """one cycle of every instance over x [n_inst*nchan, nfram] (CUDA tensor: device path; numpy / CPU tensor: host path).
        lengths: None, or n_inst frame counts <= nfram: instance i runs its cycle over its first lengths[i] frames only (0: the
        plugin did not run this cycle: no process, no read, hold unchanged), b200m_r128_run_ragged_*."""
        if lengths is None:
            self._block("run", x, self.n_inst * self.nchan, stream=stream)
        else:
            self._block("run_ragged", x, self.n_inst * self.nchan, _lengths(lengths, self.n_inst), stream=stream)

    def run_ptr(self, ptr, stride, nfram, stream=None, host=False):
        if host:
            _ck(lib().b200m_r128_run_host(self.h, C.c_void_p(ptr), stride, nfram))
        else:
            _ck(lib().b200m_r128_run_device(self.h, C.c_void_p(ptr), stride, nfram, _stream_ptr(stream)))

    def results(self, stream=None, out=None, tp=None):
        out = np.empty(self.n_inst, EBU_RESULT_DTYPE) if out is None else out
        tp = np.empty(self.n_inst, np.float32) if tp is None else tp
        _ck(lib().b200m_r128_results(self.h, _np_ptr(out), _np_ptr(tp), _stream_ptr(stream)))
        return out, tp

    def snapshot(self, stream=None):
        """the whole bank state as bytes (checkpoint)"""
        n = lib().b200m_r128_snapshot_size(self.h)
        buf = np.empty(n, np.uint8)
        _ck(lib().b200m_r128_snapshot(self.h, _np_ptr(buf), n, _stream_ptr(stream)))
        return buf

    def restore(self, blob, stream=None):
        blob = np.ascontiguousarray(blob, np.uint8)
        _ck(lib().b200m_r128_restore(self.h, _np_ptr(blob), blob.size, _stream_ptr(stream)))

    def set_dbtp(self, enable, inst=-1):
        """self->dbtp_enable (src/ebulv2.cc:316-317) of one instance, or of every instance with inst=-1: takes effect with the
        next run; a disabled instance's true-peak histories stay frozen and its hold reads -inf"""
        _ck(lib().b200m_r128_set_dbtp_inst(self.h, int(inst), int(bool(enable))))

    def set_precision(self, mode):
        """precision of the dBTP FIR (PREC_EXACT / PREC_FMA); the EBU R128 part is always exact"""
        _ck(lib().b200m_r128_set_precision(self.h, int(mode)))

    def histogram(self, inst, stream=None):
        m = np.empty(751, np.int32); s = np.empty(751, np.int32)
        _ck(lib().b200m_r128_histogram(self.h, int(inst), _np_ptr(m), _np_ptr(s), _stream_ptr(stream)))
        return m, s

    def log_enable(self, capacity, stream=None, dbtp=False):
        """the loudness log of the cycle's EBU R128 bank: Ebu_r128_proc.log_enable.  dbtp=True adds each point's dBTP, the true peak
        of its fragment (b200m_r128_log_enable); log_drain then returns R128_POINT_DTYPE"""
        if dbtp:
            _ck(lib().b200m_r128_log_enable(self.h, int(capacity), _stream_ptr(stream)))
        else:
            self.ebu.log_enable(capacity, stream)
        self._tplog = bool(dbtp) and int(capacity) > 0

    def log_drain(self, stream=None):
        """Ebu_r128_proc.log_drain of the cycle's EBU R128 bank; with the dBTP plane on (log_enable(..., dbtp=True)) the points are
        R128_POINT_DTYPE (b200m_r128_log_drain)"""
        if not getattr(self, "_tplog", False):
            return self.ebu.log_drain(stream)
        return self._drain(lib().b200m_r128_log_drain, lib().b200m_ebu_log_capacity(self.ebu.h), R128_POINT_DTYPE, stream)


def _programme_blocks(x, lengths, block, empty):
    """the blocks a programme_* function feeds its banks: (ln, blocks), ln the validated lengths (int64 [N]; `empty` is the
    message when N is 0) and blocks an iterator of (b, xb, lb) per block b: xb frames off = b * block .. off + nfram - 1 of every
    row of x (x(off, nfram) when x is callable), nfram = min(block, longest remaining), and lb each row's length in the block,
    clamp(ln - off, 0, nfram)"""
    ln = np.asarray(lengths, np.int64).ravel()
    if ln.size == 0:
        raise B200MError(empty)
    if ln.min() < 0:
        raise B200MError("lengths must be frame counts >= 0")
    if not 1 <= int(block) <= 8192:
        raise B200MError("block must be 1..8192 frames")

    def blocks():
        total = int(ln.max())
        for b, off in enumerate(range(0, total, int(block))):
            nfram = min(int(block), total - off)
            yield b, x(off, nfram) if callable(x) else x[:, off:off + nfram], np.clip(ln - off, 0, nfram)
    return ln, blocks()


def _log_points(bank, overflow):
    """bank.log_drain()'s new points as (i, j, points): points[k] is instance i[k]'s j[k]-th new point, oldest first; raises
    B200MError("<overflow>: ...") when the log lost points"""
    pts, cnt, lost = bank.log_drain()
    if lost.any():
        raise B200MError("%s: %d points lost" % (overflow, int(lost.sum())))
    i, j = np.nonzero(np.arange(pts.shape[1]) < cnt[:, None].astype(np.int64))
    return i, j, pts[i, j]


PROGRAMME_FIELDS = ("integrated", "integ_thr", "range_min", "range_max", "maxloudn_M", "maxloudn_S")
CURVE_FIELDS = (("curve_M", "loudness_M"), ("curve_S", "loudness_S"), ("curve_I", "integrated"), ("curve_range_min", "range_min"),
                ("curve_range_max", "range_max"), ("curve_TP", "dbtp"))
CURVE_LOG_POINTS = 1200        # the loudness log's capacity in programme_loudness: 60 s of fragments at 48 kHz
TPLOG_MIN_FRAGM = 256          # the log's dBTP plane needs fragments of >= 256 frames (b200m_r128_log_enable): fsamp >= 5120 Hz


ALBUM_FIELDS = ("integrated", "integ_thr", "range_min", "range_max")      # the first four of group_finish's five


def programme_loudness(x, lengths, fsamp=48000.0, nchan=2, gains=None, block=1024, dbtp=True, precision=PREC_EXACT, device=0,
                       curves=False, groups=None):
    """Whole-programme EBU R128 loudness and true peak of N clips of different lengths, in one bank.

    x: rows i * nchan + c of clip i (nchan channels, or len(gains) with per-channel weights as in EBUr128), clip i valid for its
    first lengths[i] frames: a [N * nchan, >= max(lengths)] float32 numpy array / CPU tensor (host path) or CUDA tensor (device
    path), or a callable f(offset, nfram) that returns frames offset .. offset + nfram - 1 of every row as such an array (clips
    produced block by block).  Frames past a clip's length are never read into a result.
    Integration starts before the first frame.  The clips are fed in blocks of `block` frames: block k has
    nfram = min(block, longest remaining) and clip i's length in it is clamp(lengths[i] - k * block, 0, block) (EBUr128.run with
    lengths).  Clip i's numbers are therefore bit-identical (exact mode) to a private Ebu_r128_proc + TruePeakdsp instance fed the
    clip in blocks of `block` frames with a short last block -- the reference's results depend on where blocks are cut
    (ebu_r128_proc.cc:212-216).  No padding is metered: a short clip's loudness, maxima, histograms and range stop at its end.
    Returns a dict of float32 arrays of N: integrated, integ_thr, range_min, range_max, maxloudn_M, maxloudn_S (LUFS / LU, -200
    where the reference reports nothing) and tp_max (dBTP, -inf when dbtp is False or the clip is empty).
    curves=True adds each clip's loudness curve, one point per 50 ms fragment (fragm = int(fsamp) // 20 frames), point k ending at
    frame (k + 1) * fragm of the clip: n_points (int64 [N], lengths // fragm) and curve_M, curve_S, curve_I, curve_range_min,
    curve_range_max (float32 [N, max(n_points)], NaN past a clip's n_points), each point what the clip's reading was right after
    that fragment, and curve_TP (float32 [N, max(n_points)]): the dBTP of each fragment's true peak over the clip's channels (-inf
    when dbtp is False; NaN below 5120 Hz, where the log has no dBTP plane).  The bank's loudness log holds CURVE_LOG_POINTS points per clip and is drained before it can overflow, so
    the device memory does not grow with the programme; the other fields are the same as with curves=False (in tolerance mode tp_max
    is then always the chunk-parallel FIR's, b200m_r128_log_enable).
    groups: None, or N album ids (>= 0, or -1 for a clip in no album) for album loudness: the result then also holds, for each of
    G = max(groups) + 1 albums, album_integrated, album_integ_thr, album_range_min, album_range_max (the gated statistics of the
    sum of the member clips' histograms, Ebu_r128_proc.group_reduce / group_finish after the last block), album_maxloudn_M,
    album_maxloudn_S and album_tp_max (the largest of the member clips' values) and album_n_clips (int64).  An album without
    members reads -200 and tp_max -inf.  Every other field is the same as without groups."""
    ln, blocks = _programme_blocks(x, lengths, block, "no clips")
    n = ln.size
    grp = None if groups is None else _groups(groups, n)
    if gains is not None:
        nchan = np.asarray(gains).size
    bank = EBUr128(n, fsamp, dbtp, device, nchan=nchan, gains=gains)
    try:
        bank.set_precision(precision)
        bank.control(EBUr128.START)
        if curves:
            fragm = int(fsamp) // 20
            n_points = ln // fragm
            cv = {k: np.full((n, int(n_points.max())), np.nan, np.float32) for k, _ in CURVE_FIELDS}
            pos = np.zeros(n, np.int64)
            bank.log_enable(CURVE_LOG_POINTS, dbtp=fragm >= TPLOG_MIN_FRAGM)
            per_block = int(block) // fragm + 1                 # the most fragments one block completes for an instance
            drain_every = CURVE_LOG_POINTS // per_block

            def drain():
                # a drain copies every instance's whole [CURVE_LOG_POINTS] row (NaN past its count), however few points are new
                i, j, p = _log_points(bank, "loudness log overflow")
                for k, f in CURVE_FIELDS:
                    if f in p.dtype.names:
                        cv[k][i, pos[i] + j] = p[f]
                pos[:] += np.bincount(i, minlength=n)
        for b, xb, lb in blocks:
            bank.run(xb, lengths=lb)
            if curves and (b + 1) % drain_every == 0:
                drain()
        if curves:
            drain()
        r, tp = bank.results()
        n_albums = 0 if grp is None else int(grp.max()) + 1
        if n_albums:
            import torch
            d = torch.empty((n_albums, MIX_WORDS), dtype=torch.int32, device="cuda:%d" % device)
            torch.cuda.synchronize(device)          # after host input the bank's own stream writes d: no other work may still use it
            bank.ebu.group_reduce(grp, d)
            album5 = bank.ebu.group_finish(d)
    finally:
        bank.close()
    out = {k: np.ascontiguousarray(r[k], np.float32) for k in PROGRAMME_FIELDS}
    out["tp_max"] = tp
    if curves:
        out["n_points"] = n_points
        out.update(cv)
    if grp is not None:
        member = grp >= 0
        for j, k in enumerate(ALBUM_FIELDS):
            out["album_" + k] = album5[:, j].copy() if n_albums else np.empty(0, np.float32)
        for k, v, empty in (("maxloudn_M", out["maxloudn_M"], -200.0), ("maxloudn_S", out["maxloudn_S"], -200.0), ("tp_max", tp, -np.inf)):
            a = np.full(n_albums, empty, np.float32)
            np.maximum.at(a, grp[member], v[member])
            out["album_" + k] = a
        out["album_n_clips"] = np.bincount(grp[member], minlength=n_albums).astype(np.int64)
    return out


DR_CURVE_FIELDS = (("window_rms", "rms"), ("window_peak", "peak"), ("m_rms", "m_rms"), ("peak2", "peak2"), ("dr", "dr"),
                   ("dr_total", "dr_total"), ("block_count", "block_count"))
DR_CURVE_LOG_POINTS = 16       # the window log's capacity in programme_dr14: 48 s of windows


def programme_dr14(x, lengths, rate=48000.0, n_channels=2, dr_mode=True, block=1024, device=0, curves=False, groups=None):
    """DR-14 (dr_mode=True) or TPnRMS meter readings of N whole tracks of different lengths, in one bank.

    x: rows i * n_channels + c of track i, track i valid for its first lengths[i] frames: a [N * n_channels, >= max(lengths)]
    float32 numpy array / CPU tensor (host path) or CUDA tensor (device path), or a callable f(offset, nfram) that returns frames
    offset .. offset + nfram - 1 of every row as such an array (tracks produced block by block).  Frames past a track's length are
    never read into a result.  The tracks are fed in blocks of `block` frames: block k has nfram = min(block, longest remaining)
    and track i's length in it is clamp(lengths[i] - k * block, 0, block) (DR14.run with lengths), so track i's numbers are
    bit-identical to a private dr14 plugin instance fed the track in blocks of `block` frames with a short last block.
    A track's DR counts only its whole 3 s windows (rintf (3 * rate) + 1 frames each), as the reference's does: a partial last
    window is never scored, and a track shorter than three windows reads dr 21 ("not valid").  dr_mode needs rate >= 2731 Hz
    (b200m_dr14_create: a window longer than the largest block).
    Returns a DR14_RESULT_DTYPE array of N: each track's b200m_dr14_result after its last frame (all zero for an empty track,
    which never runs).
    curves=True (DR mode only) returns (that array, curves): each track's DR curve, one point per whole 3 s window, silent ones
    included, point k (index k - 1) ending at frame k * w of the track (w = rintf (3 * rate) + 1 frames).  curves holds n_windows
    (int64 [N], lengths // w); window_rms, window_peak (each window's own RMS and peak), m_rms, peak2 (second-highest window peak)
    and dr (float32 [N, W, n_channels]); dr_total and block_count (float32 [N, W]); silent (bool [N, W]), with W = max(n_windows),
    NaN (silent False) past a track's n_windows: the b200m_dr14_point fields.  The bank's window log holds DR_CURVE_LOG_POINTS
    points per track and is drained before it can overflow, so the device memory does not grow with the tracks; the result array
    is the same as with curves=False.
    groups: None, or N album ids (>= 0, or -1 for a track in no album) for album DR (DR mode only).  One more trailing element is
    then returned, albums: a dict for G = max(groups) + 1 albums of m_rms, peak2, dr, m_peak (float32 [G, n_channels]), dr_total,
    block_count (float32 [G]) (DR14.group_reduce / group_finish after the last block: the DR of one dr14 instance that scored every
    window of every member track), n_windows and n_tracks (int64 [G]), and dr_mean (float64 [G]): the arithmetic mean of the
    member tracks' valid (1 .. 20) dr_total (dr[0] for mono), NaN if none is valid.  An album without members reads like a fresh
    plugin (m_rms and peak2 -81, dr and dr_total 21, m_peak -80).  Every other returned value is the same as without groups."""
    ln, blocks = _programme_blocks(x, lengths, block, "no tracks")
    n = ln.size
    if curves and not dr_mode:
        raise B200MError("DR curves need dr_mode (a TPnRMS bank has no 3 s windows)")
    grp = None if groups is None else _groups(groups, n)
    if grp is not None and not dr_mode:
        raise B200MError("album DR needs dr_mode (a TPnRMS bank has no 3 s windows)")
    bank = DR14(n, n_channels, rate, dr_mode, device)
    try:
        if curves:
            w = int(np.rint(np.float32(rate * 3.0))) + 1
            n_windows = ln // w
            nw = int(n_windows.max())
            cv = {k: np.full((n, nw, n_channels), np.nan, np.float32) for k, _ in DR_CURVE_FIELDS[:5]}
            cv.update({k: np.full((n, nw), np.nan, np.float32) for k, _ in DR_CURVE_FIELDS[5:]})
            silent = np.zeros((n, nw), bool)
            bank.log_enable(DR_CURVE_LOG_POINTS)
            # k blocks of `block` frames close at most (k * block - 1) // w + 1 windows of a track: no more than the log holds
            # while k * block <= DR_CURVE_LOG_POINTS * w
            drain_every = DR_CURVE_LOG_POINTS * w // int(block)

            def drain():
                i, _, p = _log_points(bank, "window log overflow")
                k = p["window"].astype(np.int64) - 1
                for name, f in DR_CURVE_FIELDS:
                    v = p[f]
                    cv[name][i, k] = v[:, :n_channels] if v.ndim == 2 else v
                silent[i, k] = p["silent"] != 0
        for b, xb, lb in blocks:
            bank.run(xb, lengths=lb)
            if curves and (b + 1) % drain_every == 0:
                drain()
        if curves:
            drain()
            cv["n_windows"] = n_windows
            cv["silent"] = silent
        res = bank.results()
        out = (res, cv) if curves else (res,)
        if grp is not None:
            out += (_dr14_albums(bank, grp, res, device),)
        return out if len(out) > 1 else res
    finally:
        bank.close()


def _dr14_albums(bank, grp, res, device):
    """programme_dr14's albums dict (see there) of the tracks of `bank` after their last block, res their results"""
    import torch
    nch, g = bank.nchan, int(grp.max()) + 1 if grp.size else 0
    if g > 0:
        rows = torch.empty((g, dr14_group_words(nch)), dtype=torch.int32, device="cuda:%d" % device)
        peaks = torch.empty((g, nch, 3), dtype=torch.float32, device="cuda:%d" % device)
        torch.cuda.synchronize(device)          # after host input the bank's own stream writes rows: no other work may still use them
        bank.group_reduce(grp, rows, peaks)
        alb = bank.group_finish(rows, peaks)
        tail = rows[:, -2:].cpu().numpy().astype(np.int64)
    else:
        alb, tail = np.empty(0, DR14_ALBUM_DTYPE), np.empty((0, 2), np.int64)
    out = {k: np.ascontiguousarray(alb[k][:, :nch]) for k in ("m_rms", "peak2", "dr", "m_peak")}
    out.update(dr_total=alb["dr_total"].copy(), block_count=alb["block_count"].copy(), n_windows=tail[:, 0].copy(),
               n_tracks=tail[:, 1].copy())
    v = (res["dr_total"] if nch > 1 else res["dr"][:, 0]).astype(np.float64)
    ok = (grp >= 0) & (v >= 1) & (v <= 20)                      # 21: not valid; 0: an empty track, which never ran
    s, c = np.zeros(g), np.zeros(g)
    np.add.at(s, grp[ok], v[ok]); np.add.at(c, grp[ok], 1)
    with np.errstate(invalid="ignore", divide="ignore"):
        out["dr_mean"] = np.where(c > 0, s / np.maximum(c, 1), np.nan)
    return out


def programme_stats(x, lengths, rate=48000.0, block=1024, device=0):
    """Whole-clip bit-meter and signal-distribution statistics of N mono clips of different lengths (file QC: the bit depth actually
    used, NaN / Inf / denormal counts, the sample distribution), in one bit-meter bank (averaging mode, integrating) and one
    SigDistHist bank (integrating).

    x: row i = clip i, valid for its first lengths[i] frames: a [N, >= max(lengths)] float32 numpy array / CPU tensor (host path) or
    CUDA tensor (device path), or a callable f(offset, nfram) that returns frames offset .. offset + nfram - 1 of every row as such an
    array.  Frames past a clip's length are never read into a result.  The clips are fed in blocks of `block` frames with clip i's
    length in block k clamp(lengths[i] - k * block, 0, block) (Bitmeter.run / SigDistHist.run with lengths), so clip i's rows are
    bit-identical to a bitmeter (averaging) and a SigDistHist plugin instance fed the whole clip.
    Returns a dict of arrays of N rows, each clip's statistics after its last frame:
      bim_hist [N, 584] int32, bim_cnt [N, 5] int32 (zero, pos, nan, inf, den), bim_minmax [N, 2] float32, bim_itime [N] int64;
      sdh_hist [N, 361] int32, sdh_max_peak [N, 2] int32, sdh_avg_tmp_var [N, 3] float64 (sum, running mean, running variance
      accumulator), sdh_itime [N] int64.
    An empty clip reads what a freshly instantiated plugin reads: zero counts and sums, bit-meter minimum +inf, peak bin -1."""
    ln, blocks = _programme_blocks(x, lengths, block, "no clips")
    n = ln.size
    bim, sdh = Bitmeter(n, rate, device), None
    try:
        sdh = SigDistHist(n, rate, device)
        bim.control(CTL_AVERAGE)
        sdh.control(CTL_START)
        for _, xb, lb in blocks:
            bim.run(xb, lengths=lb)
            sdh.run(xb, lengths=lb)
        b = bim.results_all()
        h, mp, av, it = sdh.results_all()
    finally:
        bim.close()
        if sdh is not None:
            sdh.close()
    return dict(bim_hist=b["hist"], bim_cnt=b["cnt"], bim_minmax=b["minmax"], bim_itime=b["itime"],
                sdh_hist=h, sdh_max_peak=mp, sdh_avg_tmp_var=av, sdh_itime=it)


def _ltas_db(p):
    """10 log10 (2 p) of average band powers p, -100 where sqrt (2 p) <= 1e-5 or p is NaN: the scale and floor of the spectrum's
    level ports (src/spectrumlv2.c:240-247), so a settled steady tone reads the same here and in its band's port"""
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(np.sqrt(2.0 * p) > 1e-5, 10.0 * np.log10(2.0 * p), -100.0)


def _ltas(sums, counts):
    """sums / counts, NaN where the count is 0"""
    with np.errstate(invalid="ignore", divide="ignore"):
        return np.where(counts > 0, sums / np.maximum(counts, 1), np.nan)


def spectrum_albums(sums, counts, peak_db, groups):
    """Album long-term average spectra from per-clip rows: programme_spectrum's sums, counts and peak_db, or those of several banks
    (shards on several GPUs) concatenated in clip order, e.g. with shard.gather_results.  groups: N album ids (>= 0, or -1 for a clip
    in no album).  An album's sums are its members' sums added in ascending clip index and its counts the sum of theirs, so the
    result does not depend on how the clips were split between banks.  Returns a dict for G = max(groups) + 1 albums: album_ltas
    (float64 [G, 30], summed sums / summed counts), album_ltas_db (float64 [G, 30], on the level ports' scale), album_peak_db
    (float32 [G, 30], the largest member peak_db) and album_n_clips (int64 [G]).  An album without members reads NaN, -100, -100
    and 0."""
    sums = np.asarray(sums, np.float64); counts = np.asarray(counts, np.int64); peak_db = np.asarray(peak_db, np.float32)
    n = sums.shape[0] if sums.ndim == 2 else -1
    if n < 0 or sums.shape != (n, 30) or counts.shape != (n, 30) or peak_db.shape != (n, 30):
        raise B200MError("sums, counts and peak_db must be [N, 30] rows of the same N clips")
    grp = _groups(groups, n)
    g = int(grp.max()) + 1 if n else 0
    s, c = np.zeros((g, 30)), np.zeros((g, 30), np.int64)
    pk = np.full((g, 30), -100.0, np.float32)
    for i in np.flatnonzero(grp >= 0):                 # one clip at a time, in ascending index: a fixed order of the fp64 sums
        a = grp[i]
        s[a] += sums[i]
        c[a] += counts[i]
        np.maximum(pk[a], peak_db[i], out=pk[a])
    ltas = _ltas(s, c)
    return dict(album_ltas=ltas, album_ltas_db=_ltas_db(ltas), album_peak_db=pk,
                album_n_clips=np.bincount(grp[grp >= 0], minlength=g).astype(np.int64))


def programme_spectrum(x, lengths, rate=48000.0, nchan=2, speed=1.0, block=1024, precision=PREC_EXACT, device=0, groups=None):
    """Long-term average spectrum (LTAS) of N clips of different lengths in 30 1/3-octave bands (SPEC_BAND_HZ), in one spectrum bank.

    x: rows i * nchan + c of clip i (nchan 1 or 2; the bands analyse (L + R) / 2 of a stereo clip), clip i valid for its first
    lengths[i] frames: a [N * nchan, >= max(lengths)] float32 numpy array / CPU tensor (host path) or CUDA tensor (device path), or a
    callable f(offset, nfram) that returns frames offset .. offset + nfram - 1 of every row as such an array.  Frames past a clip's
    length are never read into a result.  The clips are fed in blocks of `block` frames with clip i's length in block k
    clamp(lengths[i] - k * block, 0, block) (Spectr30.process with lengths), so clip i's numbers are bit-identical (exact mode) to one
    spectr30 instance fed only that clip in blocks of `block` frames, with the speed port at `speed` and the LTAS plane on
    (Spectr30.ltas_enable).  precision=PREC_FMA runs the tolerance-mode filters (ltas_db within 1e-4 dB of exact mode).
    Returns a dict of arrays of N rows of 30 bands:
      sums (float64) and counts (int64): the LTAS plane after the clip's last frame (Spectr30.ltas): the sum of the band's per-frame
        power v * v over the clip's frames where it is finite, and the number of those frames;
      ltas (float64): sums / counts, the band's mean power, NaN where the count is 0;
      ltas_db (float64): 10 log10 (2 ltas), -100 where sqrt (2 ltas) <= 1e-5 or ltas is NaN: the level ports' scale and floor, so a
        settled steady tone reads the same as its band's level port;
      peak_db (float32): ports 30..59 after the clip's last block, the peak hold of the level smoothed at `speed` over the whole clip
        (never reset: the reset port is held at the value the instance's handshake state already has), -100 for an empty clip.
    groups: None, or N album ids (>= 0, or -1 for a clip in no album): the dict then also holds spectrum_albums(sums, counts,
    peak_db, groups)."""
    ln, blocks = _programme_blocks(x, lengths, block, "no clips")
    n = ln.size
    grp = None if groups is None else _groups(groups, n)
    bank = Spectr30(n, nchan, rate, device)
    try:
        bank.set_precision(precision)
        bank.ltas_enable()
        spd = np.full(n, speed, np.float32)
        # a speed other than the initial 1 sets rst_h = 0 on the first run (src/spectrumlv2.c:170-177), else rst_h stays -4: a reset
        # port equal to rst_h never starts the peak-reset handshake, whose max ports read -500
        rst = np.full(n, -4.0 if spd[0] == 1.0 else 0.0, np.float32)
        for _, xb, lb in blocks:
            bank.process(xb, speed=spd, reset=rst, lengths=lb)
        sums, counts = bank.ltas()
        ports = bank.read()
    finally:
        bank.close()
    peak_db = np.ascontiguousarray(ports[:, 30:])
    peak_db[ln == 0] = -100.0
    ltas = _ltas(sums, counts)
    out = dict(sums=sums, counts=counts, ltas=ltas, ltas_db=_ltas_db(ltas), peak_db=peak_db)
    if grp is not None:
        out.update(spectrum_albums(sums, counts, peak_db, grp))
    return out


def _cor_dist(hist, sums):
    """the derived fields of correlation histogram rows (int64 [N, 200], float64 [N]): frames (the row total), mean (sums / frames),
    below0 (the fraction of frames in bins 0..99, readings with (r + 1) * 100 < 100), p1 and p5 (the lower edge of the first bin
    where the cumulative count reaches 1 % / 5 % of frames); the float fields are NaN where frames is 0"""
    frames = hist.sum(axis=1)
    live = frames > 0
    cum = np.cumsum(hist, axis=1)

    def edge(den):                                      # first k with cum[k] / frames >= 1 / den, in integers
        k = np.argmax(cum * den >= frames[:, None], axis=1)
        return np.where(live, COR_HIST_EDGES[k], np.nan)
    with np.errstate(invalid="ignore", divide="ignore"):
        mean = np.where(live, sums / np.maximum(frames, 1), np.nan)
        below0 = np.where(live, cum[:, 99] / np.maximum(frames, 1), np.nan)
    return dict(frames=frames, mean=mean, below0=below0, p1=edge(100), p5=edge(20))


def correlation_albums(hist, sums, groups):
    """Album correlation distributions from per-clip rows: programme_correlation's hist and sums, or those of several banks (shards
    on several GPUs) concatenated in clip order, e.g. with shard.gather_results.  groups: N album ids (>= 0, or -1 for a clip in no
    album).  An album's counts are the sum of its members' and its sum their sums added in ascending clip index, so the result does
    not depend on how the clips were split between banks.  Returns a dict for G = max(groups) + 1 albums: album_hist (int64 [G, 200]),
    album_frames (int64 [G]), album_sums (float64 [G]), album_mean, album_below0, album_p1, album_p5 (float64 [G], as
    programme_correlation's clip fields) and album_n_clips (int64 [G]).  An album without counted frames reads NaN."""
    hist = np.asarray(hist, np.int64); sums = np.asarray(sums, np.float64)
    n = hist.shape[0] if hist.ndim == 2 else -1
    if n < 0 or hist.shape != (n, COR_HIST_BINS) or sums.shape != (n,):
        raise B200MError("hist and sums must be [N, 200] and [N] rows of the same N clips")
    grp = _groups(groups, n)
    g = int(grp.max()) + 1 if n else 0
    h, s = np.zeros((g, COR_HIST_BINS), np.int64), np.zeros(g)
    for i in np.flatnonzero(grp >= 0):                 # one clip at a time, in ascending index: a fixed order of the fp64 sums
        a = grp[i]
        h[a] += hist[i]
        s[a] += sums[i]
    d = _cor_dist(h, s)
    return dict(album_hist=h, album_frames=d["frames"], album_sums=s, album_mean=d["mean"], album_below0=d["below0"],
                album_p1=d["p1"], album_p5=d["p5"], album_n_clips=np.bincount(grp[grp >= 0], minlength=g).astype(np.int64))


def programme_correlation(x, lengths, rate=48000.0, flp=2e3, tcf=0.3, gate_db=-70.0, block=1024, device=0, groups=None):
    """Phase-correlation distribution of N stereo clips of different lengths, in one correlation bank.

    x: rows 2i, 2i + 1 = L, R of clip i, clip i valid for its first lengths[i] frames: a [2N, >= max(lengths)] float32 numpy array /
    CPU tensor (host path) or CUDA tensor (device path), or a callable f(offset, nfram) that returns frames offset .. offset +
    nfram - 1 of every row as such an array.  Frames past a clip's length are never read into a result.  The clips are fed in blocks
    of `block` frames with clip i's length in block k clamp(lengths[i] - k * block, 0, block) (Stcorrdsp.process with lengths), so
    clip i's numbers are bit-identical to one Stcorrdsp(rate, flp, tcf) fed only that clip in blocks of `block` frames with the
    histogram plane on (Stcorrdsp.hist_enable(gate_db=gate_db)).  The plane always runs exact.
    Returns a dict of N rows:
      hist (int64 [N, 200]): the counted frames' readings in the bins of COR_HIST_EDGES; a frame counts if the correlation filters'
        power zll + zrr >= 2 * 10^(gate_db / 10) and its reading is finite;
      frames (int64): counted frames; sums (float64): the sum of their readings in frame order;
      mean (float64): sums / frames;
      below0 (float64): the fraction of counted frames in bins 0..99, readings below 0 (anti-phase);
      p1, p5 (float64): the lower edge of the bin where the cumulative count first reaches 1 % / 5 % of frames, the lowest
        correlation the clip holds for at least 1 % / 5 % of its gated time;
      reading (float32): the port reading (Stcorrdsp::read) after the clip's last block, 0 for an empty clip.
    mean, below0, p1 and p5 are NaN where frames is 0.
    groups: None, or N album ids (>= 0, or -1 for a clip in no album): the dict then also holds correlation_albums(hist, sums,
    groups)."""
    ln, blocks = _programme_blocks(x, lengths, block, "no clips")
    n = ln.size
    grp = None if groups is None else _groups(groups, n)
    bank = Stcorrdsp(n, rate, flp, tcf, device)
    try:
        bank.hist_enable(gate_db=gate_db)
        for _, xb, lb in blocks:
            bank.process(xb, lengths=lb)
        hist, sums = bank.hist()
        reading = bank.read()
    finally:
        bank.close()
    out = dict(hist=hist, sums=sums, reading=reading)
    out.update(_cor_dist(hist, sums))
    if grp is not None:
        out.update(correlation_albums(hist, sums, grp))
    return out


def pw_window(fft_bins):
    """the phasewheel bank's float32 Hann window of 2 fft_bins points, as b200m_pw_create builds it: .5 - .5 cos (2 pi i / (N - 1))
    stored as float, then times 2 / (its sum in double), stored as float (gui/fft.c:69-79,122-161)"""
    N = 2 * int(fft_bins)
    w = (0.5 - 0.5 * np.cos(2.0 * np.pi / (N - 1.0) * np.arange(N))).astype(np.float32)
    return (w.astype(np.float64) * (2.0 / w.astype(np.float64).sum())).astype(np.float32)


def pw_enbw(fft_bins):
    """the equivalent noise bandwidth of the bank's window in bins, N sum(w^2) / sum(w)^2 in float64 (about 1.5)"""
    w = pw_window(fft_bins).astype(np.float64)
    return w.size * float((w * w).sum()) / float(w.sum()) ** 2


def _stereo_band_of_bin(rate, fft_bins):
    """the 1/3-octave band (index into SPEC_BAND_HZ, -1 for none) of each bin k < fft_bins: lo <= k rate / (2 fft_bins) < hi with
    lo, hi = centre * 2^(-+1/6); DC is in no band"""
    f = np.arange(int(fft_bins)) * (float(rate) / (2.0 * int(fft_bins)))
    lo, hi = SPEC_BAND_HZ * 2.0 ** (-1.0 / 6.0), SPEC_BAND_HZ * 2.0 ** (1.0 / 6.0)
    band = np.full(f.size, -1, np.int64)
    for b in range(SPEC_BAND_HZ.size):
        band[(f >= lo[b]) & (f < hi[b])] = b
    band[0] = -1
    return band


def stereo_bands(sums, analyses, rate, fft_bins):
    """Band fields of cross-spectrum rows (sums float64 [N, 4, fft_bins] in PW_XSPEC_TERMS order, analyses [N]): a clip's or an
    album's.  A band of SPEC_BAND_HZ holds the bins k with lo <= k rate / (2 fft_bins) < hi, lo, hi = centre * 2^(-+1/6) (DC is in
    none); its sums LL, RR and C = RL_RE + i RL_IM are its bins' sums added in ascending k.  Returns a dict of:
      band_level_db (float64 [N, 30, 2]): 10 log10 (LL / (analyses * enbw)) for L and the same with RR for R, enbw = pw_enbw (fft_bins):
        a steady sine of amplitude a well inside the band reads 20 log10 a (programme_spectrum's ltas_db scale);
      band_corr (Re C / sqrt (LL RR)), band_coherence (|C|^2 / (LL RR)), band_phase (atan2 (Im C, Re C), arg R - arg L);
      band_balance_db (10 log10 (RR / LL));
      band_mono_db (10 log10 ((LL + RR + 2 Re C) / (2 (LL + RR)))): the power of (L + R) / 2 against the mean channel power, 0 dB for
        identical channels, about -3.01 dB for uncorrelated ones and -inf for exact anti-phase;
    all float64 [N, 30].  NaN where a band has no bin or a denominator is 0 (band_phase: where C is 0), -inf where a log's argument is 0."""
    sums = np.asarray(sums, np.float64); analyses = np.asarray(analyses, np.int64)
    bins = int(fft_bins)
    n = sums.shape[0] if sums.ndim == 3 else -1
    if n < 0 or sums.shape != (n, 4, bins) or analyses.shape != (n,):
        raise B200MError("sums and analyses must be [N, 4, %d] and [N] rows of the same N clips" % bins)
    band = _stereo_band_of_bin(rate, bins)
    nb = SPEC_BAND_HZ.size
    acc = np.zeros((n, 4, nb))
    for k in np.flatnonzero(band >= 0):                  # ascending k: a fixed order of the fp64 sums
        acc[:, :, band[k]] += sums[:, :, k]
    empty = np.bincount(band[band >= 0], minlength=nb) == 0
    LL, RR, CR, CI = acc[:, 0], acc[:, 1], acc[:, 2], acc[:, 3]

    def ratio(num, den):                                 # num / den, NaN where den is 0 or the band is empty
        with np.errstate(invalid="ignore", divide="ignore"):
            return np.where((den != 0) & ~empty, num / np.where(den != 0, den, 1.0), np.nan)

    def db(r):                                           # 10 log10 r, -inf at 0 (and below: rounding of an exact 0), NaN stays
        with np.errstate(invalid="ignore", divide="ignore"):
            return np.where(r > 0, 10.0 * np.log10(np.where(r > 0, r, 1.0)), np.where(np.isnan(r), np.nan, -np.inf))
    den = (analyses.astype(np.float64) * pw_enbw(bins))[:, None]
    level = np.stack([db(ratio(LL, np.broadcast_to(den, LL.shape))), db(ratio(RR, np.broadcast_to(den, RR.shape)))], axis=-1)
    with np.errstate(invalid="ignore"):
        llrr = LL * RR
        corr = ratio(CR, np.sqrt(llrr))
    coh = ratio(CR * CR + CI * CI, llrr)
    phase = np.where(empty | ((CR == 0) & (CI == 0)), np.nan, np.arctan2(CI, CR))
    return dict(band_level_db=level, band_corr=corr, band_coherence=coh, band_phase=phase,
                band_balance_db=db(ratio(RR, LL)), band_mono_db=db(ratio(LL + RR + 2.0 * CR, 2.0 * (LL + RR))))


def stereo_albums(sums, analyses, skipped, groups, rate, fft_bins):
    """Album cross-spectra from per-clip rows: programme_stereo's sums, analyses and skipped, or those of several banks (shards on
    several GPUs) concatenated in clip order, e.g. with shard.gather_results.  groups: N album ids (>= 0, or -1 for a clip in no
    album).  An album's sums are its members' sums added in ascending clip index and its counts the sum of theirs, so the result does
    not depend on how the clips were split between banks.  Returns a dict for G = max(groups) + 1 albums: album_sums (float64
    [G, 4, fft_bins]), album_analyses, album_skipped and album_n_clips (int64 [G]), and stereo_bands of the album rows with each
    field prefixed album_ (album_band_corr, ...)."""
    sums = np.asarray(sums, np.float64); analyses = np.asarray(analyses, np.int64); skipped = np.asarray(skipped, np.int64)
    bins = int(fft_bins)
    n = sums.shape[0] if sums.ndim == 3 else -1
    if n < 0 or sums.shape != (n, 4, bins) or analyses.shape != (n,) or skipped.shape != (n,):
        raise B200MError("sums, analyses and skipped must be [N, 4, %d], [N] and [N] rows of the same N clips" % bins)
    grp = _groups(groups, n)
    g = int(grp.max()) + 1 if n else 0
    s, a, k = np.zeros((g, 4, bins)), np.zeros(g, np.int64), np.zeros(g, np.int64)
    for i in np.flatnonzero(grp >= 0):                 # one clip at a time, in ascending index: a fixed order of the fp64 sums
        s[grp[i]] += sums[i]
        a[grp[i]] += analyses[i]
        k[grp[i]] += skipped[i]
    out = dict(album_sums=s, album_analyses=a, album_skipped=k,
               album_n_clips=np.bincount(grp[grp >= 0], minlength=g).astype(np.int64))
    out.update(("album_" + f, v) for f, v in stereo_bands(s, a, rate, bins).items())
    return out


def programme_stereo(x, lengths, rate=48000.0, fft_bins=2048, block=1024, device=0, groups=None):
    """Stereo image by frequency band of N stereo clips of different lengths, in one phasewheel bank: per 1/3-octave band, the
    correlation, coherence, phase, balance and the level lost in the mono downmix (stereo_bands) over the whole clip.

    x: rows 2i, 2i + 1 = L, R of clip i, clip i valid for its first lengths[i] frames: a [2N, >= max(lengths)] float32 numpy array /
    CPU tensor (host path) or CUDA tensor (device path), or a callable f(offset, nfram) that returns frames offset .. offset +
    nfram - 1 of every row as such an array.  Frames past a clip's length are never read into a result.  The clips are fed in blocks
    of `block` frames with clip i's length in block k clamp(lengths[i] - k * block, 0, block) (Phasewheel.process with lengths), so
    clip i's sums, analyses and skipped are bit-identical to one Phasewheel(1, fft_bins, rate) fed only that clip in blocks of
    `block` frames with the cross-spectrum plane on (Phasewheel.xspec_enable).
    Coverage: an analysis takes the last 2 fft_bins frames of the clip, windowed, every ceil(rate / 25) frames of the clip's own clock,
    starting from a zeroed ring (the first analyses see leading zeros).  When 2 fft_bins < ceil(rate / 25), as with fft_bins 2048 at
    192 kHz, the frames between two windows are not analysed; a clip's tail after its last analysis is not analysed either.
    Returns a dict: sums (float64 [N, 4, fft_bins], PW_XSPEC_TERMS), analyses and skipped (int64 [N]; an analysis with a non-finite
    spectrum is skipped and adds nothing), bin_hz (float64 [fft_bins], k rate / (2 fft_bins)) and the stereo_bands fields ([N, 30]).
    groups: None, or N album ids (>= 0, or -1 for a clip in no album): the dict then also holds stereo_albums(sums, analyses,
    skipped, groups, rate, fft_bins)."""
    ln, blocks = _programme_blocks(x, lengths, block, "no clips")
    n = ln.size
    grp = None if groups is None else _groups(groups, n)
    bank = Phasewheel(n, fft_bins, rate, device)
    try:
        bank.xspec_enable()
        for _, xb, lb in blocks:
            bank.process(xb, lengths=lb)
        sums, analyses, skipped = bank.xspec()
    finally:
        bank.close()
    out = dict(sums=sums, analyses=analyses, skipped=skipped, bin_hz=np.arange(int(fft_bins)) * (float(rate) / (2.0 * int(fft_bins))))
    out.update(stereo_bands(sums, analyses, rate, fft_bins))
    if grp is not None:
        out.update(stereo_albums(sums, analyses, skipped, grp, rate, fft_bins))
    return out


def _needle_dist(hist):
    """groups (the row total: finite readings) and p95_db / p99_db of needle histogram rows (int64 [..., 242]): the lower edge, in dB,
    of the first bin where the cumulative count reaches 95 % / 99 % of groups, compared in integers; -inf for bin 0, NaN where
    groups is 0"""
    groups = hist.sum(axis=-1)
    cum = np.cumsum(hist, axis=-1)
    lower = np.concatenate([[-np.inf], PPM_HIST_EDGES_DB])   # bin k's lower edge

    def edge(pct):
        k = np.argmax(cum * 100 >= pct * groups[..., None], axis=-1)
        return np.where(groups > 0, lower[k], np.nan)
    return groups, edge(95), edge(99)


def _peak_db(peak):
    """20 log10 of float32 readings, -inf where the reading is not above 0 (no finite reading: peak is -inf)"""
    p = np.asarray(peak, np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(p > 0, 20.0 * np.log10(np.where(p > 0, p, 1.0)), -np.inf)


def needle_albums(hist, stats, groups):
    """Album needle distributions from per-clip rows: programme_needle's hist and stats, or those of several banks (shards on several
    GPUs) concatenated in clip order, e.g. with shard.gather_results.  groups: N album ids (>= 0, or -1 for a clip in no album).
    Pooling is per meter position (channel, or M and S): an album's counts, nonfinite, over_groups and overs are the sums of its
    members', its longest_over and peak their maxima.  All are integer sums or maxima, so the result does not depend on how the clips
    were split between banks.  Returns a dict for G = max(groups) + 1 albums of M meters: album_hist (int64 [G, M, 242]), album_groups,
    album_nonfinite, album_over_groups, album_overs, album_longest_over (int64 [G, M]), album_peak (float32 [G, M], -inf without a
    finite reading), album_peak_db, album_p95_db, album_p99_db (float64 [G, M], as programme_needle's clip fields) and album_n_clips
    (int64 [G]).  An album without members reads 0 counts, -inf peak and NaN percentiles.  An over run that ends one clip and one
    that starts the next are counted as two overs, and the longest run is the longest within one clip."""
    hist = np.asarray(hist, np.int64); stats = np.asarray(stats)
    n = hist.shape[0] if hist.ndim == 3 else -1
    if n < 0 or hist.shape[2:] != (PPM_HIST_BINS,) or stats.dtype != PPM_HIST_STATS_DTYPE or stats.shape != hist.shape[:2]:
        raise B200MError("hist and stats must be [N, M, 242] and [N, M] (PPM_HIST_STATS_DTYPE) rows of the same N clips")
    m = hist.shape[1]
    grp = _groups(groups, n)
    g = int(grp.max()) + 1 if n else 0
    h = np.zeros((g, m, PPM_HIST_BINS), np.int64)
    tot = {k: np.zeros((g, m), np.int64) for k in ("nonfinite", "over_groups", "overs", "longest_over")}
    pk = np.full((g, m), -np.inf, np.float32)
    for i in np.flatnonzero(grp >= 0):
        a = grp[i]
        h[a] += hist[i]
        for k in ("nonfinite", "over_groups", "overs"):
            tot[k][a] += stats[k][i].astype(np.int64)
        np.maximum(tot["longest_over"][a], stats["longest_over"][i].astype(np.int64), out=tot["longest_over"][a])
        np.maximum(pk[a], stats["peak"][i], out=pk[a])
    ng, p95, p99 = _needle_dist(h)
    out = dict(album_hist=h, album_groups=ng)
    out.update({"album_" + k: v for k, v in tot.items()})
    out.update(album_peak=pk, album_peak_db=_peak_db(pk), album_p95_db=p95, album_p99_db=p99,
               album_n_clips=np.bincount(grp[grp >= 0], minlength=g).astype(np.int64))
    return out


def programme_needle(x, lengths, kind, rate=48000.0, nchan=2, limit_db=0.0, ms_gain_db=(-6.0, -6.0), block=1024, device=0,
                     groups=None):
    """Needle-meter distribution of N clips of different lengths, in one needle-meter bank of `kind` (PPM_VU, PPM_IEC1, PPM_IEC2 or
    PPM_MS).

    x: VU / IEC: rows i * nchan + c of clip i, one meter per channel; M/S: rows 2i, 2i + 1 = L, R of clip i, one M/S pair (meters M
    and S, gains ms_gain_db), nchan ignored.  Clip i is valid for its first lengths[i] frames: a [rows, >= max(lengths)] float32 numpy
    array / CPU tensor (host path) or CUDA tensor (device path), or a callable f(offset, nfram) that returns frames offset .. offset +
    nfram - 1 of every row as such an array.  Frames past a clip's length are never read into a result.  The clips are fed in blocks
    of `block` frames with clip i's length in block k clamp(lengths[i] - k * block, 0, block) (NeedleMeters.process with lengths), so
    clip i's numbers are bit-identical to one NeedleMeters fed only that clip in blocks of `block` frames with the histogram plane on
    (NeedleMeters.hist_enable(limit_db=limit_db)); a block's last nfram mod 4 frames are not metered, as in the reference.
    Returns a dict of [N, M] rows, M = nchan (M/S: 2, M then S):
      hist (int64 [N, M, 242]): every finite group reading v = g * s in the bins of PPM_HIST_EDGES;
      stats (PPM_HIST_STATS_DTYPE): the plane's statistics, for needle_albums;
      groups (int64): finite readings; seconds (float64): 4 * groups / rate; nonfinite (int64): readings that were not finite;
      peak (float32): the largest finite reading, -inf without one; peak_db (float64): 20 log10 peak, -inf where peak <= 0;
      p95_db, p99_db (float64): the lower edge of the bin where the cumulative count first reaches 95 % / 99 % of groups: the level
        the needle stays under for 95 % / 99 % of the metered time (-inf: bin 0, below -80 dB; NaN: no reading);
      over_groups (int64) and over_seconds (float64): readings at or above 10^(limit_db / 20) and their time; overs (int64): the
        separate runs of such readings; longest_over_s (float64): the longest run's time;
      reading (float32): the read() port value after the clip's last block, the highest needle of the whole clip on the level
        port's scale (0 for an empty clip).
    groups: None, or N album ids (>= 0, or -1 for a clip in no album): the dict then also holds needle_albums(hist, stats, groups)."""
    ln, blocks = _programme_blocks(x, lengths, block, "no clips")
    n = ln.size
    grp = None if groups is None else _groups(groups, n)
    ms = kind == PPM_MS
    if not ms and int(nchan) < 1:
        raise B200MError("nchan must be >= 1")
    per = 2 if ms else int(nchan)
    units = n if ms else n * per
    bank = NeedleMeters(units, kind, rate, device)
    try:
        if ms:
            bank.set_gain(*ms_gain_db)
        bank.hist_enable(limit_db=limit_db)
        for _, xb, lb in blocks:
            bank.process(xb, lengths=lb if ms else np.repeat(lb, per))     # each meter of a clip runs the clip's frames
        hist, stats = bank.hist()
        st = bank.state()
    finally:
        bank.close()
    # read() is _g * _m, and _m holds the highest needle since the clip's first block (never read in between): formed here with the
    # same fp32 multiply, because the bank's read() skips units whose clip ended before the last block
    g = np.float32(design_ppm(kind, rate)[3])
    reading = (g * st[:, 2].astype(np.float32)).astype(np.float32)
    hist = hist.reshape(n, per, PPM_HIST_BINS); stats = stats.reshape(n, per); reading = reading.reshape(n, per)
    ng, p95, p99 = _needle_dist(hist)

    def sec(groups):                                      # 4 frames per group
        return groups.astype(np.float64) * 4.0 / float(rate)
    out = dict(hist=hist, stats=stats, groups=ng, seconds=sec(ng), nonfinite=stats["nonfinite"].astype(np.int64),
               peak=stats["peak"].copy(), peak_db=_peak_db(stats["peak"]), p95_db=p95, p99_db=p99,
               over_groups=stats["over_groups"].astype(np.int64), over_seconds=sec(stats["over_groups"]),
               overs=stats["overs"].astype(np.int64), longest_over_s=sec(stats["longest_over"]), reading=reading)
    if grp is not None:
        out.update(needle_albums(hist, stats, grp))
    return out


def _truepeak_fields(pfx, cnt, stats, rate, grp=None):
    """programme_truepeak's fields of one meter ("tp": a reading per frame, "km": per 4 frames) from its rows, cnt int64 [N, M, 242]
    and stats PPM_HIST_STATS_DTYPE [N, M]; grp: album ids for needle_albums, or None"""
    fpr = 1 if pfx == "tp" else 4
    unit, what = ("_dbtp", "frames") if pfx == "tp" else ("_db", "groups")

    def sec(readings):
        return readings.astype(np.float64) * fpr / float(rate)
    ng, p95, p99 = _needle_dist(cnt)
    out = {pfx + "_hist": cnt, pfx + "_stats": stats, pfx + "_" + what: ng, pfx + "_nonfinite": stats["nonfinite"].astype(np.int64),
           pfx + "_peak": stats["peak"].copy(), pfx + "_peak" + unit: _peak_db(stats["peak"]), pfx + "_p95" + unit: p95,
           pfx + "_p99" + unit: p99, pfx + "_over_" + what: stats["over_groups"].astype(np.int64),
           pfx + "_over_seconds": sec(stats["over_groups"]), pfx + "_overs": stats["overs"].astype(np.int64),
           pfx + "_longest_over_s": sec(stats["longest_over"])}
    if grp is not None:
        out.update({pfx + "_" + k: v for k, v in needle_albums(cnt, stats, grp).items()})
    return out


def programme_truepeak(x, lengths, rate=48000.0, nchan=2, flags=TPK_TRUEPEAK | TPK_KMETER, tp_limit_db=-1.0, km_limit_db=-10.0,
                       block=1024, device=0, groups=None):
    """True-peak and K-meter distributions of N clips of different lengths, in one TruePeakKmeter bank with the histogram plane on.

    x: rows i * nchan + c of clip i, one true-peak meter and one K-meter per channel, clip i valid for its first lengths[i] frames: a
    [N * nchan, >= max(lengths)] float32 numpy array / CPU tensor (host path) or CUDA tensor (device path), or a callable f(offset,
    nfram) that returns frames offset .. offset + nfram - 1 of every row as such an array.  Frames past a clip's length are never
    read into a result.  The clips are fed in process() blocks of `block` frames with clip i's length in block k clamp(lengths[i] -
    k * block, 0, block) (TruePeakKmeter.process with lengths, repeated per channel), so clip i's numbers are bit-identical to one
    TruePeakKmeter fed only that clip in blocks of `block` frames with the plane on (hist_enable(tp_limit_db=..., km_limit_db=...)).
    flags: the meters to run (TPK_TRUEPEAK, TPK_KMETER or both); the fields of a meter the bank lacks are absent.
    Returns a dict of [N, nchan] rows.  True peak, one reading per frame (the largest of its four 4x-oversampled |out|):
      tp_hist (int64 [N, nchan, 242]): the finite readings in the bins of PPM_HIST_EDGES; tp_stats (PPM_HIST_STATS_DTYPE), for
        needle_albums; tp_frames (int64): finite readings; tp_nonfinite (int64): frames with a non-finite |out|;
      tp_peak (float32): the largest finite reading, -inf without one; tp_peak_dbtp (float64): 20 log10 tp_peak;
      tp_p95_dbtp, tp_p99_dbtp (float64): the lower edge of the bin where the cumulative count first reaches 95 % / 99 % of tp_frames
        (-inf: below -80 dB; NaN: no reading); a p99 within a dB of tp_peak_dbtp marks an over-limited master;
      tp_over_frames (int64) and tp_over_seconds (float64): frames at or above 10^(tp_limit_db / 20), e.g. the -1 dBTP ceiling of EBU
        R128; tp_overs (int64): their separate runs; tp_longest_over_s (float64): the longest run's time;
      tp_max_dbtp (float64 [N]): the largest tp_peak_dbtp over the clip's channels.
    K-meter, one reading per group of 4 frames (sqrtf(2 z2), the rms port's value had a block ended after that group; a block's last
    nfram mod 4 frames are not metered, as in the reference): km_hist, km_stats, km_groups, km_nonfinite, km_peak, km_peak_db,
      km_p95_db, km_p99_db, km_over_groups, km_over_seconds, km_overs, km_longest_over_s likewise, 4 frames per reading.
      km_limit_db is dBFS RMS on the port's sine-calibrated scale: -10 dBFS is +4 on a K-14 scale, so the default counts the time
      spent above the K-14 meter's +4 zone.
    Final readings of the clip's last block, as read() would return them with no read in between: tp_m and tp_p (true peak), km_rms
    and km_peak (K-meter) (float32 [N, nchan]; 0 for an empty clip).
    groups: None, or N album ids (>= 0, or -1 for a clip in no album): the dict then also holds needle_albums of each meter's rows
    under the keys tp_album_* and km_album_* (album_hist, album_groups, album_peak_db, album_p95_db, album_overs, ...)."""
    ln, blocks = _programme_blocks(x, lengths, block, "no clips")
    n = ln.size
    grp = None if groups is None else _groups(groups, n)
    flags = int(flags)
    if flags not in (TPK_TRUEPEAK, TPK_KMETER, TPK_TRUEPEAK | TPK_KMETER):
        raise B200MError("flags must be TPK_TRUEPEAK, TPK_KMETER or both")
    per = int(nchan)
    if per < 1:
        raise B200MError("nchan must be >= 1")
    bank = TruePeakKmeter(n * per, rate, flags, device)
    try:
        bank.hist_enable(tp_limit_db=tp_limit_db, km_limit_db=km_limit_db)
        for _, xb, lb in blocks:
            bank.process(xb, lengths=np.repeat(lb, per))        # each meter of a clip runs the clip's frames
        tc, ts, kc, ks = bank.hist()
        st = bank.state()
    finally:
        bank.close()
    out = {}
    for pfx, cnt, stats in (("tp", tc, ts), ("km", kc, ks)):
        if cnt is not None:
            out.update(_truepeak_fields(pfx, cnt.reshape(n, per, PPM_HIST_BINS), stats.reshape(n, per), rate, grp))
    if tc is not None:
        out["tp_max_dbtp"] = out["tp_peak_dbtp"].max(axis=1)
        # read() returns _m and _p; no read happens in between, so they hold the whole clip's values (0 for an empty clip: _res)
        res = st["res"].astype(bool)
        out["tp_m"] = np.where(res, np.float32(0), st["m"]).astype(np.float32).reshape(n, per)
        out["tp_p"] = np.where(res, np.float32(0), st["p"]).astype(np.float32).reshape(n, per)
    if kc is not None:
        out["km_rms"] = st["km"][:, 2].astype(np.float32).reshape(n, per)
        out["km_peak"] = st["km"][:, 3].astype(np.float32).reshape(n, per)
    return out


# ---------------------------------------------------------------------------------------------------- PCM input
PCM_S16, PCM_S24, PCM_S32, PCM_F32 = 0, 1, 2, 3     # B200M_PCM_*
PCM_MAX_CHANNELS = 32                               # B200M_PCM_MAX_CHANNELS
PCM_BYTES = (2, 3, 4, 4)                            # bytes per sample of each format
_PCM_DTYPE = {np.dtype(np.int16): PCM_S16, np.dtype(np.int32): PCM_S32, np.dtype(np.float32): PCM_F32}


def _pcm_check(fmt, nchan):
    if fmt not in (PCM_S16, PCM_S24, PCM_S32, PCM_F32):
        raise B200MError("unknown PCM format %d" % fmt)
    if not 1 <= nchan <= PCM_MAX_CHANNELS:
        raise B200MError("nchan %d outside 1..%d" % (nchan, PCM_MAX_CHANNELS))


def _pcm_layout(a, fmt=None, nchan=None):
    """(fmt, nchan) of a numpy PCM array: int16 / int32 / float32 [N, T, nchan] (PCM_S16 / S32 / F32) or uint8 [N, T, nchan, 3]
    (PCM_S24, packed little-endian); B200MError if it is neither, or if it disagrees with a given fmt or nchan"""
    if not isinstance(a, np.ndarray):
        raise B200MError("PCM data must be a numpy array, not %s" % type(a).__name__)
    if a.dtype == np.uint8 and a.ndim == 4 and a.shape[3] == 3:
        f = PCM_S24
    elif a.dtype in _PCM_DTYPE and a.ndim == 3:
        f = _PCM_DTYPE[a.dtype]
    else:
        raise B200MError("PCM data must be int16, int32 or float32 [N, T, nchan], or uint8 [N, T, nchan, 3] for packed 24-bit; "
                         "got %s %s" % (a.dtype, a.shape))
    if fmt is not None and int(fmt) != f:
        raise B200MError("PCM format %s does not match %s data" % (fmt, a.dtype))
    if nchan is not None and int(nchan) != a.shape[2]:
        raise B200MError("nchan %s does not match data of %d channels" % (nchan, a.shape[2]))
    _pcm_check(f, a.shape[2])
    if a.shape[0] == 0:
        raise B200MError("no clips")
    return f, a.shape[2]


def pcm_planar(pcm, fmt, nchan, nfram=None, stream=None):
    """Interleaved PCM already on the device to the planar float32 rows every bank reads (b200m_pcm_planar_device, one launch).

    pcm: a CUDA tensor [N, ...] of N clips, each clip's bytes contiguous (any dtype: the bytes are read as `fmt`; a uint8 [N, bytes]
    view of uploaded WAV data chunks works as it lies), holding frames [t][c] of nchan samples of PCM_S16 (int16), PCM_S24 (packed
    24-bit), PCM_S32 (int32) or PCM_F32 (float32).  nfram: the frames to convert from the start of each clip (default: all it holds).
    Returns a float32 CUDA tensor [N * nchan, nfram], row i * nchan + c = channel c of clip i scaled by 2^-(bits - 1) (PCM_F32 bit for
    bit), with a row pitch of a multiple of 64 floats.  Runs on `stream` (default: torch's current stream of pcm's device)."""
    import torch
    fmt, nchan = int(fmt), int(nchan)
    if not (isinstance(pcm, torch.Tensor) and pcm.is_cuda and pcm.dim() >= 1 and pcm.shape[0] > 0 and pcm[0].is_contiguous()):
        raise B200MError("pcm must be a CUDA tensor [N, ...] of N >= 1 clips, each clip's samples contiguous")
    _pcm_check(fmt, nchan)
    n, es = pcm.shape[0], pcm.element_size()
    clip_bytes = pcm[0].numel() * es
    in_stride = pcm.stride(0) * es if n > 1 else clip_bytes
    nfram = clip_bytes // (nchan * PCM_BYTES[fmt]) if nfram is None else int(nfram)
    if not 1 <= nfram <= MAX_BLOCK:
        raise B200MError("nfram %d outside 1..%d" % (nfram, MAX_BLOCK))
    if nfram * nchan * PCM_BYTES[fmt] > clip_bytes:
        raise B200MError("%d frames of %d channels reach past the clip's %d bytes" % (nfram, nchan, clip_bytes))
    pitch = (nfram + 63) & ~63
    out = torch.empty((n * nchan, pitch), dtype=torch.float32, device=pcm.device)
    st = C.c_void_p(torch.cuda.current_stream(pcm.device).cuda_stream) if stream is None else _stream_ptr(stream)
    _ck(lib().b200m_pcm_planar_device(pcm.device.index, C.c_void_p(pcm.data_ptr()), fmt, n, nchan, nfram, in_stride,
                                      C.c_void_p(out.data_ptr()), pitch, st))
    return out[:, :nfram]


class _PcmSource:
    """pcm_source's callable: block (offset, nfram) of the source through one of two pinned slots to the device, then pcm_planar"""

    def __init__(self, data, fmt, nchan, device):
        self.data, self.fmt, self.nchan, self.device = data, fmt, nchan, device
        self.n = None if callable(data) else data.shape[0]
        self.slots = [None, None]           # pinned uint8 buffers from host_alloc, allocated with the first block
        self.events = [None, None]          # recorded behind each slot's last copy
        self.next = 0

    def _block(self, offset, nfram):
        if callable(self.data):
            blk = self.data(offset, nfram)
            _pcm_layout(blk, self.fmt, self.nchan)
            if self.n is None:
                self.n = blk.shape[0]
            if blk.shape[0] != self.n or blk.shape[1] != nfram:
                raise B200MError("the decoder returned %s for a block of %d clips x %d frames" % (blk.shape, self.n, nfram))
            return blk
        if offset < 0 or offset + nfram > self.data.shape[1]:
            raise B200MError("block of frames %d .. %d reaches past the %d frames of the data" % (offset, offset + nfram - 1,
                                                                                             self.data.shape[1]))
        return self.data[:, offset:offset + nfram]

    def __call__(self, offset, nfram):
        import torch
        offset, nfram = int(offset), int(nfram)
        if not 1 <= nfram <= MAX_BLOCK:
            raise B200MError("nfram %d outside 1..%d" % (nfram, MAX_BLOCK))
        blk = self._block(offset, nfram)
        dev = torch.device("cuda", self.device)
        stream = torch.cuda.current_stream(dev)
        es = blk.dtype.itemsize
        clip_bytes = nfram * self.nchan * PCM_BYTES[self.fmt]
        in_stride = (clip_bytes + 15) & ~15               # each clip's chunk starts at a 16-byte boundary: 16-byte loads
        nbytes = self.n * in_stride
        s = self.next
        self.next ^= 1
        if self.events[s] is not None:
            self.events[s].synchronize()                  # the slot's previous copy has run: it may be refilled
        if self.slots[s] is None or self.slots[s].size < nbytes:
            self.slots[s] = host_alloc(1, (nbytes + 3) // 4).view(np.uint8).reshape(-1)
        rows = self.slots[s][:nbytes].view(blk.dtype).reshape(self.n, in_stride // es)
        np.copyto(rows[:, :clip_bytes // es], blk.reshape(self.n, -1))
        d = torch.empty((self.n, in_stride), dtype=torch.uint8, device=dev)
        d.view(-1).copy_(torch.from_numpy(self.slots[s][:nbytes]), non_blocking=True)
        if self.events[s] is None:
            self.events[s] = torch.cuda.Event()
        self.events[s].record(stream)
        return pcm_planar(d, self.fmt, self.nchan, nfram, stream)


def pcm_source(data, nchan=None, fmt=None, device=0):
    """The block source f(offset, nfram) that every programme_* function takes as x, fed from interleaved PCM on the host.

    data: a numpy array [N, T, nchan] of int16 (PCM_S16), int32 (PCM_S32) or float32 (PCM_F32), or uint8 [N, T, nchan, 3] of packed
    little-endian 24-bit samples (PCM_S24; e.g. an np.memmap of WAV data chunks); or a callable g(offset, nfram) that returns such an
    array of nfram frames for a decoder, with nchan and fmt given.  f(offset, nfram) copies frames offset .. offset + nfram - 1 of
    every clip, as raw bytes, into one of two pinned slots (host_alloc; each clip's chunk at a 16-byte boundary), uploads the slot
    with an asynchronous copy and converts it on the device (pcm_planar), all on torch's current stream; a slot is refilled only
    after the copy issued from it before has run.  It returns a fresh float32 CUDA tensor [N * nchan, nfram] (row i * nchan + c =
    channel c of clip i, row pitch a multiple of 64 floats), so a programme function's results are those of the same clips given as
    the float32 planar array of pcm_planar's scale.  A block past the data's T frames raises B200MError.  dtype, shape and format
    are checked here, before any device use."""
    if callable(data):
        if nchan is None or fmt is None:
            raise B200MError("a decoder callable needs nchan and fmt")
        fmt, nchan = int(fmt), int(nchan)
        _pcm_check(fmt, nchan)
    else:
        fmt, nchan = _pcm_layout(data, fmt, nchan)
    return _PcmSource(data, fmt, nchan, int(device))
