"""ctypes binding of ``libb2a.so`` (C ABI declared in ``include/b2a.h``).

The library is built in-tree by ``audiotools_b200/_build.py`` (nvcc, sm_90a) and
lives next to the sources in ``audiotools_b200/csrc/``.  There is no fallback: if
the shared object is missing or does not load, importing the engine raises.
"""
import ctypes
import os
from ctypes import POINTER, c_char_p, c_double, c_float, c_int, c_int32, c_int64, c_size_t, c_void_p

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("B2A_LIB_PATH") or os.path.join(HERE, "csrc", "libb2a.so")  # env: A/B builds only

B2A_OK = 0
PAD_MODES = {"reflect": 0, "constant": 1, "replicate": 2}
POST_NONE, POST_LOG10, POST_LN = 0, 1, 2
ROUTE_NONE, ROUTE_FFT, ROUTE_LARGE, ROUTE_DENSE = 0, 1, 2, 3  # b2a_stft_route

# name -> (restype, argtypes); must list every symbol include/b2a.h declares
SIGNATURES = {
    "b2a_version": (c_int, []),
    "b2a_last_error": (c_char_p, []),
    "b2a_stft_num_frames": (c_int64, [c_int64, c_int, c_int, c_int, c_int, c_int]),
    "b2a_spectral_workspace_bytes": (c_size_t, [c_int64, c_int64, c_int, c_int, c_int, c_int, c_int, c_int, c_int]),
    "b2a_spectral_f32": (c_int, [c_void_p, c_int64, c_int64, c_int, c_int, c_void_p, c_void_p,
                                 c_int, c_int, c_int, c_int,
                                 c_void_p, c_int, c_void_p,
                                 c_void_p, c_void_p, c_void_p, c_int, c_int,
                                 c_int, c_float, c_float,
                                 c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "b2a_lufs_num_blocks": (c_int64, [c_int64, c_double, c_double]),
    "b2a_lufs_workspace_bytes": (c_size_t, [c_int64, c_int, c_int64, c_double, c_double]),
    "b2a_lufs_f32": (c_int, [c_void_p, c_int64, c_int, c_int64, c_int64, c_double,
                             POINTER(c_double), POINTER(c_double), c_int, c_double,
                             POINTER(c_double), c_void_p, c_void_p, c_void_p,
                             c_void_p, c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
    "b2a_lufs_backward_workspace_bytes": (c_size_t, [c_int64, c_int, c_int64, c_double, c_double]),
    "b2a_lufs_backward_f32": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int64, c_int64, c_double,
                                      POINTER(c_double), POINTER(c_double), c_int, c_double, POINTER(c_double),
                                      c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "b2a_loudness_stats_num_short_term": (c_int64, [c_int64, c_double]),
    "b2a_loudness_stats_workspace_bytes": (c_size_t, [c_int64, c_int, c_int64, c_double]),
    "b2a_loudness_stats_f32": (c_int, [c_void_p, c_int64, c_int, c_int64, c_int64, c_double,
                                       POINTER(c_double), POINTER(c_double), c_int, POINTER(c_double),
                                       c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "b2a_true_peak_factor": (c_int, [c_double]),
    "b2a_true_peak_taps": (c_int, [c_int, c_void_p]),
    "b2a_true_peak_f32": (c_int, [c_void_p, c_int64, c_int, c_int64, c_int, c_void_p, c_void_p, c_void_p]),
    "b2a_limiter_workspace_bytes": (c_size_t, [c_int64, c_int, c_int64]),
    "b2a_limiter_f32": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int64, c_int, c_void_p, c_int, c_float, c_void_p,
                                c_void_p, c_void_p, c_void_p]),
    "b2a_sos_filter_workspace_bytes": (c_size_t, [c_int64, c_int, c_int64, c_int]),
    "b2a_sos_filter_f32": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int64, c_void_p, c_int64, c_int, c_int,
                                   c_void_p, c_void_p, c_void_p]),
    "b2a_sos_filter_zi_f32": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int64, c_void_p, c_int64, c_int, c_void_p,
                                      c_void_p, c_void_p, c_void_p, c_void_p]),
    "b2a_sos_filtfilt_workspace_bytes": (c_size_t, [c_int64, c_int, c_int64, c_int, c_int, c_int64]),
    "b2a_sos_filtfilt_f32": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int64, c_void_p, c_int64, c_int, c_int,
                                     c_int64, c_void_p, c_void_p, c_void_p]),
    "b2a_sos_filtfilt_backward_f32": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int64, c_void_p, c_int64, c_int,
                                              c_int, c_int64, c_void_p, c_void_p, c_void_p]),
    "b2a_rir_bands_kept": (c_int, [c_int, c_double]),
    "b2a_rir_f32": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int,
                            c_int64, c_double, c_double, c_int, c_void_p, c_void_p]),
    "b2a_rir_directional_f32": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                        c_void_p, c_int64, c_int, c_int, c_int64, c_double, c_double, c_int, c_void_p,
                                        c_void_p]),
    "b2a_rir_band_sum_f32": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int64, c_double, c_double, c_int,
                                     c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "b2a_gain_f32": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_void_p, c_void_p]),
    "b2a_fftconv_workspace_bytes": (c_size_t, [c_int64, c_int64, c_int64, c_int64]),
    "b2a_fftconv_f32": (c_int, [c_void_p, c_int64, c_int64, c_void_p, c_int64, c_int64, c_int, c_void_p, c_int,
                                c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "b2a_resample_out_len": (c_int64, [c_int64, c_int, c_int]),
    "b2a_resample_f32": (c_int, [c_void_p, c_int64, c_int64, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "b2a_pitch_shift_multi_workspace_bytes": (c_size_t, [c_int64, c_int64, c_int, c_void_p, c_int]),
    "b2a_pitch_shift_multi_f32": (c_int, [c_void_p, c_int64, c_int64, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p,
                                          c_size_t, c_void_p]),
    "b2a_pack_rows_f32": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int64, c_void_p, c_void_p]),
    "b2a_row_absmax_f32": (c_int, [c_void_p, c_int64, c_int64, c_void_p, c_void_p]),
    "b2a_limit_peak_f32": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_void_p, c_float, c_void_p]),
    "b2a_clamp_items_f32": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_void_p, c_void_p, c_void_p]),
    "b2a_mix_f32": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_void_p]),
    "b2a_quantize_f32": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_void_p, c_int, c_void_p]),
    "b2a_order_stats_f32": (c_int, [c_void_p, c_int64, c_void_p, c_int, c_void_p, c_void_p]),
    "b2a_spectral_tc_enable": (c_int, [c_int]),
    "b2a_peer_buffer_bytes": (c_size_t, [c_int, c_int]),
    "b2a_peer_buffer_create": (c_int, [c_int, c_int, c_void_p, c_void_p]),
    "b2a_peer_buffer_open": (c_int, [c_void_p, c_void_p]),
    "b2a_peer_buffer_close": (c_int, [c_void_p]),
    "b2a_peer_buffer_destroy": (c_int, [c_void_p]),
    "b2a_peer_put_f32": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "b2a_peer_collect_f32": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "b2a_peer_latest_f32": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "b2a_peer_status": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "b2a_spec_band_mask_f32": (c_int, [c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int,
                                       c_float, c_float, c_void_p]),
    "b2a_spec_rotate_f32": (c_int, [c_void_p, c_int64, c_int64, c_void_p, c_int, c_void_p]),
    "b2a_spec_mask_low_f32": (c_int, [c_void_p, c_int64, c_int64, c_void_p, c_float, c_float, c_float, c_void_p, c_void_p]),
    "b2a_pitch_shift_num_frames": (c_int, [c_int64, c_int, c_float]),
    "b2a_time_stretch_out_len": (c_int64, [c_int64, c_double]),
    "b2a_time_stretch_workspace_bytes": (c_size_t, [c_int64, c_int64, c_int, c_double]),
    "b2a_time_stretch_f32": (c_int, [c_void_p, c_int64, c_int64, c_int, c_double, c_void_p, c_void_p, c_size_t, c_void_p]),
    "b2a_spec_gate_f32": (c_int, [c_void_p, c_int64, c_int, c_int64, c_void_p, c_int64, c_int64, c_float, c_void_p, c_int,
                                  POINTER(c_float), c_int, POINTER(c_float), c_int, c_void_p, c_void_p, c_void_p]),
    "b2a_alter_drr_f32": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int, c_int, c_void_p, c_float, c_void_p]),
    "b2a_dft_matrix_floats": (c_size_t, [c_int, c_int]),
    "b2a_dft_matrix_f32": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "b2a_mel_dct_f32": (c_int, [c_void_p, c_int64, c_int, c_int64, c_void_p, c_int, c_void_p, c_void_p]),
    "b2a_stft_route": (c_int, [c_int, c_int, c_int]),
    "b2a_istft_workspace_bytes": (c_size_t, [c_int64, c_int64, c_int, c_int]),
    "b2a_istft_f32": (c_int, [c_void_p, c_int64, c_int64, c_int, c_int, c_void_p, c_void_p, c_int, c_int64, c_int64,
                              c_void_p, c_void_p, c_size_t, c_void_p]),
    "b2a_stft_backward_workspace_bytes": (c_size_t, [c_int64, c_int64, c_int, c_int, c_int, c_int, c_int]),
    "b2a_stft_backward_f32": (c_int, [c_void_p, c_int64, c_int64, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_int,
                                      c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
    "b2a_istft_backward_workspace_bytes": (c_size_t, [c_int64, c_int64]),
    "b2a_istft_backward_f32": (c_int, [c_void_p, c_int64, c_int64, c_int, c_int, c_void_p, c_void_p, c_int, c_int64,
                                       c_int64, c_void_p, c_void_p, c_size_t, c_void_p]),
    "b2a_mel_backward_f32": (c_int, [c_void_p, c_int64, c_int, c_int64, c_void_p, c_void_p, c_void_p, c_int, c_void_p,
                                     c_void_p, c_int, c_float, c_float, c_void_p, c_void_p, c_void_p]),
    "b2a_spectral_loss_supported": (c_int, [c_int, c_int, c_int]),
    "b2a_spectral_loss_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "b2a_spectral_loss_f32": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int, c_int, c_void_p, c_int, c_int, c_int,
                                      c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_float, c_float,
                                      c_float, c_float, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "b2a_fir_direct_supported": (c_int, [c_int64, c_int, c_int]),
    "b2a_fir_direct_f32": (c_int, [c_void_p, c_int64, c_int64, c_void_p, c_int64, c_int, c_int, c_void_p, c_int, c_int,
                                   c_int64, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "b2a_circconv_workspace_bytes": (c_size_t, [c_int64, c_int64, c_int64, c_int64]),
    "b2a_circconv_f32": (c_int, [c_void_p, c_int64, c_int64, c_void_p, c_int64, c_int64, c_int, c_int, c_void_p, c_void_p,
                                 c_void_p, c_size_t, c_void_p]),
    "b2a_circconv_path_workspace_bytes": (c_size_t, [c_int64, c_int64, c_int64, c_int64, c_int, c_int, c_int]),
    "b2a_circconv_path_f32": (c_int, [c_void_p, c_int64, c_int64, c_void_p, c_int64, c_int64, c_int, c_int, c_int,
                                      c_int, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "b2a_resample_backward_f32": (c_int, [c_void_p, c_int64, c_int64, c_int, c_int, c_int, c_void_p, c_void_p,
                                          c_void_p]),
    "b2a_fir_pad_fold_workspace_bytes": (c_size_t, [c_int64, c_int]),
    "b2a_fir_pad_fold_f32": (c_int, [c_void_p, c_int64, c_int64, c_void_p, c_int64, c_int, c_int, c_void_p, c_int,
                                     c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "b2a_circconv_backward_workspace_bytes": (c_size_t, [c_int64, c_int64, c_int64, c_int64]),
    "b2a_circconv_backward_f32": (c_int, [c_void_p, c_int64, c_int64, c_void_p, c_int64, c_int64, c_int, c_int,
                                          c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "b2a_peak_scale_backward_f32": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_float, c_void_p,
                                            c_void_p, c_void_p, c_void_p]),
    "b2a_spec_band_mask_out_f32": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                           c_int, c_int, c_float, c_float, c_void_p]),
    "b2a_spec_band_mask_backward_f32": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p,
                                                c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "b2a_spec_mask_low_out_f32": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_void_p, c_float, c_float, c_float,
                                          c_void_p, c_void_p]),
    "b2a_spec_mask_low_backward_f32": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_void_p, c_float, c_float,
                                               c_float, c_void_p, c_void_p, c_void_p]),
    "b2a_spec_gate_backward_f32": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int64, c_void_p, c_int64, c_void_p,
                                           c_int, POINTER(c_float), c_int, POINTER(c_float), c_int, c_void_p,
                                           c_void_p]),
    "b2a_stoi_workspace_bytes": (c_size_t, [c_int64, c_int64, c_int, c_int]),
    "b2a_stoi_f32": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int64, c_int, c_void_p, c_int, c_int, c_int,
                             c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "b2a_stoi_backward_workspace_bytes": (c_size_t, [c_int64, c_int64, c_int, c_int]),
    "b2a_stoi_backward_f32": (c_int, [c_void_p, c_void_p, c_size_t, c_int64, c_int, c_int64, c_int, c_void_p, c_int,
                                      c_int, c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
}


class B2AError(RuntimeError):
    pass


class B2ALibrary:
    """A loaded ``libb2a`` with typed entry points.  ``check(rc)`` raises ``B2AError``
    carrying ``b2a_last_error()``; error codes map to the reference's exception types
    at the AudioSignal layer."""

    def __init__(self, path: str = LIB_PATH):
        if not os.path.exists(path):
            raise ImportError(
                f"{path} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc, sm_90a).  audiotools_b200 has no CPU fallback.")
        self.path = path
        self.cdll = ctypes.CDLL(path)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(self.cdll, name)  # AttributeError if the symbol is not exported
            fn.restype = res
            fn.argtypes = args
            setattr(self, name, fn)
        # b2a_kernel_launches: ``kernel_launches.value`` reads the library's launch count with no foreign-function call
        self.kernel_launches = c_int64.in_dll(self.cdll, "b2a_kernel_launches")

    def check(self, rc: int):
        if rc != B2A_OK:
            msg = self.b2a_last_error()
            raise B2AError(f"libb2a error {rc}: {msg.decode() if msg else '?'}")

    def call(self, fn, *args) -> int:
        """Call ``fn``, an entry point that launches kernels, raise on its error code, and return the number of kernels
        it launched (read from ``b2a_kernel_launches`` around the call)."""
        n0 = self.kernel_launches.value
        self.check(fn(*args))
        return self.kernel_launches.value - n0


_LIB = None


def get_lib() -> B2ALibrary:
    global _LIB
    if _LIB is None:
        _LIB = B2ALibrary(LIB_PATH)
    return _LIB
