"""What tests/test_buffers_and_streams_gpu.py must cover, importable without a GPU.

Every public function and class of ``MODULES`` is either ``COVERED`` by a case of the GPU catalogue (the GPU
module asserts that some case names it) or ``HOST_ONLY``, with the reason it needs no case.  The symbols of
the C ABI are sorted the same way: every one not in ``EXPORTS_NOT_LAUNCHING`` or ``EXPORTS_SHARDING`` must
be reached by some case of the catalogue."""

# (module, public name) -> reason it needs no case
HOST_ONLY = {
    ("paramgen", "build_win_mats"): "NumPy window matrices on the host",
    ("paramgen", "full_window_mat"): "NumPy window matrices on the host",
    ("paramgen", "reshape_means"): "NumPy / tensor reshape, no kernel",
    ("paramgen", "StreamLayout"): "host description of the column layout",
    ("paramgen", "merlin_layout"): "host description of the column layout (used by the mlpg_batch cases)",
    ("autograd", "mlpg"): "calls MLPG.apply, which the MLPG case runs",
    ("autograd", "mlpg_batch"): "calls MLPGBatch.apply, which the MLPGBatch case runs",
    ("autograd", "unit_variance_mlpg"): "calls UnitVarianceMLPG.apply, which the UnitVarianceMLPG cases run",
    ("autograd", "modspec"): "calls ModSpec.apply, which the ModSpec case runs",
    ("autograd", "modspec_batch"): "calls ModSpecBatch.apply, which the ModSpecBatch case runs",
    ("autograd", "trajectory_log_likelihood"): "calls TrajectoryLogLikelihood.apply, which the "
                                               "TrajectoryLogLikelihood case runs",
    ("autograd", "mlpg_with_variances"): "calls MLPGWithVariances.apply, which the MLPGWithVariances case runs",
    ("preprocessing", "trim_zeros_frames"): "NumPy on the host; the device trim runs inside DTWAligner and "
                                            "apply_each2d_trim",
    ("preprocessing", "remove_zeros_frames"): "NumPy on the host, the reference's semantics",
    ("preprocessing", "minmax_scale_params"): "arithmetic on the D-vectors on the host",
    ("preprocessing", "adjust_frame_length"): "NumPy padding on the host",
    ("preprocessing", "adjust_frame_lengths"): "NumPy padding on the host",
    ("preprocessing", "adjast_frame_length"): "deprecated alias of adjust_frame_length",
    ("preprocessing", "adjast_frame_lengths"): "deprecated alias of adjust_frame_lengths",
    ("preprocessing.alignment", "IterativeDTWAligner"): "composes DTWAligner and GaussianMixture, both in the "
                                                        "catalogue",
    ("util", "apply_delta_windows"): "alias of preprocessing.delta_features",
    ("util", "adjust_frame_length"): "re-export of preprocessing.adjust_frame_length",
    ("util", "delta_features"): "re-export of preprocessing.delta_features",
    ("util", "meanstd"): "re-export of preprocessing.meanstd",
    ("util", "meanvar"): "re-export of preprocessing.meanvar",
    ("util", "minmax"): "re-export of preprocessing.minmax",
    ("util", "minmax_scale"): "re-export of preprocessing.minmax_scale",
    ("util", "remove_zeros_frames"): "re-export of preprocessing.remove_zeros_frames",
    ("util", "scale"): "re-export of preprocessing.scale",
    ("util", "trim_zeros_frames"): "re-export of preprocessing.trim_zeros_frames",
}

# (module, public name) that some case of the GPU catalogue calls
COVERED = {
    ("paramgen", "mlpg"), ("paramgen", "mlpg_batch"), ("paramgen", "mlpg_grad"), ("paramgen", "mlpg_grad_batch"),
    ("paramgen", "unit_variance_mlpg_matrix"), ("paramgen", "mlpg_gv"), ("paramgen", "mlpg_gv_batch"),
    ("paramgen", "global_variance"), ("paramgen", "gv_statistics"),
    ("paramgen", "mlpg_ms"), ("paramgen", "mlpg_ms_batch"), ("paramgen", "mlpg_mixture"),
    ("paramgen", "mlpg_mixture_batch"), ("paramgen", "trajectory_log_likelihood"),
    ("paramgen", "trajectory_log_likelihood_batch"), ("paramgen", "trajectory_sample"),
    ("paramgen", "trajectory_sample_batch"), ("paramgen", "mlpg_vjp_batch"),
    ("autograd", "MLPG"), ("autograd", "MLPGBatch"), ("autograd", "UnitVarianceMLPG"), ("autograd", "ModSpec"),
    ("autograd", "ModSpecBatch"), ("autograd", "TrajectoryLogLikelihood"), ("autograd", "MLPGWithVariances"),
    ("metrics", "melcd"), ("metrics", "mean_squared_error"), ("metrics", "lf0_mean_squared_error"),
    ("metrics", "vuv_error"),
    ("preprocessing", "delta_features"), ("preprocessing", "meanvar"), ("preprocessing", "meanstd"),
    ("preprocessing", "minmax"), ("preprocessing", "scale"), ("preprocessing", "inv_scale"),
    ("preprocessing", "minmax_scale"), ("preprocessing", "inv_minmax_scale"), ("preprocessing", "interp1d"),
    ("preprocessing", "preemphasis"), ("preprocessing", "inv_preemphasis"), ("preprocessing", "mulaw"),
    ("preprocessing", "inv_mulaw"), ("preprocessing", "mulaw_quantize"), ("preprocessing", "inv_mulaw_quantize"),
    ("preprocessing", "modspec"), ("preprocessing", "modphase"), ("preprocessing", "inv_modspec"),
    ("preprocessing", "modspec_smoothing"),
    ("preprocessing.alignment", "DTWAligner"),
    ("postfilters", "merlin_post_filter"), ("postfilters", "modspec_post_filter"), ("postfilters", "modspec_statistics"),
    ("baseline.gmm", "MLPG"), ("baseline.gmm", "MLPGBase"), ("baseline.gmm", "GaussianMixture"),
    ("util", "apply_each2d_trim"), ("util", "apply_each2d_padded"),
    ("util.linalg", "cholesky_inv"), ("util.linalg", "cholesky_inv_banded"),
}

# the package modules whose public names are checked (``__all__`` where the module has one)
MODULES = ["paramgen", "autograd", "metrics", "preprocessing", "preprocessing.alignment", "postfilters",
           "baseline.gmm", "util", "util.linalg"]

# C-ABI symbols that enqueue no device work, with the reason
EXPORTS_NOT_LAUNCHING = {
    "nnk_abi_version": "version query",
    "nnk_last_error": "error text of the last call",
    "nnk_launch_count": "launch counter",
    "nnk_status_decode": "host decode of a status word",
    "nnk_mlpg_workspace_bytes": "sizing",
    "nnk_mlpg_gv_workspace_bytes": "sizing",
    "nnk_dtw_workspace_bytes": "sizing",
    "nnk_metric_workspace_bytes": "sizing",
    "nnk_gmm_em_workspace_bytes": "sizing",
    "nnk_kmeans_workspace_bytes": "sizing",
    "nnk_postfilter_basis_elems": "sizing",
    "nnk_frame_stats_workspace_bytes": "sizing",
    "nnk_f0_interp_workspace_bytes": "sizing",
    "nnk_preemphasis_workspace_bytes": "sizing",
    "nnk_mlpg_ms_workspace_bytes": "sizing",
    "nnk_mlpg_traj_ll_workspace_bytes": "sizing",
    "nnk_mlpg_traj_sample_workspace_bytes": "sizing",
    "nnk_mlpg_vjp_workspace_bytes": "sizing",
}

# launching symbols that only multi-GPU sharding calls: tests/test_sharding_gpu.py covers what one GPU can
EXPORTS_SHARDING = {"nnk_peer_alloc", "nnk_peer_free", "nnk_peer_export", "nnk_peer_open", "nnk_peer_close",
                    "nnk_peer_copy", "nnk_segment_copy"}


# launching symbols with no stream argument: the NumPy paths of mlpg / mlpg_batch run their own copy and
# compute streams and synchronise them before returning
EXPORTS_OWN_STREAMS = {"nnk_mlpg_host", "nnk_mlpg_batch_host"}


def launching_exports(exports):
    """The symbols of ``exports`` that some catalogue case must reach."""
    return sorted(set(exports) - set(EXPORTS_NOT_LAUNCHING) - EXPORTS_SHARDING)
