"""rednose_b200 -- H100-native batched EKF engine behind commaai/rednose's filter-definition surface.

Public entry points (see DESIGN.md / INTEGRATION.md):

  codegen.gen_code            sympy filter definition -> CUDA library (reference: rednose.helpers.ekf_sym.gen_code)
  ekf_sym.EKF_sym             single-filter Python driver over the C-ABI (reference class of the same name)
  ekf_sym_pyx.EKF_sym_pyx     binding of the native C++ driver (reference: the Cython class of the same name)
  batched.BatchedEKF          B filters resident in HBM: fused step, history, RTS smoother, maha query, augment
  streaming.HostStreamer      overlapped host <-> device front-end
  scheduler.RaggedScheduler   per-filter observation streams (kind buckets, per-filter clocks)
  smoothing.TiledSmoother     forward + RTS over long histories, tiled over filters
  sharding                    multi-GPU layout helpers

The `rednose` package next to this one re-exports these under the reference's module names.
"""
__version__ = "0.1.0"
