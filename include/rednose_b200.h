/* rednose_b200 -- C-ABI of the H100-native batched EKF engine.
 *
 * This header declares (1) the plugin descriptor every generated lib<name>.so returns
 * from ekf_get(), the plain-C replacement of the reference's C++ `struct EKF` +
 * `ekf_lib_init` (rednose/helpers/ekf.h:16-42), and (2) the runtime library
 * librednose_b200.so: plugin registry (rednose/helpers/ekf_load.cc:4-39) and the
 * native single-filter driver (rednose/helpers/ekf_sym.{h,cc}).
 *
 * Per-filter entry points live in the generated <name>.h; their shapes are:
 *
 *   reference set, HOST pointers, one filter (rednose/helpers/ekf_sym.py:149-171)
 *     void <name>_predict(double *x, double *P, double *Q, double dt);                       ekf_c.c:8-33
 *     void <name>_update_<kind>(double *x, double *P, double *z, double *R, double *ea);     ekf_c.c:37-121
 *     void <name>_f_fun / _F_fun / _err_fun / _inv_err_fun / _H_mod_fun / _h_<kind> / _H_<kind> / _He_<kind>
 *     void <name>_set_<var>(double);                                                          ekf_sym.py:166-171
 *   batched additions, DEVICE pointers, B independent filters, AoS row-major float64
 *     void <name>_batch_predict(...), <name>_batch_update_<kind>(...), <name>_batch_step_<kind>(...)
 *     void <name>_batch_rts(...)   RTS smoother over a time-major history [T, B, ...]  (ekf_sym.py:651-690)
 *   batched, HOST pointers (copies inside): <name>_host_step_<kind>(...)
 *
 * All functions return void like the reference; CUDA failures are printed to stderr and
 * latched: `int <name>_cuda_status(void)` returns and clears the last cudaError_t (0 = ok).
 * There is no CPU fallback anywhere in these libraries.
 */
#ifndef REDNOSE_B200_H
#define REDNOSE_B200_H

#ifdef __cplusplus
extern "C" {
#endif

#define REDNOSE_B200_ABI_VERSION 1

/* step flags (mirrors of the driver-level normalisation calls, ekf_sym.cc:207,213) */
#define REDNOSE_NORM_AFTER_PREDICT 1
#define REDNOSE_NORM_AFTER_UPDATE 2
#define REDNOSE_Q_IS_DIAGONAL 4      /* caller promises Q is diagonal: kernels read only its diagonal */
#define REDNOSE_SHARED_R 8           /* R is one [ZDIM, ZDIM] matrix shared by the whole batch (what get_R builds, kalmanfilter.py:37-43) */

typedef void (*rednose_leaf3_fn)(double *, double *, double *);
typedef void (*rednose_leaf2_fn)(double *, double *);
typedef void (*rednose_leaf_dt_fn)(double *, double, double *);
typedef void (*rednose_predict_fn)(double *, double *, double *, double);
typedef void (*rednose_update_fn)(double *, double *, double *, double *, double *);
typedef void (*rednose_set_fn)(double);
typedef void (*rednose_batch_predict_fn)(double *x, double *P, const double *Q, const double *dt_arr, double dt, long long B, const int *quat_idxs, int n_quat, int flags, double *hx_pred, double *hP_pred, void *stream);
typedef void (*rednose_batch_update_fn)(double *x, double *P, double *z, const double *R, const double *ea, int n_obs, long long B, const int *quat_idxs, int n_quat, int flags, double *hx_filt, double *hP_filt, void *stream);
typedef void (*rednose_batch_step_fn)(double *x, double *P, const double *Q, const double *dt_arr, double dt, double *z, const double *R, const double *ea, int n_obs, long long B, const int *quat_idxs, int n_quat, int flags, double *hx_pred, double *hP_pred, double *hx_filt, double *hP_filt, void *stream);
typedef void (*rednose_host_step_fn)(double *x, double *P, const double *Q, const double *dt_arr, double dt, double *z, const double *R, const double *ea, int n_obs, long long B, const int *quat_idxs, int n_quat, int flags);

typedef void (*rednose_batch_rts_fn)(const double *hx_pred, const double *hP_pred, const double *hx_filt, const double *hP_filt, const double *t, int t_per_filter, double *xs, double *Ps, int T, long long B, const int *quat_idxs, int n_quat, int norm_quats, void *stream);

/* Plugin descriptor: replaces `struct EKF` (ekf.h:16-33).  Arrays have n_kinds entries,
 * parallel to `kinds`. */
typedef struct rednose_ekf_desc {
  int abi_version;
  const char *name;
  int dim, edim, medim;
  int n_kinds;
  const int *kinds;
  const int *zdims;
  const int *eadims;
  const int *feature_kind;  /* 1 if the kind null-space projects with He (ekf_c.c:66-76) */
  const int *maha_kind;     /* 1 if Mahalanobis gated (ekf_c.c:88-94) */
  rednose_leaf_dt_fn f_fun, F_fun;
  rednose_leaf3_fn err_fun, inv_err_fun;
  rednose_leaf2_fn H_mod_fun;
  rednose_predict_fn predict;
  const rednose_leaf3_fn *hs, *Hs, *Hes;
  const rednose_update_fn *updates;
  int n_sets;
  const char *const *set_names;
  const rednose_set_fn *sets;
  int n_extra;
  const char *const *extra_names;
  void *const *extra_fns;
  rednose_batch_predict_fn batch_predict;
  const rednose_batch_update_fn *batch_updates;
  const rednose_batch_step_fn *batch_steps;
  const rednose_host_step_fn *host_steps;
  rednose_batch_rts_fn batch_rts;   /* backward smoother over a stored history (ekf_sym.py:651-690) */
} rednose_ekf_desc;

/* ---- registry (librednose_b200.so; ekf_load.cc:4-39) ---- */
void rednose_b200_register(const rednose_ekf_desc *desc);
const rednose_ekf_desc *rednose_b200_lookup(const char *name);                 /* first registered plugin of that name (ekf_load.cc:13-20) */
/* the plugin of that name loaded from that directory: unlike the reference's name-only table, two builds of one filter
   (different directories) can be loaded side by side and a driver gets the one it asked for */
const rednose_ekf_desc *rednose_b200_lookup_in(const char *directory, const char *name);
/* dlopen(<dir>/lib<name>.so) + ekf_get() + register; idempotent per (directory, name) (ekf_load.cc:22-39); 0 on success */
int rednose_b200_load_and_register(const char *directory, const char *name);

/* ---- native single-filter driver (librednose_b200.so; rednose/helpers/ekf_sym.{h,cc} EKFSym) ----
 * The handle owns x, P, Q, the filter time (NaN = unset, ekf_sym.cc:42) and the rewind ring (512 checkpoints,
 * ekf_sym.h:18).  All numerics go through the filter library's <name>_predict / <name>_update_<kind>. */
void *rednose_ekfsym_create(const char *directory, const char *name, const double *Q, const double *x0, const double *P0, int dim_x, int dim_err, int dim_main, int dim_main_err, int N, int dim_augment, int dim_augment_err, const int *maha_test_kinds, int n_maha, const int *quaternion_idxs, int n_quat, double max_rewind_age);
void rednose_ekfsym_destroy(void *h);
void rednose_ekfsym_init_state(void *h, const double *x, const double *P, double filter_time);
double *rednose_ekfsym_x_ptr(void *h);   /* live views, valid until destroy / init_state */
double *rednose_ekfsym_P_ptr(void *h);
double rednose_ekfsym_get_filter_time(void *h);
void rednose_ekfsym_set_filter_time(void *h, double t);
void rednose_ekfsym_reset_rewind(void *h);
int rednose_ekfsym_rewind_depth(void *h);
void rednose_ekfsym_normalize_quaternions(void *h);
void rednose_ekfsym_augment(void *h);                                /* ekf_sym.py:365-391 */
void rednose_ekfsym_get_augment_times(void *h, double *out);
int rednose_ekfsym_set_global(void *h, const char *var, double val); /* 0 = ok, -1 = unknown variable */
void *rednose_ekfsym_get_extra_routine(void *h, const char *routine);
void rednose_ekfsym_predict(void *h, double t);                      /* ekf_sym.cc:196-209 */
/* ekf_sym.cc:83-117: returns 1 (outputs filled), 0 (observation too old, ignored), -1 (unknown kind) */
int rednose_ekfsym_predict_and_update_batch(void *h, double t, int kind, const double *z, const double *R, const double *ea, int n, int zdim, int eadim, int augment, double *xk1, double *xk, double *Pk1, double *Pk, double *y);

#ifdef __cplusplus
}
/* self-registration used by generated libraries (ekf.h:39-42): only if the registry is linked in */
extern "C" void rednose_b200_register(const rednose_ekf_desc *) __attribute__((weak));
static inline void rednose_b200_register_weak(const rednose_ekf_desc *d) {
  if (rednose_b200_register) rednose_b200_register(d);
}
#endif

#endif /* REDNOSE_B200_H */
