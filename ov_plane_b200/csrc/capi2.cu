// Second half of the extern "C" surface: EKFUpdate / clone / marginalize / initialize entry points, the stateless
// UpdaterHelper / UpdaterPlane helpers, UpdaterMSCKF::update, the multi-GPU shard halves, the Propagator and instrumentation.
// (compiled as part of the unity build ovp_unity.cu, after capi.cu)
#include <climits>
#include "host_math.h"

using namespace ovp;

namespace ovp {

__global__ void transpose_stack_kernel(const double *blocks, int G, int n, double *Hs, int ld) {
  // Hs[(g*n + i), j] = L_g[j, i]   for i < n, j <= n ; block g is (n+1) x (n+1) col-major
  size_t total = (size_t)G * n * (n + 1);
  for (size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
    int j = (int)(t % (n + 1));
    size_t r = t / (n + 1);
    int i = (int)(r % n), g = (int)(r / n);
    const double *L = blocks + (size_t)g * (n + 1) * (n + 1);
    Hs[(size_t)j * ld + (size_t)g * n + i] = L[(size_t)i * (n + 1) + j];
  }
}

static int small_inverse(const double *A, int s, double *Ainv) { // col-major, Gauss-Jordan with partial pivoting
  double M[9], I[9];
  for (int i = 0; i < s * s; i++) {
    M[i] = A[i];
    I[i] = 0;
  }
  for (int i = 0; i < s; i++)
    I[i * s + i] = 1;
  for (int k = 0; k < s; k++) {
    int p = k;
    for (int i = k + 1; i < s; i++)
      if (std::fabs(M[k * s + i]) > std::fabs(M[k * s + p]))
        p = i;
    if (M[k * s + p] == 0.0)
      return 1;
    if (p != k)
      for (int j = 0; j < s; j++) {
        std::swap(M[j * s + k], M[j * s + p]);
        std::swap(I[j * s + k], I[j * s + p]);
      }
    double d = M[k * s + k];
    for (int j = 0; j < s; j++) {
      M[j * s + k] /= d;
      I[j * s + k] /= d;
    }
    for (int i = 0; i < s; i++)
      if (i != k) {
        double f = M[k * s + i];
        for (int j = 0; j < s; j++) {
          M[j * s + i] -= f * M[j * s + k];
          I[j * s + i] -= f * I[j * s + k];
        }
      }
  }
  for (int i = 0; i < s * s; i++)
    Ainv[i] = I[i];
  return 0;
}

// new variable bookkeeping after its covariance rows exist
static void register_new(Ctx *c, int h, int kind, int64_t tag) {
  c->vars[h].id = c->N;
  c->order.push_back(h);
  c->N += c->vars[h].size;
  c->var_table_dirty = true;
  if (kind == OVP_KIND_LANDMARK)
    c->slam[tag] = h;
  else
    c->planes[tag] = h;
}

// StateHelper::initialize_invertible on device-staged operands (W = [H_L | H_R | res], top s rows), StateHelper.cpp:489-586
static int init_invertible_core(Ctx *c, int kind, int s, const double *value, const double *fej, int64_t tag, const int *d_cols, int n,
                                const double *W, int ldW, double sigma2, int *new_handle, bool hl_is_upper = true) {
  const int N = c->N;
  if (N + s > c->Nmax)
    return fail(c, OVP_ERR_CAPACITY, "state capacity %d exceeded", c->Nmax);
  // M_a = P[:, cols] * Hxinit^T (N x s);  Hxinit = W[0:s, s:s+n]
  MatView HxT = mv(W + (size_t)s * ldW, ldW, 1); // logical n x s
  launch_gemm1(c, make_problem(N, s, n, mv(c->dP, c->ldP, 0, nullptr, d_cols), HxT, c->dM, c->Nmax));
  // Mm = Hxinit * M_a[cols,:] + sigma2 I  (s x s) -> dscal[16..]
  double *dMm = c->dscal + 16;
  {
    MatView Hx = HxT;
    Hx.trans ^= 1;
    GemmProblem p = make_problem(s, s, n, Hx, mv(c->dM, c->Nmax, 0, d_cols, nullptr), dMm, s);
    p.diag_const = sigma2;
    launch_gemm1(c, p);
  }
  // bring the s x s pieces to the host: H_finit (upper-triangular top of H_L), Mm, resinit
  double hHL[9], hMm[9], hres[3];
  int st;
  if ((st = stage_copy2d_out(c, hHL, s * sizeof(double), W, (size_t)ldW * sizeof(double), s * sizeof(double), s)) ||
      (st = stage_copy_out(c, hMm, dMm, s * s * sizeof(double))) || (st = stage_copy_out(c, hres, W + (size_t)(s + n) * ldW, s * sizeof(double))))
    return st;
  OVP_CUDA(cudaStreamSynchronize(c->stream));
  if (hl_is_upper) // called from initialize(): the reflectors annihilated the below-diagonal entries (the storage holds reflector data there);
    for (int j = 0; j < s; j++) // a direct ovp_initialize_invertible call hands over a general square H_L (StateHelper.cpp:564)
      for (int i = j + 1; i < s; i++)
        hHL[j * s + i] = 0.0;
  double Hinv[9];
  if (small_inverse(hHL, s, Hinv))
    return fail(c, OVP_ERR_BAD_ARGS, "initialize: H_L is singular");
  // symmetric Mm from its upper part (M.selfadjointView<Upper>, :566)
  for (int j = 0; j < s; j++)
    for (int i = j + 1; i < s; i++)
      hMm[j * s + i] = hMm[i * s + j];
  double T[9], PLL[9];
  for (int i = 0; i < s; i++)
    for (int j = 0; j < s; j++) {
      double v = 0;
      for (int k = 0; k < s; k++)
        v += Hinv[k * s + i] * hMm[j * s + k]; // (Hinv * Mm)(i,j)
      T[j * s + i] = v;
    }
  for (int i = 0; i < s; i++)
    for (int j = 0; j < s; j++) {
      double v = 0;
      for (int k = 0; k < s; k++)
        v += T[k * s + i] * Hinv[k * s + j]; // (T * Hinv^T)(i,j) = sum_k T(i,k) Hinv(j,k)
      PLL[j * s + i] = v;
    }
  double dxn[3];
  for (int i = 0; i < s; i++) {
    double v = 0;
    for (int k = 0; k < s; k++)
      v += Hinv[k * s + i] * hres[k];
    dxn[i] = v;
  }
  double *dsm = c->dscal + 32; // Hinv (9) + PLL (9)
  double pack[18];
  std::memcpy(pack, Hinv, sizeof(double) * 9);
  std::memcpy(pack + 9, PLL, sizeof(double) * 9);
  if ((st = stage_copy_in(c, dsm, pack, sizeof(pack))))
    return st;
  init_grow_kernel<<<((N + s) * s + 255) / 256, 256, 0, c->stream>>>(c->dP, c->ldP, N, s, c->dM, c->Nmax, dsm, dsm + 9);
  c->launches++;
  OVP_CUDA(cudaStreamSynchronize(c->stream));
  Var v;
  v.kind = kind;
  v.size = s;
  v.nvalue = s;
  v.tag = tag;
  double nv[3], nf[3];
  for (int i = 0; i < s; i++) {
    nv[i] = value[i] + dxn[i]; // new_variable->update(H_Linv * res), :577
    nf[i] = fej[i];
  }
  st = state_append_variable(c, v, nv, nf, new_handle);
  if (st)
    return st;
  register_new(c, *new_handle, kind, tag);
  return OVP_OK;
}

// shared front half of initialize / initialize_invertible: stage W = [H_L | H_R | res] on the device
static int stage_init_system(Ctx *c, const double *H_R, const double *H_L, const double *res, int rows, int n, int s, double **W) {
  const size_t col = (size_t)rows * sizeof(double);
  StageLayout L;
  const size_t b_W = L.take(col * (s + n + 1));
  int st = ensure_stage(c, L);
  if (st)
    return st;
  *W = (double *)(c->d_stage + b_W);
  if ((st = stage_copy_in(c, *W, H_L, col * s)) || (st = stage_copy_in(c, *W + (size_t)rows * s, H_R, col * n)) ||
      (st = stage_copy_in(c, *W + (size_t)rows * (s + n), res, col)))
    return st;
  return OVP_OK;
}

} // namespace ovp

extern "C" {

int ovp_ekf_update(ovp_ctx *h, const int *handles, int k, const double *H, int rows, const double *res, const double *Rdiag) {
  Ctx *c = ovp::enter(h);
  int n = 0;
  int st = upload_cols(c, handles, k, 0, &n);
  if (st)
    return st;
  if (rows <= 0 || n <= 0)
    return fail(c, OVP_ERR_BAD_ARGS, "ekf_update: empty system");
  if (rows > c->Rcap)
    return fail(c, OVP_ERR_CAPACITY, "ekf_update: %d rows exceed capacity %d (compress first, like the reference's callers)", rows, c->Rcap);
  const size_t col = (size_t)rows * sizeof(double);
  StageLayout L;
  const size_t b_H = L.take(col * n), b_res = L.take(col), b_R = L.take(col);
  if ((st = ensure_stage(c, L)))
    return st;
  double *dH = (double *)(c->d_stage + b_H), *dres = (double *)(c->d_stage + b_res), *dR = (double *)(c->d_stage + b_R);
  if ((st = stage_copy_in(c, dH, H, col * n)) || (st = stage_copy_in(c, dres, res, col)) || (Rdiag && (st = stage_copy_in(c, dR, Rdiag, col))))
    return st;
  st = ekf_update_core(c, c->dcols, n, mv(dH, rows, 1), rows, dres, Rdiag ? dR : nullptr, -1.0, nullptr, nullptr);
  if (st)
    return st;
  return check_status_flags(c);
}

int ovp_marginalize(ovp_ctx *h, int handle) { return do_marginalize(ovp::enter(h), handle); }

int ovp_clone(ovp_ctx *h, int handle, int *new_handle) {
  Ctx *c = ovp::enter(h);
  if (!valid_handle(c, handle) || c->vars[handle].id < 0)
    return fail(c, OVP_ERR_NOT_IN_STATE, "clone: variable %d not in the state (StateHelper.cpp:387-391)", handle);
  int st = sync_host_values(c);
  if (st)
    return st;
  Var v = c->vars[handle];
  const bool imu_pose = (v.kind == OVP_KIND_IMU); // the only sub-variable clone on the path: imu->pose() (StateHelper.cpp:598)
  if (imu_pose) {
    v.kind = OVP_KIND_POSE;
    v.size = 6;
    v.nvalue = 7;
  }
  if (c->N + v.size > c->Nmax)
    return fail(c, OVP_ERR_CAPACITY, "state capacity %d exceeded", c->Nmax);
  int old = c->vars[handle].id;
  v.id = -1;
  st = state_append_variable(c, v, &c->h_val[(size_t)handle * OVP_VAL_STRIDE], &c->h_fej[(size_t)handle * OVP_VAL_STRIDE], new_handle);
  if (st)
    return st;
  clone_kernel<<<((c->N + v.size) * v.size + 255) / 256, 256, 0, c->stream>>>(c->dP, c->ldP, c->N, old, v.size);
  c->launches++;
  c->vars[*new_handle].id = c->N;
  c->order.push_back(*new_handle);
  c->N += v.size;
  c->var_table_dirty = true;
  return OVP_OK;
}

int ovp_augment_clone(ovp_ctx *h, double timestamp, const double last_w[3], int *new_handle) {
  Ctx *c = ovp::enter(h);
  if (c->clones.count(timestamp))
    return fail(c, OVP_ERR_TIME, "augment_clone: a clone at this timestamp exists (StateHelper.cpp:591-594)");
  c->timestamp = timestamp;
  int nh = -1;
  int st = ovp_clone(h, c->h_imu, &nh);
  if (st)
    return st;
  c->clones[timestamp] = nh;
  if (c->opt.do_calib_camera_timeoffset) {
    double dnc[6] = {last_w[0], last_w[1], last_w[2], c->h_val[(size_t)c->h_imu * OVP_VAL_STRIDE + 7],
                     c->h_val[(size_t)c->h_imu * OVP_VAL_STRIDE + 8], c->h_val[(size_t)c->h_imu * OVP_VAL_STRIDE + 9]};
    double *dd = c->dscal + 64;
    if ((st = stage_copy_in(c, dd, dnc, sizeof(dnc))))
      return st;
    int rows = c->N, newid = c->vars[nh].id, dtid = c->vars[c->h_dt].id;
    dt_col_kernel<<<(rows * 6 + 255) / 256, 256, 0, c->stream>>>(c->dP, c->ldP, rows, newid, dtid, dd);
    dt_row_kernel<<<(rows * 6 + 255) / 256, 256, 0, c->stream>>>(c->dP, c->ldP, rows, newid, dtid, dd);
    c->launches += 2;
    OVP_CUDA(cudaStreamSynchronize(c->stream));
  }
  if (new_handle)
    *new_handle = nh;
  return OVP_OK;
}

int ovp_marginalize_old_clone(ovp_ctx *h) {
  Ctx *c = ovp::enter(h);
  if ((int)c->clones.size() > c->opt.max_clone_size) {
    int hh = c->clones.begin()->second; // State::margtimestep(): the oldest clone
    return do_marginalize(c, hh);
  }
  return OVP_OK;
}

int ovp_marginalize_slam(ovp_ctx *h) {
  Ctx *c = ovp::enter(h);
  std::vector<int> todo;
  for (auto &kv : c->slam)
    if (c->vars[kv.second].should_marg && (int)kv.first > 4 * c->opt.max_aruco_features)
      todo.push_back(kv.second);
  for (int hh : todo) {
    int st = do_marginalize(c, hh);
    if (st)
      return st;
  }
  return OVP_OK;
}

int ovp_initialize_invertible(ovp_ctx *h, int kind, int s, const double *value, const double *fej, int64_t tag, const int *handles, int k,
                              const double *H_R, const double *H_L, const double *res, double sigma2, int *new_handle) {
  Ctx *c = ovp::enter(h);
  if (s < 1 || s > 3)
    return fail(c, OVP_ERR_BAD_ARGS, "initialize_invertible: new variable size %d not in 1..3", s);
  if ((kind == OVP_KIND_LANDMARK && c->slam.count(tag)) || (kind == OVP_KIND_VEC && c->planes.count(tag)))
    return fail(c, OVP_ERR_ALREADY_IN_STATE, "initialize_invertible: variable already in the state (StateHelper.cpp:494-498)");
  int n = 0;
  int st = upload_cols(c, handles, k, 0, &n);
  if (st)
    return st;
  double *W;
  st = stage_init_system(c, H_R, H_L, res, s, n, s, &W);
  if (st)
    return st;
  return init_invertible_core(c, kind, s, value, fej, tag, c->dcols, n, W, s, sigma2, new_handle, false);
}

} // extern "C"

namespace ovp {
// StateHelper::initialize (StateHelper.cpp:398-487) on a device-staged system W = [H_L (s) | H_R (n) | res] with `rows` rows:
// s reflectors on H_L (Givens in the reference, :434-446; orthogonal-equivalent), chi2 of the updating portion against the
// CURRENT covariance with dof = dof_rows (the reference uses the full row count, :471-472), then initialize_invertible and the
// EKF update with the remaining rows.
int initialize_core(Ctx *c, int kind, int s, const double *value, const double *fej, int64_t tag, const int *d_cols, int n, double *W,
                    int ldW, int rows, int dof_rows, double sigma2, double chi2_mult, int do_update, int *accepted, int *new_handle) {
  *accepted = 0;
  *new_handle = -1;
  if (dof_rows >= c->chi2_table_n)
    return fail(c, OVP_ERR_BAD_ARGS, "initialize: chi2 table too short for %d rows", dof_rows);
  if (rows - s > c->Rcap)
    return fail(c, OVP_ERR_CAPACITY, "initialize: %d rows exceed capacity", rows);
  householder_cols_kernel<<<1, 256, 0, c->stream>>>(W, ldW, rows, s + n + 1, s);
  c->launches++;
  OVP_CUDA(cudaGetLastError());
  const int ru = rows - s;
  double *dR = c->dvec + 3 * (size_t)c->Rcap;
  MatView HupT = mv(W + (size_t)s * ldW + s, ldW, 1);
  const double *d_resup = W + (size_t)(s + n) * ldW + s;
  double chi2 = 0.0;
  if (ru > 0) {
    launch_fill(c, dR, ru, sigma2);
    int st = ekf_update_core(c, d_cols, n, HupT, ru, d_resup, dR, -1.0, nullptr, c->dscal, false); // dry run: chi2 only (:464-475)
    if (st)
      return st;
    if ((st = stage_copy_out(c, &chi2, c->dscal, sizeof(double))))
      return st;
    OVP_CUDA(cudaStreamSynchronize(c->stream));
  }
  int st = check_status_flags(c);
  if (st)
    return st;
  if (chi2 > chi2_mult * chi2_q95(c, dof_rows))
    return OVP_OK; // accepted = 0, state untouched
  st = init_invertible_core(c, kind, s, value, fej, tag, d_cols, n, W, ldW, sigma2, new_handle);
  if (st)
    return st;
  *accepted = 1;
  if (ru > 0 && do_update) {
    st = ekf_update_core(c, d_cols, n, HupT, ru, d_resup, dR, -1.0, nullptr, nullptr);
    if (st)
      return st;
    return check_status_flags(c);
  }
  return OVP_OK;
}
} // namespace ovp

extern "C" {

int ovp_initialize(ovp_ctx *h, int kind, int s, const double *value, const double *fej, int64_t tag, const int *handles, int k,
                   const double *H_R, const double *H_L, const double *res, int rows, double sigma2, double chi2_mult, int do_update,
                   int *accepted, int *new_handle) {
  Ctx *c = ovp::enter(h);
  *accepted = 0;
  *new_handle = -1;
  if (s < 1 || s > 3 || rows < s)
    return fail(c, OVP_ERR_BAD_ARGS, "initialize: bad sizes (s=%d rows=%d)", s, rows);
  if ((kind == OVP_KIND_LANDMARK && c->slam.count(tag)) || (kind == OVP_KIND_VEC && c->planes.count(tag)))
    return fail(c, OVP_ERR_ALREADY_IN_STATE, "initialize: variable already in the state (StateHelper.cpp:403-407)");
  int n = 0;
  int st = upload_cols(c, handles, k, 0, &n);
  if (st)
    return st;
  double *W;
  st = stage_init_system(c, H_R, H_L, res, rows, n, s, &W);
  if (st)
    return st;
  return initialize_core(c, kind, s, value, fej, tag, c->dcols, n, W, rows, rows, rows, sigma2, chi2_mult, do_update, accepted, new_handle);
}

} // extern "C"

namespace ovp {
// UpdaterPlane::init_vio_plane from "plane linearisation points known" on (UpdaterPlane.cpp:297-481): for every plane of the
// batch that is NOT in the state (ascending id, std::map order) and has >= 3 features: per-feature Jacobians with
// sigma_c * const_init_multi (:384), H_cp split off H_f (:388-390), left-nullspace projection, stacking, compression and
// StateHelper::initialize(plane Vec(3), ..., const_init_chi2) (:436-446).  plane_status[i]: 1 initialised, 0 chi2-rejected,
// -1 not attempted; new_handles[i]: handle of the new plane variable or -1.  Shared by ovp_plane_init and ovp_plane_init_tracks.
int plane_init_core(Ctx *c, const ovp_feature_batch *batch, const ovp_updater_options *opt, int *plane_status, int *new_handles) {
  std::vector<std::pair<int64_t, int>> ps;
  for (int i = 0; i < batch->nplanes; i++) {
    ps.push_back({batch->plane_ids[i], i});
    plane_status[i] = -1;
    new_handles[i] = -1;
  }
  std::sort(ps.begin(), ps.end());
  for (auto &pp : ps) {
    const int64_t pid = pp.first;
    if (pid == 0 || c->planes.count(pid))
      continue;
    int nf = 0;
    for (int f = 0; f < batch->F; f++)
      nf += batch->planeid[f] == pid;
    if (nf < 3)
      continue; // assert(features.size() >= 3), UpdaterPlane.cpp:303
    MsckfExtra ex;
    ex.only_plane_id = pid;
    ex.sigma_c_scale = c->opt.const_init_multi;
    int st = msckf_prepare(c, batch, opt, &ex);
    if (st)
      return st;
    const bool graphs_before = c->use_graphs;
    c->use_graphs = false; // one-shot system
    st = msckf_launch(c);
    c->use_graphs = graphs_before; // ovp_set_use_graphs(0) must survive this call
    if (st)
      return st;
    int rowsW, ncx, rows_ref;
    const int *d_cols;
    st = msckf_last_W(c, &rowsW, &ncx, &rows_ref, &d_cols);
    if (st)
      return st;
    if (rowsW < 3)
      continue;
    const double *cp = batch->plane_cp + 3 * pp.second;
    int acc = 0, nh = -1;
    st = initialize_core(c, OVP_KIND_VEC, 3, cp, cp, pid, d_cols, ncx, c->dHT, c->Rcap, rowsW, rows_ref, 1.0, c->opt.const_init_chi2, 1, &acc, &nh);
    if (st)
      return st;
    plane_status[pp.second] = acc;
    new_handles[pp.second] = nh;
  }
  return OVP_OK;
}
} // namespace ovp

extern "C" {

int ovp_plane_init(ovp_ctx *h, const ovp_feature_batch *batch, const ovp_updater_options *opt, int *plane_status, int *new_handles) {
  Ctx *c = ovp::enter(h);
  if (!batch || !opt || !batch->plane_cp || (batch->F > 0 && !batch->planeid))
    return fail(c, OVP_ERR_BAD_ARGS, "plane_init: null batch / options / plane_cp / planeid");
  return ovp::plane_init_core(c, batch, opt, plane_status, new_handles);
}

int ovp_merge_planes_and_marginalize(ovp_ctx *h, const int64_t *f2p_feat, const int64_t *f2p_plane, int nf, const int64_t *merge_new,
                                     const int64_t *merge_old, int nm) {
  Ctx *c = ovp::enter(h);
  (void)f2p_feat;
  if (c->planes.empty())
    return OVP_OK;
  if (3 >= c->chi2_table_n)
    return fail(c, OVP_ERR_BAD_ARGS, "chi2 table not set");
  // StateHelper.cpp:661-736
  std::vector<int64_t> ids;
  for (auto &kv : c->planes)
    ids.push_back(kv.first);
  for (int64_t planeid : ids) {
    if (!c->planes.count(planeid))
      continue;
    int64_t planeid_new = -1;
    bool in_state = false;
    for (int i = 0; i < nm; i++)
      if (merge_old[i] == planeid) {
        planeid_new = merge_new[i];
        in_state = c->planes.count(planeid_new) > 0;
      }
    if (planeid_new == -1 || planeid == planeid_new)
      continue;
    if (!in_state) {
      int hh = c->planes[planeid];
      c->planes.erase(planeid);
      c->planes[planeid_new] = hh;
      c->vars[hh].tag = planeid_new;
      continue;
    }
    int st = sync_host_values(c);
    if (st)
      return st;
    int hn = c->planes[planeid_new], ho = c->planes[planeid];
    const double *cpn = &c->h_val[(size_t)hn * OVP_VAL_STRIDE], *cpo = &c->h_val[(size_t)ho * OVP_VAL_STRIDE];
    double nn = std::sqrt(cpn[0] * cpn[0] + cpn[1] * cpn[1] + cpn[2] * cpn[2]);
    double no = std::sqrt(cpo[0] * cpo[0] + cpo[1] * cpo[1] + cpo[2] * cpo[2]);
    double norm_dist = (cpn[0] * cpo[0] + cpn[1] * cpo[1] + cpn[2] * cpo[2]) / (nn * no);
    double norm_angle = (180.0 / M_PI) * std::acos(norm_dist);
    double wc = 1.0 / c->opt.sigma_plane_merge;
    double res[3], H[18];
    std::memset(H, 0, sizeof(H));
    for (int i = 0; i < 3; i++) {
      res[i] = wc * (0.0 - (cpn[i] - cpo[i]));
      H[i * 3 + i] = wc;
      H[(3 + i) * 3 + i] = -wc;
    }
    int hs[2] = {hn, ho};
    double Pm[36];
    st = ovp_get_marginal_covariance(h, hs, 2, Pm);
    if (st)
      return st;
    // S = H P H^T + I (3x3), chi2 = res^T S^-1 res on the host (6x6 problem; the EKF update itself runs on the device)
    double HP[18], S[9];
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 6; j++) {
        double v = 0;
        for (int k2 = 0; k2 < 6; k2++)
          v += H[k2 * 3 + i] * Pm[j * 6 + k2];
        HP[j * 3 + i] = v;
      }
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) {
        double v = (i == j) ? 1.0 : 0.0;
        for (int k2 = 0; k2 < 6; k2++)
          v += HP[k2 * 3 + i] * H[k2 * 3 + j];
        S[j * 3 + i] = v;
      }
    double Sinv[9];
    if (small_inverse(S, 3, Sinv))
      return fail(c, OVP_ERR_NOT_POSITIVE_DEFINITE, "plane merge: singular S");
    double chi2 = 0;
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++)
        chi2 += res[i] * Sinv[j * 3 + i] * res[j];
    double chi2_check = c->opt.plane_merge_chi2 * chi2_q95(c, 3);
    if (chi2 < chi2_check && norm_angle < c->opt.plane_merge_deg_max) {
      st = ovp_ekf_update(h, hs, 2, H, 3, res, nullptr);
      if (st)
        return st;
    }
    st = do_marginalize(c, ho);
    if (st)
      return st;
  }
  // marginalise planes no active feature refers to (:738-757)
  std::set<int64_t> active;
  for (int i = 0; i < nf; i++)
    active.insert(f2p_plane[i]);
  ids.clear();
  for (auto &kv : c->planes)
    ids.push_back(kv.first);
  for (int64_t pid : ids)
    if (!active.count(pid)) {
      int st = do_marginalize(c, c->planes[pid]);
      if (st)
        return st;
    }
  return OVP_OK;
}

// ---- stateless helpers -----------------------------------------------------------------------------------------------
} // extern "C"
namespace ovp {
// get_feature_jacobian_full of ONE feature on the staging buffer, in the layout StateHelper::initialize wants:
// W = [H_f (rows x hfc) | H_x (rows x hxc) | res (rows)], leading dimension `rows`, then the measurements' uv.
struct FeatureJacobianStage {
  int rows, hfc, hxc;
  size_t b_W, b_uv; // byte offsets into c->d_stage
  double *W(const Ctx *c) const { return (double *)(c->d_stage + b_W); }
  double *Hx(const Ctx *c) const { return W(c) + (size_t)rows * hfc; }
  double *res(const Ctx *c) const { return W(c) + (size_t)rows * (hfc + hxc); }
};
// A track that is already on the device, in the staging buffer below stage_base: the Jacobian reads its clone handles and pixels there
// and lays its own slice out from stage_base up, so the track is neither copied again nor overwritten.
struct DeviceTrack {
  const int *clone;
  const float *uv;
  size_t stage_base;
};
// The one track of get_feature_jacobian_full: 1..64 measurements (a size argument, not a track a feature kernel holds, so a longer one is a
// bad argument), each from a live pose with or without covariance columns, observed once.
static int check_jacobian_track(Ctx *c, const char *who, int m, const int *clone_handles) {
  const int off[2] = {0, m};
  return check_tracks(c, who, 1, off, clone_handles, nullptr, 1, 64, OVP_ERR_BAD_ARGS, false, true);
}
// plane_handle >= 0: plane in the state (its values come from the device tables); otherwise cp / cp_fej (may be null: no plane).
// dev (may be null): clone_handles / uv are also resident on the device there; clone_handles is still read on the host (columns).  The
// caller has checked the track (check_jacobian_track or its own check_tracks).
static int stage_feature_jacobian(Ctx *c, int m, const int *clone_handles, const float *uv, const double *p_FinG, const double *p_FinG_fej,
                                  bool has_plane, int plane_handle, const double *cp, const double *cp_fej, double sigma_px, double sigma_c,
                                  FeatureJacobianStage *j, int extra_hx_cols = 0, const DeviceTrack *dev = nullptr) {
  int st;
  const bool in_state = has_plane && plane_handle >= 0;
  const int ncal = (c->opt.do_calib_camera_pose ? 6 : 0) + (c->opt.do_calib_camera_intrinsics ? 8 : 0);
  const int rows = has_plane ? 3 * m : 2 * m;
  const int hfc = 3 + ((has_plane && !in_state) ? 3 : 0);
  const int hxc = ncal + 6 * m + (in_state ? 3 : 0) + extra_hx_cols; // extra: zero columns appended for an anchor clone (anchors.cu)
  const size_t w_bytes = (size_t)rows * (hfc + hxc + 1) * sizeof(double), uv_bytes = (size_t)m * 2 * sizeof(float);
  StageLayout L;
  L.top = dev ? dev->stage_base : 0;
  const size_t b_W = L.take(w_bytes);
  *j = {rows, hfc, hxc, b_W, dev ? 0 : L.take(uv_bytes)};
  if (dev && L.top > c->d_stage_bytes) // growing the buffer would drop the resident track: the caller reserves this slice
    return fail(c, OVP_ERR_CAPACITY, "feature_jacobian_full: %zu staging bytes needed above the resident tracks, %zu reserved", L.top,
                c->d_stage_bytes);
  if ((st = ensure_stage(c, L)))
    return st;
  OVP_CUDA(cudaMemsetAsync(j->W(c), 0, w_bytes, c->stream));
  JacArgs a;
  a.m = m;
  if (dev) {
    a.clone_handles = dev->clone;
    a.uv = dev->uv;
  } else {
    int *dcl = c->dcols + (size_t)4 * c->Rcap;
    float *duv = (float *)(c->d_stage + j->b_uv);
    if ((st = stage_copy_in(c, dcl, clone_handles, m * sizeof(int))) || (st = stage_copy_in(c, duv, uv, uv_bytes)))
      return st;
    a.clone_handles = dcl;
    a.uv = duv;
  }
  for (int i = 0; i < 3; i++) {
    a.pf[i] = p_FinG[i];
    a.pf_fej[i] = p_FinG_fej[i];
    a.cp[i] = (has_plane && cp) ? cp[i] : 0.0;
    a.cp_fej[i] = (has_plane && cp_fej) ? cp_fej[i] : 0.0;
  }
  a.has_plane = has_plane;
  a.plane_in_state = in_state;
  a.plane_handle = (in_state && !cp) ? plane_handle : -1;
  a.val = c->d_val;
  a.fej = c->d_fej;
  a.h_calib = c->h_calib;
  a.h_intr = c->h_intr;
  a.do_fej = c->opt.do_fej;
  a.do_calib_pose = c->opt.do_calib_camera_pose;
  a.do_calib_intr = c->opt.do_calib_camera_intrinsics;
  a.white_px = 1.0 / sigma_px;
  a.white_c = 1.0 / sigma_c;
  a.Hf = j->W(c);
  a.Hx = j->Hx(c);
  a.res = j->res(c);
  a.rows = rows;
  a.hf_cols = hfc;
  a.hx_cols = hxc;
  jacobian_only_kernel<<<1, 64, 0, c->stream>>>(a);
  c->launches++;
  return OVP_OK;
}
// the first hf_cols columns of H_f, then H_x and res of a staged feature Jacobian, to the host
static int read_feature_jacobian(Ctx *c, const FeatureJacobianStage &j, int hf_cols, double *H_f, double *H_x, double *res) {
  const size_t col = (size_t)j.rows * sizeof(double);
  int st;
  if ((st = stage_copy_out(c, H_f, j.W(c), col * hf_cols)) || (st = stage_copy_out(c, H_x, j.Hx(c), col * j.hxc)) ||
      (st = stage_copy_out(c, res, j.res(c), col)))
    return st;
  OVP_CUDA(cudaStreamSynchronize(c->stream));
  return OVP_OK;
}
} // namespace ovp
extern "C" {

// UpdaterHelper::get_feature_jacobian_representation (UpdaterHelper.cpp:35-193) as a context-free helper (3x3 host algebra, no
// device work): d p_FinG / d lambda for the six ov_type landmark representations and, for the anchored ones, the Jacobians
// w.r.t. the anchor clone and the camera extrinsics.  The fused device path itself runs GLOBAL_3D (every shipped config).
int ovp_feature_jacobian_representation(int representation, int do_fej, const double *p_FinG, const double *p_FinG_fej, const double *p_FinA,
                                        const double *anchor_pose7, const double *anchor_pose_fej7, const double *calib7, double *H_f,
                                        int *hf_cols, double *H_anc, double *H_calib, int *has_anchor) {
  using namespace ovp::hm;
  if (representation < 0 || representation > 5 || !H_f || !hf_cols || !has_anchor)
    return OVP_ERR_BAD_ARGS;
  auto put3 = [](double *dst, int ldrows, int c0, const M3 &B) { // column-major 3 x n target
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++)
        dst[(size_t)(c0 + j) * ldrows + i] = B(i, j);
  };
  // d p / d (theta, phi, rho) of p = (1 / rho) [cos(theta) sin(phi), sin(theta) sin(phi), cos(phi)] evaluated at p
  auto d_spherical = [](const V3 &p) {
    const double r = std::sqrt(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]);
    const double rho = 1.0 / r, phi = std::acos(rho * p[2]), th = std::atan2(p[1], p[0]);
    const double st = std::sin(th), ct = std::cos(th), sp = std::sin(phi), cp = std::cos(phi), ir = 1.0 / rho, ir2 = 1.0 / (rho * rho);
    return M3{{-ir * st * sp, ir * ct * cp, -ir2 * ct * sp, ir * ct * sp, ir * st * cp, -ir2 * st * sp, 0.0, -ir * sp, -ir2 * cp}};
  };
  *has_anchor = 0;
  *hf_cols = 3;
  if (representation == 0) {
    put3(H_f, 3, 0, eye3());
    return OVP_OK;
  }
  if (representation == 1) {
    const double *p = do_fej ? p_FinG_fej : p_FinG;
    put3(H_f, 3, 0, d_spherical(v3(p[0], p[1], p[2])));
    return OVP_OK;
  }
  if (!p_FinA || !anchor_pose7 || !anchor_pose_fej7 || !calib7 || !H_anc || !H_calib)
    return OVP_ERR_BAD_ARGS;
  const M3 R_ItoC = quat_2_Rot(V4{{calib7[0], calib7[1], calib7[2], calib7[3]}});
  const V3 p_IinC = v3(calib7[4], calib7[5], calib7[6]);
  M3 R_GtoI = quat_2_Rot(V4{{anchor_pose7[0], anchor_pose7[1], anchor_pose7[2], anchor_pose7[3]}});
  V3 p_IinG = v3(anchor_pose7[4], anchor_pose7[5], anchor_pose7[6]);
  V3 pA = v3(p_FinA[0], p_FinA[1], p_FinA[2]);
  if (do_fej) { // the best global estimate seen from the first-estimate anchor frame
    const V3 best = transpose(R_GtoI) * (transpose(R_ItoC) * (pA - p_IinC)) + p_IinG;
    R_GtoI = quat_2_Rot(V4{{anchor_pose_fej7[0], anchor_pose_fej7[1], anchor_pose_fej7[2], anchor_pose_fej7[3]}});
    p_IinG = v3(anchor_pose_fej7[4], anchor_pose_fej7[5], anchor_pose_fej7[6]);
    pA = R_ItoC * (R_GtoI * (best - p_IinG)) + p_IinC;
  }
  const M3 R_ItoG = transpose(R_GtoI), R_CtoG = R_ItoG * transpose(R_ItoC);
  const V3 dA = pA - p_IinC;
  put3(H_anc, 3, 0, (-1.0) * (R_ItoG * skew(transpose(R_ItoC) * dA)));
  put3(H_anc, 3, 3, eye3());
  put3(H_calib, 3, 0, (-1.0) * (R_CtoG * skew(dA)));
  put3(H_calib, 3, 3, (-1.0) * R_CtoG);
  *has_anchor = 1;
  if (representation == 2) {
    put3(H_f, 3, 0, R_CtoG);
  } else if (representation == 3) {
    put3(H_f, 3, 0, R_CtoG * d_spherical(pA));
  } else if (representation == 4) { // lambda = (x/z, y/z, 1/z)
    const double rho = 1.0 / pA[2], al = pA[0] / pA[2], be = pA[1] / pA[2], ir = 1.0 / rho, ir2 = 1.0 / (rho * rho);
    put3(H_f, 3, 0, R_CtoG * M3{{ir, 0.0, -ir2 * al, 0.0, ir, -ir2 * be, 0.0, 0.0, -ir2}});
  } else { // lambda = 1/z along the fixed initial bearing
    const double rho = 1.0 / pA[2];
    const V3 d = R_CtoG * ((-(1.0 / (rho * rho))) * (rho * pA));
    for (int i = 0; i < 3; i++)
      H_f[i] = d[i];
    *hf_cols = 1;
  }
  return OVP_OK;
}

int ovp_feature_jacobian_full(ovp_ctx *h, int m, const int *clone_handles, const float *uv, const double *p_FinG, const double *p_FinG_fej,
                              int64_t planeid, const double *cp, const double *cp_fej, double sigma_px, double sigma_c, double *H_f,
                              int *hf_cols, double *H_x, int *hx_cols, double *res, int *rows_out, int *x_order, int *x_order_n) {
  Ctx *c = ovp::enter(h);
  int st = check_jacobian_track(c, "feature_jacobian_full", m, clone_handles);
  if (st)
    return st;
  const bool has_plane = planeid != 0;
  const bool in_state = has_plane && c->planes.count(planeid);
  FeatureJacobianStage j;
  st = stage_feature_jacobian(c, m, clone_handles, uv, p_FinG, p_FinG_fej, has_plane, in_state ? c->planes[planeid] : -1, cp, cp_fej,
                              sigma_px, sigma_c, &j);
  if (st || (st = read_feature_jacobian(c, j, j.hfc, H_f, H_x, res)))
    return st;
  *hf_cols = j.hfc;
  *hx_cols = j.hxc;
  *rows_out = j.rows;
  int no = 0;
  if (c->opt.do_calib_camera_pose)
    x_order[no++] = c->h_calib;
  if (c->opt.do_calib_camera_intrinsics)
    x_order[no++] = c->h_intr;
  for (int i = 0; i < m; i++)
    x_order[no++] = clone_handles[i];
  if (in_state)
    x_order[no++] = c->planes[planeid];
  *x_order_n = no;
  return OVP_OK;
}

static int nullspace_common(Ctx *c, double *H_f, int hf_cols, double *H_x, int hx_cols, double *H_cp, double *res, int rows, int *rows_out) {
  if (rows < hf_cols || hf_cols < 1)
    return fail(c, OVP_ERR_BAD_ARGS, "nullspace_project: need rows >= H_f.cols() (assert, UpdaterHelper.cpp:518)");
  int ncp = H_cp ? 3 : 0;
  int ncols = hf_cols + hx_cols + ncp + 1;
  // W = [H_f | H_x | H_cp | res], leading dimension rows
  const size_t col = (size_t)rows * sizeof(double);
  StageLayout L;
  const size_t b_W = L.take(col * ncols);
  int st = ensure_stage(c, L);
  if (st)
    return st;
  double *W = (double *)(c->d_stage + b_W), *Wx = W + (size_t)rows * hf_cols, *Wcp = Wx + (size_t)rows * hx_cols, *Wres = Wcp + (size_t)rows * ncp;
  if ((st = stage_copy_in(c, W, H_f, col * hf_cols)) || (st = stage_copy_in(c, Wx, H_x, col * hx_cols)) ||
      (H_cp && (st = stage_copy_in(c, Wcp, H_cp, col * 3))) || (st = stage_copy_in(c, Wres, res, col)))
    return st;
  householder_cols_kernel<<<1, 256, 0, c->stream>>>(W, rows, rows, ncols, hf_cols);
  c->launches++;
  OVP_CUDA(cudaGetLastError());
  int ro = rows - hf_cols;
  // copy back rows [hf_cols, rows) compacted to ld = ro (none when H_f is square)
  const size_t rcol = (size_t)ro * sizeof(double);
  if ((st = stage_copy2d_out(c, H_x, rcol, Wx + hf_cols, col, rcol, hx_cols)) ||
      (H_cp && (st = stage_copy2d_out(c, H_cp, rcol, Wcp + hf_cols, col, rcol, 3))) || (st = stage_copy_out(c, res, Wres + hf_cols, rcol)))
    return st;
  OVP_CUDA(cudaStreamSynchronize(c->stream));
  *rows_out = ro;
  return OVP_OK;
}
int ovp_nullspace_project_inplace(ovp_ctx *h, double *H_f, int hf_cols, double *H_x, int hx_cols, double *res, int rows, int *rows_out) {
  return nullspace_common(ovp::enter(h), H_f, hf_cols, H_x, hx_cols, nullptr, res, rows, rows_out);
}
int ovp_plane_nullspace_project_inplace(ovp_ctx *h, double *H_f, int hf_cols, double *H_x, int hx_cols, double *H_cp, double *res, int rows,
                                        int *rows_out) {
  return nullspace_common(ovp::enter(h), H_f, hf_cols, H_x, hx_cols, H_cp, res, rows, rows_out);
}

static int compress_common(Ctx *c, double *H_x, int cols, double *H_cp, double *res, int rows, int *rows_out) {
  *rows_out = rows;
  if (rows <= cols)
    return OVP_OK; // fat matrix: nothing to do (UpdaterHelper.cpp:551-552)
  int ncp = H_cp ? 3 : 0;
  int nc1 = cols + ncp + 1;
  if (nc1 > c->Rcap)
    return fail(c, OVP_ERR_CAPACITY, "measurement_compress: %d columns exceed capacity %d", nc1, c->Rcap);
  if (rows > c->max_meas_rows)
    return fail(c, OVP_ERR_CAPACITY, "measurement_compress: %d rows exceed capacity %d", rows, c->max_meas_rows);
  int ld = (rows + 7) & ~7;
  launch_fill(c, c->dHs, (size_t)ld * nc1, 0.0);
  const size_t col = (size_t)rows * sizeof(double), dcol = (size_t)ld * sizeof(double); // stacked [H_x | H_cp | res], leading dimension ld
  int st;
  if ((st = stage_copy2d_in(c, c->dHs, dcol, H_x, col, col, cols)) ||
      (H_cp && (st = stage_copy2d_in(c, c->dHs + (size_t)ld * cols, dcol, H_cp, col, col, 3))) ||
      (st = stage_copy_in(c, c->dHs + (size_t)ld * (cols + ncp), res, col)) || (st = gram_of_stacked(c, rows, nc1, ld)))
    return st;
  st = chol_partial(c, c->wsG.S, c->wsG.cap, nc1, cols, c->gram_tol);
  if (st)
    return st;
  // R = L[0:cols,0:cols]^T ; carried columns = L[cols.., 0:cols]^T
  std::vector<double> L((size_t)nc1 * cols);
  if ((st = stage_copy2d_out(c, L.data(), (size_t)nc1 * sizeof(double), c->wsG.S, (size_t)c->wsG.cap * sizeof(double), (size_t)nc1 * sizeof(double),
                             cols)))
    return st;
  OVP_CUDA(cudaStreamSynchronize(c->stream));
  const int r = cols; // min(rows, cols)
  for (int j = 0; j < cols; j++)
    for (int i = 0; i < r; i++)
      H_x[(size_t)j * r + i] = (i <= j) ? L[(size_t)i * nc1 + j] : 0.0;
  if (H_cp)
    for (int j = 0; j < 3; j++)
      for (int i = 0; i < r; i++)
        H_cp[(size_t)j * r + i] = L[(size_t)i * nc1 + cols + j];
  for (int i = 0; i < r; i++)
    res[i] = L[(size_t)i * nc1 + cols + ncp];
  *rows_out = r;
  return OVP_OK;
}
int ovp_measurement_compress_inplace(ovp_ctx *h, double *H_x, int cols, double *res, int rows, int *rows_out) {
  return compress_common(ovp::enter(h), H_x, cols, nullptr, res, rows, rows_out);
}
int ovp_plane_measurement_compress_inplace(ovp_ctx *h, double *H_x, int cols, double *H_cp, double *res, int rows, int *rows_out) {
  return compress_common(ovp::enter(h), H_x, cols, H_cp, res, rows, rows_out);
}

// ---- UpdaterMSCKF ------------------------------------------------------------------------------------------------------
// an empty landmark list is the plain update (same plan, same key)
static const MsckfExtra *landmark_extra(const ovp_plane_landmarks *lm, MsckfExtra &ex) {
  if (!lm || lm->n == 0)
    return nullptr;
  ex.landmarks = lm;
  return &ex;
}
int ovp_msckf_update_landmarks(ovp_ctx *h, const ovp_feature_batch *batch, const ovp_plane_landmarks *landmarks, const ovp_updater_options *opt,
                               int *feat_status, double *feat_chi2, int *plane_status, double *plane_chi2, int *hx_order, int *hx_order_n) {
  Ctx *c = ovp::enter(h);
  if (!batch || !opt)
    return fail(c, OVP_ERR_BAD_ARGS, "null batch / options");
  MsckfExtra ex;
  return msckf_update_impl(c, batch, opt, feat_status, feat_chi2, plane_status, plane_chi2, hx_order, hx_order_n, landmark_extra(landmarks, ex));
}
int ovp_msckf_update(ovp_ctx *h, const ovp_feature_batch *batch, const ovp_updater_options *opt, int *feat_status, double *feat_chi2,
                     int *plane_status, double *plane_chi2, int *hx_order, int *hx_order_n) {
  return ovp_msckf_update_landmarks(h, batch, nullptr, opt, feat_status, feat_chi2, plane_status, plane_chi2, hx_order, hx_order_n);
}

static int shard_cols(Ctx *c, const int *all_clone_handles, int n_clones, std::vector<int> &cols) {
  std::vector<std::pair<int, int>> clones;
  for (int i = 0; i < n_clones; i++) {
    int hh = all_clone_handles[i];
    if (!is_clone(c, hh, true))
      return fail(c, OVP_ERR_BAD_ARGS, "shard: handle %d is not a clone in the state", hh);
    clones.push_back({c->vars[hh].id, 6});
  }
  cols = compact_cols(c, std::move(clones));
  return OVP_OK;
}
int ovp_msckf_shard_columns(ovp_ctx *h, const int *all_clone_handles, int n_clones, int *n_cols) {
  std::vector<int> cols;
  int st = shard_cols(&h->c, all_clone_handles, n_clones, cols);
  if (st)
    return st;
  *n_cols = (int)cols.size();
  return OVP_OK;
}
int ovp_msckf_shard_compress(ovp_ctx *h, const ovp_feature_batch *batch, const ovp_updater_options *opt, const int *all_clone_handles,
                             int n_clones, double *d_out, int *feat_status, double *feat_chi2) {
  Ctx *c = ovp::enter(h);
  std::vector<int> cols;
  int st = shard_cols(c, all_clone_handles, n_clones, cols);
  if (st)
    return st;
  MsckfExtra ex;
  ex.forced_cols = &cols;
  ex.d_export = d_out;
  if (batch->F == 0) {
    size_t n1 = cols.size() + 1;
    OVP_CUDA(cudaMemsetAsync(d_out, 0, n1 * n1 * sizeof(double), c->stream));
    OVP_CUDA(cudaStreamSynchronize(c->stream));
    return OVP_OK;
  }
  return msckf_update_impl(c, batch, opt, feat_status, feat_chi2, nullptr, nullptr, nullptr, nullptr, &ex);
}
int ovp_msckf_update_gathered(ovp_ctx *h, const double *d_blocks, int G, const int *all_clone_handles, int n_clones) {
  Ctx *c = ovp::enter(h);
  std::vector<int> cols;
  int st = shard_cols(c, all_clone_handles, n_clones, cols);
  if (st)
    return st;
  const int n = (int)cols.size();
  const int rows = G * n, nc1 = n + 1;
  if (rows > c->max_meas_rows || nc1 > c->Rcap)
    return fail(c, OVP_ERR_CAPACITY, "gathered system %d x %d exceeds capacity", rows, nc1);
  if ((st = stage_copy_in(c, c->dcols, cols.data(), n * sizeof(int))))
    return st;
  int ld = (rows + 7) & ~7;
  launch_fill(c, c->dHs, (size_t)ld * nc1, 0.0);
  transpose_stack_kernel<<<c->num_sms * 4, 256, 0, c->stream>>>(d_blocks, G, n, c->dHs, ld);
  c->launches++;
  st = gram_of_stacked(c, rows, nc1, ld);
  if (st)
    return st;
  st = gram_factor_update(c, c->dcols, n, n, c->gram_tol, -1.0, nullptr, nullptr, false);
  if (st)
    return st;
  return check_status_flags(c);
}

} // extern "C"
#include "capi_nccl.inc"
extern "C" {

// ---- Propagator ----------------------------------------------------------------------------------------------------------
int ovp_propagator_set_noise(ovp_ctx *h, double sigma_w, double sigma_wb, double sigma_a, double sigma_ab, double gravity_mag) {
  Ctx *c = ovp::enter(h);
  c->sigma_w = sigma_w;
  c->sigma_wb = sigma_wb;
  c->sigma_a = sigma_a;
  c->sigma_ab = sigma_ab;
  c->gravity[0] = 0;
  c->gravity[1] = 0;
  c->gravity[2] = gravity_mag;
  return OVP_OK;
}
int ovp_propagator_feed_imu(ovp_ctx *h, double timestamp, const double wm[3], const double am[3]) {
  ImuSample s;
  s.t = timestamp;
  for (int i = 0; i < 3; i++) {
    s.wm[i] = wm[i];
    s.am[i] = am[i];
  }
  h->c.imu_data.push_back(s);
  return OVP_OK;
}

} // extern "C"

namespace ovp {
using namespace hm;

static ImuSample interpolate_data(const ImuSample &a, const ImuSample &b, double t) { // Propagator.h:146-156
  double lambda = (t - a.t) / (b.t - a.t);
  ImuSample d;
  d.t = t;
  for (int i = 0; i < 3; i++) {
    d.am[i] = (1 - lambda) * a.am[i] + lambda * b.am[i];
    d.wm[i] = (1 - lambda) * a.wm[i] + lambda * b.wm[i];
  }
  return d;
}
static std::vector<ImuSample> select_imu_readings(const std::vector<ImuSample> &imu, double time0, double time1) { // Propagator.cpp:226-341
  std::vector<ImuSample> prop;
  if (imu.empty())
    return prop;
  for (size_t i = 0; i + 1 < imu.size(); i++) {
    if (imu[i + 1].t > time0 && imu[i].t < time0) {
      prop.push_back(interpolate_data(imu[i], imu[i + 1], time0));
      continue;
    }
    if (imu[i].t >= time0 && imu[i + 1].t <= time1) {
      prop.push_back(imu[i]);
      continue;
    }
    if (imu[i + 1].t > time1) {
      if (imu[i].t > time1 && i == 0) {
        break;
      } else if (imu[i].t > time1) {
        prop.push_back(interpolate_data(imu[i - 1], imu[i], time1));
      } else {
        prop.push_back(imu[i]);
      }
      if (prop.back().t != time1)
        prop.push_back(interpolate_data(imu[i], imu[i + 1], time1));
      break;
    }
  }
  if (prop.empty())
    return prop;
  for (size_t i = 0; i + 1 < prop.size(); i++)
    if (std::abs(prop[i + 1].t - prop[i].t) < 1e-12) {
      prop.erase(prop.begin() + i);
      i--;
    }
  return prop;
}

struct ImuMean {
  V4 q;
  V3 p, v, bg, ba;
};

// Propagator.cpp:490-569
static void predict_mean_rk4(const ImuMean &x, const V3 &g, double dt, const V3 &w1, const V3 &a1, const V3 &w2, const V3 &a2, V4 &nq, V3 &nv,
                             V3 &np) {
  V3 w_hat = w1, a_hat = a1;
  V3 w_alpha = (1.0 / dt) * (w2 - w1);
  V3 a_jerk = (1.0 / dt) * (a2 - a1);
  V4 q_0 = x.q;
  V3 p_0 = x.p, v_0 = x.v;
  V4 dq_0{{0, 0, 0, 1}};
  auto add4 = [](const V4 &a, double s, const V4 &b) { return V4{{a[0] + s * b[0], a[1] + s * b[1], a[2] + s * b[2], a[3] + s * b[3]}}; };
  V4 q0_dot = half_omega_times(w_hat, dq_0);
  V3 p0_dot = v_0;
  M3 R0 = quat_2_Rot(quat_multiply(dq_0, q_0));
  V3 v0_dot = transpose(R0) * a_hat - g;
  V4 k1_q{{dt * q0_dot[0], dt * q0_dot[1], dt * q0_dot[2], dt * q0_dot[3]}};
  V3 k1_p = dt * p0_dot, k1_v = dt * v0_dot;
  w_hat = w_hat + (0.5 * dt) * w_alpha;
  a_hat = a_hat + (0.5 * dt) * a_jerk;
  V4 dq_1 = quatnorm(add4(dq_0, 0.5, k1_q));
  V3 v_1 = v_0 + 0.5 * k1_v;
  V4 q1_dot = half_omega_times(w_hat, dq_1);
  M3 R1 = quat_2_Rot(quat_multiply(dq_1, q_0));
  V3 v1_dot = transpose(R1) * a_hat - g;
  V4 k2_q{{dt * q1_dot[0], dt * q1_dot[1], dt * q1_dot[2], dt * q1_dot[3]}};
  V3 k2_p = dt * v_1, k2_v = dt * v1_dot;
  V4 dq_2 = quatnorm(add4(dq_0, 0.5, k2_q));
  V3 v_2 = v_0 + 0.5 * k2_v;
  V4 q2_dot = half_omega_times(w_hat, dq_2);
  M3 R2 = quat_2_Rot(quat_multiply(dq_2, q_0));
  V3 v2_dot = transpose(R2) * a_hat - g;
  V4 k3_q{{dt * q2_dot[0], dt * q2_dot[1], dt * q2_dot[2], dt * q2_dot[3]}};
  V3 k3_p = dt * v_2, k3_v = dt * v2_dot;
  w_hat = w_hat + (0.5 * dt) * w_alpha;
  a_hat = a_hat + (0.5 * dt) * a_jerk;
  V4 dq_3 = quatnorm(add4(dq_0, 1.0, k3_q));
  V3 v_3 = v_0 + k3_v;
  V4 q3_dot = half_omega_times(w_hat, dq_3);
  M3 R3 = quat_2_Rot(quat_multiply(dq_3, q_0));
  V3 v3_dot = transpose(R3) * a_hat - g;
  V4 k4_q{{dt * q3_dot[0], dt * q3_dot[1], dt * q3_dot[2], dt * q3_dot[3]}};
  V3 k4_p = dt * v_3, k4_v = dt * v3_dot;
  V4 s = dq_0;
  s = add4(s, 1.0 / 6.0, k1_q);
  s = add4(s, 1.0 / 3.0, k2_q);
  s = add4(s, 1.0 / 3.0, k3_q);
  s = add4(s, 1.0 / 6.0, k4_q);
  V4 dq = quatnorm(s);
  nq = quat_multiply(dq, q_0);
  np = p_0 + (1.0 / 6.0) * k1_p + (1.0 / 3.0) * k2_p + (1.0 / 3.0) * k3_p + (1.0 / 6.0) * k4_p;
  nv = v_0 + (1.0 / 6.0) * k1_v + (1.0 / 3.0) * k2_v + (1.0 / 3.0) * k3_v + (1.0 / 6.0) * k4_v;
}
// Propagator.cpp:456-488
static void predict_mean_discrete(const ImuMean &x, const V3 &g, bool imu_avg, double dt, const V3 &w1, const V3 &a1, const V3 &w2, const V3 &a2,
                                  V4 &nq, V3 &nv, V3 &np) {
  V3 w_hat = w1, a_hat = a1;
  if (imu_avg) {
    w_hat = 0.5 * (w1 + w2);
    a_hat = 0.5 * (a1 + a2);
  }
  double w_norm = norm(w_hat);
  M3 R = quat_2_Rot(x.q);
  V4 ho = half_omega_times(w_hat, x.q); // 0.5 * Omega(w) q
  V4 q;
  if (w_norm > 1e-20) {
    double cs = std::cos(0.5 * w_norm * dt), sn = (1 / w_norm) * std::sin(0.5 * w_norm * dt);
    for (int i = 0; i < 4; i++)
      q[i] = cs * x.q[i] + sn * 2.0 * ho[i];
  } else {
    for (int i = 0; i < 4; i++)
      q[i] = x.q[i] + dt * ho[i];
  }
  nq = quatnorm(q);
  nv = x.v + dt * (transpose(R) * a_hat) - dt * g;
  np = x.p + dt * x.v + (0.5 * dt * dt) * (transpose(R) * a_hat) - (0.5 * dt * dt) * g;
}

} // namespace ovp

extern "C" {

// Propagator::fast_state_propagate (Propagator.cpp:128-224): IMU-rate odometry prediction on a COPY of the IMU marginal (15 x 15
// read back from the device covariance); nothing in the state changes.  state_plus = [q(4) p(3) v_local(3) w(3)], covariance 12 x 12
// (column-major) over [theta p v_local w].  *ok = 0 when fewer than two IMU samples cover the interval (:147-148).
int ovp_fast_state_propagate(ovp_ctx *h, double timestamp, double *state_plus13, double *cov144, int *ok) {
  using namespace ovp::hm;
  Ctx *c = ovp::enter(h);
  *ok = 0;
  int st = sync_host_values(c);
  if (st)
    return st;
  const double *iv = &c->h_val[(size_t)c->h_imu * OVP_VAL_STRIDE];
  const double t_off = c->h_val[(size_t)c->h_dt * OVP_VAL_STRIDE];
  double P15[225];
  st = ovp_get_marginal_covariance(h, &c->h_imu, 1, P15); // column-major, symmetric
  if (st)
    return st;
  std::vector<ImuSample> prop = select_imu_readings(c->imu_data, c->timestamp + t_off, timestamp + t_off);
  if (prop.size() < 2)
    return OVP_OK;
  M15 cov;
  for (int i = 0; i < 15; i++)
    for (int j = 0; j < 15; j++)
      cov(i, j) = P15[15 * j + i];
  V4 q = {{iv[0], iv[1], iv[2], iv[3]}};
  V3 p = v3(iv[4], iv[5], iv[6]), v = v3(iv[7], iv[8], iv[9]);
  const V3 bg = v3(iv[10], iv[11], iv[12]), ba = v3(iv[13], iv[14], iv[15]);
  const V3 g = v3(c->gravity[0], c->gravity[1], c->gravity[2]);
  const M3 I3 = eye3();
  auto smp = [](const double *x) { return v3(x[0], x[1], x[2]); };
  for (size_t i = 0; i + 1 < prop.size(); i++) {
    const double dt = prop[i + 1].t - prop[i].t;
    const V3 w_hat = 0.5 * (smp(prop[i + 1].wm) + smp(prop[i].wm)) - bg, a_hat = 0.5 * (smp(prop[i + 1].am) + smp(prop[i].am)) - ba;
    const M3 R = quat_2_Rot(q), RT = transpose(R);
    const M3 E = exp_so3((-dt) * w_hat), EJ = (-dt) * (E * Jr_so3((-dt) * w_hat));
    M15 F;
    double G[15][12];
    std::memset(G, 0, sizeof(G));
    auto setG = [&](int i0, int j0, const M3 &B) {
      for (int a = 0; a < 3; a++)
        for (int b = 0; b < 3; b++)
          G[i0 + a][j0 + b] = B(a, b);
    };
    F.setBlock3(0, 0, E);
    F.setBlock3(0, 9, EJ);
    F.setBlock3(9, 9, I3);
    F.setBlock3(6, 0, (-1.0) * (RT * skew(dt * a_hat)));
    F.setBlock3(6, 6, I3);
    F.setBlock3(6, 12, (-dt) * RT);
    F.setBlock3(12, 12, I3);
    F.setBlock3(3, 0, (-0.5) * (RT * skew((dt * dt) * a_hat)));
    F.setBlock3(3, 6, dt * I3);
    F.setBlock3(3, 12, (-0.5 * dt * dt) * RT);
    F.setBlock3(3, 3, I3);
    setG(0, 0, EJ);
    setG(6, 3, (-dt) * RT);
    setG(3, 3, (-0.5 * dt * dt) * RT);
    setG(9, 6, I3);
    setG(12, 9, I3);
    double qc[12];
    for (int k = 0; k < 3; k++) {
      qc[k] = c->sigma_w * c->sigma_w / dt;
      qc[3 + k] = c->sigma_a * c->sigma_a / dt;
      qc[6 + k] = c->sigma_wb * c->sigma_wb * dt;
      qc[9 + k] = c->sigma_ab * c->sigma_ab * dt;
    }
    M15 Qd;
    for (int a = 0; a < 15; a++)
      for (int b = 0; b < 15; b++) {
        double s = 0;
        for (int k = 0; k < 12; k++)
          s += G[a][k] * qc[k] * G[b][k];
        Qd(a, b) = s;
      }
    M15 FP = mulT(mul(F, cov), F);
    for (int a = 0; a < 15; a++)
      for (int b = 0; b < 15; b++)
        cov(a, b) = FP(a, b) + 0.5 * (Qd(a, b) + Qd(b, a));
    const V3 Ra = RT * a_hat;
    const V3 pn = p + dt * v + (0.5 * dt * dt) * Ra - (0.5 * dt * dt) * g, vn = v + dt * Ra - dt * g;
    q = rot_2_quat(E * R);
    p = pn;
    v = vn;
  }
  const M3 Rq = quat_2_Rot(q);
  const V3 vl = Rq * v;
  const size_t n = prop.size();
  const V3 wl = 0.5 * (smp(prop[n - 1].wm) + smp(prop[n - 2].wm)) - bg;
  for (int k = 0; k < 4; k++)
    state_plus13[k] = q[k];
  for (int k = 0; k < 3; k++) {
    state_plus13[4 + k] = p[k];
    state_plus13[7 + k] = vl[k];
    state_plus13[10 + k] = wl[k];
  }
  M15 Phi;
  for (int i = 0; i < 15; i++)
    Phi(i, i) = 1.0;
  Phi.setBlock3(6, 6, Rq);
  M15 rc = mulT(mul(Phi, cov), Phi);
  std::memset(cov144, 0, 144 * sizeof(double));
  for (int i = 0; i < 9; i++)
    for (int j = 0; j < 9; j++)
      cov144[12 * j + i] = rc(i, j);
  const double dtl = prop[n - 1].t - prop[n - 2].t;
  for (int k = 0; k < 3; k++)
    cov144[12 * (9 + k) + 9 + k] = c->sigma_w * c->sigma_w / dtl;
  *ok = 1;
  return OVP_OK;
}

int ovp_propagate_and_clone(ovp_ctx *h, double timestamp, double *Phi15, double *Q15, int *new_handle) {
  using namespace ovp::hm;
  Ctx *c = ovp::enter(h);
  if (c->timestamp == timestamp)
    return fail(c, OVP_ERR_TIME, "propagate_and_clone: same timestep as the last update (Propagator.cpp:41-44)");
  if (c->timestamp > timestamp)
    return fail(c, OVP_ERR_TIME, "propagate_and_clone: backwards in time (Propagator.cpp:47-51)");
  int st = sync_host_values(c);
  if (st)
    return st;
  double *iv = &c->h_val[(size_t)c->h_imu * OVP_VAL_STRIDE];
  double *ifej = &c->h_fej[(size_t)c->h_imu * OVP_VAL_STRIDE];
  double t_off = c->h_val[(size_t)c->h_dt * OVP_VAL_STRIDE];
  if (!c->have_last_prop_time_offset) {
    c->last_prop_time_offset = t_off;
    c->have_last_prop_time_offset = true;
  }
  double time0 = c->timestamp + c->last_prop_time_offset;
  double time1 = timestamp + t_off;
  std::vector<ImuSample> prop = select_imu_readings(c->imu_data, time0, time1);
  M15 Phi, Qs;
  for (int i = 0; i < 15; i++)
    Phi(i, i) = 1.0;
  V3 g = v3(c->gravity[0], c->gravity[1], c->gravity[2]);
  const int th = 0, p_id = 3, v_id = 6, bg = 9, ba = 12;
  if (prop.size() > 1) {
    for (size_t i = 0; i + 1 < prop.size(); i++) {
      // predict_and_compute, Propagator.cpp:343-454
      ImuMean x;
      ImuMean xf;
      for (int k = 0; k < 4; k++) {
        x.q[k] = iv[k];
        xf.q[k] = ifej[k];
      }
      for (int k = 0; k < 3; k++) {
        x.p[k] = iv[4 + k];
        x.v[k] = iv[7 + k];
        x.bg[k] = iv[10 + k];
        x.ba[k] = iv[13 + k];
        xf.p[k] = ifej[4 + k];
        xf.v[k] = ifej[7 + k];
      }
      double dt = prop[i + 1].t - prop[i].t;
      V3 w_hat = v3(prop[i].wm[0], prop[i].wm[1], prop[i].wm[2]) - x.bg;
      V3 a_hat = v3(prop[i].am[0], prop[i].am[1], prop[i].am[2]) - x.ba;
      V3 w_hat2 = v3(prop[i + 1].wm[0], prop[i + 1].wm[1], prop[i + 1].wm[2]) - x.bg;
      V3 a_hat2 = v3(prop[i + 1].am[0], prop[i + 1].am[1], prop[i + 1].am[2]) - x.ba;
      V4 nq;
      V3 nv, np;
      if (c->opt.use_rk4_integration)
        predict_mean_rk4(x, g, dt, w_hat, a_hat, w_hat2, a_hat2, nq, nv, np);
      else
        predict_mean_discrete(x, g, c->opt.imu_avg != 0, dt, w_hat, a_hat, w_hat2, a_hat2, nq, nv, np);
      M15 F;
      double G[15][12];
      std::memset(G, 0, sizeof(G));
      auto setG = [&](int i0, int j0, const M3 &B) {
        for (int a = 0; a < 3; a++)
          for (int b = 0; b < 3; b++)
            G[i0 + a][j0 + b] = B(a, b);
      };
      M3 I3 = eye3();
      if (c->opt.do_fej) {
        M3 Rfej = quat_2_Rot(xf.q);
        M3 RfT = transpose(Rfej);
        M3 dR = quat_2_Rot(nq) * RfT;
        M3 Jr = Jr_so3((-dt) * w_hat);
        M3 dRJ = (-dt) * (dR * Jr);
        F.setBlock3(th, th, dR);
        F.setBlock3(th, bg, dRJ);
        F.setBlock3(bg, bg, I3);
        F.setBlock3(v_id, th, (-1.0) * (skew(nv - xf.v + dt * g) * RfT));
        F.setBlock3(v_id, v_id, I3);
        F.setBlock3(v_id, ba, (-dt) * RfT);
        F.setBlock3(ba, ba, I3);
        F.setBlock3(p_id, th, (-1.0) * (skew(np - xf.p - dt * xf.v + (0.5 * dt * dt) * g) * RfT));
        F.setBlock3(p_id, v_id, dt * I3);
        F.setBlock3(p_id, ba, (-0.5 * dt * dt) * RfT);
        F.setBlock3(p_id, p_id, I3);
        setG(th, 0, dRJ);
        setG(v_id, 3, (-dt) * RfT);
        setG(p_id, 3, (-0.5 * dt * dt) * RfT);
        setG(bg, 6, I3);
        setG(ba, 9, I3);
      } else {
        M3 R = quat_2_Rot(x.q);
        M3 RT = transpose(R);
        M3 E = exp_so3((-dt) * w_hat);
        M3 Jr = Jr_so3((-dt) * w_hat);
        M3 EJ = (-dt) * (E * Jr);
        F.setBlock3(th, th, E);
        F.setBlock3(th, bg, EJ);
        F.setBlock3(bg, bg, I3);
        F.setBlock3(v_id, th, (-1.0) * (RT * skew(dt * a_hat)));
        F.setBlock3(v_id, v_id, I3);
        F.setBlock3(v_id, ba, (-dt) * RT);
        F.setBlock3(ba, ba, I3);
        F.setBlock3(p_id, th, (-0.5) * (RT * skew((dt * dt) * a_hat)));
        F.setBlock3(p_id, v_id, dt * I3);
        F.setBlock3(p_id, ba, (-0.5 * dt * dt) * RT);
        F.setBlock3(p_id, p_id, I3);
        setG(th, 0, EJ);
        setG(v_id, 3, (-dt) * RT);
        setG(p_id, 3, (-0.5 * dt * dt) * RT);
        setG(bg, 6, I3);
        setG(ba, 9, I3);
      }
      double qc[12];
      for (int k = 0; k < 3; k++) {
        qc[k] = c->sigma_w * c->sigma_w / dt;
        qc[3 + k] = c->sigma_a * c->sigma_a / dt;
        qc[6 + k] = c->sigma_wb * c->sigma_wb * dt;
        qc[9 + k] = c->sigma_ab * c->sigma_ab * dt;
      }
      M15 Qd;
      for (int a = 0; a < 15; a++)
        for (int b = 0; b < 15; b++) {
          double s = 0;
          for (int k = 0; k < 12; k++)
            s += G[a][k] * qc[k] * G[b][k];
          Qd(a, b) = s;
        }
      for (int a = 0; a < 15; a++)
        for (int b = a + 1; b < 15; b++) {
          double m = 0.5 * (Qd(a, b) + Qd(b, a));
          Qd(a, b) = Qd(b, a) = m;
        }
      // state mean + FEJ are both replaced by the propagated mean (:448-453)
      for (int k = 0; k < 4; k++)
        iv[k] = nq[k];
      for (int k = 0; k < 3; k++) {
        iv[4 + k] = np[k];
        iv[7 + k] = nv[k];
      }
      for (int k = 0; k < 16; k++)
        ifej[k] = iv[k];
      // Phi_summed = F Phi ; Qd_summed = F Qd_summed F^T + Qdi, symmetrised (:100-102)
      Phi = mul(F, Phi);
      M15 FQ = mul(F, Qs);
      Qs = mulT(FQ, F);
      for (int a = 0; a < 225; a++)
        Qs.a[a] += Qd.a[a];
      for (int a = 0; a < 15; a++)
        for (int b = a + 1; b < 15; b++) {
          double m = 0.5 * (Qs(a, b) + Qs(b, a));
          Qs(a, b) = Qs(b, a) = m;
        }
    }
  }
  double last_w[3] = {0, 0, 0};
  if (prop.size() > 1)
    for (int k = 0; k < 3; k++)
      last_w[k] = prop[prop.size() - 2].wm[k] - iv[10 + k];
  else if (!prop.empty())
    for (int k = 0; k < 3; k++)
      last_w[k] = prop.back().wm[k] - iv[10 + k];
  st = push_host_values(c, c->h_imu);
  if (st)
    return st;
  // column-major copies for the device
  double PhiC[225], QC[225];
  for (int i = 0; i < 15; i++)
    for (int j = 0; j < 15; j++) {
      PhiC[j * 15 + i] = Phi(i, j);
      QC[j * 15 + i] = Qs(i, j);
    }
  int hi = c->h_imu;
  st = ovp_ekf_propagation(h, &hi, 1, &hi, 1, PhiC, 15, 15, QC);
  if (st)
    return st;
  c->last_prop_time_offset = t_off;
  int nh = -1;
  st = ovp_augment_clone(h, timestamp, last_w, &nh);
  if (st)
    return st;
  if (Phi15)
    std::memcpy(Phi15, PhiC, sizeof(PhiC));
  if (Q15)
    std::memcpy(Q15, QC, sizeof(QC));
  if (new_handle)
    *new_handle = nh;
  return OVP_OK;
}

// ---- instrumentation -----------------------------------------------------------------------------------------------------
int64_t ovp_launch_count(ovp_ctx *h) { return h->c.launches; }
void *ovp_stream(ovp_ctx *h) { return (void *)h->c.stream; }
int ovp_last_timing(ovp_ctx *h, double *ms4) {
  for (int i = 0; i < 4; i++)
    ms4[i] = h->c.last_ms[i];
  return OVP_OK;
}
int ovp_synchronize(ovp_ctx *h) {
  Ctx *c = ovp::enter(h);
  OVP_CUDA(cudaStreamSynchronize(c->stream));
  return OVP_OK;
}
int ovp_selftest_dgemm_tflops(ovp_ctx *h, int n, int iters, double *tflops) {
  Ctx *c = ovp::enter(h);
  if (n < 64 || iters < 1)
    return fail(c, OVP_ERR_BAD_ARGS, "selftest: bad sizes");
  double *A, *B, *C;
  size_t e = (size_t)n * n;
  OVP_CUDA(cudaMalloc(&A, e * sizeof(double)));
  OVP_CUDA(cudaMalloc(&B, e * sizeof(double)));
  OVP_CUDA(cudaMalloc(&C, e * sizeof(double)));
  dmma_selftest_fill<<<(unsigned)((e + 255) / 256), 256, 0, c->stream>>>(A, e, 1.0);
  dmma_selftest_fill<<<(unsigned)((e + 255) / 256), 256, 0, c->stream>>>(B, e, 0.5);
  GemmProblem p = make_problem(n, n, n, mv(A, n), mv(B, n), C, n);
  for (int i = 0; i < 3; i++)
    launch_gemm1(c, p);
  cudaEventRecord(c->ev[2], c->stream);
  for (int i = 0; i < iters; i++)
    launch_gemm1(c, p);
  cudaEventRecord(c->ev[3], c->stream);
  OVP_CUDA(cudaStreamSynchronize(c->stream));
  float ms = 0;
  cudaEventElapsedTime(&ms, c->ev[2], c->ev[3]);
  *tflops = 2.0 * (double)n * n * n * iters / (ms * 1e-3) / 1e12;
  cudaFree(A);
  cudaFree(B);
  cudaFree(C);
  return OVP_OK;
}

} // extern "C"

// ---- prepared-batch variant of UpdaterMSCKF::update, snapshots and per-kernel profiling (measurement support) ----------
extern "C" {

int ovp_msckf_prepare_landmarks(ovp_ctx *h, const ovp_feature_batch *batch, const ovp_plane_landmarks *landmarks, const ovp_updater_options *opt) {
  Ctx *c = ovp::enter(h);
  if (!batch || !opt)
    return fail(c, OVP_ERR_BAD_ARGS, "null batch / options");
  MsckfExtra ex;
  return msckf_prepare(c, batch, opt, landmark_extra(landmarks, ex));
}
int ovp_msckf_prepare(ovp_ctx *h, const ovp_feature_batch *batch, const ovp_updater_options *opt) {
  return ovp_msckf_prepare_landmarks(h, batch, nullptr, opt);
}
int ovp_msckf_launch(ovp_ctx *h) { return msckf_launch(ovp::enter(h)); }
int ovp_msckf_finish(ovp_ctx *h, int *feat_status, double *feat_chi2, int *plane_status, double *plane_chi2, int *hx_order, int *hx_order_n) {
  Ctx *c = ovp::enter(h);
  if (hx_order_n)
    *hx_order_n = 0;
  return msckf_finish(c, feat_status, feat_chi2, plane_status, plane_chi2, hx_order, hx_order_n);
}

int ovp_snapshot(ovp_ctx *h) {
  Ctx *c = ovp::enter(h);
  size_t pe = (size_t)c->ldP * c->Nmax, ve = (size_t)c->max_handles * OVP_VAL_STRIDE;
  if (!c->snapP) {
    OVP_CUDA(cudaMalloc(&c->snapP, pe * sizeof(double)));
    OVP_CUDA(cudaMalloc(&c->snap_val, ve * sizeof(double)));
    OVP_CUDA(cudaMalloc(&c->snap_fej, ve * sizeof(double)));
  }
  OVP_CUDA(cudaMemcpyAsync(c->snapP, c->dP, (size_t)c->ldP * c->N * sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
  OVP_CUDA(cudaMemcpyAsync(c->snap_val, c->d_val, c->vars.size() * OVP_VAL_STRIDE * sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
  OVP_CUDA(cudaMemcpyAsync(c->snap_fej, c->d_fej, c->vars.size() * OVP_VAL_STRIDE * sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
  c->snapN = c->N;
  return OVP_OK;
}
int ovp_restore(ovp_ctx *h) {
  Ctx *c = ovp::enter(h);
  if (c->snapN != c->N)
    return fail(c, OVP_ERR_BAD_ARGS, "restore: no snapshot of a %d-row state", c->N);
  OVP_CUDA(cudaMemcpyAsync(c->dP, c->snapP, (size_t)c->ldP * c->N * sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
  OVP_CUDA(cudaMemcpyAsync(c->d_val, c->snap_val, c->vars.size() * OVP_VAL_STRIDE * sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
  OVP_CUDA(cudaMemcpyAsync(c->d_fej, c->snap_fej, c->vars.size() * OVP_VAL_STRIDE * sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
  c->launches += 3;
  c->host_values_stale = true;
  return OVP_OK;
}

int ovp_set_profiling(ovp_ctx *h, int on) {
  Ctx *c = ovp::enter(h);
  cudaStreamSynchronize(c->stream);
  c->profiling = on != 0;
  c->prof_recs.clear();
  c->ev_used = 0;
  c->prof_pending = nullptr;
  return OVP_OK;
}
// per kernel class [gemm, gram, potrf, feature, other]: total ms, launch count, algorithmic work (flops or bytes)
int ovp_profile_report(ovp_ctx *h, double *ms, int64_t *count, double *work) {
  Ctx *c = ovp::enter(h);
  OVP_CUDA(cudaStreamSynchronize(c->stream));
  for (int i = 0; i < PROF_N; i++) {
    ms[i] = 0;
    count[i] = 0;
    work[i] = 0;
  }
  for (auto &r : c->prof_recs) {
    float t = 0;
    cudaEventElapsedTime(&t, r.e0, r.e1);
    ms[r.id] += t;
    count[r.id]++;
    work[r.id] += r.work;
  }
  c->prof_recs.clear();
  c->ev_used = 0;
  return OVP_OK;
}
int ovp_set_use_graphs(ovp_ctx *h, int on) {
  h->c.use_graphs = on != 0;
  return OVP_OK;
}
int ovp_set_rank_tolerance(ovp_ctx *h, double tol) {
  Ctx *c = ovp::enter(h);
  if (!(tol > 0.0 && tol < 1e-3))
    return fail(c, OVP_ERR_BAD_ARGS, "rank tolerance %g outside (0, 1e-3)", tol);
  OVP_CUDA(cudaStreamSynchronize(c->stream));
  free_prepared(c); // the captured graph holds the tolerance by value
  c->gram_tol = tol;
  return OVP_OK;
}
int ovp_transfer_bytes(ovp_ctx *h, int64_t *h2d, int64_t *d2h) {
  *h2d = h->c.h2d_bytes;
  *d2h = h->c.d2h_bytes;
  return OVP_OK;
}

} // extern "C"

// ---- UpdaterZeroVelocity::try_update (update/UpdaterZeroVelocity.cpp:68-318) -------------------------------------------------------------
// With the flags the reference hard-codes (:113-116): measurements w_true = 0, a_true = 0 for every IMU interval between the state time and
// `timestamp`; chi2 against the IMU marginal inflated by the bias random walk; accepted when the disparity check passes, or when chi2 and
// the velocity pass; then the bias propagation (Phi = I, so EKFPropagation changes exactly the six diagonal entries P_ii += Q_ii) and ONE
// StateHelper::EKFUpdate with the diagonal R.  FeatureHelper::compute_disparity (front end) is upstream: its outputs are arguments.
// H is laid out over the whole IMU variable (15 columns, zeros for p and v): the reference's {q, bg, ba} sub-variable order gives the same
// products.  The small host-side linear algebra (chi2 of a <= few-hundred-row system against a 15 x 15 marginal) needs no GPU.
namespace ovp {
__global__ void add_diag6_kernel(double *P, int ld, int id0, const double *q6) {
  const int j = threadIdx.x;
  if (j < 6)
    P[(size_t)(id0 + j) * ld + id0 + j] += q6[j];
}
} // namespace ovp
extern "C" {
int ovp_zupt_feed_imu(ovp_ctx *h, double timestamp, const double wm[3], const double am[3]) {
  ImuSample s;
  s.t = timestamp;
  for (int i = 0; i < 3; i++) {
    s.wm[i] = wm[i];
    s.am[i] = am[i];
  }
  h->c.zupt_imu.push_back(s);
  return OVP_OK;
}
int ovp_zupt_try_update(ovp_ctx *h, const ovp_zupt_options *zo, double timestamp, double average_disparity, int num_features, int *accepted,
                        double *chi2_out) {
  using namespace ovp::hm;
  Ctx *c = ovp::enter(h);
  if (!zo || !accepted)
    return fail(c, OVP_ERR_BAD_ARGS, "zupt_try_update: null argument");
  *accepted = 0;
  if (chi2_out)
    *chi2_out = 0.0;
  if (c->zupt_imu.empty() || c->timestamp == timestamp) { // :71-80
    c->zupt_last_state_timestamp = 0.0;
    return OVP_OK;
  }
  int st = sync_host_values(c);
  if (st)
    return st;
  const double *iv = &c->h_val[(size_t)c->h_imu * OVP_VAL_STRIDE];
  const double *ifej = &c->h_fej[(size_t)c->h_imu * OVP_VAL_STRIDE];
  const double t_off_new = c->h_val[(size_t)c->h_dt * OVP_VAL_STRIDE];
  if (!c->zupt_have_offset) {
    c->zupt_last_offset = t_off_new;
    c->zupt_have_offset = true;
  }
  const double time0 = c->timestamp + c->zupt_last_offset, time1 = timestamp + t_off_new;
  std::vector<ImuSample> rec = select_imu_readings(c->zupt_imu, time0, time1);
  c->zupt_last_offset = t_off_new;
  if (rec.size() < 2) {
    c->zupt_last_state_timestamp = 0.0;
    return OVP_OK;
  }
  const int m = 6 * ((int)rec.size() - 1);
  if (m > c->Rcap)
    return fail(c, OVP_ERR_CAPACITY, "zupt: %d measurement rows exceed capacity %d", m, c->Rcap);
  std::vector<double> H((size_t)m * 15, 0.0), res(m, 0.0), Rd(m, 0.0);
  double Rv[9], Rj[9];
  quat_to_rot(iv, Rv);
  quat_to_rot(c->opt.do_fej ? ifej : iv, Rj);
  const double g[3] = {0.0, 0.0, zo->gravity_mag};
  double Rg[3], Rjg[3];
  mat3_vec(Rv, g, Rg);
  mat3_vec(Rj, g, Rjg);
  double sk[9];
  skew3(Rjg, sk);
  double dt_summed = 0.0;
  for (size_t i = 0; i + 1 < rec.size(); i++) {
    const double dt = rec[i + 1].t - rec[i].t;
    for (int j = 0; j < 3; j++) {
      const double a_hat = rec[i].am[j] - iv[13 + j];
      res[6 * i + j] = -(rec[i].wm[j] - iv[10 + j]);
      res[6 * i + 3 + j] = -(a_hat - Rg[j]);
      H[(size_t)(9 + j) * m + 6 * i + j] = -1.0;
      for (int l = 0; l < 3; l++)
        H[(size_t)l * m + 6 * i + 3 + j] = -sk[3 * j + l];
      H[(size_t)(12 + j) * m + 6 * i + 3 + j] = -1.0;
      Rd[6 * i + j] = zo->zupt_noise_multiplier * (c->sigma_w * c->sigma_w / dt);
      Rd[6 * i + 3 + j] = zo->zupt_noise_multiplier * (c->sigma_a * c->sigma_a / dt);
    }
    dt_summed += dt;
  }
  double Qb[6];
  for (int j = 0; j < 3; j++) {
    Qb[j] = dt_summed * c->sigma_wb; // sigma, not sigma^2: exactly what the reference does (:186-187)
    Qb[3 + j] = dt_summed * c->sigma_ab;
  }
  // chi2 = res^T (H P_marg H^T + R)^-1 res with the inflated IMU marginal (:189-193), on the host
  double Pm[225];
  st = ovp_get_marginal_covariance(h, &c->h_imu, 1, Pm);
  if (st)
    return st;
  for (int j = 0; j < 6; j++)
    Pm[(9 + j) * 15 + 9 + j] += Qb[j];
  std::vector<double> T((size_t)m * 15), S((size_t)m * m);
  for (int i = 0; i < m; i++)
    for (int j = 0; j < 15; j++) {
      double a = 0.0;
      for (int k = 0; k < 15; k++)
        a += H[(size_t)k * m + i] * Pm[j * 15 + k];
      T[(size_t)j * m + i] = a;
    }
  for (int i = 0; i < m; i++)
    for (int j = 0; j <= i; j++) {
      double a = (i == j) ? Rd[i] : 0.0;
      for (int k = 0; k < 15; k++)
        a += T[(size_t)k * m + i] * H[(size_t)k * m + j];
      S[(size_t)j * m + i] = a;
    }
  std::vector<double> y(res);
  for (int j = 0; j < m; j++) { // Cholesky (lower, in place) and forward substitution in one sweep
    double d = S[(size_t)j * m + j];
    if (!(d > 0.0))
      return fail(c, OVP_ERR_NOT_POSITIVE_DEFINITE, "zupt: innovation covariance not positive definite");
    d = std::sqrt(d);
    S[(size_t)j * m + j] = d;
    y[j] /= d;
    for (int i = j + 1; i < m; i++) {
      S[(size_t)j * m + i] /= d;
      y[i] -= S[(size_t)j * m + i] * y[j];
    }
    for (int k = j + 1; k < m; k++) {
      const double lkj = S[(size_t)j * m + k];
      for (int i = k; i < m; i++)
        S[(size_t)k * m + i] -= S[(size_t)j * m + i] * lkj;
    }
  }
  double chi2 = 0.0;
  for (int i = 0; i < m; i++)
    chi2 += y[i] * y[i];
  if (chi2_out)
    *chi2_out = chi2;
  const double chi2_check = chi2_q95(c, m);
  const bool disparity_passed = average_disparity < zo->zupt_max_disparity && num_features > 20; // :219
  const double vnorm = std::sqrt(iv[7] * iv[7] + iv[8] * iv[8] + iv[9] * iv[9]);
  if (!disparity_passed && (chi2 > zo->chi2_multipler * chi2_check || vnorm > zo->zupt_max_velocity)) {
    c->zupt_last_state_timestamp = 0.0;
    return OVP_OK;
  }
  // accepted (:253-264): bias propagation, then the update, then move the state time forward
  if ((st = stage_copy_in(c, c->dscal + 32, Qb, sizeof(Qb))))
    return st;
  add_diag6_kernel<<<1, 32, 0, c->stream>>>(c->dP, c->ldP, c->vars[c->h_imu].id + 9, c->dscal + 32);
  c->launches++;
  st = ovp_ekf_update(h, &c->h_imu, 1, H.data(), m, res.data(), Rd.data());
  if (st)
    return st;
  c->timestamp = timestamp;
  c->zupt_last_state_timestamp = timestamp;
  *accepted = 1;
  return OVP_OK;
}
}

// ---- UpdaterSLAM entry points (slam_host.inc) ----------------------------------------------------------------------------
namespace ovp {
int slam_update_impl(Ctx *c, int F, const int *meas_offset, const int *meas_clone, const float *uv, const int64_t *featid,
                     const int64_t *planeid, const ovp_updater_options *opt, int use_plane, int *feat_status, double *feat_chi2);

// The tracks of slam_delayed_init_core already on the device (ovp_slam_delayed_init_tracks): feature f's clone handles and pixels start at
// measurement at[f] of clone / uv, and the staging buffer holds them below stage_base.
struct DeviceTracks {
  const int *clone;
  const float *uv;
  const int *at;
  size_t stage_base;
};
static bool is_relative(int rep);
static bool landmark_set_from_xyz(int rep, const double *p, double *v);
static int landmark_store_bearing(Ctx *c, int h, const double *b); // anchors.cu
static int stage_feature_jacobian_rep(Ctx *c, int m, const int *clone_handles, const float *uv, int representation, int anchor_clone_handle,
                                      const double *p_F, const double *p_F_fej, double sigma_px, FeatureJacobianStage *jo, int *k_out,
                                      int *extra_out, const DeviceTrack *dev = nullptr); // anchors.cu
// UpdaterSLAM::delayed_init, estimator half (UpdaterSLAM.cpp:225-372): per feature, in order, get_feature_jacobian_full with the
// plane constraint when the plane is in the state, StateHelper::initialize(landmark, ..., chi2_multipler); when that fails WITH a
// plane, detach the landmark from the plane and retry from the pre-refinement position (:310-359).  An ArUco tag takes the context's
// ArUco options on both tries (slam_options_of).  A feature whose representation (landmark_rep_of) is not GLOBAL_3D has no plane (its
// caller refuses it otherwise) and is initialised once, with the Jacobians of stage_feature_jacobian_rep (:230-304): anchored (2..5) in the
// clone of its last measurement, from p_FinA (its value and first estimate are set_from_xyz(p_FinA)); rep 1 from p_FinG.  Rep 5 takes the
// Jacobians of rep 4, projects the two bearing columns out and initialises a 1-wide landmark from the remaining 2m - 2 rows.  Shared by
// ovp_slam_delayed_init (dev == nullptr: each attempt stages its track from meas_clone / uv; p_FinA == nullptr, GLOBAL_3D only) and
// ovp_slam_delayed_init_tracks (uv unused).
static int slam_delayed_init_core(Ctx *c, int F, const int *meas_offset, const int *meas_clone, const float *uv, const DeviceTracks *dev,
                                  const double *p_FinG, const double *p_FinG_original, const int64_t *featid, const int64_t *planeid,
                                  const ovp_updater_options *opt, int use_plane, int *feat_status, int *new_handles,
                                  const double *p_FinA = nullptr) {
  for (int f = 0; f < F; f++) {
    feat_status[f] = 0;
    new_handles[f] = -1;
  }
  for (int f = 0; f < F; f++) {
    const int m = meas_offset[f + 1] - meas_offset[f];
    const int *cl = meas_clone + meas_offset[f];
    if (c->slam.count(featid[f]))
      return fail(c, OVP_ERR_ALREADY_IN_STATE, "delayed_init: feature %lld already has a landmark", (long long)featid[f]);
    const int ph = slam_plane_of(c, featid[f], planeid ? planeid[f] : 0, use_plane);
    DeviceTrack dt{};
    if (dev)
      dt = {dev->clone + dev->at[f], dev->uv + 2 * (size_t)dev->at[f], dev->stage_base};
    const ovp_updater_options &fo = slam_options_of(c, featid[f], *opt); // an ArUco tag's own (UpdaterSLAM.cpp:257, 302-304)
    const int rep = landmark_rep_of(c, featid[f]);
    if (rep != 0) {
      if (ph >= 0 || (is_relative(rep) && !p_FinA)) // refused up front by both callers
        return fail(c, OVP_ERR_BAD_ARGS, "delayed_init: feature %lld in representation %d", (long long)featid[f], rep);
      const int anc = is_relative(rep) ? cl[m - 1] : -1; // FeatureInitializer's anchor of a mono track: the last measurement's clone
      const double *pF = is_relative(rep) ? p_FinA + 3 * (size_t)f : p_FinG + 3 * (size_t)f;
      FeatureJacobianStage j;
      int k = 3, extra = 0;
      // the single-depth form takes the Jacobians of ANCHORED_MSCKF_INVERSE_DEPTH (UpdaterSLAM.cpp:233-236)
      int st = stage_feature_jacobian_rep(c, m, cl, dev ? nullptr : uv + 2 * (size_t)meas_offset[f], rep == 5 ? 4 : rep, anc, pF, pF, fo.sigma_pix,
                                          &j, &k, &extra, dev ? &dt : nullptr);
      if (st)
        return st;
      std::vector<int> xo;
      if (c->opt.do_calib_camera_pose)
        xo.push_back(c->h_calib);
      if (c->opt.do_calib_camera_intrinsics)
        xo.push_back(c->h_intr);
      for (int i = 0; i < m; i++)
        xo.push_back(cl[i]);
      if (extra)
        xo.push_back(anc);
      int n = 0;
      if ((st = upload_cols(c, xo.data(), (int)xo.size(), 0, &n)))
        return st;
      if (n != j.hxc)
        return fail(c, OVP_ERR_BAD_ARGS, "delayed_init: internal column mismatch %d vs %d", n, j.hxc);
      if (c->var_table_dirty && (st = upload_var_table(c)))
        return st;
      double v[4]; // Landmark::set_from_xyz (:283-289)
      landmark_set_from_xyz(rep, pF, v);
      double *W = j.W(c);
      int s = 3, rows = j.rows;
      if (rep == 5) { // H_f's last column joins the state side, its two bearing columns are projected out of [H_x | H_rho | r] (:260-283):
        // the landmark is initialised from the last 2m - 2 rows of [H_rho | H_x | r] with s = 1, and the chi2 takes their 2m - 2 dof
        householder_cols_kernel<<<1, 256, 0, c->stream>>>(W, j.rows, j.rows, 3 + n + 1, 2);
        c->launches++;
        OVP_CUDA(cudaGetLastError());
        W += 2 * (size_t)j.rows + 2;
        s = 1;
        rows = j.rows - 2;
      }
      int acc = 0, nh = -1;
      if ((st = initialize_core(c, OVP_KIND_LANDMARK, s, v, v, featid[f], c->dcols, n, W, j.rows, rows, rows, 1.0, fo.chi2_multipler, 1, &acc, &nh)))
        return st;
      if (acc) {
        feat_status[f] = 1;
        new_handles[f] = nh;
        c->vars[nh].rep = rep;
        c->vars[nh].anchor = anc;
        if (rep == 5 && (st = landmark_store_bearing(c, nh, v + 1))) // the bearing it was created with, value and first estimate
          return st;
      }
      continue;
    }
    auto attempt = [&](const double *pf, int plane_h, int *acc, int *nh) -> int {
      FeatureJacobianStage j;
      int st = stage_feature_jacobian(c, m, cl, dev ? nullptr : uv + 2 * (size_t)meas_offset[f], pf, pf, plane_h >= 0, plane_h, nullptr, nullptr,
                                      fo.sigma_pix, c->opt.sigma_constraint, &j, 0, dev ? &dt : nullptr);
      if (st)
        return st;
      std::vector<int> xo;
      if (c->opt.do_calib_camera_pose)
        xo.push_back(c->h_calib);
      if (c->opt.do_calib_camera_intrinsics)
        xo.push_back(c->h_intr);
      for (int i = 0; i < m; i++)
        xo.push_back(cl[i]);
      if (plane_h >= 0)
        xo.push_back(plane_h);
      int n = 0;
      st = upload_cols(c, xo.data(), (int)xo.size(), 0, &n);
      if (st)
        return st;
      if (n != j.hxc)
        return fail(c, OVP_ERR_BAD_ARGS, "delayed_init: internal column mismatch %d vs %d", n, j.hxc);
      if (c->var_table_dirty) {
        st = upload_var_table(c);
        if (st)
          return st;
      }
      return initialize_core(c, OVP_KIND_LANDMARK, 3, pf, pf, featid[f], c->dcols, n, j.W(c), j.rows, j.rows, j.rows, 1.0, fo.chi2_multipler,
                             1, acc, nh);
    };
    int acc = 0, nh = -1;
    int st = attempt(p_FinG + 3 * (size_t)f, ph, &acc, &nh);
    if (st)
      return st;
    if (acc) {
      feat_status[f] = 1;
      new_handles[f] = nh;
      if (ph >= 0)
        c->slam_to_plane[featid[f]] = planeid[f];
    } else if (ph >= 0) {
      c->slam_to_plane[featid[f]] = 0;
      const double *po = (p_FinG_original ? p_FinG_original : p_FinG) + 3 * (size_t)f;
      st = attempt(po, -1, &acc, &nh);
      if (st)
        return st;
      if (acc) {
        feat_status[f] = 3;
        new_handles[f] = nh;
      }
    }
  }
  return OVP_OK;
}
} // namespace ovp
extern "C" {
int ovp_slam_update(ovp_ctx *h, int F, const int *meas_offset, const int *meas_clone, const float *uv, const int64_t *featid,
                    const int64_t *planeid, const ovp_updater_options *opt, int use_plane_constraint, int *feat_status, double *feat_chi2) {
  Ctx *c = ovp::enter(h);
  if (F > 0 && (!meas_offset || !meas_clone || !uv || !featid || !opt))
    return fail(c, OVP_ERR_BAD_ARGS, "slam_update: null argument");
  return slam_update_impl(c, F, meas_offset, meas_clone, uv, featid, planeid, opt, use_plane_constraint, feat_status, feat_chi2);
}
int ovp_slam_delayed_init(ovp_ctx *h, int F, const int *meas_offset, const int *meas_clone, const float *uv, const double *p_FinG,
                          const double *p_FinG_original, const int64_t *featid, const int64_t *planeid, const ovp_updater_options *opt,
                          int use_plane_constraint, int *feat_status, int *new_handles) {
  Ctx *c = ovp::enter(h);
  if (F > 0 && (!meas_offset || !meas_clone || !uv || !featid || !opt || !p_FinG || !feat_status || !new_handles))
    return fail(c, OVP_ERR_BAD_ARGS, "slam_delayed_init: null argument");
  // every track is checked before the first landmark is initialised (each one's Jacobian takes 1..64 measurements)
  int st = check_tracks(c, "slam_delayed_init", F, meas_offset, meas_clone, nullptr, 1, 64, OVP_ERR_BAD_ARGS, false, true);
  if (st)
    return st;
  for (int f = 0; f < F; f++) // the reference initialises such a landmark from p_FinA, which this entry point does not take
    if (landmark_rep_of(c, featid[f]) != 0)
      return fail(c, OVP_ERR_BAD_ARGS, "slam_delayed_init: feature %lld takes representation %d (ovp_set_landmark_options); landmarks outside "
                  "GLOBAL_3D are initialised from the triangulation's p_FinA by ovp_slam_delayed_init_tracks", (long long)featid[f],
                  landmark_rep_of(c, featid[f]));
  return slam_delayed_init_core(c, F, meas_offset, meas_clone, uv, nullptr, p_FinG, p_FinG_original, featid, planeid, opt, use_plane_constraint,
                                feat_status, new_handles);
}
int ovp_set_aruco_options(ovp_ctx *h, const ovp_updater_options *aruco) {
  Ctx *c = &h->c; // host-only: the kernels take the options as launch arguments
  if (!aruco) {
    c->has_aruco = false;
    return OVP_OK;
  }
  if (!(aruco->sigma_pix > 0.0) || !(aruco->chi2_multipler > 0.0))
    return fail(c, OVP_ERR_BAD_ARGS, "set_aruco_options: sigma_pix (%g) and chi2_multipler (%g) must be positive", aruco->sigma_pix,
                aruco->chi2_multipler);
  c->aruco = *aruco;
  c->has_aruco = true;
  return OVP_OK;
}
int ovp_slam_handle(ovp_ctx *h, int64_t featid) {
  auto it = h->c.slam.find(featid);
  return it == h->c.slam.end() ? -1 : it->second;
}
int ovp_slam_should_marg(ovp_ctx *h, int64_t featid) {
  auto it = h->c.slam.find(featid);
  return it == h->c.slam.end() ? -1 : (h->c.vars[it->second].should_marg ? 1 : 0);
}
int64_t ovp_slam_plane_of(ovp_ctx *h, int64_t featid) { /* State::_features_SLAM_to_PLANE; -1 = no entry */
  auto it = h->c.slam_to_plane.find(featid);
  return it == h->c.slam_to_plane.end() ? -1 : it->second;
}
}

