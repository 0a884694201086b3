// Gaussian-kernel vector field utilities shared by the alignment and by st.tdr:
//   U^T = exp(-beta |x - z|^2)            (con_K, spateo/alignment/methods/utils.py:1132-1158)
//   field evaluation on query points      (BA_transform, spateo/alignment/transform.py:93-103;
//                                          _gp_velocity, spateo/tdr/morphometrics/morphofield/gaussian_process.py:109-117)
#include "common.cuh"

namespace {

__global__ void rbf_kernel_T_kernel(const float* __restrict__ x, int64_t n, int64_t ldx, const float* __restrict__ z,
                                    int K, float beta, float* __restrict__ UT) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int k = blockIdx.y;
  if (i >= ldx) return;
  float v = 0.f;
  if (i < n) {
    const float d0 = x[i] - z[k * 3 + 0], d1 = x[ldx + i] - z[k * 3 + 1], d2 = x[2 * ldx + i] - z[k * 3 + 2];
    v = expf(-beta * (d0 * d0 + d1 * d1 + d2 * d2));
  }
  UT[(int64_t)k * ldx + i] = v;
}

// out[i][:] = sum_k exp(-beta |q_i - z_k|^2) Coff[k][:]   (fp64; K*D*2 doubles staged in shared memory)
__global__ void field_eval_kernel(const double* __restrict__ q, int64_t n, int D, const double* __restrict__ z,
                                  const double* __restrict__ Coff, int K, double beta, double* __restrict__ out) {
  extern __shared__ double shf[];
  double* zs = shf;
  double* cs = shf + (size_t)K * D;
  for (int t = threadIdx.x; t < K * D; t += blockDim.x) {
    zs[t] = z[t];
    cs[t] = Coff[t];
  }
  __syncthreads();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double qi[3] = {0, 0, 0}, acc[3] = {0, 0, 0};
  for (int d = 0; d < D; ++d) qi[d] = q[i * D + d];
  for (int k = 0; k < K; ++k) {
    double d2 = 0;
    for (int d = 0; d < D; ++d) {
      const double df = qi[d] - zs[k * D + d];
      d2 += df * df;
    }
    const double w = exp(-beta * d2);
    for (int d = 0; d < D; ++d) acc[d] += w * cs[k * D + d];
  }
  for (int d = 0; d < D; ++d) out[i * D + d] = acc[d];
}


// Differential geometry of the Gaussian-process field, one thread per query point, everything in registers (fp64):
//   velocity  (_gp_velocity, gaussian_process.py:102-127), Jacobian (Jacobian_GP_gaussian_kernel, GPVectorField.py:143-190),
//   acceleration / curvature / curl / torsion / divergence (GPVectorField.py:12-125), det J (differential_geometry.py:336).
struct GeomOut {
  double *V, *J, *acc, *acc_mat, *curv, *curv_mat, *curl, *torsion, *div, *det;
};

// Field value at one raw point for an spb_field_desc, shared by field_geometry_kernel and field_integrate_kernel:
//   field_normalize  xn = (x - mean_transformed) / scale_transformed
//   field_sum        vel += sum_k exp(-beta |xn - z_k|^2) Coff[k] over kn control points of zs / cs (JAC: the Jacobian's
//                    sum over the same terms, J[a][b] += w Coff[k][a] (xn - z_k)[b])
//   field_velocity   velocity in raw units / velocity_divisor (10000 for the GP field, 1 for a plain RBF field)
template <int D>
__device__ __forceinline__ void field_normalize(const spb_field_desc& f, const double (&x)[D], double (&xn)[D]) {
#pragma unroll
  for (int d = 0; d < D; ++d) xn[d] = (x[d] - f.mean_transformed[d]) / f.scale_transformed;
}

template <int D, bool JAC>
__device__ __forceinline__ void field_sum(const double* zs, const double* cs, int kn, double beta, const double (&xn)[D],
                                          double (&vel)[D], double (*J)[D]) {
  for (int k = 0; k < kn; ++k) {
    double df[D], d2 = 0.0;
#pragma unroll
    for (int d = 0; d < D; ++d) {
      df[d] = xn[d] - zs[k * D + d];
      d2 += df[d] * df[d];
    }
    const double w = exp(-beta * d2);
#pragma unroll
    for (int a = 0; a < D; ++a) {
      const double wc = w * cs[k * D + a];
      vel[a] += wc;
      if constexpr (JAC) {
#pragma unroll
        for (int b = 0; b < D; ++b) J[a][b] += wc * df[b];
      }
    }
  }
}

template <int D>
__device__ __forceinline__ void field_velocity(const spb_field_desc& f, const double (&x)[D], const double (&xn)[D],
                                               const double (&vel)[D], double (&v)[D]) {
#pragma unroll
  for (int d = 0; d < D; ++d) {
    if (f.nonrigid_only) {
      v[d] = vel[d] * f.scale_fixed + (f.scale_fixed - f.scale_transformed) * xn[d];
    } else {
      double r = f.t[d];
#pragma unroll
      for (int e = 0; e < D; ++e) r += xn[e] * f.R[d * 3 + e];
      v[d] = (vel[d] + r) * f.scale_fixed + f.mean_fixed[d] - x[d];
    }
    v[d] /= f.velocity_divisor;
  }
}

template <int D>
__global__ void field_geometry_kernel(spb_field_desc f, const double* __restrict__ X, int64_t n,
                                      const double* __restrict__ z, const double* __restrict__ Coff, GeomOut o) {
  extern __shared__ double shf[];
  double* zs = shf;
  double* cs = shf + (size_t)f.K * D;
  for (int t = threadIdx.x; t < f.K * D; t += blockDim.x) {
    zs[t] = z[t];
    cs[t] = Coff[t];
  }
  __syncthreads();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double x[D], xn[D], vel[D], J[D][D];
#pragma unroll
  for (int d = 0; d < D; ++d) {
    x[d] = X[i * D + d];
    vel[d] = 0.0;
#pragma unroll
    for (int e = 0; e < D; ++e) J[d][e] = 0.0;
  }
  field_normalize<D>(f, x, xn);
  field_sum<D, true>(zs, cs, f.K, f.beta, xn, vel, J);
  const double jscale = -2.0 * f.beta * (f.scale_fixed / f.scale_transformed);
#pragma unroll
  for (int a = 0; a < D; ++a)
#pragma unroll
    for (int b = 0; b < D; ++b) J[a][b] *= jscale;
  double v[D];
  field_velocity<D>(f, x, xn, vel, v);
  double a[D], vv = 0.0, va = 0.0, aa = 0.0;
#pragma unroll
  for (int d = 0; d < D; ++d) {
    double s = 0.0;
#pragma unroll
    for (int e = 0; e < D; ++e) s += J[d][e] * v[e];
    a[d] = s;
  }
#pragma unroll
  for (int d = 0; d < D; ++d) {
    vv += v[d] * v[d];
    va += v[d] * a[d];
    aa += a[d] * a[d];
  }
  if (o.V)
    for (int d = 0; d < D; ++d) o.V[i * D + d] = v[d];
  if (o.J)
    for (int p = 0; p < D; ++p)
      for (int q = 0; q < D; ++q) o.J[(i * D + p) * D + q] = J[p][q];
  if (o.acc) o.acc[i] = sqrt(aa);
  if (o.acc_mat)
    for (int d = 0; d < D; ++d) o.acc_mat[i * D + d] = a[d];
  if (o.curv || o.curv_mat) {
    const double nv = sqrt(vv);
    if (f.curvature_formula == 1) {
      if (o.curv) o.curv[i] = sqrt(vv * aa) / (nv * nv * nv);
    } else {
      double c2 = 0.0;
      const double nv4 = (nv * nv) * (nv * nv);
      for (int d = 0; d < D; ++d) {
        const double c = (a[d] * vv - v[d] * va) / nv4;
        if (o.curv_mat) o.curv_mat[i * D + d] = c;
        c2 += c * c;
      }
      if (o.curv) o.curv[i] = sqrt(c2);
    }
  }
  if (o.curl) {
    if (D == 2) {
      o.curl[i] = J[1][0] - J[0][1];
    } else if (D == 3) {
      o.curl[i * 3 + 0] = J[2 % D][1] - J[1][2 % D];
      o.curl[i * 3 + 1] = J[0][2 % D] - J[2 % D][0];
      o.curl[i * 3 + 2] = J[1][0] - J[0][1];
    }
  }
  if (o.torsion && D == 3) {
    // tau = outer(v, a) . (J a) / |outer(v, a)|_F^2 = v (a . J a) / (|v|^2 |a|^2)
    double Ja[D], aJa = 0.0;
    for (int d = 0; d < D; ++d) {
      double s = 0.0;
      for (int e = 0; e < D; ++e) s += J[d][e] * a[e];
      Ja[d] = s;
    }
    for (int d = 0; d < D; ++d) aJa += a[d] * Ja[d];
    const double nrm = sqrt(vv * aa);
    for (int d = 0; d < D; ++d) o.torsion[i * D + d] = v[d] * aJa / (nrm * nrm);
  }
  if (o.div) {
    double tr = 0.0;
    for (int d = 0; d < D; ++d) tr += J[d][d];
    o.div[i] = tr;
  }
  if (o.det) {
    double dt;
    if (D == 1) dt = J[0][0];
    else if (D == 2) dt = J[0][0] * J[1][1] - J[0][1] * J[1][0];
    else
      dt = J[0][0] * (J[1][1] * J[2 % D][2 % D] - J[1][2 % D] * J[2 % D][1]) -
           J[0][1] * (J[1][0] * J[2 % D][2 % D] - J[1][2 % D] * J[2 % D][0]) +
           J[0][2 % D] * (J[1][0] * J[2 % D][1] - J[1][1] * J[2 % D][0]);
    o.det[i] = dt;
  }
}


// ---- trajectories dx/dt = v(x): scipy.integrate.solve_ivp(method="RK45") restated per thread ----------------------
// (scipy/integrate/_ivp/rk.py RungeKutta / RK45, common.py select_initial_step / norm, ivp.py solve_ivp's event and
// t_eval handling; the field function and its terminal event are those dynamo's fate / integrate_vf_ivp hand to it).
constexpr int FI_THREADS = 128;
constexpr int FI_TILE = 1024;  // control points per shared-memory tile: 2 * 1024 * 3 doubles = 48 KB at D = 3

// Dormand-Prince 5(4): rk.py class RK45 (A, B, E and the dense-output matrix P)
__constant__ double kA[6][5] = {
    {0, 0, 0, 0, 0},
    {1.0 / 5, 0, 0, 0, 0},
    {3.0 / 40, 9.0 / 40, 0, 0, 0},
    {44.0 / 45, -56.0 / 15, 32.0 / 9, 0, 0},
    {19372.0 / 6561, -25360.0 / 2187, 64448.0 / 6561, -212.0 / 729, 0},
    {9017.0 / 3168, -355.0 / 33, 46732.0 / 5247, 49.0 / 176, -5103.0 / 18656}};
__constant__ double kB[6] = {35.0 / 384, 0, 500.0 / 1113, 125.0 / 192, -2187.0 / 6784, 11.0 / 84};
__constant__ double kE[7] = {-71.0 / 57600, 0, 71.0 / 16695, -71.0 / 1920, 17253.0 / 339200, -22.0 / 525, 1.0 / 40};
__constant__ double kP[7][4] = {
    {1, -8048581381.0 / 2820520608, 8663915743.0 / 2820520608, -12715105075.0 / 11282082432},
    {0, 0, 0, 0},
    {0, 131558114200.0 / 32700410799, -68118460800.0 / 10900136933, 87487479700.0 / 32700410799},
    {0, -1754552775.0 / 470086768, 14199869525.0 / 1410260304, -10690763975.0 / 1880347072},
    {0, 127303824393.0 / 49829197408, -318862633887.0 / 49829197408, 701980252875.0 / 199316789632},
    {0, -282668133.0 / 205662961, 2019193451.0 / 616988883, -1453857185.0 / 822651844},
    {0, 40617522.0 / 29380423, -110615467.0 / 29380423, 69997945.0 / 29380423}};

// v(x) for every thread of the block. With K > FI_TILE the control points pass through shared memory tile by tile, so
// every thread of the block must call this the same number of times (field_integrate_kernel runs its threads in lockstep).
template <int D>
__device__ __forceinline__ void integrate_eval(const spb_field_desc& f, const double* __restrict__ z,
                                               const double* __restrict__ Coff, double* zs, double* cs,
                                               const double (&x)[D], double (&v)[D]) {
  double xn[D], vel[D];
#pragma unroll
  for (int d = 0; d < D; ++d) vel[d] = 0.0;
  field_normalize<D>(f, x, xn);
  if (f.K <= FI_TILE) {
    field_sum<D, false>(zs, cs, f.K, f.beta, xn, vel, nullptr);
  } else {
    for (int k0 = 0; k0 < f.K; k0 += FI_TILE) {
      const int kn = min(FI_TILE, f.K - k0);
      __syncthreads();
      for (int t = threadIdx.x; t < kn * D; t += blockDim.x) {
        zs[t] = z[(size_t)k0 * D + t];
        cs[t] = Coff[(size_t)k0 * D + t];
      }
      __syncthreads();
      field_sum<D, false>(zs, cs, kn, f.beta, xn, vel, nullptr);
    }
  }
  field_velocity<D>(f, x, xn, vel, v);
}

template <int D>
__device__ __forceinline__ double rms_norm(const double (&x)[D]) {  // common.py norm: ||x|| / sqrt(n)
  double s = 0.0;
#pragma unroll
  for (int d = 0; d < D; ++d) s += x[d] * x[d];
  return sqrt(s) / sqrt((double)D);
}

// dynamo's terminal event np.all(abs(f(x)) < 1e-5) - 1: 0 once every velocity component is below 1e-5, else -1
template <int D>
__device__ __forceinline__ int slow_event(const double (&v)[D]) {
  bool all = true;
#pragma unroll
  for (int d = 0; d < D; ++d) all = all && fabs(v[d]) < 1e-5;
  return all ? 0 : -1;
}

// RkDenseOutput._call_impl: y_old + h Q p(x), Q = K^T P, p = cumprod([x] * 4), x = (t - t_old) / h
template <int D>
__device__ __forceinline__ void dense_eval(const double (&k)[7][D], const double (&y_old)[D], double t_old, double h,
                                           double t, double (&y)[D]) {
  const double x = (t - t_old) / h;
  const double p1 = x, p2 = p1 * x, p3 = p2 * x, p4 = p3 * x;
#pragma unroll
  for (int d = 0; d < D; ++d) {
    double q[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      double s = 0.0;
#pragma unroll
      for (int r = 0; r < 7; ++r) s += k[r][d] * kP[r][c];
      q[c] = s;
    }
    y[d] = h * (q[0] * p1 + q[1] * p2 + q[2] * p3 + q[3] * p4) + y_old[d];
  }
}

struct IntegrateArgs {
  const double *X0, *z, *Coff;
  int64_t n;
  double t_bound, rtol, atol, max_step;
  int32_t n_out, max_accepted;
  double *out, *t_stop;
  int32_t *steps, *status;
};

// One thread per trajectory, each with its own adaptive step sequence; the block advances one step attempt (six field
// evaluations) per loop trip until none of its threads is still integrating. A thread writes grid sample j (time
// j * t_bound / (n_out - 1), the last exactly t_bound: np.linspace) from the dense output of the step that passes it,
// and after the stop fills the remaining samples with the state at the stop.
template <int D>
__global__ void __launch_bounds__(FI_THREADS, 3) field_integrate_kernel(spb_field_desc f, IntegrateArgs a) {
  extern __shared__ double shf[];
  const int kt = min(f.K, FI_TILE);
  double* zs = shf;
  double* cs = shf + (size_t)kt * D;
  if (f.K <= FI_TILE) {
    for (int t = threadIdx.x; t < f.K * D; t += blockDim.x) {
      zs[t] = a.z[t];
      cs[t] = a.Coff[t];
    }
    __syncthreads();
  }
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t ic = i < a.n ? i : a.n - 1;  // threads past n integrate a copy of the last cell and write nothing
  const double dir = a.t_bound > 0 ? 1.0 : -1.0;
  const double grid_dt = a.t_bound / (a.n_out - 1);
  double* out = a.out + (size_t)ic * a.n_out * D;

  double y[D], k[7][D];
#pragma unroll
  for (int d = 0; d < D; ++d) y[d] = a.X0[ic * D + d];
  integrate_eval<D>(f, a.z, a.Coff, zs, cs, y, k[0]);

  // select_initial_step (error estimator order 4)
  double h_abs;
  {
    double sy[D], sf[D];
#pragma unroll
    for (int d = 0; d < D; ++d) {
      const double scale = a.atol + fabs(y[d]) * a.rtol;
      sy[d] = y[d] / scale;
      sf[d] = k[0][d] / scale;
    }
    const double interval = fabs(a.t_bound), d0 = rms_norm<D>(sy), d1 = rms_norm<D>(sf);
    double h0 = (d0 < 1e-5 || d1 < 1e-5) ? 1e-6 : 0.01 * d0 / d1;
    h0 = fmin(h0, interval);
    double y1[D], f1[D];
#pragma unroll
    for (int d = 0; d < D; ++d) y1[d] = y[d] + h0 * dir * k[0][d];
    integrate_eval<D>(f, a.z, a.Coff, zs, cs, y1, f1);
#pragma unroll
    for (int d = 0; d < D; ++d) sf[d] = (f1[d] - k[0][d]) / (a.atol + fabs(y[d]) * a.rtol);
    const double d2 = rms_norm<D>(sf) / h0;
    const double h1 = (d1 <= 1e-15 && d2 <= 1e-15) ? fmax(1e-6, h0 * 1e-3) : pow(0.01 / fmax(d1, d2), 1.0 / 5);
    h_abs = fmin(fmin(100 * h0, h1), fmin(interval, a.max_step));
  }

  double t = 0.0, min_step = 0.0;
  int g_old = slow_event<D>(k[0]);
  int j = 0, accepted = 0, rejected = 0, stat = 2;  // 2: still integrating
  bool in_step = false, step_rejected = false;
  double y_stop[D];  // state at the stop, written to the samples after it
  while (__syncthreads_or(i < a.n && stat == 2)) {
    const bool was_live = stat == 2;
    double h = 0.0, t_new = t;
    if (stat == 2 && !in_step) {  // RungeKutta._step_impl entry
      if (accepted >= a.max_accepted) {
        stat = -1;
      } else {
        min_step = 10 * fabs(nextafter(t, dir * INFINITY) - t);
        h_abs = h_abs > a.max_step ? a.max_step : (h_abs < min_step ? min_step : h_abs);
        in_step = true;
        step_rejected = false;
      }
    }
    if (stat == 2 && h_abs < min_step) stat = -1;  // TOO_SMALL_STEP
    if (stat == 2) {
      t_new = t + h_abs * dir;
      if (dir * (t_new - a.t_bound) > 0) t_new = a.t_bound;
      h = t_new - t;
      h_abs = fabs(h);
    } else if (was_live) {  // failed this trip: the solver stops at its last accepted state
#pragma unroll
      for (int d = 0; d < D; ++d) y_stop[d] = y[d];
    }
    // rk_step: five stages, then f_new at y_new (FSAL: k[6] becomes the next step's k[0]). Threads that have stopped
    // evaluate at their frozen state (h = 0) to keep the block in lockstep.
    double y_new[D];
#pragma unroll
    for (int s = 1; s <= 6; ++s) {
      double xs[D];
#pragma unroll
      for (int d = 0; d < D; ++d) {
        double acc = 0.0;
        if (s < 6) {
#pragma unroll
          for (int r = 0; r < s; ++r) acc += k[r][d] * kA[s][r];
          xs[d] = y[d] + acc * h;
        } else {
#pragma unroll
          for (int r = 0; r < 6; ++r) acc += k[r][d] * kB[r];
          y_new[d] = xs[d] = y[d] + h * acc;
        }
      }
      integrate_eval<D>(f, a.z, a.Coff, zs, cs, xs, k[s]);
    }
    if (stat != 2) continue;
    double en[D];
#pragma unroll
    for (int d = 0; d < D; ++d) {
      double e = 0.0;
#pragma unroll
      for (int r = 0; r < 7; ++r) e += k[r][d] * kE[r];
      en[d] = e * h / (a.atol + fmax(fabs(y[d]), fabs(y_new[d])) * a.rtol);
    }
    const double error_norm = rms_norm<D>(en);
    if (!(error_norm < 1)) {
      h_abs *= fmax(0.2, 0.9 * pow(error_norm, -1.0 / 5));
      step_rejected = true;
      ++rejected;
      continue;
    }
    double factor = error_norm == 0 ? 10.0 : fmin(10.0, 0.9 * pow(error_norm, -1.0 / 5));
    if (step_rejected) factor = fmin(1.0, factor);
    h_abs *= factor;
    ++accepted;
    in_step = false;
    if (dir * (t_new - a.t_bound) >= 0) stat = 0;
    // solve_ivp's event handling. With direction 0 the event is active when g is 0 at either end of the step. Its
    // root is brentq's on the step's dense output; g takes only the values -1 and 0, so brentq returns at its endpoint
    // checks: t_old when g(y_old) = 0, otherwise t_new (where g(sol(t_new)) rounds back to -1 there is no bracket and
    // scipy raises; the trajectory stops at t_new as well).
    const int g_new = slow_event<D>(k[6]);
    double t_end_step = t_new;
    if (g_old == 0 || g_new == 0) {
      stat = 1;
      t_end_step = g_old == 0 ? t : t_new;
      if (g_old == 0) {
#pragma unroll
        for (int d = 0; d < D; ++d) y_stop[d] = y[d];
      } else {
        dense_eval<D>(k, y, t, h, t_new, y_stop);
      }
    }
    g_old = g_new;
    for (; j < a.n_out; ++j) {  // t_eval times up to the end of this step (searchsorted side='right' / 'left')
      const double tj = j == a.n_out - 1 ? a.t_bound : j * grid_dt;
      if (dir * (tj - t_end_step) > 0) break;
      double ys[D];
      dense_eval<D>(k, y, t, h, tj, ys);
      if (i < a.n)
#pragma unroll
        for (int d = 0; d < D; ++d) out[(size_t)j * D + d] = ys[d];
    }
    t = t_end_step;
#pragma unroll
    for (int d = 0; d < D; ++d) {
      y[d] = y_new[d];
      k[0][d] = k[6][d];
    }
  }
  if (i >= a.n) return;
  for (; j < a.n_out; ++j)
#pragma unroll
    for (int d = 0; d < D; ++d) out[(size_t)j * D + d] = y_stop[d];
  a.t_stop[i] = t;
  a.steps[2 * i] = accepted;
  a.steps[2 * i + 1] = rejected;
  a.status[i] = stat;
}

}  // namespace

#define ST ((cudaStream_t)stream)

extern "C" int spb_rbf_kernel_T(const float* x, int64_t n, int64_t ldx, const float* z, int32_t K, float beta, float* UT,
                                void* stream) {
  dim3 grid((unsigned)((ldx + 255) / 256), (unsigned)K);
  rbf_kernel_T_kernel<<<grid, 256, 0, ST>>>(x, n, ldx, z, K, beta, UT);
  SPB_CHECK_LAUNCH();
  return 0;
}

extern "C" int spb_field_eval(const double* q, int64_t n, int32_t D, const double* z, const double* Coff, int32_t K,
                              double beta, double* out, void* stream) {
  if (n <= 0) return 0;
  if (D < 1 || D > 3) return SPB_EINVAL;
  const size_t smem = sizeof(double) * 2 * (size_t)K * D;
  if (smem > 96 * 1024) return SPB_EUNSUPPORTED;
  static bool attr_set[SPB_MAX_DEVICES] = {};  // the opt-in is per device (one process may drive several GPUs)
  const int dev_ = spb_current_device();
  if (!attr_set[dev_]) {
    cudaError_t e = cudaFuncSetAttribute(field_eval_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
    if (e != cudaSuccess) return (int)e;
    attr_set[dev_] = true;
  }
  field_eval_kernel<<<(unsigned)((n + 127) / 128), 128, smem, ST>>>(q, n, D, z, Coff, K, beta, out);
  SPB_CHECK_LAUNCH();
  return 0;
}


extern "C" int spb_field_geometry(const spb_field_desc* f, const double* X, int64_t n, const double* z,
                                  const double* Coff, double* V, double* J, double* acc, double* acc_mat, double* curv,
                                  double* curv_mat, double* curl, double* torsion, double* div, double* det,
                                  void* stream) {
  if (n <= 0) return 0;
  if (f == nullptr || f->D < 2 || f->D > 3 || f->K < 1) return SPB_EINVAL;
  if (torsion != nullptr && f->D != 3) return SPB_EINVAL;
  const size_t smem = sizeof(double) * 2 * (size_t)f->K * f->D;
  if (smem > 96 * 1024) return SPB_EUNSUPPORTED;
  static bool attr_set[SPB_MAX_DEVICES] = {};  // the opt-in is per device (one process may drive several GPUs)
  const int dev_ = spb_current_device();
  if (!attr_set[dev_]) {
    cudaError_t e = cudaFuncSetAttribute(field_geometry_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
    if (e != cudaSuccess) return (int)e;
    e = cudaFuncSetAttribute(field_geometry_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
    if (e != cudaSuccess) return (int)e;
    attr_set[dev_] = true;
  }
  GeomOut o{V, J, acc, acc_mat, curv, curv_mat, curl, torsion, div, det};
  const unsigned grid = (unsigned)((n + 127) / 128);
  if (f->D == 2)
    field_geometry_kernel<2><<<grid, 128, smem, ST>>>(*f, X, n, z, Coff, o);
  else
    field_geometry_kernel<3><<<grid, 128, smem, ST>>>(*f, X, n, z, Coff, o);
  SPB_CHECK_LAUNCH();
  return 0;
}

extern "C" int spb_field_integrate(const spb_field_desc* f, const double* X0, int64_t n, const double* z,
                                   const double* Coff, double t_end, int32_t n_out, double rtol, double atol,
                                   double max_step, double* out, double* t_stop, int32_t* steps, int32_t* status,
                                   void* stream) {
  if (n <= 0) return 0;
  if (f == nullptr || f->D < 2 || f->D > 3 || f->K < 1 || n_out < 2 || !(t_end != 0.0) || !isfinite(t_end) ||
      !(rtol > 0.0) || !(atol > 0.0) || !(max_step > 0.0) || n_out > INT32_MAX / 100)
    return SPB_EINVAL;
  if (X0 == nullptr || z == nullptr || Coff == nullptr || out == nullptr || t_stop == nullptr || steps == nullptr ||
      status == nullptr)
    return SPB_EINVAL;
  IntegrateArgs a{X0, z, Coff, n, t_end, rtol, atol, max_step, n_out, 100 * (n_out - 1), out, t_stop, steps, status};
  const size_t smem = sizeof(double) * 2 * (size_t)min(f->K, FI_TILE) * f->D;
  const unsigned grid = (unsigned)((n + FI_THREADS - 1) / FI_THREADS);
  if (f->D == 2)
    field_integrate_kernel<2><<<grid, FI_THREADS, smem, ST>>>(*f, a);
  else
    field_integrate_kernel<3><<<grid, FI_THREADS, smem, ST>>>(*f, a);
  SPB_CHECK_LAUNCH();
  return 0;
}

extern "C" int spb_field_eval_host(const double* q_host, int64_t n, int32_t D, const double* z_host,
                                   const double* Coff_host, int32_t K, double beta, double* out_host) {
  double *q = nullptr, *z = nullptr, *c = nullptr, *o = nullptr;
  cudaError_t e;
  int rc = 0;
  if ((e = cudaMalloc(&q, sizeof(double) * n * D)) != cudaSuccess) return (int)e;
  if ((e = cudaMalloc(&z, sizeof(double) * K * D)) != cudaSuccess) { cudaFree(q); return (int)e; }
  if ((e = cudaMalloc(&c, sizeof(double) * K * D)) != cudaSuccess) { cudaFree(q); cudaFree(z); return (int)e; }
  if ((e = cudaMalloc(&o, sizeof(double) * n * D)) != cudaSuccess) { cudaFree(q); cudaFree(z); cudaFree(c); return (int)e; }
  cudaMemcpy(q, q_host, sizeof(double) * n * D, cudaMemcpyHostToDevice);
  cudaMemcpy(z, z_host, sizeof(double) * K * D, cudaMemcpyHostToDevice);
  cudaMemcpy(c, Coff_host, sizeof(double) * K * D, cudaMemcpyHostToDevice);
  rc = spb_field_eval(q, n, D, z, c, K, beta, o, nullptr);
  if (rc == 0) {
    e = cudaMemcpy(out_host, o, sizeof(double) * n * D, cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) rc = (int)e;
  }
  cudaFree(q); cudaFree(z); cudaFree(c); cudaFree(o);
  return rc;
}
