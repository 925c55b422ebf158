// TEST INFRASTRUCTURE - NOT PRODUCT CODE, never loaded by the package.
//
// The pieces of the forward dynamics' derivatives that are new in csrc/: the product kernel of
// tiny-differentiable-simulator_b200/csrc/tds_fd_derivatives.cu (double and dual) and the DER instances of csrc/tds_stepw.cu reading qdd in
// fp64 from StepIO::g_out, both compiled FOR THE HOST with single-lane meanings of the CUDA built-ins and called lane after lane as
// tds_launch_fdd and tds_launch_dynamics_derivatives(_jvp) launch them on the GPU.  The DER instances' host build and its set-up come from
// tests/cpp/dynamics_derivatives_host.cpp, whose entry points stay as they are.  Nothing outside tests/ builds or loads it.
//   g++ -std=c++17 -O1 -shared -fPIC -I<csrc> -I<include> -I/usr/local/cuda/include tests/cpp/fd_derivatives_host.cpp -o ...
#include "dynamics_derivatives_host.cpp"

#define TDS_FDD_KERNEL_ONLY 1
#include "../../tiny-differentiable-simulator_b200/csrc/tds_fd_derivatives.cu"

namespace {
// host [n][rows] -> device layout [rows][ns] (null: zeros)
std::vector<double> fdd_soa(const double* x, int n, size_t rows, int ns) {
  std::vector<double> o(rows * ns + 1, 0.0);
  if (x)
    for (int e = 0; e < n; ++e)
      for (size_t r = 0; r < rows; ++r) o[r * ns + e] = x[(size_t)e * rows + r];
  return o;
}
void fdd_aos(double* y, const std::vector<double>& o, int n, size_t rows, int ns) {
  if (y)
    for (int e = 0; e < n; ++e)
      for (size_t r = 0; r < rows; ++r) y[(size_t)e * rows + r] = o[r * ns + e];
}
}  // namespace

extern "C" {

// d tau / dq and d tau / dqd [n][n_qd][n_qd] as tdsemu_dynamics_derivatives, with qdd [n][n_qd] read in fp64 (not rounded) through
// StepIO::g_out; with m >= 1 instead their tangents [n][n_qd][n_qd][m] along t_q [n][n_q][m], t_qd and t_qdd [n][n_qd][m] and t_par
// [n][k][m] (each may be null) as tdsemu_dynamics_derivatives_jvp.
int tdsemu_der_qdd64(const double* model, int n_model, int n, const double* q, const double* qd, const double* qdd, const double* g, int k,
                     const int* ids, const double* values, int m, const double* t_q, const double* t_qd, const double* t_qdd, const double* t_par,
                     double* dq, double* dqd) {
  Setup* S = new Setup;
  int rc = setup(*S, model, n_model, n, q, qd, nullptr, k, ids, values, m > 0 ? 16 : 8);
  if (rc) { delete S; return rc; }
  const int n_q = S->D.n_q, nd = S->D.n_qd, nn = nd * nd, ns = S->ns, mm = m > 0 ? m : 1;
  const std::vector<double> sqdd = fdd_soa(qdd, n, nd, ns);
  std::vector<double> o0((size_t)nn * mm * ns + 1, -1.0), o1((size_t)nn * mm * ns + 1, -1.0);
  StepIO io = io_of(*S);
  io.g_out = sqdd.data();
  io.jac = o0.data(); io.g_in = o1.data(); io.jac_n_in = mm; io.jac_dir0 = 0;
  std::vector<char> scratch((size_t)mm * ((n + 31) / 32) * S->D.x_total * 32 * 4 + 64);
  if (m == 0) {
    if (k > 0) run_grid<double, true, false>(S->D, io, 1, scratch.data(), S->pm, g);
    else run_grid<double, false, false>(S->D, io, 1, scratch.data(), tdsw::NoPar{}, g);
  } else {
    std::vector<double> ti((size_t)(n_q + 2 * nd) * m * ns, 0.0), tp((size_t)(k > 0 ? k : 1) * m * ns, 0.0);
    for (int e = 0; e < n; ++e) {
      if (t_q) for (int c = 0; c < n_q * m; ++c) ti[(size_t)c * ns + e] = t_q[(size_t)e * n_q * m + c];
      if (t_qd) for (int c = 0; c < nd * m; ++c) ti[((size_t)n_q * m + c) * ns + e] = t_qd[(size_t)e * nd * m + c];
      if (t_qdd) for (int c = 0; c < nd * m; ++c) ti[((size_t)(n_q + nd) * m + c) * ns + e] = t_qdd[(size_t)e * nd * m + c];
      if (t_par) for (int c = 0; c < k * m; ++c) tp[(size_t)c * ns + e] = t_par[(size_t)e * k * m + c];
    }
    const tdsw::JvpTan jv{(t_q || t_qd || t_qdd) ? ti.data() : nullptr, t_par ? tp.data() : nullptr, m};
    if (k > 0) {
      tdsw::ParMapJvp a;
      static_cast<ParMap&>(a) = S->pm;
      a.jv = jv;
      run_grid<tds::Dual<double>, true, true>(S->D, io, m, scratch.data(), a, g);
    } else {
      run_grid<tds::Dual<double>, false, true>(S->D, io, m, scratch.data(), tdsw::NoParJvp{jv}, g);
    }
  }
  fdd_aos(dq, o0, n, (size_t)nn * mm, ns);
  fdd_aos(dqd, o1, n, (size_t)nn * mm, ns);
  delete S;
  return 0;
}

// The product kernel: dq = -Mi Aq, dqd = -Mi Aqd, dtau = Mi [n][n_qd][n_qd] from Mi, Aq, Aqd [n][n_qd][n_qd] by the value instance; with
// m >= 1 instead their tangents [n][n_qd][n_qd][m] from the tangents dMi, dAq, dAqd [n][n_qd][n_qd][m] (each may be null: zero) by the
// dual instance.  Any output may be null.
int tdsemu_fdd(int n, int nd, const double* Mi, const double* Aq, const double* Aqd, int m, const double* dMi, const double* dAq,
               const double* dAqd, double* dq, double* dqd, double* dtau) {
  const int ns = (n + 31) & ~31, mm = m > 0 ? m : 1;
  const size_t nn = (size_t)nd * nd;
  const std::vector<double> sM = fdd_soa(Mi, n, nn, ns), sAq = fdd_soa(Aq, n, nn, ns), sAqd = fdd_soa(Aqd, n, nn, ns);
  const std::vector<double> sdM = fdd_soa(dMi, n, nn * mm, ns), sdAq = fdd_soa(dAq, n, nn * mm, ns), sdAqd = fdd_soa(dAqd, n, nn * mm, ns);
  std::vector<double> o0(nn * mm * ns + 1, -1.0), o1(nn * mm * ns + 1, -1.0), o2(nn * mm * ns + 1, -1.0);
  TdsFddCall c;
  memset(&c, 0, sizeof(c));
  c.n_qd = nd; c.m = mm; c.j0 = 0; c.m_out = mm;
  c.Mi = sM.data(); c.Aq = sAq.data(); c.Aqd = sAqd.data();
  if (m > 0) { c.dMi = dMi ? sdM.data() : nullptr; c.dAq = dAq ? sdAq.data() : nullptr; c.dAqd = dAqd ? sdAqd.data() : nullptr; }
  c.dq = dq ? o0.data() : nullptr; c.dqd = dqd ? o1.data() : nullptr; c.dtau = dtau ? o2.data() : nullptr;
  emu_blockDim = {128, 1, 1};
  for (int j = 0; j < mm; ++j)
    for (int e = 0; e < n; ++e)
      for (int col = 0; col < ((dq || dqd) ? nd : 0) + (dtau ? nd : 0); ++col) {
        emu_threadIdx = {(unsigned)(e % 128), 0, 0};
        emu_blockIdx = {(unsigned)(e / 128), (unsigned)col, (unsigned)j};
        if (m > 0) fdd_product_kernel<tds::Dual<double>>(c, n, ns);
        else fdd_product_kernel<double>(c, n, ns);
      }
  fdd_aos(dq, o0, n, nn * mm, ns);
  fdd_aos(dqd, o1, n, nn * mm, ns);
  fdd_aos(dtau, o2, n, nn * mm, ns);
  return 0;
}

}  // extern "C"
