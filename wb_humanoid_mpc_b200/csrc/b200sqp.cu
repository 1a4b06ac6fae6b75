// C ABI implementation (include/b200sqp.h).  Host C++ orchestration + kernel launches; no CPU fallback.
#include "../../include/b200sqp.h"

#include <cuda_runtime.h>
#include <dlfcn.h>

#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <memory>
#include <new>
#include <string>
#include <type_traits>
#include <vector>

#include "riccati.cuh"
#include "riccati_cluster.cuh"
#include "riccati_wb.cuh"
#ifdef B200SQP_WITH_WB
#include "wb_solver.cuh"
#include "wb_builder.cuh"
#include "wb_fleet.cuh"
#include "wb_sim.cuh"
#include "cen_dynamics.cuh"
#include "wb_torque.cuh"
#include "wb_torque_cost.cuh"
#include "wb_mrt.cuh"
#include "wb_devio.cuh"
#include "wb_query.cuh"
#include "cen_kernels.cuh"
#include "cen_host.cuh"
#include "wb_gains.cuh"
#endif

namespace {
thread_local std::string g_err;
int fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_err = buf;
  return code;
}
#define CUDA_TRY(expr)                                                                             \
  do {                                                                                             \
    cudaError_t e_ = (expr);                                                                       \
    if (e_ != cudaSuccess) return fail(e_ == cudaErrorMemoryAllocation ? B200SQP_ENOMEM : B200SQP_ENODEV, "%s: %s", #expr, \
                                       cudaGetErrorString(e_));                                    \
  } while (0)

int select_device(int device) {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) return fail(B200SQP_ENODEV, "no CUDA device available (%s); b200sqp has no CPU fallback", cudaGetErrorString(e));
  if (device < 0 || device >= n) return fail(B200SQP_EINVAL, "device %d out of range (%d devices)", device, n);
  CUDA_TRY(cudaSetDevice(device));
  return 0;
}

cudaError_t set_riccati_smem_attributes(int nx, int numax) {
  const int one = static_cast<int>(b200sqp::riccati_smem_doubles(nx, numax) * sizeof(double));
  const int clu = static_cast<int>(b200sqp::riccati_cluster_smem_doubles(nx, numax) * sizeof(double));
  cudaError_t e = cudaFuncSetAttribute(b200sqp::riccati_kernel<0, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, one);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(b200sqp::riccati_cluster_kernel<0, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, clu);
  if (nx == 58 && numax == 23) {
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(b200sqp::ricwb::riccati_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(b200sqp::ricwb::BWD_SMEM_BYTES));
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(b200sqp::ricwb::riccati_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(b200sqp::ricwb::FWD_SMEM_BYTES));
    if (e == cudaSuccess) e = cudaFuncSetAttribute(b200sqp::riccati_kernel<58, 23>, cudaFuncAttributeMaxDynamicSharedMemorySize, one);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(b200sqp::riccati_cluster_kernel<58, 23>, cudaFuncAttributeMaxDynamicSharedMemorySize, clu);
  }
  return e;
}

// K2 dispatch: the cluster variant (RC SMs per instance) for small batches; for the whole-body sizes the two-kernel form of riccati_wb.cuh
// (backward factorisation with a helper warp + separate forward substitution); the generic one-CTA kernel for every other size.
// B200SQP_NO_CLUSTER=1 skips the cluster variant, B200SQP_K2_LEGACY=1 forces the generic kernel (tests exercise all three).
// Returns the number of kernels launched.
int launch_riccati(const b200sqp::QpDeviceView& v, cudaStream_t st) {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  }
  const char* no = std::getenv("B200SQP_NO_CLUSTER");
  // the cluster variant is used while at most half of the SMs are taken by clusters (B <= 16 on an H100, where it is 7-9 % faster than the
  // one-CTA kernels for every such B; where the crossover lies above that bound has not been measured on the H100)
  const bool cluster = !(no && no[0] == '1') && v.B * b200sqp::RC * 2 <= sms;
  const bool wb = (v.nx == 58 && v.numax == 23);   // the whole-body sizes have a compile-time instantiation
  if (cluster) {
    const size_t smem = b200sqp::riccati_cluster_smem_doubles(v.nx, v.numax) * sizeof(double);
    if (wb) b200sqp::riccati_cluster_kernel<58, 23><<<v.B * b200sqp::RC, 256, smem, st>>>(v);
    else b200sqp::riccati_cluster_kernel<0, 0><<<v.B * b200sqp::RC, 256, smem, st>>>(v);
  } else {
    const char* legacy = std::getenv("B200SQP_K2_LEGACY");
    if (wb && !(legacy && legacy[0] == '1')) {
      // two instances per CTA (c and c + ceil(B / 2)) once the batch is larger than the SM count, so that it runs in one wave up to twice
      // that; one per CTA below, so that no SM idles
      const int pairOff = v.B > sms ? (v.B + 1) / 2 : 0;
      b200sqp::ricwb::riccati_bwd_kernel<<<pairOff ? pairOff : v.B, b200sqp::ricwb::BWD_THREADS, b200sqp::ricwb::BWD_SMEM_BYTES, st>>>(v, pairOff);
      b200sqp::ricwb::riccati_fwd_kernel<<<v.B, b200sqp::ricwb::FWD_THREADS, b200sqp::ricwb::FWD_SMEM_BYTES, st>>>(v);
      return 2;
    }
    const size_t smem = b200sqp::riccati_smem_doubles(v.nx, v.numax) * sizeof(double);
    if (wb) b200sqp::riccati_kernel<58, 23><<<v.B, 256, smem, st>>>(v);
    else b200sqp::riccati_kernel<0, 0><<<v.B, 256, smem, st>>>(v);
  }
  return 1;
}

// a failed allocation, reported as the error of the entry point that made it
int failAlloc(const char* entry, cudaError_t e) {
  return fail(e == cudaErrorMemoryAllocation ? B200SQP_ENOMEM : B200SQP_ENODEV, "%s: %s", entry, cudaGetErrorString(e));
}
}  // namespace

namespace b200sqp {
// The device and pinned allocations of one lifetime.  Each allocation stores its pointer in a field of the caller and records that field;
// release(from) frees what was allocated since mark() returned `from`, newest first, and sets each recorded field back to null.  The first
// error is sticky -- later allocations do nothing, so a group of them is checked once with error() -- until release() clears it.
class MemOwner {
 public:
  MemOwner() = default;
  MemOwner(const MemOwner&) = delete;
  MemOwner& operator=(const MemOwner&) = delete;
  ~MemOwner() { release(); }
  template <class T>
  void device(T*& field, size_t count, bool zero = false) {
    add(slot(field), count * sizeof(T), false, zero);
  }
  template <class T>
  void pinned(T*& field, size_t count) {
    add(slot(field), count * sizeof(T), true, false);
  }
  cudaError_t error() const { return err_; }
  size_t mark() const { return live_.size(); }
  void release(size_t from = 0) {
    for (; live_.size() > from; live_.pop_back()) {
      void** field = live_.back().field;
      if (live_.back().pinned) cudaFreeHost(*field);
      else cudaFree(*field);
      *field = nullptr;
    }
    err_ = cudaSuccess;
  }

 private:
  struct Entry {
    void** field;
    bool pinned;
  };
  template <class T>
  static void** slot(T*& field) {   // (const-qualified T: the device arrays a kernel only reads)
    return reinterpret_cast<void**>(const_cast<std::remove_const_t<T>**>(&field));
  }
  void add(void** field, size_t bytes, bool pinned, bool zero) {
    if (err_ != cudaSuccess) return;
    void* p = nullptr;
    err_ = pinned ? cudaMallocHost(&p, bytes) : cudaMalloc(&p, bytes);
    if (err_ != cudaSuccess) return;
    *field = p;
    live_.push_back({field, pinned});
    if (zero) err_ = cudaMemset(p, 0, bytes);
  }
  std::vector<Entry> live_;
  cudaError_t err_ = cudaSuccess;
};
}  // namespace b200sqp

struct b200sqp_qp_t {
  int device = 0;
  b200sqp::QpDeviceView v{};   // the arrays and sizes; a solve sets nu, keepP and reg on its copy
  bool hasNu = false;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  bool uploaded = false, solved = false, keptP = false;
  b200sqp::MemOwner mem;
};

extern "C" {

const char* b200sqp_last_error(void) { return g_err.c_str(); }
const char* b200sqp_version(void) { return "b200sqp 0.1 (sm_90a, fp64)"; }

int b200sqp_qp_create(int device, int batch, int N, int nx, int nu_max, b200sqp_qp* out) {
  if (!out || batch <= 0 || N <= 0 || nx <= 0 || nx > 64 || nu_max <= 0 || nu_max > 32)
    return fail(B200SQP_EINVAL, "qp_create: need batch,N > 0, 0 < nx <= 64 and 0 < nu_max <= 32 (got %d,%d,%d,%d)", batch, N, nx, nu_max);
  if (int rc = select_device(device)) return rc;
  if (!b200sqp::riccati_sizes_supported(nx, nu_max))
    return fail(B200SQP_EINVAL, "qp_create: nx=%d nu_max=%d needs %zu B (one-CTA kernel) and %zu B (cluster kernel) of shared memory (limit %zu B)",
                nx, nu_max, b200sqp::riccati_smem_doubles(nx, nu_max) * sizeof(double),
                b200sqp::riccati_cluster_smem_doubles(nx, nu_max) * sizeof(double), b200sqp::RIC_SMEM_BYTES_MAX);
  b200sqp_qp_t* qp = new (std::nothrow) b200sqp_qp_t;
  if (!qp) return fail(B200SQP_ENOMEM, "host allocation failed");
  qp->device = device;
  b200sqp::QpDeviceView& v = qp->v;
  v.B = batch;
  v.N = N;
  v.nx = nx;
  v.numax = nu_max;
  b200sqp::MemOwner& m = qp->mem;
  b200sqp::forEachQpArray(v, true, [&](auto*& a, b200sqp::RowKind k, int w) { m.device(a, b200sqp::batchRows(k, batch, N + 1) * w); });
  cudaError_t e = m.error();
  if (e == cudaSuccess) e = cudaEventCreate(&qp->ev0);
  if (e == cudaSuccess) e = cudaEventCreate(&qp->ev1);
  if (e == cudaSuccess) e = set_riccati_smem_attributes(nx, nu_max);
  if (e != cudaSuccess) {
    b200sqp_qp_destroy(qp);
    return failAlloc("qp_create", e);
  }
  *out = qp;
  return 0;
}

void b200sqp_qp_destroy(b200sqp_qp qp) {
  if (!qp) return;
  cudaSetDevice(qp->device);
  if (qp->ev0) cudaEventDestroy(qp->ev0);
  if (qp->ev1) cudaEventDestroy(qp->ev1);
  delete qp;   // (its owner frees the arrays)
}

int b200sqp_qp_upload(b200sqp_qp qp, const double* A, const double* B, const double* b, const double* Q, const double* S,
                      const double* R, const double* q, const double* r, const int32_t* nu, const double* dx0) {
  if (!qp || !A || !B || !b || !Q || !S || !R || !q || !r || !dx0) return fail(B200SQP_EINVAL, "qp_upload: null argument");
  CUDA_TRY(cudaSetDevice(qp->device));
  const b200sqp::QpDeviceView& v = qp->v;
  const size_t bn = static_cast<size_t>(v.B) * v.N, bn1 = static_cast<size_t>(v.B) * (v.N + 1);
  const int nx = v.nx, nm = v.numax;
  // (the inputs are const in the view the kernels read)
  auto up = [&](const void* d, const void* h, size_t bytes) { return cudaMemcpy(const_cast<void*>(d), h, bytes, cudaMemcpyHostToDevice); };
  CUDA_TRY(up(v.A, A, bn * nx * nx * sizeof(double)));
  CUDA_TRY(up(v.Bm, B, bn * nx * nm * sizeof(double)));
  CUDA_TRY(up(v.b, b, bn * nx * sizeof(double)));
  CUDA_TRY(up(v.Q, Q, bn1 * nx * nx * sizeof(double)));
  CUDA_TRY(up(v.S, S, bn * nm * nx * sizeof(double)));
  CUDA_TRY(up(v.R, R, bn * nm * nm * sizeof(double)));
  CUDA_TRY(up(v.q, q, bn1 * nx * sizeof(double)));
  CUDA_TRY(up(v.r, r, bn * nm * sizeof(double)));
  CUDA_TRY(up(v.dx0, dx0, static_cast<size_t>(v.B) * nx * sizeof(double)));
  qp->hasNu = nu != nullptr;
  if (nu) {
    for (size_t i = 0; i < bn; ++i)
      if (nu[i] < 0 || nu[i] > nm) return fail(B200SQP_EINVAL, "qp_upload: nu[%zu]=%d outside [0,%d]", i, nu[i], nm);
    CUDA_TRY(up(v.nu, nu, bn * sizeof(int)));
  }
  qp->uploaded = true;
  qp->solved = false;
  return 0;
}

int b200sqp_qp_solve(b200sqp_qp qp, double reg_prim, int keep_P, void* stream) {
  if (!qp) return fail(B200SQP_EINVAL, "qp_solve: null handle");
  if (!qp->uploaded) return fail(B200SQP_ESTATE, "qp_solve: no problem uploaded");
  CUDA_TRY(cudaSetDevice(qp->device));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t bn = static_cast<size_t>(qp->v.B) * qp->v.N;
  b200sqp::QpDeviceView v = qp->v;
  if (!qp->hasNu) v.nu = nullptr;
  v.keepP = keep_P;
  v.reg = reg_prim;
  CUDA_TRY(cudaEventRecord(qp->ev0, st));
  CUDA_TRY(cudaMemsetAsync(v.K, 0, bn * v.numax * v.nx * sizeof(double), st));
  CUDA_TRY(cudaMemsetAsync(v.kff, 0, bn * v.numax * sizeof(double), st));
  launch_riccati(v, st);
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaEventRecord(qp->ev1, st));
  qp->solved = true;
  qp->keptP = keep_P != 0;
  return 0;
}

int b200sqp_qp_download(b200sqp_qp qp, double* dx, double* du, double* K, double* k, double* P, double* p, int32_t* status) {
  if (!qp) return fail(B200SQP_EINVAL, "qp_download: null handle");
  if (!qp->solved) return fail(B200SQP_ESTATE, "qp_download: nothing solved yet");
  if ((P || p) && !qp->keptP) return fail(B200SQP_ESTATE, "qp_download: cost-to-go requested but solve ran with keep_P = 0");
  CUDA_TRY(cudaSetDevice(qp->device));
  CUDA_TRY(cudaDeviceSynchronize());
  const b200sqp::QpDeviceView& v = qp->v;
  const size_t bn = static_cast<size_t>(v.B) * v.N, bn1 = static_cast<size_t>(v.B) * (v.N + 1);
  const int nx = v.nx, nm = v.numax;
  auto dn = [&](double* h, const double* d, size_t n) { return h ? cudaMemcpy(h, d, n * sizeof(double), cudaMemcpyDeviceToHost) : cudaSuccess; };
  CUDA_TRY(dn(dx, v.dx, bn1 * nx));
  CUDA_TRY(dn(du, v.du, bn * nm));
  CUDA_TRY(dn(K, v.K, bn * nm * nx));
  CUDA_TRY(dn(k, v.kff, bn * nm));
  CUDA_TRY(dn(P, v.P, bn1 * nx * nx));
  CUDA_TRY(dn(p, v.p, bn1 * nx));
  std::vector<int> st(v.B);
  CUDA_TRY(cudaMemcpy(st.data(), v.status, v.B * sizeof(int), cudaMemcpyDeviceToHost));
  int bad = 0;
  for (int i = 0; i < v.B; ++i) {
    if (status) status[i] = st[i];
    bad += st[i] != 0;
  }
  if (bad) return fail(B200SQP_EQP, "[b200sqp] Failed to solve QP for %d of %d instances", bad, v.B);
  return 0;
}

int b200sqp_qp_last_ms(b200sqp_qp qp, float* ms) {
  if (!qp || !ms) return fail(B200SQP_EINVAL, "qp_last_ms: null argument");
  if (!qp->solved) return fail(B200SQP_ESTATE, "qp_last_ms: nothing solved yet");
  CUDA_TRY(cudaSetDevice(qp->device));
  CUDA_TRY(cudaEventSynchronize(qp->ev1));
  CUDA_TRY(cudaEventElapsedTime(ms, qp->ev0, qp->ev1));
  return 0;
}

void b200sqp_default_settings(b200sqp_settings* s) {
  if (!s) return;
  // sqp::Settings defaults (SqpSettings.h:42-86) overridden by G1 task.info:77-94
  s->sqp_iteration = 1;
  s->delta_tol = 1e-4;
  s->cost_tol = 1e-4;
  s->alpha_decay = 0.5;
  s->alpha_min = 1e-4;
  s->gamma_c = 1e-6;
  s->g_max = 1e-2;
  s->g_min = 1e-6;
  s->armijo_factor = 1e-4;
  s->reg_prim = 1e-12;
  s->use_feedback_policy = 0;
  s->global_step = 0;
  s->create_value_function = 0;
}

void b200sqp_default_rollout_settings(b200sqp_rollout_settings* rs) {
  if (!rs) return;
  // the rollout block of the G1 whole-body task.info (robot_models/unitree_g1/g1_wb_mpc/config/mpc/task.info:97-105)
  rs->abs_tol = 1e-5;
  rs->rel_tol = 1e-3;
  rs->time_step = 0.015;
  rs->max_steps_per_second = 10000;
}

}  // extern "C"

#ifdef B200SQP_WITH_WB
#include "wb_capi.inc"
#include "fleet_capi.inc"
#endif
