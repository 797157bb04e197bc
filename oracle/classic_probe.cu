// TEST INFRASTRUCTURE ONLY: classic.cu's own sin / cos helpers (epb::M<R>) behind a C ABI, so
// that a host model of the classic_control steps can take every sin and cos value from the
// device for the same argument, and the helpers themselves can be measured against a
// high-precision reference.  Nothing is restated here: the kernels call the engine's functions,
// compiled with classic.cu's own flags (oracle/classic_lib.py).
//
// Every launcher maps n arguments x[i] to s[i] (sin) and / or c[i] (cos) on `stream` and
// returns the launch's cudaError_t.  sin_ writes s only, cos_ c only.
#include "../envpool_b200/csrc/classic.cu"

namespace {

enum Fn { kSincosSmall, kSin, kCos, kSincos };

template <typename R, int F>
__global__ void trig_kernel(const R* __restrict__ x, R* __restrict__ s, R* __restrict__ c,
                            int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const R v = x[i];
  if (F == kSincosSmall) {
    R sn, cs;
    epb::M<R>::sincos_small_(v, &sn, &cs);
    s[i] = sn;
    c[i] = cs;
  } else if (F == kSin) {
    s[i] = epb::M<R>::sin_(v);
  } else if (F == kCos) {
    c[i] = epb::M<R>::cos_(v);
  } else {
    R sn, cs;
    epb::M<R>::sincos_(v, &sn, &cs);
    s[i] = sn;
    c[i] = cs;
  }
}

template <typename R, int F>
int launch(const R* x, R* s, R* c, int n, cudaStream_t stream) {
  if (n <= 0) return 0;
  trig_kernel<R, F><<<(n + 255) / 256, 256, 0, stream>>>(x, s, c, n);
  return (int)cudaGetLastError();
}

}  // namespace

#define EPB_PROBE(name, R, F)                                                       \
  extern "C" int name(const R* x, R* s, R* c, int n, cudaStream_t stream) {         \
    return launch<R, F>(x, s, c, n, stream);                                        \
  }
EPB_PROBE(classic_probe_sincos_small_f64, double, kSincosSmall)
EPB_PROBE(classic_probe_sin_f64, double, kSin)
EPB_PROBE(classic_probe_cos_f64, double, kCos)
EPB_PROBE(classic_probe_sincos_f64, double, kSincos)
EPB_PROBE(classic_probe_sincos_small_f32, float, kSincosSmall)
EPB_PROBE(classic_probe_sin_f32, float, kSin)
EPB_PROBE(classic_probe_cos_f32, float, kCos)
EPB_PROBE(classic_probe_sincos_f32, float, kSincos)
#undef EPB_PROBE
