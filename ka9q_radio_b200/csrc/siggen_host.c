/* siggen_host.c -- the host half of the sig_gen carrier (csrc/siggen.cuh): the exact angle of the oscillator step as
 * set_osc rounds it.  C rather than CUDA because it needs binary128 arithmetic (libquadmath). */
#include <math.h>
#include <quadmath.h>
#include <stdbool.h>
#include <stdint.h>

/* sincospi as the reference states it (sincospi.c): reduce x to [0, 2), then to [0, 0.25] by symmetry, then libm's sin
 * and cos of pi z.  Every reduction step is exact, so the doubles are those set_osc's cispi (misc.h:273-277) stores. */
static double mod2(double x) {
  x -= floor(x * 0.5) * 2.0;
  if (x < 0)
    x += 2.0;
  if (x >= 2.0)
    x -= 2.0;
  return x;
}
static void ref_sincospi(double x, double *s, double *c) {
  double const y = mod2(x);
  int const q = (int)(2.0 * y);
  double z = y - 0.5 * q;
  bool flip = false;
  if (z > 0.25) {
    z = 0.5 - z;
    flip = true;
  }
  double const piz = 3.141592653589793238462643383279502884 * z;
  double ss = sin(piz), cc = cos(piz);
  if (flip) {
    double const t = ss;
    ss = cc;
    cc = t;
  }
  switch (q) {
  case 0: *s = ss; *c = cc; break;
  case 1: *s = cc; *c = -ss; break;
  case 2: *s = -ss; *c = -cc; break;
  default: *s = -cc; *c = ss; break;
  }
}

/* The angle of the phasor set_osc(f) steps by, cispi(2 f) rounded to doubles (osc.c:37-44), in cycles mod 1, as a
 * 128-bit fraction: out[0] the low and out[1] the high 64 bits.  f = 0 leaves the step at 1 (angle 0), as set_osc does. */
void kgpu_siggen_angle128(double f, uint64_t *out) {
  out[0] = out[1] = 0;
  if (f == 0)
    return;
  double s, c;
  ref_sincospi(2 * f, &s, &c);
  __float128 a = atan2q((__float128)s, (__float128)c) / (2 * M_PIq);
  if (a < 0)
    a += 1;
  __float128 const x = ldexpq(a, 64), h = floorq(x);
  out[1] = (uint64_t)h;
  out[0] = (uint64_t)floorq(ldexpq(x - h, 64));
}
