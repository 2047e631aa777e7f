/* Oracle (TEST INFRASTRUCTURE): plain-C restatement of box voting (Detectron's TEST.BBOX_VOTE) as include/frcnn_b200.h defines
 * it for frcnn_box_vote_host / frcnn_detect_post_vote: scalar, single thread, every fp32 operation a separate IEEE round-to-nearest
 * op (build with -ffp-contract=off), the fp64 sums in the header's order (32 partials by candidate index mod 32, then the xor
 * butterfly), exp / log / pow in fp64.
 *
 * top: [n_top,5], all: [n_all,5] rows (x1,y1,x2,y2,score).  out: [n_top,5], the voted rows in top's order.  method: the
 * FRCNN_BOX_VOTE_* code.  variant: 0 is the definition; the bits select deliberate mistakes that the tests must catch
 * (1: ov > thresh instead of >=, 2: areas without the '+1', 4: fp32 instead of fp64 accumulation). */
#include <math.h>
#include <stddef.h>

enum { ID = 0, AVG = 1, IOU_AVG = 2, GENERALIZED_AVG = 3, QUASI_SUM = 4, TEMP_AVG = 5 };
enum { ACC = 7 };   /* S, X1, Y1, X2, Y2, M0, M1 */

static float area_(const float* u, int plus1) {
  const float one = plus1 ? 1.0f : 0.0f;
  return ((u[2] - u[0]) + one) * ((u[3] - u[1]) + one);
}

/* the overlap of the header, 0 when the boxes do not overlap */
static float overlap_(const float* t, const float* a, int plus1) {
  const float one = plus1 ? 1.0f : 0.0f;
  const float iw = (fminf(t[2], a[2]) - fmaxf(t[0], a[0])) + one;
  if (!(iw > 0.0f)) return 0.0f;
  const float ih = (fminf(t[3], a[3]) - fmaxf(t[1], a[1])) + one;
  if (!(ih > 0.0f)) return 0.0f;
  const float inter = iw * ih;
  return inter / ((area_(t, plus1) + area_(a, plus1)) - inter);
}

static double rnd_(double v, int f32) { return f32 ? (double)(float)v : v; }

void oracle_box_vote(const float* top, int n_top, const float* all, int n_all, float thresh, int method, float beta, int variant,
                     float* out) {
  const int strict = variant & 1, plus1 = !(variant & 2), f32 = (variant & 4) != 0;
  for (int i = 0; i < n_top; ++i) {
    const float* t = top + (size_t)i * 5;
    double P[ACC][32];
    int n = 0;
    for (int q = 0; q < ACC; ++q)
      for (int l = 0; l < 32; ++l) P[q][l] = 0.0;
    for (int k = 0; k < n_all; ++k) {
      const float* a = all + (size_t)k * 5;
      const float ov = overlap_(t, a, plus1);
      if (strict ? !(ov > thresh) : !(ov >= thresh)) continue;
      const int l = k & 31;
      const double s = (double)a[4];
      double term[ACC] = {s, s * (double)a[0], s * (double)a[1], s * (double)a[2], s * (double)a[3], 0.0, 0.0};
      if (method == IOU_AVG) {
        term[5] = (double)ov * s;
        term[6] = (double)ov;
      } else if (method == GENERALIZED_AVG) {
        term[5] = exp((double)beta * s);
      } else if (method == TEMP_AVG) {
        const double qq = 1.0 - s, m = fmax(s, qq), b = (double)beta;
        const double e0 = exp(log(s / m) / b), e1 = exp(log(qq / m) / b);
        term[5] = e0 / (e0 + e1);
      }
      for (int q = 0; q < ACC; ++q) P[q][l] = rnd_(P[q][l] + rnd_(term[q], f32), f32);
      n += 1;
    }
    double R[ACC];
    for (int q = 0; q < ACC; ++q) {
      for (int o = 16; o; o >>= 1) {
        double nx[32];
        for (int l = 0; l < 32; ++l) nx[l] = rnd_(P[q][l] + P[q][l ^ o], f32);
        for (int l = 0; l < 32; ++l) P[q][l] = nx[l];
      }
      R[q] = P[q][0];
    }
    float* o = out + (size_t)i * 5;
    o[0] = t[0]; o[1] = t[1]; o[2] = t[2]; o[3] = t[3]; o[4] = t[4];
    if (n == 0) continue;
    if (R[0] != 0.0) {
      o[0] = (float)(R[1] / R[0]); o[1] = (float)(R[2] / R[0]); o[2] = (float)(R[3] / R[0]); o[3] = (float)(R[4] / R[0]);
    }
    const double dn = (double)n, b = (double)beta;
    switch (method) {
      case AVG: o[4] = (float)(R[0] / dn); break;
      case IOU_AVG: o[4] = (float)(R[5] / R[6]); break;
      case GENERALIZED_AVG: o[4] = (float)(log(R[5] / dn) / b); break;
      case QUASI_SUM: o[4] = (float)(R[0] / (b == 1.0 ? dn : b == 2.0 ? dn * dn : b == 0.5 ? sqrt(dn) : pow(dn, b))); break;
      case TEMP_AVG: o[4] = (float)(R[5] / dn); break;
      default: break;
    }
  }
}
