/* CPU oracle for the halo-exchange / jacobi3d hot path of cwpearson/stencil -- plain C (+OpenMP).
 *
 * TEST INFRASTRUCTURE ONLY (see oracle/__init__.py): used by tests/ as the checker and by
 * bench.py as the timed CPU baseline ("port").  The product (stencil_b200/, src/, include/)
 * never links or loads this file.
 *
 * All citations are relative to the reference checkout.  Layout: x fastest, unpitched rows
 * (src/local_domain.cu:187-203), element (x,y,z) of an allocation with raw size (nx,ny,nz)
 * lives at byte offset ((z*ny + y)*nx + x)*elem_size.
 *
 * Parity status: pinned for data movement (golden vectors of test/test_cuda_pack.cu and
 * test/test_cuda_packer.cu, cross-checked against oracle/np_oracle.py); jacobi numerics are
 * unpinned in the reference (no test, SURVEY.md 8c) -- this file and np_oracle.py are two
 * independent restatements of bin/jacobi3d.cu:40-85 that must agree bit for bit.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#ifdef _OPENMP
#include <omp.h>
#endif

typedef struct {
  int64_t x, y, z;
} so_vec;

int so_num_threads(void) {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}

void so_set_num_threads(int n) {
#ifdef _OPENMP
  omp_set_num_threads(n);
#else
  (void)n;
#endif
}

/* strided -> strided copy of the box [spos, spos+ext) of src into [dpos, dpos+ext) of dst.
 * translate_grid, src/copy.cu:34-77.  pack (src/pack_kernel.cu:3-59) is the special case where
 * dst is a dense (ext.x, ext.y, ext.z) array at dpos 0; unpack (:61-108) the mirror. */
void so_translate(uint8_t *dst, so_vec draw, so_vec dpos, const uint8_t *src, so_vec sraw, so_vec spos, so_vec ext,
                  int64_t es) {
  const int64_t row = ext.x * es;
  if (row <= 0 || ext.y <= 0 || ext.z <= 0) return;
#pragma omp parallel for collapse(2) schedule(static)
  for (int64_t z = 0; z < ext.z; ++z) {
    for (int64_t y = 0; y < ext.y; ++y) {
      const uint8_t *s = src + (((spos.z + z) * sraw.y + (spos.y + y)) * sraw.x + spos.x) * es;
      uint8_t *d = dst + (((dpos.z + z) * draw.y + (dpos.y + y)) * draw.x + dpos.x) * es;
      memcpy(d, s, (size_t)row);
    }
  }
}

void so_pack(uint8_t *buf, const uint8_t *src, so_vec sraw, so_vec spos, so_vec ext, int64_t es) {
  so_vec zero = {0, 0, 0};
  so_translate(buf, ext, zero, src, sraw, spos, ext, es);
}

void so_unpack(uint8_t *dst, so_vec draw, so_vec dpos, const uint8_t *buf, so_vec ext, int64_t es) {
  so_vec zero = {0, 0, 0};
  so_translate(dst, draw, dpos, buf, ext, zero, ext, es);
}

/* A batch of box copies -- one halo exchange in a single address space is a list of these
 * (plan of src/stencil.cu:327-412 computed by oracle/geometry.py:plan_sends). */
typedef struct {
  uint8_t *dst;
  const uint8_t *src;
  so_vec draw, dpos, sraw, spos, ext;
  int64_t es;
} so_copy;

void so_translate_many(const so_copy *c, int64_t n) {
  for (int64_t i = 0; i < n; ++i) so_translate(c[i].dst, c[i].draw, c[i].dpos, c[i].src, c[i].sraw, c[i].spos, c[i].ext, c[i].es);
}

/* ------------------------------------------------------------------------------------------- jacobi
 * stencil_kernel, bin/jacobi3d.cu:40-85.  dist() (:31-33) = int64(sqrtf(float(d2))).
 * A row (fixed y,z) can only touch a sphere of radius R around c if (y-cy)^2+(z-cz)^2 < (R+1)^2
 * (then some x has floor(sqrt(d2)) <= R); rows that cannot are processed by the branch-free loop.
 * This is an exact pre-filter: for rows it rejects, d2 >= (R+1)^2 for every x so sqrtf(d2) >= R+1.
 */
#define SO_JACOBI(NAME, T)                                                                                              \
  void NAME(T *dst, const T *src, so_vec raw, so_vec acc_origin, so_vec lo, so_vec hi, so_vec clo, so_vec chi) {        \
    const int64_t ex = chi.x - clo.x;                                                                                   \
    const int64_t hx = clo.x + ex / 3, cx = clo.x + ex * 2 / 3;                                                         \
    const int64_t cy = (clo.y + chi.y) / 2, cz = (clo.z + chi.z) / 2;                                                   \
    const int64_t R = ex / 10;                                                                                          \
    const int64_t sx = 1, sy = raw.x, sz = raw.x * raw.y;                                                               \
    if (hi.x <= lo.x || hi.y <= lo.y || hi.z <= lo.z) return;                                                           \
    _Pragma("omp parallel for collapse(2) schedule(static)") for (int64_t z = lo.z; z < hi.z; ++z) {                    \
      for (int64_t y = lo.y; y < hi.y; ++y) {                                                                           \
        const int64_t base = ((z - acc_origin.z) * raw.y + (y - acc_origin.y)) * raw.x - acc_origin.x;                  \
        const T *s = src + base;                                                                                        \
        T *d = dst + base;                                                                                              \
        const int64_t dyz = (y - cy) * (y - cy) + (z - cz) * (z - cz);                                                  \
        if (dyz >= (R + 1) * (R + 1)) {                                                                                 \
          for (int64_t x = lo.x; x < hi.x; ++x) {                                                                       \
            T v = (T)0;                                                                                                 \
            v += s[x + sx];                                                                                             \
            v += s[x - sx];                                                                                             \
            v += s[x + sy];                                                                                             \
            v += s[x - sy];                                                                                             \
            v += s[x + sz];                                                                                             \
            v += s[x - sz];                                                                                             \
            d[x] = v / (T)6;                                                                                            \
          }                                                                                                             \
        } else {                                                                                                        \
          for (int64_t x = lo.x; x < hi.x; ++x) {                                                                       \
            const int64_t dh = (x - hx) * (x - hx) + dyz, dc = (x - cx) * (x - cx) + dyz;                               \
            if ((int64_t)sqrtf((float)dh) <= R) {                                                                       \
              d[x] = (T)1;                                                                                              \
            } else if ((int64_t)sqrtf((float)dc) <= R) {                                                                \
              d[x] = (T)0;                                                                                              \
            } else {                                                                                                    \
              T v = (T)0;                                                                                               \
              v += s[x + sx];                                                                                           \
              v += s[x - sx];                                                                                           \
              v += s[x + sy];                                                                                           \
              v += s[x - sy];                                                                                           \
              v += s[x + sz];                                                                                           \
              v += s[x - sz];                                                                                           \
              d[x] = v / (T)6;                                                                                          \
            }                                                                                                           \
          }                                                                                                             \
        }                                                                                                               \
      }                                                                                                                 \
    }                                                                                                                   \
  }

SO_JACOBI(so_jacobi_f32, float)
SO_JACOBI(so_jacobi_f64, double)

/* init_kernel, bin/jacobi3d.cu:18-29: compute region := (HOT+COLD)/2 = 0.5 */
#define SO_FILL(NAME, T)                                                                                                \
  void NAME(T *dst, so_vec raw, so_vec pos, so_vec ext, T v) {                                                          \
    _Pragma("omp parallel for collapse(2) schedule(static)") for (int64_t z = 0; z < ext.z; ++z) {                      \
      for (int64_t y = 0; y < ext.y; ++y) {                                                                             \
        T *d = dst + ((pos.z + z) * raw.y + (pos.y + y)) * raw.x + pos.x;                                               \
        for (int64_t x = 0; x < ext.x; ++x) d[x] = v;                                                                   \
      }                                                                                                                 \
    }                                                                                                                   \
  }
SO_FILL(so_fill_f32, float)
SO_FILL(so_fill_f64, double)

/* sum over a box of (a-b)^2 in double (the new FP64 residual requirement, SURVEY.md 8d).
 * Deterministic: per-(z,y)-row partial sums added in row order by one thread at the end. */
#define SO_SQDIFF(NAME, T)                                                                                              \
  double NAME(const T *a, const T *b, so_vec raw, so_vec pos, so_vec ext) {                                             \
    const int64_t rows = ext.y * ext.z;                                                                                 \
    if (rows <= 0 || ext.x <= 0) return 0.0;                                                                            \
    double *part = (double *)malloc(sizeof(double) * (size_t)rows);                                                     \
    _Pragma("omp parallel for schedule(static)") for (int64_t r = 0; r < rows; ++r) {                                   \
      const int64_t z = r / ext.y, y = r % ext.y;                                                                       \
      const int64_t o = ((pos.z + z) * raw.y + (pos.y + y)) * raw.x + pos.x;                                            \
      double acc = 0.0;                                                                                                 \
      for (int64_t x = 0; x < ext.x; ++x) {                                                                             \
        const double d = (double)a[o + x] - (double)b[o + x];                                                           \
        acc += d * d;                                                                                                   \
      }                                                                                                                 \
      part[r] = acc;                                                                                                    \
    }                                                                                                                   \
    double tot = 0.0;                                                                                                   \
    for (int64_t r = 0; r < rows; ++r) tot += part[r];                                                                  \
    free(part);                                                                                                         \
    return tot;                                                                                                         \
  }
SO_SQDIFF(so_sqdiff_f32, float)
SO_SQDIFF(so_sqdiff_f64, double)
