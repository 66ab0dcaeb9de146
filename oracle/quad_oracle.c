/* TEST INFRASTRUCTURE -- NOT PRODUCT CODE.  Three precisions of the quadrotor oracle, see quad_oracle_impl.h.
 * Build: see oracle/Makefile (gcc -O2 -ffp-contract=off: numpy does not fuse multiply-add in its scalar/ufunc loops).
 */
#include <math.h>
#include "quad_oracle.h"

/* Obstacle map of Quadrotor._check_collision (env.py:248-260): summed-area table of non-zero cells, set by
 * qo_set_map() for the next env_step calls (test infrastructure: a process-global is enough). */
static const int *qo_sat = 0;
static int qo_rows = 0, qo_cols = 0, qo_xoff = 0, qo_yoff = 0;
void qo_set_map(const int *sat, int rows, int cols, int xoff, int yoff)
{
    qo_sat = sat; qo_rows = rows; qo_cols = cols; qo_xoff = xoff; qo_yoff = yoff;
}
static int qo_slice(double v, int len)
{
    long long x = (long long)v;
    if (x < 0) { x += len; if (x < 0) x = 0; }
    if (x > len) x = len;
    return (int)x;
}
/* `np.any(map[y_min:y_max+1, x_min:x_max+1])` for the window swept between two positions */
static int qo_any_obstacle(double xo, double yo, double xn, double yn)
{
    const double x_min = floor(xo < xn ? xo : xn), x_max = ceil(xo > xn ? xo : xn);
    const double y_min = floor(yo < yn ? yo : yn), y_max = ceil(yo > yn ? yo : yn);
    const int ys = qo_slice(y_min, qo_rows), ye = qo_slice(y_max + 1.0, qo_rows);
    const int xs = qo_slice(x_min, qo_cols), xe = qo_slice(x_max + 1.0, qo_cols);
    if (!(ys < ye && xs < xe)) return 0;
    const int W = qo_cols + 1;
    return (qo_sat[ye * W + xe] - qo_sat[ys * W + xe] - qo_sat[ye * W + xs] + qo_sat[ys * W + xs]) > 0;
}
/* the same, exported for tests that check the window against a literal numpy slice of the map */
int qo_map_any_obstacle(double xo, double yo, double xn, double yn) { return qo_any_obstacle(xo, yo, xn, yn); }

#define QO_CAT2(a, b) a##b
#define QO_CAT(a, b) QO_CAT2(a, b)

/* ---- all float32: a simulator that was never reset() (velocity-task generator) ---- */
#define T float
#define TV float
#define QO_NAME(x) QO_CAT(qo_f32_, x)
#define QO_SQRTT sqrtf
#define QO_SQRTV sqrtf
#define QO_ATAN2T atan2f
#define QO_FLOORT floorf
#define QO_CEILT ceilf
#include "quad_oracle_impl.h"
#undef T
#undef TV
#undef QO_NAME
#undef QO_SQRTT
#undef QO_SQRTV
#undef QO_ATAN2T
#undef QO_FLOORT
#undef QO_CEILT

/* ---- mixed: float32 state with float64 velocity vectors (after reset()) ---- */
#define T float
#define TV double
#define QO_NAME(x) QO_CAT(qo_mix_, x)
#define QO_SQRTT sqrtf
#define QO_SQRTV sqrt
#define QO_ATAN2T atan2f
#define QO_FLOORT floorf
#define QO_CEILT ceilf
#include "quad_oracle_impl.h"
#undef T
#undef TV
#undef QO_NAME
#undef QO_SQRTT
#undef QO_SQRTV
#undef QO_ATAN2T
#undef QO_FLOORT
#undef QO_CEILT

/* ---- all float64: arbiter ---- */
#define T double
#define TV double
#define QO_NAME(x) QO_CAT(qo_f64_, x)
#define QO_SQRTT sqrt
#define QO_SQRTV sqrt
#define QO_ATAN2T atan2
#define QO_FLOORT floor
#define QO_CEILT ceil
#include "quad_oracle_impl.h"
