// k5_atan2 of K5's contract (k5_winding.cu): atan2 written with IEEE + - * / sqrt and comparisons only, so that the device, the CPU
// emulation and a numpy restatement agree bit for bit.  Shared by K5 and by the refit's pseudonormal angles (k8_refit.cu).
#pragma once
#include "dg_device.cuh"

namespace dgb {

namespace k5 {
constexpr double PI = 3.1415926535897931160E+00, PI_LO = 1.2246467991473531772E-16;
constexpr double PI_2 = 1.5707963267948965580E+00, PI_4 = 7.8539816339744827900E-01, PI3_4 = 2.3561944901923448370E+00;
constexpr double FOUR_PI = 12.566370614359172;
constexpr double AT0 = 3.33333333333329318027e-01, AT1 = -1.99999999998764832476e-01, AT2 = 1.42857142725034663711e-01,
                 AT3 = -1.11111104054623557880e-01, AT4 = 9.09088713343650656196e-02, AT5 = -7.69187620504482999495e-02,
                 AT6 = 6.66107313738753120669e-02, AT7 = -5.83357013379057348645e-02, AT8 = 4.97687799461593236017e-02,
                 AT9 = -3.65315727442169155270e-02, AT10 = 1.62858201153657823623e-02;
}  // namespace k5

// sign bit without a bit cast: a zero is negative iff 1/v is -inf
DG_HD bool k5_neg(double v) { return v < 0.0 || (v == 0.0 && 1.0 / v < 0.0); }

// atan(t) for 0 <= t <= 2^60 (fdlibm's reduction and polynomial)
DG_HD double k5_atan_pos(double t)
{
    using namespace k5;
    double x, hi = 0.0, lo = 0.0;
    int id;
    if (t < 0.4375) {
        if (t < 0x1p-29) return t;
        id = -1; x = t;
    } else if (t < 0.6875) {
        id = 0; x = (2.0 * t - 1.0) / (2.0 + t); hi = 4.63647609000806093515e-01; lo = 2.26987774529616870924e-17;
    } else if (t < 1.1875) {
        id = 1; x = (t - 1.0) / (t + 1.0); hi = 7.85398163397448278999e-01; lo = 3.06161699786838301793e-17;
    } else if (t < 2.4375) {
        id = 2; x = (t - 1.5) / (1.0 + 1.5 * t); hi = 9.82793723247329054082e-01; lo = 1.39033110312309984516e-17;
    } else {
        id = 3; x = -1.0 / t; hi = 1.57079632679489655800e+00; lo = 6.12323399573676603587e-17;
    }
    const double z = x * x, w = z * z;
    const double s1 = z * (AT0 + w * (AT2 + w * (AT4 + w * (AT6 + w * (AT8 + w * AT10)))));
    const double s2 = w * (AT1 + w * (AT3 + w * (AT5 + w * (AT7 + w * AT9))));
    if (id < 0) return x - x * (s1 + s2);
    return hi - ((x * (s1 + s2) - lo) - x);
}

DG_HD double k5_atan2(double y, double x)
{
    using namespace k5;
    if (x != x || y != y) return x + y;
    const double ax = (x < 0.0) ? -x : x, ay = (y < 0.0) ? -y : y;
    const bool nx = k5_neg(x), ny = k5_neg(y);
    if (ay == 0.0) return nx ? (ny ? -PI : PI) : y;
    if (ax == 0.0) return ny ? -PI_2 : PI_2;
    if (ax == INFINITY) {
        if (ay == INFINITY) return nx ? (ny ? -PI3_4 : PI3_4) : (ny ? -PI_4 : PI_4);
        return nx ? (ny ? -PI : PI) : (ny ? -0.0 : 0.0);
    }
    if (ay == INFINITY) return ny ? -PI_2 : PI_2;
    const double q = ay / ax;
    if (q > 0x1p60) return ny ? -PI_2 : PI_2;
    const double z = (nx && q < 0x1p-60) ? 0.0 : k5_atan_pos(q);
    if (!nx) return ny ? -z : z;
    const double r = PI - (z - PI_LO);
    return ny ? -r : r;
}

}  // namespace dgb
