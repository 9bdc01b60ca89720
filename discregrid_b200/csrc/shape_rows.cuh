// The 32 rows of shape_function_ (cubic_lagrange_discrete_grid.cpp:339-580) at one reference-cell point xi = (X, Y, Z), as one __device__
// definition shared by shape_functions_kernel (K2, dg_shape_functions) and K11's vector-Jacobian product (k11_field_grad.cu).
//
// shape_rows(X, Y, Z, row) calls row(j, N_j, D_j0, D_j1, D_j2) for j = 0 .. 31 in that order.  N_j is the expression K2's value sum
// multiplies c_j by, e.g. (facc*mxmy)*_1mz; D_jk the scaled derivative row its gradient sum multiplies c_j by, e.g. (xmA*mymz)*0.015625
// (corners, == /64 exactly) or (...)*(9.0/64.0) (edges): the same expressions, in the same operation order, as interpolate_kernel's
// DG_CORNER / DG_EDGE terms.  interpolate_kernel keeps its own copy of them, interleaved with its coefficient loads.
#pragma once

namespace dgb {
namespace {

template <class Row>
__device__ __forceinline__ void shape_rows(const double X, const double Y, const double Z, Row&& row)
{
    const double x2 = X * X, y2 = Y * Y, z2 = Z * Z;
    const double _1mx = 1.0 - X, _1my = 1.0 - Y, _1mz = 1.0 - Z;
    const double _1px = 1.0 + X, _1py = 1.0 + Y, _1pz = 1.0 + Z;
    const double _1m3x = 1.0 - 3.0 * X, _1m3y = 1.0 - 3.0 * Y, _1m3z = 1.0 - 3.0 * Z;
    const double _1p3x = 1.0 + 3.0 * X, _1p3y = 1.0 + 3.0 * Y, _1p3z = 1.0 + 3.0 * Z;
    const double mxmy = _1mx * _1my, mxpy = _1mx * _1py, pxmy = _1px * _1my, pxpy = _1px * _1py;
    const double mxmz = _1mx * _1mz, mxpz = _1mx * _1pz, pxmz = _1px * _1mz, pxpz = _1px * _1pz;
    const double mymz = _1my * _1mz, mypz = _1my * _1pz, pymz = _1py * _1mz, pypz = _1py * _1pz;
    const double _1mx2 = 1.0 - x2, _1my2 = 1.0 - y2, _1mz2 = 1.0 - z2;
    const double facc = 1.0 / 64.0 * (9.0 * (x2 + y2 + z2) - 19.0);
    const double fx = 9.0 / 64.0 * _1mx2, fy = 9.0 / 64.0 * _1my2, fz = 9.0 / 64.0 * _1mz2;
    const double fxm = fx * _1m3x, fxp = fx * _1p3x, fym = fy * _1m3y, fyp = fy * _1p3y, fzm = fz * _1m3z, fzp = fz * _1p3z;
    const double A = 9.0 * (3.0 * x2 + y2 + z2) - 19.0, B = 9.0 * (x2 + 3.0 * y2 + z2) - 19.0, C = 9.0 * (x2 + y2 + 3.0 * z2) - 19.0;
    const double _18x = 18.0 * X, _18y = 18.0 * Y, _18z = 18.0 * Z;
    const double xmA = _18x - A, xpA = _18x + A, ymB = _18y - B, ypB = _18y + B, zmC = _18z - C, zpC = _18z + C;
    const double _3m9x2 = 3.0 - 9.0 * x2, _3m9y2 = 3.0 - 9.0 * y2, _3m9z2 = 3.0 - 9.0 * z2;
    const double _2x = 2.0 * X, _2y = 2.0 * Y, _2z = 2.0 * Z;
    const double mX = -_3m9x2 - _2x, pX = _3m9x2 - _2x, Xm = _1mx2 * _1m3x, Xp = _1mx2 * _1p3x;
    const double mY = -_3m9y2 - _2y, pY = _3m9y2 - _2y, Ym = _1my2 * _1m3y, Yp = _1my2 * _1p3y;
    const double mZ = -_3m9z2 - _2z, pZ = _3m9z2 - _2z, Zm = _1mz2 * _1m3z, Zp = _1mz2 * _1p3z;
#define DG_ROW(j, n, dx, dy, dz, SC) row(j, (n), SC(dx), SC(dy), SC(dz));
#define DG_SC_C(v) ((v) * 0.015625)   /* == /64.0 exactly */
#define DG_SC_E(v) ((v) * (9.0 / 64.0))
    DG_ROW(0, facc * mxmy * _1mz, xmA * mymz, mxmz * ymB, mxmy * zmC, DG_SC_C)
    DG_ROW(1, facc * pxmy * _1mz, xpA * mymz, pxmz * ymB, pxmy * zmC, DG_SC_C)
    DG_ROW(2, facc * mxpy * _1mz, xmA * pymz, mxmz * ypB, mxpy * zmC, DG_SC_C)
    DG_ROW(3, facc * pxpy * _1mz, xpA * pymz, pxmz * ypB, pxpy * zmC, DG_SC_C)
    DG_ROW(4, facc * mxmy * _1pz, xmA * mypz, mxpz * ymB, mxmy * zpC, DG_SC_C)
    DG_ROW(5, facc * pxmy * _1pz, xpA * mypz, pxpz * ymB, pxmy * zpC, DG_SC_C)
    DG_ROW(6, facc * mxpy * _1pz, xmA * pypz, mxpz * ypB, mxpy * zpC, DG_SC_C)
    DG_ROW(7, facc * pxpy * _1pz, xpA * pypz, pxpz * ypB, pxpy * zpC, DG_SC_C)
    DG_ROW(8, fxm * mymz, mX * mymz, -Xm * _1mz, -Xm * _1my, DG_SC_E)
    DG_ROW(9, fxp * mymz, pX * mymz, -Xp * _1mz, -Xp * _1my, DG_SC_E)
    DG_ROW(10, fxm * mypz, mX * mypz, -Xm * _1pz, Xm * _1my, DG_SC_E)
    DG_ROW(11, fxp * mypz, pX * mypz, -Xp * _1pz, Xp * _1my, DG_SC_E)
    DG_ROW(12, fxm * pymz, mX * pymz, Xm * _1mz, -Xm * _1py, DG_SC_E)
    DG_ROW(13, fxp * pymz, pX * pymz, Xp * _1mz, -Xp * _1py, DG_SC_E)
    DG_ROW(14, fxm * pypz, mX * pypz, Xm * _1pz, Xm * _1py, DG_SC_E)
    DG_ROW(15, fxp * pypz, pX * pypz, Xp * _1pz, Xp * _1py, DG_SC_E)
    DG_ROW(16, fym * mxmz, -Ym * _1mz, mY * mxmz, -Ym * _1mx, DG_SC_E)
    DG_ROW(17, fyp * mxmz, -Yp * _1mz, pY * mxmz, -Yp * _1mx, DG_SC_E)
    DG_ROW(18, fym * pxmz, Ym * _1mz, mY * pxmz, -Ym * _1px, DG_SC_E)
    DG_ROW(19, fyp * pxmz, Yp * _1mz, pY * pxmz, -Yp * _1px, DG_SC_E)
    DG_ROW(20, fym * mxpz, -Ym * _1pz, mY * mxpz, Ym * _1mx, DG_SC_E)
    DG_ROW(21, fyp * mxpz, -Yp * _1pz, pY * mxpz, Yp * _1mx, DG_SC_E)
    DG_ROW(22, fym * pxpz, Ym * _1pz, mY * pxpz, Ym * _1px, DG_SC_E)
    DG_ROW(23, fyp * pxpz, Yp * _1pz, pY * pxpz, Yp * _1px, DG_SC_E)
    DG_ROW(24, fzm * mxmy, -Zm * _1my, -Zm * _1mx, mZ * mxmy, DG_SC_E)
    DG_ROW(25, fzp * mxmy, -Zp * _1my, -Zp * _1mx, pZ * mxmy, DG_SC_E)
    DG_ROW(26, fzm * mxpy, -Zm * _1py, Zm * _1mx, mZ * mxpy, DG_SC_E)
    DG_ROW(27, fzp * mxpy, -Zp * _1py, Zp * _1mx, pZ * mxpy, DG_SC_E)
    DG_ROW(28, fzm * pxmy, Zm * _1my, -Zm * _1px, mZ * pxmy, DG_SC_E)
    DG_ROW(29, fzp * pxmy, Zp * _1my, -Zp * _1px, pZ * pxmy, DG_SC_E)
    DG_ROW(30, fzm * pxpy, Zm * _1py, Zm * _1px, mZ * pxpy, DG_SC_E)
    DG_ROW(31, fzp * pxpy, Zp * _1py, Zp * _1px, pZ * pxpy, DG_SC_E)
#undef DG_ROW
#undef DG_SC_C
#undef DG_SC_E
}

}  // namespace
}  // namespace dgb
