// tests/cpp/volume_oracle.cpp -- TEST INFRASTRUCTURE: the CPU oracle (oracle/dg_oracle.cpp, included unchanged) plus the volume map
// restated over the oracle's interpolate, written from the contract (DESIGN section 3, "Volume map"; the header of k3_density.cu) and not
// from the kernel: every Gauss point of the 16^3 rule is visited in the reference's order, the ones outside the ball return 0.0 without an
// interpolation, as the volume function does.  Built into build/bin/liborcvolume.so; the product never loads it.
#include "../../oracle/dg_oracle.cpp"

extern "C" {

void orc_volume_map(const double* gd, const uint32_t* res, const double* nodes, const uint32_t* cells, const uint32_t* cell_map, double h,
                    double scale, int no_reduction, uint64_t l_begin, uint64_t l_end, double* out, int nthreads)
{
    const Grid g = mkgrid(gd, res);
    CubicKernel ker; ker.set(h);
    const double w_zero = ker.W(0.0, 0.0, 0.0);                                      // CubicKernel::setRadius: m_W_zero = W(0)
    const double cell_diag = norm3_eigen(g.cell[0], g.cell[1], g.cell[2]);
    const double c0 = 0.5 * (h - (-h)), c1 = 0.5 * ((-h) + h);                        // integrate() over [-h, h]^3
    auto gamma = [&](double d) -> double {
        if (d <= 0.0) return 1.0;
        if (d < h) return ker.W(d, 0.0, 0.0) / w_zero;
        return 0.0;
    };
#ifdef _OPENMP
    if (nthreads > 0) omp_set_num_threads(nthreads);
#endif
#pragma omp parallel for schedule(dynamic, 16)
    for (long long l = (long long)l_begin; l < (long long)l_end; l++) {
        double x[3];
        index_to_node_position(g, (unsigned)l, x);
        bool keep = true;
        if (!no_reduction) {                                                          // GenerateDensityMap's predicate
            double xc[3];
            for (int d = 0; d < 3; d++) xc[d] = std::min(std::max(x[d], g.mn[d]), g.mx[d]);
            const double dist = interpolate(g, nodes, cells, cell_map, xc, nullptr);
            if (dist == DBL_MAX) keep = false;
            else keep = (-6.0 * h < dist + cell_diag) && (dist - cell_diag < 2.0 * h);
        }
        if (!keep) { out[l - l_begin] = DBL_MAX; continue; }
        const double dist = interpolate(g, nodes, cells, cell_map, x, nullptr);
        if (dist > (1.0 + 1.0) * h) { out[l - l_begin] = 0.0; continue; }
        double r = 0.0;
        for (int i = 0; i < 16; i++) {
            const double wi = GW16[i];
            const double yx = c0 * GA16[i] + c1;
            for (int j = 0; j < 16; j++) {
                const double wij = wi * GW16[j];
                const double yy = c0 * GA16[j] + c1;
                for (int k = 0; k < 16; k++) {
                    const double wijk = wij * GW16[k];
                    const double yz = c0 * GA16[k] + c1;
                    double gv = 0.0;
                    if (!((yx * yx + yy * yy) + yz * yz > h * h)) {
                        const double xs[3] = {x[0] + yx, x[1] + yy, x[2] + yz};
                        gv = gamma(interpolate(g, nodes, cells, cell_map, xs, nullptr));
                    }
                    r += wijk * gv;
                }
            }
        }
        r *= c0 * c0 * c0;
        out[l - l_begin] = scale * r;
    }
}

}  // extern "C"
