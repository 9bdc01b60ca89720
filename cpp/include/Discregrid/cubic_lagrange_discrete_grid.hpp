// Discregrid::CubicLagrangeDiscreteGrid -- the reference's public surface and members
// (discregrid/include/Discregrid/cubic_lagrange_discrete_grid.hpp:8-72) with the hot path on the H100:
//
//   addFunction(MeshSignedDistanceFunction)  -> dg_add_function_sdf (K1)   replaces the OpenMP node loop :806-831
//   addFunction(MeshSignedDistanceFunction, verbose, MeshDistanceBandPredicate)
//                                            -> dg_add_function_sdf_band (K1, narrow band: DBL_MAX where |distance| > band, :811-817)
//   addReducedBandField(MeshSignedDistanceFunction, MeshDistanceBandPredicate)
//                                            -> dg_reduced_band_create (the same band + reduceField(always true), on the GPU)
//   addFunction(DensityMapFunction)          -> dg_density_map  (K3)   (GenerateDensityMap's functor + predicate)
//   addReducedDensityMap(DensityMapFunction) -> dg_reduced_density_map_create (K3 + both of GenerateDensityMap's reduceField calls, on the GPU)
//   addFunction(VolumeMapFunction)           -> dg_volume_map   (K3's volume-map kernel: SPH boundary volumes; not in the reference)
//   addReducedVolumeMap(VolumeMapFunction)   -> dg_reduced_volume_map_create (the volume map + reduceField(0, p0) + reduceField(id, 0 <= v))
//   addFunction(DeviceFunction, verbose, DeviceSamplePredicate)
//                                            -> dg_add_function_device (the caller's own GPU code on batches of node positions)
//   reduceField(field, DeviceNodePredicate)  -> dg_reduce_field_device (the caller's predicate on the GPU, reduceField's passes there)
//   addReducedFunction(DeviceFunction, DeviceSamplePredicate*, DeviceNodePredicate*)
//                                            -> dg_reduced_function_create (both calls in one, the dense field kept on the GPU)
//   interpolate(field, x, grad*)             -> dg_interpolate_batch (K2), also batched: interpolate(field, n, x, phi, grad)
//   interpolate(field, n, x, phi, grad, hess) -> dg_interpolate_hessian_batch (K2's Hessian mode; not in the reference)
//   isosurface(field, iso, subdivisions)     -> dg_isosurface_create (K6: the level set as a TriangleMesh; not in the reference)
//   isosurface_vjp(field, iso, s, n, ...)    -> dg_isosurface_vjp_device (K13: its vertices' gradient in the trainable field's node values)
//   raycast(field, n, o, d, iso, t0, t1, ...) -> dg_field_raycast (K7: first crossings along rays and segments; not in the reference)
//   connectivity table of addFunction        -> dg_build_cells  (GPU)  replaces the serial loop :833-886
//
// m_nodes / m_cells / m_cell_map hold exactly what the reference would have produced, so save()/load() stay
// byte-compatible (.cdf/.cdm, :678-778) and reduceField() (host bookkeeping, restated from :1065-1174) keeps working.
// Device copies of fields are caches owned by this object, dropped by addFunction / load / reduceField.  The reduced calls keep the
// library's handle on their result until the field's first deviceField(), which builds the device copy from it without the host
// (dg_field_create_reduced); until then the handle's arrays stay in GPU memory.
//
// addFunction takes the reference's opaque std::function.  Functors of the two types the reference's own tools build are
// recognised with std::function::target<>() and run on the GPU, and so are DeviceFunction / DeviceSamplePredicate /
// DeviceNodePredicate, which carry the caller's own GPU code in batched form.  Any other callable cannot run on a GPU: it throws
// std::invalid_argument unless DISCREGRID_B200_ALLOW_HOST_CALLBACK is defined, in which case YOUR callback is invoked
// once per node on the host (node positions still come from the GPU); that path is never part of any reported number.
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <exception>
#include <functional>
#include <iostream>
#include <limits>
#include <map>
#include <numeric>
#include <stdexcept>
#include "discrete_grid.hpp"
#include "geometry/TriangleMeshDistance.h"
#include "discregrid_b200.h"

#if defined(__GNUC__) && !defined(__clang__)
#define DG_NO_CONTRACT __attribute__((optimize("fp-contract=off")))
#else
#define DG_NO_CONTRACT
#endif

namespace Discregrid {

class CubicLagrangeDiscreteGrid;

// std::vector whose resize() leaves trivially-constructible elements uninitialised.  The field arrays (947 MB of coefficients and a
// 2 GiB connectivity table at 256^3) are written exactly once, by the library: value-initialising them first would touch every page
// serially before the real fill does.  Same interface as std::vector; the members are private in the reference too
// (cubic_lagrange_discrete_grid.hpp:69-71), so no caller sees the allocator.
template <class T>
struct FieldAllocator : std::allocator<T> {
    template <class U> struct rebind { using other = FieldAllocator<U>; };
    using std::allocator<T>::allocator;
    FieldAllocator() = default;
    template <class U> FieldAllocator(FieldAllocator<U> const&) noexcept {}
    template <class U> void construct(U* p) noexcept { ::new (static_cast<void*>(p)) U; }
    template <class U, class... A> void construct(U* p, A&&... a) { ::new (static_cast<void*>(p)) U(std::forward<A>(a)...); }
};
template <class T> using FieldVector = std::vector<T, FieldAllocator<T>>;

// GenerateDensityMap's density functor + sample predicate (cmd/generate_density_map/main.cpp:96-133) as a recognisable type
struct DensityMapFunction {
    const CubicLagrangeDiscreteGrid* grid;
    unsigned int sdf_field_id;
    double smoothing_length, rest_density;
    bool no_reduction;
    double operator()(Eigen::Vector3d const&) const { throw std::logic_error("DensityMapFunction is evaluated by addFunction on the GPU"); }
};

// The volume map of Bender et al. 2019 (SPlisHSPlasH's boundary representation) as a recognisable type: scale * the 16^3-point Gauss
// quadrature of an inside indicator over the ball of radius h around each node, on the SDF in field sdf_field_id, with GenerateDensityMap's
// sample predicate unless no_reduction (include/discregrid_b200.h, dg_volume_map)
struct VolumeMapFunction {
    const CubicLagrangeDiscreteGrid* grid;
    unsigned int sdf_field_id;
    double smoothing_length, scale;
    bool no_reduction;
    VolumeMapFunction(const CubicLagrangeDiscreteGrid* grid_, unsigned int sdf_field_id_, double smoothing_length_, double scale_ = 0.8,
                      bool no_reduction_ = false)
        : grid(grid_), sdf_field_id(sdf_field_id_), smoothing_length(smoothing_length_), scale(scale_), no_reduction(no_reduction_) {}
    double operator()(Eigen::Vector3d const&) const { throw std::logic_error("VolumeMapFunction is evaluated by addFunction on the GPU"); }
};

// The caller's own GPU code as recognisable types (include/discregrid_b200.h, dg_device_function & co.): f is called once per chunk of node
// ids, in ascending order, on the calling thread, with device pointers (positions d_x: n x 3; masks: n bytes, nonzero = keep) and the
// cudaStream_t the library works on (as void*); it enqueues its work there or finishes it before returning, and returns 0 (nonzero aborts
// the call; an exception it throws is rethrown by the grid method).  The reference-signature call operators only exist so that the types
// convert to ContinuousFunction / SamplePredicate / Predicate; they throw.
struct DeviceFunction {
    std::function<int(const double* d_x, const std::uint8_t* d_sample_keep, std::uint64_t n, double* d_values, void* stream)> f;
    double operator()(Eigen::Vector3d const&) const { throw std::logic_error("DeviceFunction is evaluated in batches on the GPU by addFunction"); }
};
struct DeviceSamplePredicate {
    std::function<int(const double* d_x, std::uint64_t n, std::uint8_t* d_keep, void* stream)> f;
    bool operator()(Eigen::Vector3d const&) const { throw std::logic_error("DeviceSamplePredicate is evaluated in batches on the GPU by addFunction"); }
};
struct DeviceNodePredicate {
    std::function<int(const double* d_x, const double* d_values, std::uint64_t n, std::uint8_t* d_keep, void* stream)> f;
    bool operator()(Eigen::Vector3d const&, double) const { throw std::logic_error("DeviceNodePredicate is evaluated in batches on the GPU by reduceField"); }
};

namespace detail {
// C trampolines for the device callbacks: an exception thrown by a callback is kept and the call aborted (nonzero)
struct DeviceCallbackContext {
    DeviceFunction const* func = nullptr;
    DeviceSamplePredicate const* sample = nullptr;
    DeviceNodePredicate const* node = nullptr;
    std::exception_ptr error;
    template <class F> int run(F&& f)
    {
        try { return f(); } catch (...) { error = std::current_exception(); return -1; }
    }
    static int func_cb(void* u, const double* x, const std::uint8_t* keep, std::uint64_t n, double* v, void* s)
    {
        auto* c = static_cast<DeviceCallbackContext*>(u);
        return c->run([&] { return c->func->f(x, keep, n, v, s); });
    }
    static int sample_cb(void* u, const double* x, std::uint64_t n, std::uint8_t* keep, void* s)
    {
        auto* c = static_cast<DeviceCallbackContext*>(u);
        return c->run([&] { return c->sample->f(x, n, keep, s); });
    }
    static int node_cb(void* u, const double* x, const double* v, std::uint64_t n, std::uint8_t* keep, void* s)
    {
        auto* c = static_cast<DeviceCallbackContext*>(u);
        return c->run([&] { return c->node->f(x, v, n, keep, s); });
    }
    dg_device_function func_ptr() const { return func ? &func_cb : nullptr; }
    dg_device_sample_predicate sample_ptr() const { return sample ? &sample_cb : nullptr; }
    dg_device_node_predicate node_ptr() const { return node ? &node_cb : nullptr; }
    void rethrow() const { if (error) std::rethrow_exception(error); }
};
}  // namespace detail

class CubicLagrangeDiscreteGrid : public DiscreteGrid {
public:
    CubicLagrangeDiscreteGrid(std::string const& filename) { load(filename); }
    CubicLagrangeDiscreteGrid(Eigen::AlignedBox3d const& domain, std::array<unsigned int, 3> const& resolution) : DiscreteGrid(domain, resolution) {}
    CubicLagrangeDiscreteGrid(const CubicLagrangeDiscreteGrid&) = delete;
    CubicLagrangeDiscreteGrid& operator=(const CubicLagrangeDiscreteGrid&) = delete;
    ~CubicLagrangeDiscreteGrid() override { invalidate(); }

    // ---- save / load: byte layout of cubic_lagrange_discrete_grid.cpp:678-719 / 721-778 (serialize.hpp:12-25)
    void save(std::string const& filename) const override
    {
        std::ofstream out(filename, std::ios::binary);
        auto put = [&](const void* p, std::size_t n) { out.write(static_cast<const char*>(p), (std::streamsize)n); };
        put(m_domain.min().data(), 24); put(m_domain.max().data(), 24);
        put(m_resolution.data(), 12); put(m_cell_size.data(), 24); put(m_inv_cell_size.data(), 24);
        put(&m_n_cells, 8); put(&m_n_fields, 8);
        std::size_t n = m_nodes.size(); put(&n, 8);
        for (auto const& v : m_nodes) { n = v.size(); put(&n, 8); put(v.data(), 8 * n); }
        n = m_cells.size(); put(&n, 8);
        for (auto const& v : m_cells) { n = v.size(); put(&n, 8); put(v.data(), 128 * n); }
        n = m_cell_map.size(); put(&n, 8);
        for (auto const& v : m_cell_map) { n = v.size(); put(&n, 8); put(v.data(), 4 * n); }
    }
    void load(std::string const& filename) override
    {
        invalidate();
        std::ifstream in(filename, std::ios::binary);
        if (!in.good()) { std::cerr << "ERROR: Discrete grid can not be loaded. Input file does not exist!" << std::endl; return; }
        auto get = [&](void* p, std::size_t n) { in.read(static_cast<char*>(p), (std::streamsize)n); };
        get(m_domain.min().data(), 24); get(m_domain.max().data(), 24);
        get(m_resolution.data(), 12); get(m_cell_size.data(), 24); get(m_inv_cell_size.data(), 24);
        get(&m_n_cells, 8); get(&m_n_fields, 8);
        std::size_t n = 0; get(&n, 8); m_nodes.resize(n);
        for (auto& v : m_nodes) { get(&n, 8); v.resize(n); get(v.data(), 8 * n); }
        get(&n, 8); m_cells.resize(n);
        for (auto& v : m_cells) { get(&n, 8); v.resize(n); get(v.data(), 128 * n); }
        get(&n, 8); m_cell_map.resize(n);
        for (auto& v : m_cell_map) { get(&n, 8); v.resize(n); get(v.data(), 4 * n); }
    }

    // ---- addFunction (cubic_lagrange_discrete_grid.cpp:780-899)
    unsigned int addFunction(ContinuousFunction const& func, bool verbose = false, SamplePredicate const& pred = nullptr) override
    {
        const dg_grid_desc d = desc();
        std::uint64_t n_nodes = 0;
        check(dg_grid_num_nodes(d.resolution, &n_nodes));
        auto const* dev_func = func.target<DeviceFunction>();
        auto const* dev_pred = pred ? pred.target<DeviceSamplePredicate>() : nullptr;
        if (dev_func || dev_pred) {
            if (!dev_func || (pred && !dev_pred))
                throw std::invalid_argument("addFunction: a DeviceFunction takes a DeviceSamplePredicate (or none), and a DeviceSamplePredicate only goes "
                                            "with a DeviceFunction");
            // the whole of :780-899 in one library call: the caller's code on the GPU, connectivity + cell map by the library's host threads
            FieldVector<double> coeffs(n_nodes);
            FieldVector<std::array<unsigned int, 32>> cells(m_n_cells);
            FieldVector<unsigned int> cell_map(m_n_cells);
            detail::DeviceCallbackContext ctx;
            ctx.func = dev_func; ctx.sample = dev_pred;
            const int rc = dg_add_function_device(&d, ctx.func_ptr(), &ctx, ctx.sample_ptr(), &ctx, 0, coeffs.data(),
                                                  reinterpret_cast<std::uint32_t*>(cells.data()), cell_map.data(), m_last_add_function_ms);
            ctx.rethrow();
            check(rc);
            if (verbose) std::cout << "Construction: " << n_nodes << " nodes sampled on the GPU in " << m_last_add_function_ms[0] << " ms" << std::endl;
            invalidate();
            m_nodes.push_back(std::move(coeffs)); m_cells.push_back(std::move(cells)); m_cell_map.push_back(std::move(cell_map));
            return static_cast<unsigned int>(m_n_fields++);
        }
        if (auto const* sdf = func.target<MeshSignedDistanceFunction>()) {
            auto const* band = pred ? pred.target<MeshDistanceBandPredicate>() : nullptr;
            if (pred && !band)
                throw std::invalid_argument("addFunction: a sample predicate is only supported with DensityMapFunction, or as MeshDistanceBandPredicate "
                                            "with MeshSignedDistanceFunction");
            if (band && band->md != sdf->md)
                throw std::invalid_argument("addFunction: the MeshDistanceBandPredicate must use the same TriangleMeshDistance as the MeshSignedDistanceFunction");
            if (band && sdf->md->group())
                throw std::invalid_argument("addFunction: narrow-band sampling runs on one GPU; it is not available after TriangleMeshDistance::useGpus(n > 1)");
            // the whole of :780-899 in one library call: node loop on the GPU; connectivity (:833-886) and cell map (:888-891) written by
            // the library's host threads into these arrays while the GPU works
            FieldVector<double> coeffs(n_nodes);
            FieldVector<std::array<unsigned int, 32>> cells(m_n_cells);
            FieldVector<unsigned int> cell_map(m_n_cells);
            if (sdf->md->group())             // TriangleMeshDistance::useGpus(n): the same call spread over n GPUs
                check(dg_add_function_sdf_multi(sdf->md->group(), &d, sdf->sign, coeffs.data(), reinterpret_cast<std::uint32_t*>(cells.data()), cell_map.data(),
                                                m_last_add_function_ms));
            else if (band)
                check(dg_add_function_sdf_band(sdf->md->handle(), &d, sdf->sign, band->band, coeffs.data(), reinterpret_cast<std::uint32_t*>(cells.data()),
                                               cell_map.data(), m_last_add_function_ms));
            else
                check(dg_add_function_sdf(sdf->md->handle(), &d, sdf->sign, coeffs.data(), reinterpret_cast<std::uint32_t*>(cells.data()), cell_map.data(),
                                          m_last_add_function_ms));
            if (verbose) std::cout << "Construction: " << n_nodes << " nodes sampled on the GPU in " << m_last_add_function_ms[0] << " ms" << std::endl;
            invalidate();
            m_nodes.push_back(std::move(coeffs)); m_cells.push_back(std::move(cells)); m_cell_map.push_back(std::move(cell_map));
            return static_cast<unsigned int>(m_n_fields++);
        }
        FieldVector<double> coeffs(n_nodes);
        if (auto const* dm = func.target<DensityMapFunction>()) {
            check(dg_density_map(dm->grid->deviceField(dm->sdf_field_id), dm->smoothing_length, dm->rest_density, dm->no_reduction ? 1 : 0,
                                 0, n_nodes, coeffs.data()));
        } else if (auto const* vm = func.target<VolumeMapFunction>()) {
            check(dg_volume_map(vm->grid->deviceField(vm->sdf_field_id), vm->smoothing_length, vm->scale, vm->no_reduction ? 1 : 0, 0, n_nodes,
                                coeffs.data()));
        } else {
#ifdef DISCREGRID_B200_ALLOW_HOST_CALLBACK
            FieldVector<double> x(3 * n_nodes);
            check(dg_node_positions(&d, 0, n_nodes, x.data()));
            for (std::uint64_t l = 0; l < n_nodes; l++) {
                const Eigen::Vector3d p(x[3 * l], x[3 * l + 1], x[3 * l + 2]);
                coeffs[l] = (!pred || pred(p)) ? func(p) : std::numeric_limits<double>::max();
            }
#else
            (void)pred;
            throw std::invalid_argument("CubicLagrangeDiscreteGrid::addFunction: only MeshSignedDistanceFunction / DensityMapFunction / VolumeMapFunction run on the GPU "
                                        "(define DISCREGRID_B200_ALLOW_HOST_CALLBACK to have other callables invoked per node on the host)");
#endif
        }
        if (verbose) std::cout << "Construction: " << n_nodes << " nodes sampled on the GPU" << std::endl;
        return addSampledFunction(std::move(coeffs));
    }
    // new: addFunction(func, verbose, pred) followed by reduceField(id, always true) in one library call (dg_reduced_band_create).  The field
    // holds exactly what those two calls leave; the dense field never reaches the host, only the survivors and the cell map do.
    unsigned int addReducedBandField(MeshSignedDistanceFunction const& func, MeshDistanceBandPredicate const& pred, bool verbose = false)
    {
        if (pred.md != func.md)
            throw std::invalid_argument("addReducedBandField: the MeshDistanceBandPredicate must use the same TriangleMeshDistance as the MeshSignedDistanceFunction");
        if (func.md->group())
            throw std::invalid_argument("addReducedBandField: narrow-band sampling runs on one GPU; it is not available after TriangleMeshDistance::useGpus(n > 1)");
        const dg_grid_desc d = desc();
        dg_reduced_band* r = nullptr;
        check(dg_reduced_band_create(func.md->handle(), &d, func.sign, pred.band, 0u, &r, m_last_reduced_band_ms));
        ReducedHandle hold(r);
        FieldVector<double> coeffs; FieldVector<std::array<unsigned int, 32>> cells; FieldVector<unsigned int> cell_map;
        take_reduced(r, coeffs, cells, cell_map);
        if (verbose) std::cout << "Construction: " << coeffs.size() << " nodes kept, " << cells.size() << " cells, on the GPU in " << m_last_reduced_band_ms[6] << " ms" << std::endl;
        invalidate();
        m_nodes.push_back(std::move(coeffs)); m_cells.push_back(std::move(cells)); m_cell_map.push_back(std::move(cell_map));
        keep_reduced(static_cast<unsigned int>(m_n_fields), hold);
        return static_cast<unsigned int>(m_n_fields++);
    }
    // new: addFunction(func, verbose, sample) followed by reduceField(id, reduce) in one library call (dg_reduced_function_create); sample /
    // reduce may be nullptr (every node sampled / always true).  The field holds exactly what those two calls leave; the dense field stays
    // on the GPU, only the survivors and the cell map reach the host.  Returns the new field id.
    unsigned int addReducedFunction(DeviceFunction const& func, DeviceSamplePredicate const* sample = nullptr, DeviceNodePredicate const* reduce = nullptr,
                                    bool verbose = false)
    {
        const dg_grid_desc d = desc();
        detail::DeviceCallbackContext ctx;
        ctx.func = &func; ctx.sample = sample; ctx.node = reduce;
        dg_reduced_band* r = nullptr;
        const int rc = dg_reduced_function_create(&d, ctx.func_ptr(), &ctx, ctx.sample_ptr(), &ctx, ctx.node_ptr(), &ctx, 0, 0u, &r, m_last_reduced_function_ms);
        ctx.rethrow();
        check(rc);
        ReducedHandle hold(r);
        FieldVector<double> coeffs; FieldVector<std::array<unsigned int, 32>> cells; FieldVector<unsigned int> cell_map;
        take_reduced(r, coeffs, cells, cell_map);
        if (verbose) std::cout << "Construction: " << coeffs.size() << " nodes kept, " << cells.size() << " cells, in " << m_last_reduced_function_ms[6] << " ms" << std::endl;
        invalidate();
        m_nodes.push_back(std::move(coeffs)); m_cells.push_back(std::move(cells)); m_cell_map.push_back(std::move(cell_map));
        keep_reduced(static_cast<unsigned int>(m_n_fields), hold);
        return static_cast<unsigned int>(m_n_fields++);
    }
    // new: GenerateDensityMap with reduction in one library call (dg_reduced_density_map_create).  Leaves exactly what
    //   id = addFunction(f, verbose);  reduceField(f.sdf_field_id, p0);  reduceField(id, p1);
    // leave, with the tool's predicates p0(x, v) = -6h < v + cell_diag && v - cell_diag < 2h and p1(x, v) = 0 <= v && v <= 3 rho0
    // (main.cpp:139-140): the SDF field is replaced by its reduction, the reduced density field is appended and its id returned.  The dense
    // density field never reaches the host; only the survivors and the cell maps do.
    unsigned int addReducedDensityMap(DensityMapFunction const& f, bool verbose = false)
    {
        if (f.grid != this) throw std::invalid_argument("addReducedDensityMap: the DensityMapFunction must sample this grid's own SDF field");
        if (f.no_reduction) throw std::invalid_argument("addReducedDensityMap: the DensityMapFunction has no_reduction set (use addFunction)");
        return addReducedNodeMap("addReducedDensityMap", "density", dg_reduced_density_map_create, f.sdf_field_id, f.smoothing_length,
                                 f.rest_density, m_last_reduced_density_ms, verbose);
    }
    // new: the volume map with reduction in one library call (dg_reduced_volume_map_create).  Leaves exactly what
    //   id = addFunction(f, verbose);  reduceField(f.sdf_field_id, p0);  reduceField(id, p1);
    // leave, with GenerateDensityMap's p0 (as above) and p1(x, v) = 0 <= v.  The dense volume field never reaches the host.
    unsigned int addReducedVolumeMap(VolumeMapFunction const& f, bool verbose = false)
    {
        if (f.grid != this) throw std::invalid_argument("addReducedVolumeMap: the VolumeMapFunction must sample this grid's own SDF field");
        if (f.no_reduction) throw std::invalid_argument("addReducedVolumeMap: the VolumeMapFunction has no_reduction set (use addFunction)");
        return addReducedNodeMap("addReducedVolumeMap", "volume", dg_reduced_volume_map_create, f.sdf_field_id, f.smoothing_length, f.scale,
                                 m_last_reduced_volume_ms, verbose);
    }
    // appends a field from node values + the closed-form connectivity (:833-886, built on the GPU) + identity cell map (:888-891)
    unsigned int addSampledFunction(FieldVector<double> coeffs)
    {
        invalidate();
        m_nodes.push_back(std::move(coeffs));
        m_cells.emplace_back(m_n_cells);
        check(dg_build_cells(m_resolution.data(), 0, m_n_cells, reinterpret_cast<std::uint32_t*>(m_cells.back().data())));
        m_cell_map.emplace_back(m_n_cells);
        std::iota(m_cell_map.back().begin(), m_cell_map.back().end(), 0u);
        return static_cast<unsigned int>(m_n_fields++);
    }

    std::size_t nCells() const { return m_n_cells; }

    // ---- interpolate (cubic_lagrange_discrete_grid.cpp:977-1063), scalar form kept for source compatibility
    double interpolate(unsigned int field_id, Eigen::Vector3d const& xi, Eigen::Vector3d* gradient = nullptr) const override
    {
        double phi = 0.0, g[3] = {0, 0, 0};
        // the reference leaves *gradient untouched when it returns DBL_MAX before the loop (:981-982, :993-994)
        check(dg_interpolate_batch(deviceField(field_id), xi.data(), 1, &phi, gradient ? g : nullptr));
        if (gradient && !(phi == std::numeric_limits<double>::max() && !in_kept_cell(field_id, xi))) *gradient = Eigen::Vector3d(g[0], g[1], g[2]);
        return phi;
    }
    // batched form (new; the one to use): x = n x 3, phi = n, grad = n x 3 or nullptr
    void interpolate(unsigned int field_id, std::size_t n, const double* x, double* phi, double* grad = nullptr) const
    {
        check(dg_interpolate_batch(deviceField(field_id), x, n, phi, grad));
    }
    // batched value + gradient + Hessian (new, beyond the reference): phi = n, grad = n x 3 (the bits of the form above), hess = n x 3 x 3
    // row-major and exactly symmetric, all three required (dg_interpolate_hessian_batch)
    void interpolate(unsigned int field_id, std::size_t n, const double* x, double* phi, double* grad, double* hess) const
    {
        check(dg_interpolate_hessian_batch(deviceField(field_id), x, n, phi, grad, hess));
    }
    // the level set {phi = iso} of a field by marching tetrahedra on a lattice that subdivides every cell `subdivisions` times (new, beyond
    // the reference; contract in k6_isosurface.cu): outward-oriented triangles for an SDF, coincident vertices not welded.  edge_ids, when
    // given, receives the lattice edge of every vertex (dg_isosurface_copy_edges), what isosurface_vjp takes
    TriangleMesh isosurface(unsigned int field_id, double iso = 0.0, unsigned int subdivisions = 1, std::vector<std::uint64_t>* edge_ids = nullptr) const
    {
        dg_isosurface* s = nullptr;
        check(dg_isosurface_create(deviceField(field_id), iso, subdivisions, &s, nullptr));
        std::uint64_t nv = 0, nt = 0;
        dg_isosurface_sizes(s, &nv, &nt);
        std::vector<double> v(3 * nv);
        std::vector<std::uint32_t> t(3 * nt);
        int rc = dg_isosurface_copy(s, v.data(), t.data());
        if (rc == DG_OK && edge_ids) {
            edge_ids->resize((std::size_t)nv);
            rc = dg_isosurface_copy_edges(s, edge_ids->data());
        }
        dg_isosurface_destroy(s);
        check(rc);
        return TriangleMesh(v.data(), t.data(), (std::size_t)nv, (std::size_t)nt);
    }
    // the first crossing of {phi = iso} along n rays (new, beyond the reference; contract in k7_raycast.cu): origins and directions n x 3,
    // t in [t_min, t_max] (a segment x0 -> x1 is the ray (x0, x1 - x0) on [0, 1]); outputs t_lo, t_hi (the bracket) and status = DG_RAY_MISS /
    // DG_RAY_ENTER / DG_RAY_LEAVE, all n (dg_field_raycast)
    void raycast(unsigned int field_id, std::size_t n, const double* origins, const double* directions, double iso, double t_min, double t_max,
                 double* t_lo, double* t_hi, std::int32_t* status) const
    {
        check(dg_field_raycast(deviceField(field_id), origins, directions, n, iso, t_min, t_max, t_lo, t_hi, status));
    }

    // ---- trainable fields (new, beyond the reference; contract in k11_field_grad.cu).  One trainable device field per field id, made at first
    // use from the members (dg_field_create_trainable, which synchronises) and dropped with the other device copies.  Device pointers, `stream`
    // a cudaStream_t (NULL: the legacy default stream); neither call synchronises the host.
    // setNodesDevice: the trainable field takes the n_nodes values at d_nodes (dg_field_set_nodes_device); n_nodes must be the field's count
    void setNodesDevice(unsigned int field_id, const double* d_nodes, std::size_t n_nodes, void* stream = nullptr)
    {
        check(dg_field_set_nodes_device(trainableField(field_id), d_nodes, n_nodes, stream));
    }
    // interpolate_vjp: d_grad_nodes [nodes] = the gradient in the trainable field's node values of sum_q d_grad_phi[q] phi(x_q) +
    // d_grad_grad[q] . grad(x_q) over the n points d_x [n x 3] (dg_interpolate_vjp_device; either upstream may be NULL, not both)
    void interpolate_vjp(unsigned int field_id, std::size_t n, const double* d_x, const double* d_grad_phi, const double* d_grad_grad,
                         double* d_grad_nodes, void* stream = nullptr)
    {
        check(dg_interpolate_vjp_device(trainableField(field_id), d_x, n, d_grad_phi, d_grad_grad, d_grad_nodes, stream));
    }
    // raycast_vjp: the gradients of the first crossings (t_lo, t_hi from raycast on device arrays) in the origins, the directions and, when
    // d_grad_nodes is given, the trainable field's node values, for the upstream gradients d_grad_t_lo and d_grad_t_hi [n] (either may be
    // NULL, not both); every output [n x 3], [n x 3], [nodes] may be NULL (dg_field_raycast_vjp_device; contract in k12_raycast_grad.cu).
    // With d_grad_nodes the rays must have been cast on trainableField(field_id) holding the same values; without it on deviceField(field_id).
    void raycast_vjp(unsigned int field_id, std::size_t n, const double* d_origins, const double* d_directions, const double* d_t_lo,
                     const std::int32_t* d_status, const double* d_grad_t_lo, const double* d_grad_t_hi, double* d_grad_origins,
                     double* d_grad_directions, double* d_grad_nodes, void* stream = nullptr)
    {
        const dg_field* f = d_grad_nodes ? trainableField(field_id) : deviceField(field_id);
        check(dg_field_raycast_vjp_device(f, n, d_origins, d_directions, d_t_lo, d_status, d_grad_t_lo, d_grad_t_hi, d_grad_origins,
                                          d_grad_directions, d_grad_nodes, stream));
    }
    // isosurface_vjp: d_grad_nodes [nodes] = the gradient in the trainable field's node values of sum_v d_grad_vertices[v] . V_v over the n
    // vertices on the lattice edges d_edge_ids [n] of isosurface(field_id, iso, subdivisions) extracted on trainableField(field_id) holding
    // the same values (dg_isosurface_vjp_device; contract in k13_isosurface_grad.cu)
    void isosurface_vjp(unsigned int field_id, double iso, unsigned int subdivisions, std::size_t n, const std::uint64_t* d_edge_ids,
                        const double* d_grad_vertices, double* d_grad_nodes, void* stream = nullptr)
    {
        check(dg_isosurface_vjp_device(trainableField(field_id), iso, subdivisions, n, d_edge_ids, d_grad_vertices, d_grad_nodes, stream));
    }
    // the trainable field itself, for the library's other calls on its current values (dg_interpolate_batch_device, ...)
    dg_field* trainableField(unsigned int field_id)
    {
        auto it = m_trainable.find(field_id);
        if (it != m_trainable.end()) return it->second;
        const dg_grid_desc d = desc();
        dg_field* f = nullptr;
        check(dg_field_create_trainable(&d, m_nodes.at(field_id).data(), m_nodes[field_id].size(),
                                        reinterpret_cast<const std::uint32_t*>(m_cells[field_id].data()), m_cells[field_id].size(),
                                        m_cell_map[field_id].data(), &f));
        m_trainable[field_id] = f;
        return f;
    }

    // ---- split API (:901-975): shape functions on the GPU (dg_shape_functions), index algebra on the host
    DG_NO_CONTRACT bool determineShapeFunctions(unsigned int field_id, Eigen::Vector3d const& x, std::array<unsigned int, 32>& cell, Eigen::Vector3d& c0,
                                                Eigen::Matrix<double, 32, 1>& N, Eigen::Matrix<double, 32, 3>* dN = nullptr) const override
    {
        if (!m_domain.contains(x)) return false;
        unsigned mi[3];
        for (int d = 0; d < 3; d++) {
            mi[d] = static_cast<unsigned int>((x[d] - m_domain.min()[d]) * m_inv_cell_size[d]);
            if (mi[d] >= m_resolution[d]) mi[d] = m_resolution[d] - 1;
        }
        const unsigned i = multiToSingleIndex({{mi[0], mi[1], mi[2]}});
        const unsigned i_ = m_cell_map[field_id][i];
        if (i_ == std::numeric_limits<unsigned int>::max()) return false;
        double xi[3];
        for (int d = 0; d < 3; d++) {
            const double lo = m_domain.min()[d] + static_cast<double>(mi[d]) * m_cell_size[d];
            const double hi = lo + m_cell_size[d];
            const double denom = hi - lo;
            c0[d] = 2.0 / denom;
            const double c1 = (hi + lo) / denom;
            xi[d] = c0[d] * x[d] - c1;
        }
        cell = m_cells[field_id][i_];
        double Nb[32], dNb[96];
        check(dg_shape_functions(xi, 1, Nb, dN ? dNb : nullptr));
        for (int j = 0; j < 32; j++) N[j] = Nb[j];
        if (dN) for (int j = 0; j < 32; j++) for (int d = 0; d < 3; d++) (*dN)(j, d) = dNb[3 * j + d];
        return true;
    }
    DG_NO_CONTRACT double interpolate(unsigned int field_id, Eigen::Vector3d const&, const std::array<unsigned int, 32>& cell, const Eigen::Vector3d& c0,
                                      const Eigen::Matrix<double, 32, 1>& N, Eigen::Vector3d* gradient = nullptr, Eigen::Matrix<double, 32, 3>* dN = nullptr) const override
    {
        double phi = 0.0;
        if (gradient) gradient->setZero();
        for (unsigned j = 0; j < 32u; ++j) {
            const double c = m_nodes[field_id][cell[j]];
            if (c == std::numeric_limits<double>::max()) { if (gradient) gradient->setZero(); return std::numeric_limits<double>::max(); }
            phi = phi + c * N[j];
            if (gradient) for (int d = 0; d < 3; d++) (*gradient)[d] = (*gradient)[d] + c * (*dN)(j, d);
        }
        if (gradient) for (int d = 0; d < 3; d++) (*gradient)[d] = (*gradient)[d] * c0[d];
        return phi;
    }

    // ---- reduceField (:1065-1174): the predicate is evaluated here; cells / nodes / cell map are rewritten by dg_reduce_field
    // and end up exactly as the reference leaves them (kept cells in order, surviving nodes in its Z-curve order)
    void reduceField(unsigned int field_id, Predicate pred) override;

    void forEachCell(unsigned int, std::function<void(unsigned int, Eigen::AlignedBox3d const&, unsigned int)> const& cb) const
    {
        const unsigned n = m_resolution[0] * m_resolution[1] * m_resolution[2];
        for (unsigned i = 0; i < n; ++i) cb(i, subdomain(i), 0);
    }

    // ---- accessors used by tools / tests
    FieldVector<double> const& nodeData(unsigned int f) const { return m_nodes[f]; }
    FieldVector<std::array<unsigned int, 32>> const& cellData(unsigned int f) const { return m_cells[f]; }
    FieldVector<unsigned int> const& cellMap(unsigned int f) const { return m_cell_map[f]; }
    // ms since entry of the last addFunction(MeshSignedDistanceFunction): total, node pipeline, index tables, pre-fault; workers
    const double* lastAddFunctionTimings() const { return m_last_add_function_ms; }
    // ms of the last addReducedBandField: sampling, cells, nodes, sort, write-back; tie path (1.0 / 0.0); total
    const double* lastReducedBandTimings() const { return m_last_reduced_band_ms; }
    // ms of the last addReducedDensityMap: upload + pack, density; cells, nodes, sort, write-back of field 0 then of field 1; tie paths; total
    const double* lastReducedDensityTimings() const { return m_last_reduced_density_ms; }
    // ms of the last addReducedVolumeMap, in the same layout ([1] is the volume sampling)
    const double* lastReducedVolumeTimings() const { return m_last_reduced_volume_ms; }
    // ms of the last addReducedFunction / reduceField(DeviceNodePredicate): positions + callbacks (reduceField: with the upload), cells, nodes,
    // sort, write-back; tie path (1.0 / 0.0); total; inside the callbacks
    const double* lastReducedFunctionTimings() const { return m_last_reduced_function_ms; }
    std::size_t nFields() const { return m_n_fields; }
    dg_grid_desc desc() const
    {
        dg_grid_desc d; std::memset(&d, 0, sizeof d);
        for (int k = 0; k < 3; k++) { d.domain_min[k] = m_domain.min()[k]; d.domain_max[k] = m_domain.max()[k]; d.resolution[k] = m_resolution[k];
                                      d.cell_size[k] = m_cell_size[k]; d.inv_cell_size[k] = m_inv_cell_size[k]; }
        return d;
    }
    // the device field of field_id, made at first use: from the handle a reduced call kept for it (dg_field_create_reduced, device to device;
    // the handle is released) or else by uploading the members (dg_field_create).  Making it synchronises the device.
    const dg_field* deviceField(unsigned int field_id) const
    {
        auto it = m_dev.find(field_id);
        if (it != m_dev.end()) return it->second;
        dg_field* f = nullptr;
        auto kept = m_reduced.find(field_id);
        if (kept != m_reduced.end()) {
            check(dg_field_create_reduced(kept->second, &f));
            dg_reduced_band_destroy(kept->second);
            m_reduced.erase(kept);
        } else {
            const dg_grid_desc d = desc();
            check(dg_field_create(&d, m_nodes.at(field_id).data(), m_nodes[field_id].size(), reinterpret_cast<const std::uint32_t*>(m_cells[field_id].data()),
                                  m_cells[field_id].size(), m_cell_map[field_id].data(), &f));
        }
        m_dev[field_id] = f;
        return f;
    }

private:
    // the shared body of addReducedDensityMap / addReducedVolumeMap: `entry` is the library's one-call route, timings its 13 stage times
    typedef int (*ReducedNodeMapEntry)(const dg_grid_desc*, const double*, std::uint64_t, const std::uint32_t*, std::uint64_t, const std::uint32_t*,
                                       double, double, std::uint32_t, dg_reduced_band**, dg_reduced_band**, double*);
    unsigned int addReducedNodeMap(const char* who, const char* what, ReducedNodeMapEntry entry, unsigned int id, double h, double param,
                                   double* timings, bool verbose)
    {
        if (id >= m_n_fields) throw std::invalid_argument(std::string(who) + ": no SDF field with that id");
        if (m_cell_map[id].size() != m_n_cells) throw std::invalid_argument(std::string(who) + ": the SDF field's cell map must cover every grid cell");
        const dg_grid_desc d = desc();
        dg_reduced_band* r[2] = {nullptr, nullptr};
        check(entry(&d, m_nodes[id].data(), m_nodes[id].size(), reinterpret_cast<const std::uint32_t*>(m_cells[id].data()), m_cells[id].size(),
                    m_cell_map[id].data(), h, param, 0u, &r[0], &r[1], timings));
        ReducedHandle hold0(r[0]), hold1(r[1]);
        FieldVector<double> coeffs[2];
        FieldVector<std::array<unsigned int, 32>> cells[2];
        FieldVector<unsigned int> cell_map[2];
        for (int k = 0; k < 2; k++)           // both copied before anything changes, so a failure leaves the grid as it was
            take_reduced(r[k], coeffs[k], cells[k], cell_map[k]);
        if (verbose)
            std::cout << "Construction: " << what << " map sampled and both fields reduced on the GPU in " << timings[12] << " ms ("
                      << coeffs[0].size() << " SDF nodes and " << coeffs[1].size() << " " << what << " nodes kept)" << std::endl;
        invalidate();
        m_nodes[id] = std::move(coeffs[0]); m_cells[id] = std::move(cells[0]); m_cell_map[id] = std::move(cell_map[0]);
        m_nodes.push_back(std::move(coeffs[1])); m_cells.push_back(std::move(cells[1])); m_cell_map.push_back(std::move(cell_map[1]));
        keep_reduced(id, hold0);
        keep_reduced(static_cast<unsigned int>(m_n_fields), hold1);
        return static_cast<unsigned int>(m_n_fields++);
    }
    std::vector<FieldVector<double>> m_nodes;
    std::vector<FieldVector<std::array<unsigned int, 32>>> m_cells;
    std::vector<FieldVector<unsigned int>> m_cell_map;
    double m_last_add_function_ms[6] = {0, 0, 0, 0, 0, 0};
    double m_last_reduced_band_ms[7] = {0, 0, 0, 0, 0, 0, 0};
    double m_last_reduced_density_ms[13] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    double m_last_reduced_volume_ms[13] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    double m_last_reduced_function_ms[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    mutable std::map<unsigned int, dg_field*> m_dev;
    // the handles the reduced calls returned, kept until their field's first deviceField or the next invalidate(): a field made from a
    // handle needs no upload.  Owned like m_dev.
    mutable std::map<unsigned int, dg_reduced_band*> m_reduced;
    std::map<unsigned int, dg_field*> m_trainable;          // trainableField's, owned like m_dev

    // owns a dg_reduced_band until keep_reduced takes it; destroys it on every other path
    struct ReducedHandle {
        dg_reduced_band* r;
        explicit ReducedHandle(dg_reduced_band* p) : r(p) {}
        ReducedHandle(const ReducedHandle&) = delete;
        ReducedHandle& operator=(const ReducedHandle&) = delete;
        ~ReducedHandle() { dg_reduced_band_destroy(r); }
    };
    void keep_reduced(unsigned int field_id, ReducedHandle& h)
    {
        dg_reduced_band*& slot = m_reduced[field_id];
        dg_reduced_band_destroy(slot);
        slot = h.r;
        h.r = nullptr;
    }

    // the arrays of a dg_reduced_band handle (which stays with the caller)
    void take_reduced(dg_reduced_band* r, FieldVector<double>& coeffs, FieldVector<std::array<unsigned int, 32>>& cells, FieldVector<unsigned int>& cell_map) const
    {
        std::uint64_t n_nodes = 0, n_cells = 0;
        check(dg_reduced_band_sizes(r, &n_nodes, &n_cells));
        coeffs.resize(n_nodes); cells.resize(n_cells); cell_map.resize(m_n_cells);
        check(dg_reduced_band_copy(r, coeffs.data(), reinterpret_cast<std::uint32_t*>(cells.data()), cell_map.data()));
    }

    static void check(int rc) { if (rc != DG_OK) throw std::runtime_error(std::string("discregrid_b200: ") + dg_last_error()); }
    void invalidate()
    {
        for (auto& kv : m_dev) dg_field_destroy(kv.second);
        m_dev.clear();
        for (auto& kv : m_reduced) dg_reduced_band_destroy(kv.second);
        m_reduced.clear();
        for (auto& kv : m_trainable) dg_field_destroy(kv.second);
        m_trainable.clear();
    }
    bool in_kept_cell(unsigned int field_id, Eigen::Vector3d const& x) const
    {
        if (!m_domain.contains(x)) return false;
        unsigned mi[3];
        for (int d = 0; d < 3; d++) { mi[d] = static_cast<unsigned int>((x[d] - m_domain.min()[d]) * m_inv_cell_size[d]); if (mi[d] >= m_resolution[d]) mi[d] = m_resolution[d] - 1; }
        return m_cell_map[field_id][multiToSingleIndex({{mi[0], mi[1], mi[2]}})] != std::numeric_limits<unsigned int>::max();
    }
};

inline void CubicLagrangeDiscreteGrid::reduceField(unsigned int field_id, Predicate pred)
{
    if (auto const* dev = pred.target<DeviceNodePredicate>()) {
        // the predicate on the GPU and every pass there (dg_reduce_field_device); the field is replaced only once the result is in
        const dg_grid_desc d = desc();
        detail::DeviceCallbackContext ctx;
        ctx.node = dev;
        dg_reduced_band* r = nullptr;
        const int rc = dg_reduce_field_device(&d, m_nodes[field_id].data(), m_nodes[field_id].size(), reinterpret_cast<const std::uint32_t*>(m_cells[field_id].data()),
                                              m_cells[field_id].size(), ctx.node_ptr(), &ctx, 0, 0u, &r, m_last_reduced_function_ms);
        ctx.rethrow();
        check(rc);
        ReducedHandle hold(r);
        FieldVector<double> coeffs; FieldVector<std::array<unsigned int, 32>> cells; FieldVector<unsigned int> cell_map;
        take_reduced(r, coeffs, cells, cell_map);
        invalidate();
        m_nodes[field_id] = std::move(coeffs); m_cells[field_id] = std::move(cells); m_cell_map[field_id] = std::move(cell_map);
        keep_reduced(field_id, hold);
        return;
    }
    invalidate();
    auto& coeffs = m_nodes[field_id];
    auto& cells = m_cells[field_id];
    const dg_grid_desc d = desc();
    std::vector<double> pos(3 * coeffs.size());
    check(dg_node_positions(&d, 0, coeffs.size(), pos.data()));              // indexToNodePosition for every node (:604-665)
    const double dbl_max = std::numeric_limits<double>::max();
    std::vector<std::uint8_t> keep(coeffs.size());                            // the predicate is the caller's: evaluated here, serially (:1069-1074)
    for (std::size_t l = 0; l < coeffs.size(); ++l)
        keep[l] = (pred(Eigen::Vector3d(pos[3 * l], pos[3 * l + 1], pos[3 * l + 2]), coeffs[l]) && coeffs[l] != dbl_max) ? 1 : 0;
    std::vector<double>().swap(pos);
    auto& cell_map = m_cell_map[field_id];
    cell_map.resize(m_n_cells);
    // surviving cells, surviving nodes in Z-curve order, renumbered connectivity, cell map (:1076-1173) -- the library's index passes
    std::uint64_t n_nodes = 0, n_cells = 0;
    check(dg_reduce_field(&d, coeffs.data(), coeffs.size(), keep.data(), reinterpret_cast<std::uint32_t*>(cells.data()), cells.size(),
                          cell_map.data(), 0u, &n_nodes, &n_cells, nullptr));
    coeffs.resize(n_nodes);
    cells.resize(n_cells);
}

}  // namespace Discregrid
