// Discregrid::TriangleMeshDistance with the reference's public surface (geometry/TriangleMeshDistance.h:75-208),
// implemented on the H100 through the C-ABI (include/discregrid_b200.h).  construct() builds the reference's
// sphere tree + pseudonormals on the host and uploads them once (dg_mesh_create); signed_distance / unsigned_distance run
// in the sm_90a traversal kernel -- one point per call for source compatibility, or batched with the *_batch overloads
// (the form to use: a launch per point is dominated by latency).
// Differences, all deliberate: unconstructed / empty mesh throws std::runtime_error instead of exit(-1)
// (:318-321, :338-341); the raw-pointer construct() sizes its arrays correctly (the reference over-allocates 3x and
// injects degenerate triangles, :232-249).
#pragma once
#include <array>
#include <cstdint>
#include <limits>
#include <stdexcept>
#include <string>
#include <vector>
#include "../mesh/triangle_mesh.hpp"
#include "discregrid_b200.h"

namespace Discregrid {

enum class NearestEntity { V0, V1, V2, E01, E12, E02, F };
// new: where signed distances take their sign from.  Pseudonormal is the reference's rule (right for closed manifold meshes only); Winding
// takes it from the generalized winding number (inside iff w > 0.5), which also holds for open and non-manifold meshes.  One GPU only.
enum class SignMode { Pseudonormal = DG_SIGN_PSEUDONORMAL, Winding = DG_SIGN_WINDING };

template <typename FLOAT>
class Vec3r {
public:
    std::array<FLOAT, 3> v;
    Vec3r() {}
    template <typename FLOAT_I> Vec3r(const FLOAT_I& x, const FLOAT_I& y, const FLOAT_I& z) { v[0] = static_cast<FLOAT>(x); v[1] = static_cast<FLOAT>(y); v[2] = static_cast<FLOAT>(z); }
    template <typename SIZE_T> const FLOAT& operator[](const SIZE_T& i) const { return v[i]; }
    template <typename SIZE_T> FLOAT& operator[](const SIZE_T& i) { return v[i]; }
};
using Vec3d = Vec3r<double>;

struct Result {
    double distance = std::numeric_limits<double>::max();
    Vec3d nearest_point;
    Discregrid::NearestEntity nearest_entity;
    int triangle_id = -1;
};

class TriangleMeshDistance {
public:
    TriangleMeshDistance() = default;
    TriangleMeshDistance(const TriangleMeshDistance&) = delete;
    TriangleMeshDistance& operator=(const TriangleMeshDistance&) = delete;
    ~TriangleMeshDistance() { if (m_group) dg_mesh_group_destroy(m_group); if (m_mesh) dg_mesh_destroy(m_mesh); }

    template <typename FLOAT, typename INT, typename SIZE_T>
    TriangleMeshDistance(const FLOAT* vertices, const SIZE_T n_vertices, const INT* triangles, const SIZE_T n_triangles) { construct(vertices, n_vertices, triangles, n_triangles); }
    template <typename IndexableVector3double, typename IndexableVector3int>
    TriangleMeshDistance(const std::vector<IndexableVector3double>& vertices, const std::vector<IndexableVector3int>& triangles) { construct(vertices, triangles); }
    TriangleMeshDistance(const TriangleMesh& mesh) { construct(mesh.vertex_data(), mesh.face_data()); }

    template <typename FLOAT, typename INT, typename SIZE_T>
    void construct(const FLOAT* vertices, const SIZE_T n_vertices, const INT* triangles, const SIZE_T n_triangles)
    {
        std::vector<double> V(3 * (size_t)n_vertices); std::vector<uint32_t> F(3 * (size_t)n_triangles);
        for (size_t i = 0; i < V.size(); i++) V[i] = (double)vertices[i];
        for (size_t i = 0; i < F.size(); i++) F[i] = (uint32_t)triangles[i];
        upload(V, F);
    }
    template <typename IndexableVector3double, typename IndexableVector3int>
    void construct(const std::vector<IndexableVector3double>& vertices, const std::vector<IndexableVector3int>& triangles)
    {
        std::vector<double> V(3 * vertices.size()); std::vector<uint32_t> F(3 * triangles.size());
        for (size_t i = 0; i < vertices.size(); i++) for (int d = 0; d < 3; d++) V[3 * i + d] = (double)vertices[i][d];
        for (size_t i = 0; i < triangles.size(); i++) for (int d = 0; d < 3; d++) F[3 * i + d] = (uint32_t)triangles[i][d];
        upload(V, F);
    }

    template <typename IndexableVector3double> Result unsigned_distance(const IndexableVector3double& p) const { return unsigned_distance(std::array<double, 3>{{(double)p[0], (double)p[1], (double)p[2]}}); }
    Result unsigned_distance(const std::array<double, 3>& p) const { Result r; query(p.data(), 1, 0, &r); return r; }
    template <typename IndexableVector3double> Result signed_distance(const IndexableVector3double& p) const { return signed_distance(std::array<double, 3>{{(double)p[0], (double)p[1], (double)p[2]}}); }
    Result signed_distance(const std::array<double, 3>& p) const { Result r; query(p.data(), 1, 1, &r); return r; }

    // batched forms (new): points = n x 3 doubles, xyzxyz
    std::vector<Result> signed_distance_batch(const double* points, size_t n) const { std::vector<Result> r(n); query(points, n, 1, r.data()); return r; }
    std::vector<Result> unsigned_distance_batch(const double* points, size_t n) const { std::vector<Result> r(n); query(points, n, 0, r.data()); return r; }

    bool is_constructed() const { return m_mesh != nullptr; }
    const dg_mesh* handle() const { require(); return m_mesh; }
    // new: spread addFunction over n GPUs of this node (`GenerateSDF --gpus N`): the device records are replicated once, by peer copies
    void useGpus(int n_gpus)
    {
        require();
        if (m_group) { dg_mesh_group_destroy(m_group); m_group = nullptr; }
        if (n_gpus > 1 && dg_mesh_group_create(m_mesh, n_gpus, nullptr, &m_group) != DG_OK) throw std::runtime_error(std::string("TriangleMeshDistance: ") + dg_last_error());
    }
    dg_mesh_group* group() const { return m_group; }
    // new: the sign mode of signed_distance and of the grid calls built on it (MeshSignedDistanceFunction, MeshDistanceBandPredicate);
    // beta >= 1 or infinity (the exact sum).  Not to be called while another thread uses this object.  The winding mode runs on one GPU:
    // it throws after useGpus(n > 1), and useGpus(n > 1) throws in it.
    void setSignMode(SignMode mode, double beta = 2.0)
    {
        require();
        if (mode == SignMode::Winding && m_group) throw std::runtime_error("TriangleMeshDistance: the winding sign mode runs on one GPU; it is not available after useGpus(n > 1)");
        if (dg_mesh_set_sign_mode(m_mesh, (int)mode, beta) != DG_OK) throw std::runtime_error(std::string("TriangleMeshDistance: ") + dg_last_error());
        m_sign_mode = mode;
    }
    SignMode signMode() const { return m_sign_mode; }
    // new: moves the vertices (the count of the construction) and refits the tree, pseudonormals and winding records on the GPU; the
    // triangles and the tree's leaf order stay, so construct again after large deformations.  Not to be called while another thread uses
    // this object.  The multi-GPU replicas would go stale: it throws after useGpus(n > 1).
    template <typename IndexableVector3double> void refit(const std::vector<IndexableVector3double>& vertices)
    {
        std::vector<double> V(3 * vertices.size());
        for (size_t i = 0; i < vertices.size(); i++) for (int k = 0; k < 3; k++) V[3 * i + k] = (double)vertices[i][k];
        refit_check();
        if (dg_mesh_refit(m_mesh, V.data(), vertices.size()) != DG_OK) throw std::runtime_error(std::string("TriangleMeshDistance: ") + dg_last_error());
    }
    // the same from n_vertices x 3 doubles in the mesh's device memory, read on `stream` (cudaStream_t) after the work queued there
    void refit(const double* d_vertices, size_t n_vertices, void* stream = nullptr)
    {
        refit_check();
        if (dg_mesh_refit_device(m_mesh, d_vertices, n_vertices, stream) != DG_OK) throw std::runtime_error(std::string("TriangleMeshDistance: ") + dg_last_error());
    }
    // new: generalized winding number at a point (1 inside a closed surface, 0 outside), or at n points (xyzxyz) into w[n]
    template <typename IndexableVector3double> double winding_number(const IndexableVector3double& p, double beta = 2.0) const
    {
        const double x[3] = {(double)p[0], (double)p[1], (double)p[2]};
        double w = 0.0;
        winding_number(x, 1, &w, beta);
        return w;
    }
    void winding_number(const double* points, size_t n, double* w, double beta = 2.0) const
    {
        require();
        if (dg_mesh_winding_number(m_mesh, points, n, beta, w) != DG_OK) throw std::runtime_error(std::string("TriangleMeshDistance: ") + dg_last_error());
    }
    // new: the first hit of n rays (origins, directions: xyzxyz) on the triangles, t in [t_min, t_max] (a segment x0 -> x1 is the ray
    // (x0, x1 - x0) on [0, 1]); outputs t, triangle_id, barycentric (3 per ray; may be NULL) and status = DG_RAY_MISS / DG_RAY_ENTER /
    // DG_RAY_LEAVE, all n (dg_mesh_raycast; contract in k9_mesh_raycast.cu).  Runs on the mesh's GPU, also after useGpus(n > 1).
    void raycast(size_t n, const double* origins, const double* directions, double t_min, double t_max, double* t, int32_t* triangle_id,
                 double* barycentric, int32_t* status) const
    {
        require();
        if (dg_mesh_raycast(m_mesh, origins, directions, n, t_min, t_max, t, triangle_id, barycentric, status) != DG_OK)
            throw std::runtime_error(std::string("TriangleMeshDistance: ") + dg_last_error());
    }
    // the same on arrays in the mesh's device memory, asynchronous on `stream` (cudaStream_t)
    void raycast(size_t n, const double* d_origins, const double* d_directions, double t_min, double t_max, double* d_t, int32_t* d_triangle_id,
                 double* d_barycentric, int32_t* d_status, void* stream) const
    {
        require();
        if (dg_mesh_raycast_device(m_mesh, d_origins, d_directions, n, t_min, t_max, d_t, d_triangle_id, d_barycentric, d_status, stream) != DG_OK)
            throw std::runtime_error(std::string("TriangleMeshDistance: ") + dg_last_error());
    }
    // new: the distance query on n points in the mesh's device memory with the barycentric weights (3 per point) of the nearest point on
    // its triangle's vertices; every output may be NULL; asynchronous on `stream` (dg_mesh_distance_bary_device; contract in
    // k10_distance_grad.cu).  Follows setSignMode when is_signed.
    void nearest(size_t n, const double* d_points, bool is_signed, double* d_distance, double* d_nearest_point, int32_t* d_nearest_entity,
                 int32_t* d_triangle_id, double* d_barycentric, void* stream) const
    {
        require();
        if (dg_mesh_distance_bary_device(m_mesh, d_points, n, is_signed ? 1 : 0, d_distance, d_nearest_point, d_nearest_entity, d_triangle_id,
                                         d_barycentric, stream) != DG_OK)
            throw std::runtime_error(std::string("TriangleMeshDistance: ") + dg_last_error());
    }
    // new: the gradients of sum(grad_distance * distance) for the outputs of nearest(): d_grad_points (n x 3) and d_grad_vertices
    // (n_vertices x 3, overwritten, summed in a fixed order), each may be NULL; on `stream` (dg_mesh_distance_vjp_device)
    void distance_vjp(size_t n, const double* d_points, const double* d_distance, const double* d_nearest_point, const int32_t* d_triangle_id,
                      const double* d_barycentric, const double* d_grad_distance, double* d_grad_points, double* d_grad_vertices, void* stream) const
    {
        require();
        if (dg_mesh_distance_vjp_device(m_mesh, n, d_points, d_distance, d_nearest_point, d_triangle_id, d_barycentric, d_grad_distance,
                                        d_grad_points, d_grad_vertices, stream) != DG_OK)
            throw std::runtime_error(std::string("TriangleMeshDistance: ") + dg_last_error());
    }
    // new: the gradients of the first hits (t, barycentric from raycast on device arrays) in the origins, the directions and the vertices,
    // for the upstream gradients d_grad_t [n] and d_grad_barycentric [n x 3] (either may be NULL, not both), taken at the positions
    // d_vertices [n_vertices x 3] the rays were cast against; every output [n x 3], [n x 3], [n_vertices x 3] may be NULL, the vertex
    // gradient is overwritten and summed in a fixed order; on `stream` (dg_mesh_raycast_vjp_device; contract in k12_raycast_grad.cu)
    void raycast_vjp(size_t n, const double* d_directions, const double* d_t, const int32_t* d_triangle_id, const double* d_barycentric,
                     const double* d_vertices, const double* d_grad_t, const double* d_grad_barycentric, double* d_grad_origins,
                     double* d_grad_directions, double* d_grad_vertices, void* stream) const
    {
        require();
        if (dg_mesh_raycast_vjp_device(m_mesh, n, d_directions, d_t, d_triangle_id, d_barycentric, d_vertices, d_grad_t, d_grad_barycentric,
                                       d_grad_origins, d_grad_directions, d_grad_vertices, stream) != DG_OK)
            throw std::runtime_error(std::string("TriangleMeshDistance: ") + dg_last_error());
    }

private:
    dg_mesh* m_mesh = nullptr;
    dg_mesh_group* m_group = nullptr;
    SignMode m_sign_mode = SignMode::Pseudonormal;
    void require() const { if (!m_mesh) throw std::runtime_error("DistanceTriangleMesh error: not constructed."); }
    void refit_check() const
    {
        require();
        if (m_group) throw std::runtime_error("TriangleMeshDistance: refit is not available after useGpus(n > 1): the replicas on the other GPUs would go stale");
    }
    void upload(const std::vector<double>& V, const std::vector<uint32_t>& F)
    {
        if (m_group) { dg_mesh_group_destroy(m_group); m_group = nullptr; }
        if (m_mesh) { dg_mesh_destroy(m_mesh); m_mesh = nullptr; }
        m_sign_mode = SignMode::Pseudonormal;
        if (F.empty()) throw std::runtime_error("DistanceTriangleMesh error: Empty triangle list.");
        if (dg_mesh_create(V.data(), V.size() / 3, F.data(), F.size() / 3, &m_mesh) != DG_OK) throw std::runtime_error(std::string("TriangleMeshDistance: ") + dg_last_error());
    }
    void query(const double* pts, size_t n, int is_signed, Result* out) const
    {
        require();
        std::vector<double> d(n), q(3 * n); std::vector<int32_t> e(n), t(n);
        if (dg_mesh_distance(m_mesh, pts, n, is_signed, d.data(), q.data(), e.data(), t.data()) != DG_OK) throw std::runtime_error(std::string("TriangleMeshDistance: ") + dg_last_error());
        for (size_t i = 0; i < n; i++) { out[i].distance = d[i]; out[i].nearest_point = Vec3d(q[3 * i], q[3 * i + 1], q[3 * i + 2]); out[i].nearest_entity = (NearestEntity)e[i]; out[i].triangle_id = t[i]; }
    }
};

// The functor GenerateSDF passes to addFunction (cmd/generate_sdf/main.cpp:94-102), as a TYPE the grid can recognise through
// std::function::target<>() (the reference uses an anonymous lambda, which a GPU cannot run -- SURVEY F6/H1).  Calling it
// evaluates one point through the batch API, like the reference lambda.
struct MeshSignedDistanceFunction {
    const TriangleMeshDistance* md;
    double sign;                                    // -1.0 for --invert
    explicit MeshSignedDistanceFunction(const TriangleMeshDistance& m, bool invert = false) : md(&m), sign(invert ? -1.0 : 1.0) {}
    double operator()(Eigen::Vector3d const& xi) const { const double d = md->signed_distance(xi).distance; return sign == 1.0 ? d : sign * d; }
};

// new: the narrow-band sample predicate x -> |md.signed_distance(x).distance| <= band as a recognisable type.  A valid SamplePredicate on its
// own; handed to addFunction next to a MeshSignedDistanceFunction over the same md, the band is sampled on the GPU (DBL_MAX outside it).
struct MeshDistanceBandPredicate {
    const TriangleMeshDistance* md;
    double band;
    MeshDistanceBandPredicate(const TriangleMeshDistance& m, double w) : md(&m), band(w) {}
    bool operator()(Eigen::Vector3d const& xi) const { return std::abs(md->signed_distance(xi).distance) <= band; }
};

}  // namespace Discregrid
