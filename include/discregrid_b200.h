/* =====================================================================================
 * discregrid_b200.h -- C-ABI of the H100-native (sm_90a) Discregrid hot path.
 *
 * Plain C, plain pointers and sizes, no torch / Eigen / STL types.  This is the drop-in
 * boundary: the reference (InteractiveComputerGraphics/Discregrid @ ddf20dc) has no FFI of its
 * own -- its boundary is the C++ class API -- so each entry point names the reference
 * function(s) it replaces (paths relative to the reference root):
 *
 *   geometry/TriangleMeshDistance.h = discregrid/include/Discregrid/geometry/TriangleMeshDistance.h
 *   cubic_lagrange_discrete_grid.cpp = discregrid/src/cubic_lagrange_discrete_grid.cpp
 *   discrete_grid.{hpp,cpp}          = discregrid/include/Discregrid/discrete_grid.hpp, discregrid/src/discrete_grid.cpp
 *
 * Conventions
 *   - every function returns DG_OK (0) or a negative dg_status; dg_last_error() gives the message of
 *     the calling thread's last failure.  The library never calls exit() (the reference does:
 *     TriangleMeshDistance.h:318-321, 338-341).
 *   - "host" entry points take host pointers and include the H2D/D2H copies; "_device" entry points
 *     take device pointers of the CURRENT CUDA device plus a cudaStream_t (passed as void*, NULL =
 *     default stream), are asynchronous on that stream, and are what bench.py times with CUDA events.
 *   - there is NO CPU fallback: without a CUDA device every compute entry point fails with
 *     DG_ERR_NO_DEVICE.
 *   - arithmetic is IEEE fp64, round-to-nearest, no FMA contraction, in the reference's operation
 *     order (SURVEY.md appendix A), so results are bit-identical to the reference's x86-64 build.
 *   - the sentinel for "no value" is DBL_MAX, as in the reference
 *     (cubic_lagrange_discrete_grid.cpp:817, 981-982, 993-994, 1015-1018, 1050-1054).
 * ===================================================================================== */
#ifndef DISCREGRID_B200_H
#define DISCREGRID_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DG_ABI_VERSION 1

#if defined(__GNUC__)
#define DG_API __attribute__((visibility("default")))
#else
#define DG_API
#endif

typedef enum dg_status {
    DG_OK = 0,
    DG_ERR_INVALID = -1,     /* bad argument (NULL, empty mesh, zero resolution, range out of bounds ...) */
    DG_ERR_NO_DEVICE = -2,   /* no usable CUDA device: there is no CPU fallback */
    DG_ERR_CUDA = -3,        /* a CUDA runtime call failed; dg_last_error() has the cudaError string */
    DG_ERR_NOMEM = -4,       /* host or device allocation failed */
    DG_ERR_SELFTEST = -5,    /* device self-test failed (e.g. library built with FMA contraction on) */
    DG_ERR_IO = -6,          /* a file could not be opened or read */
    DG_ERR_CALLBACK = -7     /* a caller-supplied callback returned nonzero; dg_last_error() names the callback and the chunk */
} dg_status;

/* TriangleMeshDistance.h:75 -- same numbering */
typedef enum dg_nearest_entity { DG_V0 = 0, DG_V1, DG_V2, DG_E01, DG_E12, DG_E02, DG_F } dg_nearest_entity;

/* Grid geometry = the DiscreteGrid members (discrete_grid.hpp:93-98).  cell_size / inv_cell_size are passed
 * verbatim from the host object (never recomputed on the device); dg_grid_init fills them the way the
 * DiscreteGrid constructor does (discrete_grid.hpp:22-29). */
typedef struct dg_grid_desc {
    double   domain_min[3];
    double   domain_max[3];
    uint32_t resolution[3];
    uint32_t _pad;
    double   cell_size[3];
    double   inv_cell_size[3];
} dg_grid_desc;

typedef struct dg_mesh  dg_mesh;    /* device-resident TriangleMeshDistance (BVH + triangles + pseudonormals) */
typedef struct dg_field dg_field;   /* device-resident field of a CubicLagrangeDiscreteGrid (one m_nodes/m_cells/m_cell_map entry) */

/* ---- library ------------------------------------------------------------------------------- */
DG_API int         dg_abi_version(void);
DG_API const char* dg_last_error(void);
/* Number of CUDA devices visible (0 if none / no driver). */
DG_API int         dg_device_count(void);
/* cudaSetDevice for this library's CUDA runtime instance (call it with LOCAL_RANK in a one-process-per-GPU job). */
DG_API int         dg_set_device(int device);
/* Runs the device self-test (FMA-contraction probe + trivial kernel) on the current device. */
DG_API int         dg_selftest(void);
/* Measures the fp64 issue rate of the current device for the library's instruction mix (DMUL + DADD, no FMA contraction -- the
 * numerical contract forbids fused operations): Tflop/s.  bench.py uses it as the measured denominator of the fp64 rooflines. */
DG_API int         dg_fp64_rate_probe(double* tflops);
/* Kernels launched by this library in this process since load / last reset (all streams). */
DG_API uint64_t    dg_kernel_launch_count(void);
DG_API void        dg_kernel_launch_count_reset(void);

/* ---- grid helpers (host, no GPU) ----------------------------------------------------------------
 * replaces: DiscreteGrid ctor discrete_grid.hpp:22-29; node count cubic_lagrange_discrete_grid.cpp:790-796;
 * GenerateSDF's asymmetric domain padding cmd/generate_sdf/main.cpp:83-91. */
DG_API int dg_grid_init(const double domain_min[3], const double domain_max[3], const uint32_t resolution[3], dg_grid_desc* out);
DG_API int dg_grid_num_nodes(const uint32_t resolution[3], uint64_t* n_nodes);
DG_API int dg_generate_sdf_domain(const double* vertices, uint64_t n_vertices, double domain_min[3], double domain_max[3]);

/* ---- OBJ reader (host, no GPU; SURVEY 8f N4) ---------------------------------------------------------
 * replaces the parser of Discregrid::TriangleMesh(path) (src/mesh/triangle_mesh.cpp:90-124): "v x y z" and "f a[/..] b[/..] c[/..]"
 * lines, everything else ignored; same doubles as the stream extraction (correctly rounded), indices made 0-based.  The arrays
 * are allocated by the library and released with dg_obj_free.  DG_ERR_IO when the file cannot be read, DG_ERR_INVALID for a face
 * index the reference's std::stoi would throw on. */
DG_API int dg_obj_read(const char* path, double** vertices, uint64_t* n_vertices, uint32_t** triangles, uint64_t* n_triangles);
DG_API void dg_obj_free(double* vertices, uint32_t* triangles);

/* ---- mesh / distance ------------------------------------------------------------------------------
 * dg_mesh_create replaces TriangleMeshDistance::construct / _construct / _build_tree
 * (TriangleMeshDistance.h:251-267, 336-441, 443-512): builds the reference's bounding-sphere tree (same
 * split, same std::sort order, same spheres) and the angle-weighted pseudonormals on the host, re-lays
 * them out for the GPU and uploads them ONCE.  vertices: n_vertices x 3 doubles (xyzxyz), triangles:
 * n_triangles x 3 uint32 (0-based).  Fails with DG_ERR_INVALID on an empty triangle list or an index
 * out of range (the reference exits / reads out of bounds). */
DG_API int dg_mesh_create(const double* vertices, uint64_t n_vertices, const uint32_t* triangles, uint64_t n_triangles, dg_mesh** out);
DG_API int dg_mesh_destroy(dg_mesh* mesh);
/* info[0]=n_vertices, [1]=n_triangles, [2]=max stack depth, [3]=watertight flags (bit0: edge with one
 * triangle, bit1: edge with >2 triangles -- the two warnings of TriangleMeshDistance.h:422-438),
 * [4]=device bytes, [5]=host build microseconds, [6]=upload microseconds, [7]=the CUDA device the mesh lives on */
DG_API int dg_mesh_info(const dg_mesh* mesh, uint64_t info[8]);
/* Test/diagnostic: copies the host-built tree in the reference's node numbering (pre-order; left == -1 marks
 * a leaf whose `right` is the triangle id).  spheres: n_nodes x 8 (cl.xyz, rl, cr.xyz, rr), kids: n_nodes x 2.
 * n_nodes = 2*n_triangles-1.  Any pointer may be NULL. */
DG_API int dg_mesh_tree(const dg_mesh* mesh, double* spheres, int32_t* kids);
/* Test/diagnostic: pseudonormals in the reference's arrays (TriangleMeshDistance.h:122-124). */
DG_API int dg_mesh_pseudonormals(const dg_mesh* mesh, double* tri /*nT x3*/, double* edge /*nT x3x3*/, double* vert /*nV x3*/);

/* Batched TriangleMeshDistance::signed_distance / unsigned_distance (TriangleMeshDistance.h:269-328) for n
 * points (n x 3 doubles).  Outputs (each nullable): distance[n], nearest_point[n x 3], nearest_entity[n]
 * (dg_nearest_entity), triangle_id[n] -- the fields of Discregrid::Result (TriangleMeshDistance.h:80-86). */
DG_API int dg_mesh_distance(const dg_mesh* mesh, const double* points, uint64_t n, int is_signed,
                     double* distance, double* nearest_point, int32_t* nearest_entity, int32_t* triangle_id);
DG_API int dg_mesh_distance_device(const dg_mesh* mesh, const double* d_points, uint64_t n, int is_signed,
                            double* d_distance, double* d_nearest_point, int32_t* d_nearest_entity,
                            int32_t* d_triangle_id, void* stream);

/* ---- sign modes and generalized winding numbers (K5, k5_winding.cu; beyond the reference) -----------------------------------------
 * The reference signs every distance with the angle-weighted pseudonormal at the nearest entity (TriangleMeshDistance.h:269-308), which is
 * right only for closed manifold meshes (dg_mesh_info[3] reports open and non-manifold edges).  The winding mode takes the sign from the
 * generalized winding number w(x) instead (Barill et al. 2018): inside iff w > 0.5.  w is the sum of the triangles' solid angles / 4 pi,
 * evaluated over the mesh's sphere tree with a far-field expansion for clusters farther than beta times their radius; the numerical
 * contract (operation order, the library's own atan2, the fold order) is stated in k5_winding.cu.  beta >= 1 or +inf (exact sum over all
 * triangles); NaN or < 1: DG_ERR_INVALID.  The default beta is 2.
 *   dg_mesh_set_sign_mode: DG_SIGN_PSEUDONORMAL (the default, the reference's rule) or DG_SIGN_WINDING, with the beta the signed entry
 *       points then use.  Must not be called while another call uses the same mesh.  In the winding mode these single-GPU entry points take
 *       the sign from w: dg_mesh_distance[_device] with is_signed (nearest point, entity and triangle id are those of the unsigned query),
 *       dg_sample_sdf[_device], dg_add_function_sdf, dg_sample_sdf_band_device, dg_add_function_sdf_band, dg_reduced_band_create: K1 runs
 *       with sign = +1 and a node pass writes sign * (w > 0.5 ? -d : d); the DBL_MAX sentinels are those of the pseudonormal mode.
 *       dg_mesh_group_create, dg_add_function_sdf_multi, dg_sample_sdf_multi_device and the slab / interleaved entry points refuse a mesh in
 *       the winding mode (DG_ERR_INVALID).
 *   dg_mesh_winding_number[_device]: w[n] for points x[n x 3], host arrays or device pointers on `stream`.
 * The winding records (the vertices per triangle in leaf order, 72 B, and a 256-byte cluster pair per internal node) are built on the host
 * and uploaded at their first use; a mesh that never uses them allocates nothing more. */
#define DG_SIGN_PSEUDONORMAL 0   /* the reference's rule; default */
#define DG_SIGN_WINDING      1
DG_API int dg_mesh_set_sign_mode(dg_mesh* mesh, int mode, double beta);
DG_API int dg_mesh_winding_number(const dg_mesh* mesh, const double* x, uint64_t n, double beta, double* w);
DG_API int dg_mesh_winding_number_device(const dg_mesh* mesh, const double* d_x, uint64_t n, double beta, double* d_w, void* stream);

/* ---- refit to new vertex positions (K8, k8_refit.cu; beyond the reference) ---------------------------------------------------------
 * dg_mesh_refit replaces the mesh's vertices with `vertices` (n_vertices x 3 doubles, the count of the build) and recomputes on the device
 * every record the kernels read: leaf records and shadows, the sphere tree's spheres and fp32 records, the bounding-box centre and half
 * extent, the pseudonormals and, when they exist, the winding records.  The triangles and the tree's leaf order stay those of
 * dg_mesh_create, so spheres grow with large deformations and queries slow down: rebuild with dg_mesh_create when they do.  Query
 * results after a refit are the reference's query rule over the refit tree and pseudonormals; the numerical contract (sums bottom-up,
 * the library's own acos for the pseudonormal angles) is stated in k8_refit.cu.  The watertight flags, the stack depth, the sign mode and
 * beta are unchanged.
 *   dg_mesh_refit_device: d_vertices on the mesh's device, read on `stream` after the work already queued there; returns when the refit
 *       has finished (it reads back the centre and half extent).  No host<->device copy proportional to the mesh.
 *   dg_mesh_refit: uploads the host array, then runs the device form.
 * Topology tables and scratch are allocated at the first refit and kept (dg_mesh_info[4] counts them).  DG_ERR_INVALID, before anything is
 * written: NULL mesh, NULL vertices with n_vertices > 0, n_vertices different from the build's, a mesh on another device, a mesh a live
 * dg_mesh_group replicates.  Like dg_mesh_set_sign_mode, a refit must not overlap any other call that uses the mesh, including work queued
 * on other streams.  A CUDA error after records have started to be written leaves the mesh failed: every later call on it except
 * dg_mesh_destroy returns DG_ERR_INVALID.  After a refit dg_mesh_tree and dg_mesh_pseudonormals report the refit records (a vertex no
 * triangle uses has NaN pseudonormals, as after dg_mesh_create). */
DG_API int dg_mesh_refit(dg_mesh* mesh, const double* vertices, uint64_t n_vertices);
DG_API int dg_mesh_refit_device(dg_mesh* mesh, const double* d_vertices, uint64_t n_vertices, void* stream);

/* ---- K1: addFunction node loop with the GenerateSDF functor -------------------------------------------
 * replaces the hot loop cubic_lagrange_discrete_grid.cpp:806-817 with
 * func = sign * md.signed_distance(x).distance (cmd/generate_sdf/main.cpp:97,101; sign = -1 for --invert):
 *     out[l - l_begin] = sign * signed_distance(indexToNodePosition(l)).distance,  l in [l_begin, l_end)
 * indexToNodePosition = cubic_lagrange_discrete_grid.cpp:604-665.  Node ids are the reference's (uint32 in
 * the file format); 64-bit here only so ranges can be expressed without overflow.
 * A sub-range is what a rank computes when the grid is sharded across GPUs (SURVEY 8e).
 * The host form overlaps kernel chunks, D2H DMA (pooled pinned double buffer) and the copy into `out_host`; for ranges of 32 MiB and more
 * (environment: DG_HOST_HELPERS_MIN_BYTES) a few worker threads (a quarter of the usable CPUs, DG_HOST_THREADS) pre-fault `out_host` and
 * share that copy, as in dg_add_function_sdf; calls are serialised per process.  The _device form is asynchronous on `stream` and may be
 * issued concurrently on several streams. */
DG_API int dg_sample_sdf(const dg_mesh* mesh, const dg_grid_desc* grid, double sign, uint64_t l_begin, uint64_t l_end, double* out_host);
DG_API int dg_sample_sdf_device(const dg_mesh* mesh, const dg_grid_desc* grid, double sign, uint64_t l_begin, uint64_t l_end,
                         double* d_out, void* stream);
/* The WHOLE of CubicLagrangeDiscreteGrid::addFunction with the GenerateSDF functor (cubic_lagrange_discrete_grid.cpp:780-899) into
 * the three arrays the reference appends to m_nodes / m_cells / m_cell_map: nodes_host[n_nodes] (the node loop :806-817, on the GPU),
 * cells_host[n_cells x 32] (connectivity :833-886) and cell_map_host[n_cells] (identity :888-891) -- the two index tables are written
 * by host threads straight into the caller's memory WHILE the GPU samples the nodes, so the call ends one D2H piece after the last
 * kernel chunk.  cells_host / cell_map_host may be NULL (skipped).  timings_ms: NULL or 6 doubles = total, node pipeline done,
 * index tables done, coefficient array pre-faulted (all ms since entry), worker threads used, 0.
 * This is what the C++ facade's addFunction(MeshSignedDistanceFunction) calls and what bench.py times as `e2e`. */
DG_API int dg_add_function_sdf(const dg_mesh* mesh, const dg_grid_desc* grid, double sign, double* nodes_host, uint32_t* cells_host,
                        uint32_t* cell_map_host, double* timings_ms);
/* ---- K1, narrow band: addFunction(func, verbose, pred) with the band predicate ----------------------------------------------------
 * replaces the node loop cubic_lagrange_discrete_grid.cpp:806-817 with func as above and
 *     pred(x) = std::abs(md.signed_distance(x).distance) <= band      (fp64, the reference's own distance)
 * i.e. out = sign * distance where pred holds and DBL_MAX (:817) elsewhere -- the pattern GenerateDensityMap uses
 * (cmd/generate_density_map/main.cpp:119-147) and what reduceField (:1065-1174) then sparsifies.  In-band nodes hold exactly the bits
 * dg_sample_sdf writes.  A classifier first drops the blocks of nodes that provably lie farther than `band` from every triangle (their
 * nodes get DBL_MAX without a tree query); only the rest is sampled.  band must be >= 0 (negative or NaN: DG_ERR_INVALID); +inf keeps
 * every node.
 *   dg_sample_sdf_band_device: nodes [l_begin, l_end) into d_out, asynchronous on `stream` like dg_sample_sdf_device (its scratch is
 *       allocated and freed in stream order); nodes outside the range are never written.
 *   dg_add_function_sdf_band: the whole addFunction into host arrays, as dg_add_function_sdf (same pipeline, same timings_ms). */
DG_API int dg_sample_sdf_band_device(const dg_mesh* mesh, const dg_grid_desc* grid, double sign, double band, uint64_t l_begin, uint64_t l_end,
                              double* d_out, void* stream);
DG_API int dg_add_function_sdf_band(const dg_mesh* mesh, const dg_grid_desc* grid, double sign, double band, double* nodes_host,
                             uint32_t* cells_host, uint32_t* cell_map_host, double* timings_ms);
/* ---- multi-GPU from ONE process (SURVEY 8b: `dg_sample_sdf(..., n_gpus, ...)`; 8e) -------------------------------------------
 * A dg_mesh_group replicates the device records of `mesh` on n_gpus - 1 further GPUs (peer copies from the mesh's device; the host
 * build is not repeated).  devices: NULL = the mesh's device first, then the lowest other ids; else n_gpus ids with devices[0] == the
 * mesh's device.  The group borrows `mesh` (destroy the group first).  n_gpus = 1 is valid (same code path on one GPU).
 *   dg_add_function_sdf_multi : dg_add_function_sdf across the group -- plane pairs of the four node arrays dealt round-robin to
 *       2 x n_gpus parts, one host thread and two streams per GPU, every part DMA'd to its final place in nodes_host (directly if that
 *       memory is page-locked, else through pinned staging); index tables by host threads meanwhile.  No collective: the exchange
 *       target is host memory.  This is what `GenerateSDF --gpus N` calls.
 *   dg_sample_sdf_multi_device: the coefficient array device-resident on EVERY GPU of the group (d_out[i] = n_nodes doubles in
 *       device i's memory): one launch per GPU into its slot of an exchange buffer, ONE in-place ncclAllGather per device
 *       (ncclCommInitAll, grouped calls; libnccl.so.2 is loaded at first use), one unpack kernel into the reference's node order. */
typedef struct dg_mesh_group dg_mesh_group;
DG_API int dg_mesh_group_create(const dg_mesh* mesh, int n_gpus, const int* devices, dg_mesh_group** out);
DG_API int dg_mesh_group_destroy(dg_mesh_group* group);
DG_API int dg_mesh_group_size(const dg_mesh_group* group);
DG_API int dg_add_function_sdf_multi(dg_mesh_group* group, const dg_grid_desc* grid, double sign, double* nodes_host, uint32_t* cells_host,
                              uint32_t* cell_map_host, double* timings_ms);
DG_API int dg_sample_sdf_multi_device(dg_mesh_group* group, const dg_grid_desc* grid, double sign, double* const* d_out);
/* Slab sharding of the same loop for one-process-per-GPU jobs (SURVEY 8e, "P1"): part `part` of `n_parts` samples, in ONE launch,
 * whole slow-plane PAIRS of each of the four row-major node arrays (vertex / x-edge nodes: z-slabs; y-edge nodes: x-slabs; z-edge
 * nodes: y-slabs), i.e. no partially filled bricks and a single launch tail per rank.  Results are written at their final positions
 * of the full coefficient array d_full (n_nodes doubles).  ranges[8] = the four [l_begin, l_end) node ranges of this part (some may
 * be empty); dg_slab_ranges computes them on the host (no GPU) for the exchange step. */
DG_API int dg_slab_ranges(const dg_grid_desc* grid, uint32_t part, uint32_t n_parts, uint64_t ranges[8]);
DG_API int dg_sample_sdf_slab_device(const dg_mesh* mesh, const dg_grid_desc* grid, double sign, uint32_t part, uint32_t n_parts,
                              double* d_full, void* stream);
/* Interleaved slab sharding (SURVEY H7 / 8e P1): the slow-plane pairs of every node array are dealt round-robin -- pair p belongs to
 * part p % n_parts -- which balances the spatially varying cost almost perfectly and still needs ONE launch per rank and no masked
 * bricks.  A part writes its pairs compactly into its slot of an exchange buffer of n_parts x slot_elems doubles
 * (dg_interleaved_slot_elems); after ONE all-gather of the slots, dg_interleaved_unpack_device scatters them into the
 * reference's node order.  n_parts <= 16. */
DG_API int dg_interleaved_slot_elems(const dg_grid_desc* grid, uint32_t n_parts, uint64_t* slot_elems);
DG_API int dg_sample_sdf_interleaved_device(const dg_mesh* mesh, const dg_grid_desc* grid, double sign, uint32_t part, uint32_t n_parts,
                                     double* d_slot, void* stream);
DG_API int dg_interleaved_unpack_device(const dg_grid_desc* grid, uint32_t n_parts, const double* d_slots, double* d_nodes, void* stream);
/* the same layout on the host (no GPU): for node ids l in [l_begin, l_end), the part that samples node l and its position inside
 * that part's slot (either output may be NULL) -- for hosts that consume or exchange slots themselves */
DG_API int dg_interleaved_node_slots(const dg_grid_desc* grid, uint32_t n_parts, uint64_t l_begin, uint64_t l_end, uint32_t* part_out,
                              uint64_t* pos_out);
/* indexToNodePosition for l in [l_begin, l_end) -> x[(l-l_begin)*3 ..] (cubic_lagrange_discrete_grid.cpp:604-665) */
DG_API int dg_node_positions(const dg_grid_desc* grid, uint64_t l_begin, uint64_t l_end, double* x_host);
/* Cell connectivity table of addFunction (cubic_lagrange_discrete_grid.cpp:833-886) for cells
 * [c_begin, c_end): cells_host[(c-c_begin)*32 + j]. */
DG_API int dg_build_cells(const uint32_t resolution[3], uint64_t c_begin, uint64_t c_end, uint32_t* cells_host);

/* ---- fields / K2: interpolate ------------------------------------------------------------------------
 * dg_field_create uploads one field (m_nodes[f], m_cells[f], m_cell_map[f] of
 * cubic_lagrange_discrete_grid.hpp:69-71) and builds the device layout: one contiguous 256-byte block of the
 * 32 coefficients per kept cell.  cells == NULL means the closed-form table addFunction builds
 * (cubic_lagrange_discrete_grid.cpp:833-886, n_cells_kept must then equal nx*ny*nz); cell_map == NULL means identity
 * (:888-891).  After reduceField() pass the reduced arrays (cell_map entries UINT32_MAX = removed cell). */
DG_API int dg_field_create(const dg_grid_desc* grid, const double* nodes, uint64_t n_nodes, const uint32_t* cells,
                    uint64_t n_cells_kept, const uint32_t* cell_map, dg_field** out);
/* same, coefficient array already on the device (e.g. straight out of dg_sample_sdf_device); unreduced only.  Returns once the
 * field is built on `stream` (it reads one fact about the coefficients back: see dg_density_map) */
DG_API int dg_field_create_device(const dg_grid_desc* grid, const double* d_nodes, uint64_t n_nodes, void* stream, dg_field** out);
DG_API int dg_field_destroy(dg_field* field);
/* info[0]=n_nodes, [1]=n_cells_kept, [2]=device bytes, [3]=the CUDA device the field lives on */
DG_API int dg_field_info(const dg_field* field, uint64_t info[4]);

/* Batched CubicLagrangeDiscreteGrid::interpolate(field_id, x, gradient*) (cubic_lagrange_discrete_grid.cpp:977-1063;
 * identical arithmetic to determineShapeFunctions + split interpolate, :901-975) for n points x[n x 3].
 * phi[n]; grad[n x 3] nullable (value-only path :1006-1023).  Out-of-domain / removed cell / missing coefficient
 * -> phi = DBL_MAX and grad = 0 exactly as the reference. */
DG_API int dg_interpolate_batch(const dg_field* field, const double* x, uint64_t n, double* phi, double* grad);
DG_API int dg_interpolate_batch_device(const dg_field* field, const double* d_x, uint64_t n, double* d_phi, double* d_grad, void* stream);
/* Value, gradient and Hessian in one pass (beyond the reference, which has no Hessian): phi[n] and grad[n x 3] have the bits of
 * dg_interpolate_batch with a gradient; hess[n x 3 x 3] is the row-major Hessian in x, exactly symmetric (the numerical contract is
 * in k2_interp.cu).  Sentinel points get phi = DBL_MAX, grad = 0 and hess = +0.0.  phi, grad and hess are all required when n > 0.
 * The _device form takes device pointers and runs on `stream` (a cudaStream_t; NULL = legacy default stream), asynchronously. */
DG_API int dg_interpolate_hessian_batch(const dg_field* field, const double* x, uint64_t n, double* phi, double* grad, double* hess);
DG_API int dg_interpolate_hessian_batch_device(const dg_field* field, const double* d_x, uint64_t n, double* d_phi, double* d_grad, double* d_hess,
                                               void* stream);
/* shape_function_ (cubic_lagrange_discrete_grid.cpp:339-580) for n reference-cell points xi[n x 3]:
 * N[n x 32], dN[n x 32 x 3] (nullable). */
DG_API int dg_shape_functions(const double* xi, uint64_t n, double* N, double* dN);

/* ---- K11: trainable fields (beyond the reference) -----------------------------------------------------
 * dg_field_create_trainable takes dg_field_create's arguments and checks, and makes an ordinary dg_field (interpolate, Hessian, isosurface,
 * raycast, density and volume maps all take it) that also keeps what it needs to replace its node values and to sum their gradient: its
 * cell table (when cells is given), the node -> (cell, slot) incidence table and a per-cell DBL_MAX flag (counted in dg_field_info[2]).
 * Refused when 32 * n_cells_kept >= 2^32.  Synchronises the device.
 * dg_field_set_nodes[_device] replaces the field's n_nodes node values (n_nodes must be the field's count) and repacks its blocks; the
 * _device form takes a device pointer and queues the work on `stream` with no host synchronisation.  Refused for a field not made by
 * dg_field_create_trainable.
 * dg_interpolate_vjp[_device]: for n points x[n x 3] and the upstream gradients grad_phi[n] of phi and grad_grad[n x 3] of grad (either
 * may be NULL, not both), grad_nodes[n_nodes] = the gradient with respect to the node values of sum_q grad_phi[q] phi(x_q) +
 * grad_grad[q] . grad(x_q), with K2's phi and grad on the field's current values.  Queries where K2 returns its sentinel contribute
 * nothing.  grad_nodes is always overwritten (zeros for n = 0); its bits depend only on the field's topology, x and the upstream gradients
 * (the summation order is in k11_field_grad.cu).  n must be below 2^32 - 1.  The _device form runs on `stream` with stream-ordered
 * scratch and no host synchronisation; the host form uploads every input in one piece and returns when grad_nodes is written. */
DG_API int dg_field_create_trainable(const dg_grid_desc* grid, const double* nodes, uint64_t n_nodes, const uint32_t* cells,
                                     uint64_t n_cells_kept, const uint32_t* cell_map, dg_field** out);
DG_API int dg_field_set_nodes(dg_field* field, const double* nodes, uint64_t n_nodes);
DG_API int dg_field_set_nodes_device(dg_field* field, const double* d_nodes, uint64_t n_nodes, void* stream);
DG_API int dg_interpolate_vjp(const dg_field* field, const double* x, uint64_t n, const double* grad_phi, const double* grad_grad,
                              double* grad_nodes);
DG_API int dg_interpolate_vjp_device(const dg_field* field, const double* d_x, uint64_t n, const double* d_grad_phi, const double* d_grad_grad,
                                     double* d_grad_nodes, void* stream);

/* ---- K3: GenerateDensityMap node function ---------------------------------------------------------
 * replaces addFunction(density_func, verbose, pred) of cmd/generate_density_map/main.cpp:96-133 with
 * GaussQuadrature::integrate(p=30 -> 16^3 points, gauss_quadrature.cpp:5927-5960) and CubicKernel::W
 * (sph_kernel.hpp:22-42) over nodes [l_begin, l_end) of the grid of `sdf` (its field 0):
 * out = DBL_MAX where the predicate rejects (unless no_reduction), 0 where dist > 2h, else rho0 * integral.
 * Quadrature points outside the kernel support are skipped only where that is exact, which the field's creation decides from its
 * coefficients: a field holding NaN, +-inf or magnitudes near DBL_MAX (or an h too small for them) gets the reference's NaN. */
DG_API int dg_density_map(const dg_field* sdf, double h, double rho0, int no_reduction, uint64_t l_begin, uint64_t l_end, double* out_host);
DG_API int dg_density_map_device(const dg_field* sdf, double h, double rho0, int no_reduction, uint64_t l_begin, uint64_t l_end,
                          double* d_out, void* stream);

/* ---- K3: volume map (Bender et al. 2019, "Volume Maps: An Implicit Boundary Representation for SPH"; not in the reference) ----------
 * The SPH boundary volume of an SDF, as SPlisHSPlasH builds it with addFunction over the SDF grid, in 3D and in fp64, over nodes
 * [l_begin, l_end) of the grid of `sdf` (any field: dense or reduced).  With d(y) = interpolate(sdf, y):
 *   out = DBL_MAX where GenerateDensityMap's sample predicate rejects the node (unless no_reduction), 0 where d(x) > 2h, else
 *   scale * GaussQuadrature::integrate(g, [-h, h]^3, p = 30) (16^3 points, the reference's order), with g(xi) = 0 outside the ball
 *   |xi| <= h and gamma(d(x + xi)) inside it; gamma(t) = 1 for t <= 0, W((t, 0, 0)) / W(0) for t < h (CubicKernel, radius h), 0 otherwise
 *   (DBL_MAX and NaN included).
 * The full contract is in k3_density.cu and DESIGN section 3.  h must be finite and > 0 and scale finite (else DG_ERR_INVALID), the range
 * inside the grid's nodes, out non-NULL when the range is not empty.  The _device form writes d_out on `stream` and returns at once. */
DG_API int dg_volume_map(const dg_field* sdf, double h, double scale, int no_reduction, uint64_t l_begin, uint64_t l_end, double* out_host);
DG_API int dg_volume_map_device(const dg_field* sdf, double h, double scale, int no_reduction, uint64_t l_begin, uint64_t l_end,
                                double* d_out, void* stream);

/* ---- reduceField (SURVEY 8f, N3) -------------------------------------------------------------------
 * replaces the body of CubicLagrangeDiscreteGrid::reduceField (cubic_lagrange_discrete_grid.cpp:1065-1174) after the predicate has
 * been evaluated: keep_node[l] != 0 <=> pred(x_l, c_l) && c_l != DBL_MAX (:1069-1074).  Rewrites IN PLACE, exactly as the
 * reference leaves its members: cells (n_cells_in x 32; first *n_cells_out rows = surviving cells, renumbered), nodes (first
 * *n_nodes_out coefficients = surviving nodes in the reference's Z-curve order) and cell_map (resolution product entries; 0xffffffff
 * for removed cells).
 * flags: DG_REDUCE_REFERENCE_SORT makes the plain single-threaded std::sort call instead of its multithreaded replay (same result).
 * timings_ms: NULL or 5 doubles (ms spent on cells, node compaction, sort, write-back; 1.0 if surviving nodes shared Morton keys,
 * i.e. the node order depended on how std::sort leaves equal keys). */
#define DG_REDUCE_REFERENCE_SORT 1u
/* DG_REDUCE_HOST_PASSES (or the environment variable DG_REDUCE_FIELD_HOST=1): every pass on the host threads.  Default: the index passes run
 * on the GPU (k4_reduce.cu: cell flags, cell map + row compaction, node marks, Z-curve keys, renumbering and coefficient gather); the host
 * keeps the reference's serial swap-walk compaction and the sort whose order among equal keys is std::sort's.  Without a CUDA device the
 * default fails with DG_ERR_NO_DEVICE -- nothing switches silently. */
#define DG_REDUCE_HOST_PASSES 2u
DG_API int dg_reduce_field(const dg_grid_desc* grid, double* nodes, uint64_t n_nodes, const uint8_t* keep_node, uint32_t* cells,
                    uint64_t n_cells_in, uint32_t* cell_map, uint32_t flags, uint64_t* n_nodes_out, uint64_t* n_cells_out,
                    double* timings_ms);

/* ---- reduced narrow band: addFunction(band) + reduceField(always true) in one call -----------------------------------------------
 * replaces
 *     id = addFunction(func, verbose, pred);  reduceField(id, [](Vector3d const&, double) { return true; });
 * with func and pred as for dg_add_function_sdf_band: the result is exactly what the reference holds afterwards -- the same nodes in the
 * same Z-curve order (including the order among equal keys), the same renumbered cells and the same cell map -- bit for bit what
 * dg_add_function_sdf_band followed by dg_reduce_field gives.  Everything the size of the grid stays on the current device (dense band
 * coefficients, cell flags, node marks, the swap-walk positions); the host holds one count per 1024 flags and the survivors' keys.  The
 * results stay on the device in the handle (created on, and only usable from, the current device) until dg_reduced_band_copy copies
 * them into the caller's arrays, sized with dg_reduced_band_sizes.
 *   band: >= 0 (negative or NaN: DG_ERR_INVALID); +inf keeps every node.  Grids of 2^31 nodes or more are refused before anything is
 *       allocated (as dg_reduce_field).  One GPU.
 *   flags: 0 or DG_REDUCE_REFERENCE_SORT (as for dg_reduce_field).
 *   timings_ms: NULL or 7 doubles = ms of band sampling, kept cells, node compaction, sort, write-back; 1.0 if surviving nodes shared
 *       Morton keys (dg_reduce_field's tie path); total ms.  Every stage ends with a device synchronise.
 *   dg_reduced_band_copy: nodes[n_nodes], cells[n_cells x 32], cell_map[nx*ny*nz] (0xffffffff = removed cell); nodes / cells may be NULL
 *       only when their count is 0.
 * dg_reduced_band: a reduced field kept on its device (also returned by dg_reduced_density_map_create). */
typedef struct dg_reduced_band dg_reduced_band;
DG_API int dg_reduced_band_create(const dg_mesh* mesh, const dg_grid_desc* grid, double sign, double band, uint32_t flags,
                           dg_reduced_band** out, double* timings_ms);
DG_API int dg_reduced_band_sizes(const dg_reduced_band* result, uint64_t* n_nodes, uint64_t* n_cells);
DG_API int dg_reduced_band_copy(const dg_reduced_band* result, double* nodes, uint32_t* cells, uint32_t* cell_map);
DG_API int dg_reduced_band_destroy(dg_reduced_band* result);
/* An interpolation field (the packed layout of dg_field_create) made from the reduced field held by a dg_reduced_band handle
 * (dg_reduced_band_create, dg_reduced_density_map_create, dg_reduced_function_create, dg_reduce_field_device), entirely on the
 * handle's device: nothing is copied to or from the host and the rows are not re-checked (the library made them).  The field has the
 * grid the handle was made for, and dg_field_info gives what it gives for dg_field_create of the handle's dg_reduced_band_copy.
 * Synchronous: when it returns, the field does not depend on the handle, which may be destroyed.  The handle must live on the current
 * device (DG_ERR_INVALID otherwise).  A handle with no kept cell gives a field whose every query returns DBL_MAX. */
DG_API int dg_field_create_reduced(const dg_reduced_band* r, dg_field** out);

/* ---- level sets: the surface {phi = iso} of a field as a triangle mesh (not in the reference) -------------------------------------------
 * Marching tetrahedra on a lattice that subdivides every grid cell `subdivisions` times; the lattice values are the bits of the value-only
 * dg_interpolate_batch.  The full contract -- lattice, validity (finite and != DBL_MAX; a point in a removed cell of a reduced field is
 * invalid), the Kuhn split, the case table and orientation (normals from the negative to the non-negative side: outward for an SDF), vertex
 * arithmetic and the order of vertices and triangles -- is stated in discregrid_b200/csrc/k6_isosurface.cu and DESIGN.md section 3.
 * Coincident vertices are not welded; no normals are output.  One GPU (the field's), synchronous on the legacy default stream.  The result
 * stays on the device in the handle until dg_isosurface_copy[_device]; vertices[n_vertices x 3] and triangles[n_triangles x 3] (0-based
 * indices, the layout dg_mesh_create takes).  A field with no kept cell, or an iso above or below every value, gives 0 / 0.
 *   iso: finite (NaN or +-inf: DG_ERR_INVALID).  subdivisions: 1..16.  A lattice of 2^31 points or more, and a result of 2^32 vertices or
 *       triangles or more, are refused (DG_ERR_INVALID), the lattice before anything is allocated.  The field must live on the current device.
 *   timings_ms: NULL or 5 doubles = ms of values, classify, scans, emit, total.  Every stage ends with a device synchronise.
 *   dg_isosurface_copy / _copy_device: outputs may be NULL only when their count is 0.  _copy_device is asynchronous on `stream`; let it
 *       finish before dg_isosurface_destroy. */
typedef struct dg_isosurface dg_isosurface;
DG_API int dg_isosurface_create(const dg_field* field, double iso, uint32_t subdivisions, dg_isosurface** out, double* timings_ms);
DG_API int dg_isosurface_sizes(const dg_isosurface* s, uint64_t* n_vertices, uint64_t* n_triangles);
DG_API int dg_isosurface_copy(const dg_isosurface* s, double* vertices, uint32_t* triangles);
DG_API int dg_isosurface_copy_device(const dg_isosurface* s, double* d_vertices, uint32_t* d_triangles, void* stream);
DG_API int dg_isosurface_destroy(dg_isosurface* s);
/* dg_isosurface_copy_edges[_device]: edge_ids[n_vertices], the lattice edge 7 * lin(p) + d of every vertex (lin and d as in the contract),
 *   ascending because the vertices are ordered by it; what dg_isosurface_vjp takes.  The rules of dg_isosurface_copy[_device]: NULL only
 *   when there are no vertices, the _device form asynchronous on `stream`. */
DG_API int dg_isosurface_copy_edges(const dg_isosurface* s, uint64_t* edge_ids);
DG_API int dg_isosurface_copy_edges_device(const dg_isosurface* s, uint64_t* d_edge_ids, void* stream);

/* ---- differentiable level sets (K13, k13_isosurface_grad.cu; beyond the reference) ---------------------------------------------------
 * dg_isosurface_vjp[_device]: for n vertices of dg_isosurface_create(field, iso, subdivisions), given by their edge ids (or any edges of
 * that lattice), and the upstream gradient grad_vertices[n x 3] of their positions, grad_nodes[n_nodes] = the gradient with respect to the
 * field's node values.  The field must be made by dg_field_create_trainable and hold the forward's node values.  Each vertex moves along its
 * edge with t = (iso - f_p) / (f_q - f_p); a vertex whose lattice values are DBL_MAX or not finite, or whose difference is 0 or not finite,
 * gets 0.  grad_nodes is always overwritten (zeros for n = 0); it is summed as K11 sums interpolate's VJP, over the 2n edge endpoints, so its
 * bits depend only on the field's topology and values, iso, subdivisions, the edge ids and grad_vertices (the contract is in
 * k13_isosurface_grad.cu and DESIGN.md section 3).  First order only; not differentiable in iso.  The edge ids are checked on the device
 * first (one synchronise).  Device scratch of about 150 B per vertex is taken and released in stream order.  The _device form is queued on
 * `stream`; the host form uploads every input in one piece and returns when grad_nodes is written.
 *   DG_ERR_INVALID, before anything is written: NULL field; NULL edge_ids or grad_vertices with n > 0; NULL grad_nodes on a field with nodes;
 *   a field not made by dg_field_create_trainable or on another device; iso not finite; subdivisions outside 1..16; a lattice of 2^31 points
 *   or more; n >= 2^31; an edge id that is not an edge of the lattice (lin(p) >= points, or p + delta_d outside it). */
DG_API int dg_isosurface_vjp(const dg_field* field, double iso, uint32_t subdivisions, uint64_t n, const uint64_t* edge_ids,
                             const double* grad_vertices, double* grad_nodes);
DG_API int dg_isosurface_vjp_device(const dg_field* field, double iso, uint32_t subdivisions, uint64_t n, const uint64_t* d_edge_ids,
                                    const double* d_grad_vertices, double* d_grad_nodes, void* stream);

/* ---- ray casts: the first crossing of {phi = iso} along rays and segments (not in the reference) -----------------------------------------
 * For each ray i (origin origins[3 i..], direction directions[3 i..]) and t in [t_min, t_max] clipped to the domain: the first crossing of
 * the level set, isolated cell by cell with Bernstein bounds of the interpolant's restriction to the line, so a feature thinner than any step
 * is not missed.  The values along the ray are the bits of the value-only dg_interpolate_batch; the full contract (clip, segments, samples,
 * pruning, descent, bisection) is stated in discregrid_b200/csrc/k7_raycast.cu and DESIGN.md section 3.  A segment x0 -> x1 is the ray
 * (x0, x1 - x0) with t_min = 0, t_max = 1.
 *   t_lo[i], t_hi[i]: the final bisection bracket; status[i] = DG_RAY_ENTER when phi(x(t_lo)) >= iso > phi(x(t_hi)), DG_RAY_LEAVE for the
 *       reverse (a ray that starts inside reports its first LEAVE), DG_RAY_MISS with t_lo = t_hi = +inf when no crossing is found.
 *   iso: finite.  t_min <= t_max, neither NaN (either may be infinite).  Arrays may be NULL only when n is 0.  The field must live on the
 *       current device.  Otherwise DG_ERR_INVALID.
 *   dg_field_raycast: host arrays, synchronous.  dg_field_raycast_device: device arrays, asynchronous on `stream`. */
#define DG_RAY_MISS  0
#define DG_RAY_ENTER 1
#define DG_RAY_LEAVE 2
DG_API int dg_field_raycast(const dg_field* field, const double* origins, const double* directions, uint64_t n, double iso, double t_min,
                            double t_max, double* t_lo, double* t_hi, int32_t* status);
DG_API int dg_field_raycast_device(const dg_field* field, const double* d_origins, const double* d_directions, uint64_t n, double iso,
                                   double t_min, double t_max, double* d_t_lo, double* d_t_hi, int32_t* d_status, void* stream);

/* ---- ray casts on a mesh: the first hit of rays and segments on the triangles themselves (not in the reference) --------------------
 * For each ray i (origin origins[3 i..], direction directions[3 i..]) and t in [t_min, t_max]: the triangle hit first, by the watertight
 * ray/triangle test of Woop, Benthin and Wald (JCGT 2013) in fp64 on the vertices as given, with two conditions that reject hits off a
 * triangle for rays lying in its plane.  The full contract is stated in discregrid_b200/csrc/k9_mesh_raycast.cu and DESIGN.md section 3.
 * A ray through a shared edge or vertex of a closed mesh is not lost between its triangles.  A segment x0 -> x1 is the ray (x0, x1 - x0)
 * with t_min = 0, t_max = 1.  A ray misses if its origin or direction is not finite, or its direction is 0.
 *   t[i]: the least accepted t (the lower triangle id wins a tie; -0.0 == +0.0); triangle_id[i]: the original triangle index;
 *       barycentric[3 i..]: the weights of vertices 0, 1, 2 of that triangle (may be NULL); status[i] = DG_RAY_ENTER when the ray crosses
 *       the triangle from the side a ray enters a closed, outward-oriented mesh from, DG_RAY_LEAVE otherwise.  A miss: DG_RAY_MISS, t = +inf,
 *       triangle_id = -1, barycentric NaN.  The result does not depend on the traversal: it equals a loop over every triangle, bit for bit.
 *   t_min <= t_max, neither NaN (either may be infinite).  Arrays other than barycentric may be NULL only when n is 0.  The mesh must live on
 *       the current device and not be left unusable by a failed refit.  Otherwise DG_ERR_INVALID, before anything is written.
 *   The vertices are read from the winding-number records (dg_mesh_winding_number): the first call on a mesh builds them (328 B per
 *   triangle) and returns after their upload.  Either sign mode; a mesh that a dg_mesh_group borrows may be cast; after dg_mesh_refit the
 *   cast sees the refit positions.  One GPU, the mesh's.
 *   dg_mesh_raycast: host arrays, synchronous.  dg_mesh_raycast_device: device arrays, asynchronous on `stream`. */
DG_API int dg_mesh_raycast(const dg_mesh* mesh, const double* origins, const double* directions, uint64_t n, double t_min, double t_max,
                           double* t, int32_t* triangle_id, double* barycentric, int32_t* status);
DG_API int dg_mesh_raycast_device(const dg_mesh* mesh, const double* d_origins, const double* d_directions, uint64_t n, double t_min,
                                  double t_max, double* d_t, int32_t* d_triangle_id, double* d_barycentric, int32_t* d_status, void* stream);

/* ---- differentiable mesh distance (K10, k10_distance_grad.cu; beyond the reference) -------------------------------------------------
 * dg_mesh_distance_bary[_device]: dg_mesh_distance[_device] that also writes barycentric[n x 3], the weights of the nearest point on the
 *     vertices F[t][0], F[t][1], F[t][2] of its triangle t: (fl(fl(1 - s) - t'), s, t') with (s, t') the parameters of the leaf test, so that
 *     nearest_point = v0 + s (v1 - v0) + t' (v2 - v0) as the query computes it; one-hot on a vertex, on the edge for an edge.  NaN when no
 *     triangle was accepted (triangle_id -1, distance DBL_MAX).  Distance, nearest point, entity and triangle id are bit for bit those of
 *     dg_mesh_distance[_device], in both sign modes.  Every output is nullable.  Refusals as dg_mesh_distance: NULL mesh, NULL points with
 *     n > 0, a mesh on another device and a mesh left unusable by a failed refit (DG_ERR_INVALID).
 * dg_mesh_distance_vjp[_device]: for the outputs of that call (points, distance, nearest_point, triangle_id, barycentric; either sign mode)
 *     and an upstream gradient grad_distance[n], the gradient with respect to the points, grad_points[n x 3] = (g / d) (x - p) (0 where
 *     d == 0 or triangle_id == -1), and with respect to the vertices, grad_vertices[n_vertices x 3] = the sum over queries of
 *     -w_i * grad_points on vertex F[t][i] (envelope theorem).  Both nullable; grad_vertices is overwritten (0 where nothing arrives; n = 0
 *     writes zeros).  The vertex sums are in a fixed order stated in k10_distance_grad.cu: the same bits on every run, stream and device.
 *     Only the given outputs and the mesh's triangles are read, not its vertex positions, so the gradient stays right after a later refit.
 *     First order only.  The _device form is queued on `stream` after one synchronise that checks the triangle ids; the host form uploads
 *     every input in one piece and returns when done.  The first call with grad_vertices builds the topology tables dg_mesh_refit uses
 *     (kept, counted in dg_mesh_info[4]); device scratch of about 130 B per query is taken and released in stream order.
 *     DG_ERR_INVALID, before anything is written: NULL mesh; a NULL input with n > 0; n >= 2^32 - 1; a mesh on another device; a mesh left
 *     unusable by a failed refit; a triangle id outside [-1, n_triangles) (checked on the device, reported by the call). */
DG_API int dg_mesh_distance_bary(const dg_mesh* mesh, const double* points, uint64_t n, int is_signed, double* distance, double* nearest_point,
                                 int32_t* nearest_entity, int32_t* triangle_id, double* barycentric);
DG_API int dg_mesh_distance_bary_device(const dg_mesh* mesh, const double* d_points, uint64_t n, int is_signed, double* d_distance,
                                        double* d_nearest_point, int32_t* d_nearest_entity, int32_t* d_triangle_id, double* d_barycentric,
                                        void* stream);
DG_API int dg_mesh_distance_vjp(const dg_mesh* mesh, uint64_t n, const double* points, const double* distance, const double* nearest_point,
                                const int32_t* triangle_id, const double* barycentric, const double* grad_distance, double* grad_points,
                                double* grad_vertices);
DG_API int dg_mesh_distance_vjp_device(const dg_mesh* mesh, uint64_t n, const double* d_points, const double* d_distance,
                                       const double* d_nearest_point, const int32_t* d_triangle_id, const double* d_barycentric,
                                       const double* d_grad_distance, double* d_grad_points, double* d_grad_vertices, void* stream);

/* ---- differentiable ray casts (K12, k12_raycast_grad.cu; beyond the reference) ------------------------------------------------------
 * The vector-Jacobian products of the two ray casts above.  The contract (operation order, validity, summation order) is stated in
 * discregrid_b200/csrc/k12_raycast_grad.cu and DESIGN.md section 3; the results depend only on the inputs, the same bits on every run and
 * stream.  First order only.  Every output is nullable and asking for none is a no-op.  n < 2^32 - 1.  Arrays may be NULL only when n is 0
 * (the upstream gradients as stated below).  Device scratch is taken and released in stream order.  The _device forms are queued on
 * `stream`; the host forms upload every input in one piece, run the device form and return when done.
 * dg_mesh_raycast_vjp[_device]: for the outputs of dg_mesh_raycast (directions, t, triangle_id, barycentric) and the upstream gradients
 *     grad_t[n] and grad_barycentric[n x 3] (either may be NULL for zeros, not both): grad_origins[n x 3], grad_directions[n x 3] and
 *     grad_vertices[n_vertices x 3].  vertices[n_vertices x 3] are the positions the forward cast against (the mesh may have been refit
 *     since): the gradient is taken there.  A ray with triangle id -1, or whose triangle is degenerate or parallel to it (n . d == 0), gets 0.
 *     grad_vertices is overwritten (0 where nothing arrives) and is summed as K10 sums the distance gradient.  The triangle ids are checked
 *     on the device first (one synchronise); DG_ERR_INVALID, before anything is written: NULL mesh, a NULL input, both upstreams NULL, a mesh
 *     on another device or left unusable by a failed refit, n too large, a triangle id outside [-1, n_triangles).
 * dg_field_raycast_vjp[_device]: for the rays (origins, directions) and the outputs t_lo and status of dg_field_raycast, and the upstream
 *     gradients grad_t_lo[n] and grad_t_hi[n] (either may be NULL for zeros, not both; both ends of the bracket follow the crossing, so they
 *     are added): grad_origins[n x 3], grad_directions[n x 3] on any field (dense, reduced, a kept reduced handle), and grad_nodes[n_nodes],
 *     overwritten, only on a field made by dg_field_create_trainable (DG_ERR_INVALID on any other).  The field must hold the node values of
 *     the forward.  A miss, a crossing where the field is DBL_MAX or not finite, or a ray tangent to the level set (grad phi . d == 0) gets 0.
 *     DG_ERR_INVALID, before anything is written: NULL field, a NULL input, both upstreams NULL, a field on another device, n too large. */
DG_API int dg_mesh_raycast_vjp(const dg_mesh* mesh, uint64_t n, const double* directions, const double* t, const int32_t* triangle_id,
                               const double* barycentric, const double* vertices, const double* grad_t, const double* grad_barycentric,
                               double* grad_origins, double* grad_directions, double* grad_vertices);
DG_API int dg_mesh_raycast_vjp_device(const dg_mesh* mesh, uint64_t n, const double* d_directions, const double* d_t,
                                      const int32_t* d_triangle_id, const double* d_barycentric, const double* d_vertices,
                                      const double* d_grad_t, const double* d_grad_barycentric, double* d_grad_origins,
                                      double* d_grad_directions, double* d_grad_vertices, void* stream);
DG_API int dg_field_raycast_vjp(const dg_field* field, uint64_t n, const double* origins, const double* directions, const double* t_lo,
                                const int32_t* status, const double* grad_t_lo, const double* grad_t_hi, double* grad_origins,
                                double* grad_directions, double* grad_nodes);
DG_API int dg_field_raycast_vjp_device(const dg_field* field, uint64_t n, const double* d_origins, const double* d_directions,
                                       const double* d_t_lo, const int32_t* d_status, const double* d_grad_t_lo, const double* d_grad_t_hi,
                                       double* d_grad_origins, double* d_grad_directions, double* d_grad_nodes, void* stream);

/* ---- reduced density map: GenerateDensityMap with reduction in one call -----------------------------------------------------------
 * GenerateDensityMap with reduction (cmd/generate_density_map/main.cpp:117-147) in one call:
 *   id = addFunction(density_func, verbose, pred);  reduceField(0, p0);  reduceField(id, p1);
 * on the SDF field (sdf_nodes, sdf_cells, sdf_cell_map) of `grid`, with
 *   p0(x, v) = -6h < v + cell_diag && v - cell_diag < 2h,   p1(x, v) = 0 <= v && v <= 3 rho0,   cell_diag = cellSize().norm().
 * The two handles hold exactly what those calls leave, bit for bit what dg_density_map (no_reduction = 0), dg_build_cells + identity map
 * and dg_reduce_field on each field give: *sdf_out the reduced SDF field, *density_out the reduced density field, each with its nodes in
 * the reference's Z-curve order (including the order among equal keys), renumbered cells and cell map.  Read them with
 * dg_reduced_band_sizes / _copy, free them with dg_reduced_band_destroy.  Every array the size of the grid stays on the current device;
 * the packed SDF field that K3 reads is freed before the reductions start.  One GPU.
 *   sdf_nodes: n_nodes = the grid's node count (a field that is already reduced: DG_ERR_INVALID, as dg_reduce_field).
 *   sdf_cells: n_cells <= nx*ny*nz rows of 32 node ids (an id >= n_nodes: DG_ERR_INVALID); sdf_cell_map: nx*ny*nz entries, each
 *       0xffffffff or < n_cells.  When n_cells < nx*ny*nz the reduced SDF cell map holds i at every i >= n_cells, as reduceField leaves it.
 *   h: > 0 (NaN refused, as dg_density_map).  flags: 0 or DG_REDUCE_REFERENCE_SORT.  Grids of 2^31 nodes or more are refused before
 *       anything is allocated.
 *   timings_ms: NULL or 13 doubles = ms of upload + pack; density sampling; for field 0 then field 1: kept cells, node compaction, sort,
 *       write-back; the tie flags of field 0 and field 1 (1.0 when survivors shared Morton keys); total ms.  Every stage ends with a device
 *       synchronise; field 0's cell flags, computed before packing because they check the rows, count as its kept cells. */
DG_API int dg_reduced_density_map_create(const dg_grid_desc* grid, const double* sdf_nodes, uint64_t n_nodes,
                                         const uint32_t* sdf_cells, uint64_t n_cells, const uint32_t* sdf_cell_map,
                                         double h, double rho0, uint32_t flags,
                                         dg_reduced_band** sdf_out, dg_reduced_band** density_out, double* timings_ms);

/* ---- reduced volume map: the volume map with reduction in one call ------------------------------------------------------------------
 * What a volume-map generator that reduces its fields as GenerateDensityMap does leaves, in one call:
 *   id = addFunction(volume_func, verbose, pred);  reduceField(0, p0);  reduceField(id, p1);
 * with volume_func and pred those of dg_volume_map (no_reduction = 0), p0 GenerateDensityMap's (above) and p1(x, v) = 0 <= v (which,
 * as in every reduceField, also drops DBL_MAX).  Arguments, outputs, rules and timings_ms (13 doubles; [1] is the volume sampling) are
 * those of dg_reduced_density_map_create, with scale in place of rho0: h finite and > 0, scale finite, else DG_ERR_INVALID. */
DG_API int dg_reduced_volume_map_create(const dg_grid_desc* grid, const double* sdf_nodes, uint64_t n_nodes,
                                        const uint32_t* sdf_cells, uint64_t n_cells, const uint32_t* sdf_cell_map,
                                        double h, double scale, uint32_t flags,
                                        dg_reduced_band** sdf_out, dg_reduced_band** volume_out, double* timings_ms);

/* ---- user functions on the GPU: addFunction(func, verbose, pred) and reduceField(id, pred) with batched device callbacks ----------------
 * The reference's addFunction and reduceField take any callable.  These entry points take the caller's OWN GPU code instead, as batched
 * callbacks: the library generates the node positions x = indexToNodePosition(l) (cubic_lagrange_discrete_grid.cpp:604-665, the bits of
 * dg_node_positions) for contiguous id ranges [b, e) ("chunks") on the device and calls the callbacks once per chunk, in ascending order, ON
 * THE CALLING THREAD, with n = e - b and device pointers of the current device:
 *   d_x            n x 3 doubles, the positions of nodes b .. e-1 (valid until the callback's work on `stream` has run)
 *   d_sample_keep  n bytes written by the sample predicate of the same chunk, or NULL without one; a function may skip the nodes whose byte
 *                  is 0 -- the library writes DBL_MAX there anyway (:817)
 *   d_values       function: n doubles to write (node b first); node predicate: the chunk's values, DBL_MAX where the sample predicate rejected
 *   d_keep         n bytes to write: nonzero = keep.  A node predicate's mask is ANDed with v != DBL_MAX (:1073) on the device.
 *   stream         the cudaStream_t the library works on: enqueue the work there, or finish it before returning.  It is one stream per
 *                  device, kept for the life of the process (calls from several threads share it), and it is a blocking stream: its work
 *                  -- the first positions and every callback's work on it -- starts after everything queued on the legacy default stream
 *                  (NULL; torch's default stream) before the call.  Work the caller queued on OTHER streams is not waited for: order it first
 *                  (e.g. cudaStreamSynchronize, or a cudaStreamWaitEvent on `stream` in the first callback).  When the call returns, all
 *                  its work on `stream` has finished.
 * A callback returns 0, or nonzero to abort the call: the call then returns DG_ERR_CALLBACK (dg_last_error() names the callback and the chunk),
 * produces no handle and leaves the output arrays' contents unspecified.  Callbacks may call the library's _device entry points (e.g.
 * dg_mesh_distance_device on d_x); they must not call the entry point that is calling them.
 * chunk_nodes: ids per chunk, 0 = 2^24 (positions of one chunk: 384 MiB).  The values do not depend on it.  One GPU (the current device);
 * grids of 2^31 nodes or more are refused before anything is allocated. */
typedef int (*dg_device_function)(void* user, const double* d_x, const uint8_t* d_sample_keep, uint64_t n, double* d_values, void* stream);
typedef int (*dg_device_sample_predicate)(void* user, const double* d_x, uint64_t n, uint8_t* d_keep, void* stream);
typedef int (*dg_device_node_predicate)(void* user, const double* d_x, const double* d_values, uint64_t n, uint8_t* d_keep, void* stream);
/* addFunction(func, verbose, pred) (:780-899) into the caller's three arrays, as dg_add_function_sdf fills them: nodes_host[n_nodes] = func(x)
 * where pred(x) holds (pred NULL: everywhere) and DBL_MAX elsewhere (:806-817); cells_host[n_cells x 32] and cell_map_host[n_cells] (each
 * nullable) are written by host threads while the callbacks run.  func must not be NULL.
 * timings_ms: NULL or 6 doubles = total, node pipeline done, index tables done, coefficient array pre-faulted (all ms since entry), worker
 * threads used, ms spent inside the callbacks (host time from call to return; work they only enqueue counts in the node pipeline). */
DG_API int dg_add_function_device(const dg_grid_desc* grid, dg_device_function func, void* fu, dg_device_sample_predicate pred, void* pu,
                                  uint64_t chunk_nodes, double* nodes_host, uint32_t* cells_host, uint32_t* cell_map_host, double* timings_ms);
/* id = addFunction(func, verbose, sample_pred); reduceField(id, reduce_pred); in one call: the dense values stay on the device, the rows come
 * from the closed form, and the handle holds exactly what those two calls leave (nodes in the reference's Z-curve order, including the order
 * among equal keys; renumbered cells; cell map) -- bit for bit dg_add_function_device followed by dg_reduce_field with
 * keep = reduce_pred && v != DBL_MAX.  Read it with dg_reduced_band_sizes / _copy, free it with dg_reduced_band_destroy.
 *   func: required.  sample_pred: NULL = every node sampled.  reduce_pred: NULL = always true.  flags: 0 or DG_REDUCE_REFERENCE_SORT.
 *   Per chunk the callbacks run in the order sample_pred, func, reduce_pred.
 *   timings_ms: NULL or 8 doubles = ms of positions + callbacks (synchronised), kept cells, node compaction, sort, write-back; 1.0 if surviving
 *       nodes shared Morton keys; total ms; ms spent inside the callbacks (part of [0]). */
DG_API int dg_reduced_function_create(const dg_grid_desc* grid, dg_device_function func, void* fu, dg_device_sample_predicate sample_pred, void* su,
                                      dg_device_node_predicate reduce_pred, void* ru, uint64_t chunk_nodes, uint32_t flags, dg_reduced_band** out,
                                      double* timings_ms);
/* reduceField(id, pred) (:1065-1174) of a dense field held on the host (nodes[n_nodes], its rows cells[n_cells x 32]), e.g. one just loaded:
 * the field and its rows are uploaded, the rows checked on the device (an id >= n_nodes: DG_ERR_INVALID), pred evaluated per chunk, and the
 * handle holds exactly what dg_reduce_field leaves with keep = pred && v != DBL_MAX (the cell map holds i at every i >= n_cells, as
 * reduceField leaves it).  pred: required.  n_nodes must be the grid's node count (a field that is already reduced: DG_ERR_INVALID, as
 * dg_reduce_field); n_cells <= nx*ny*nz.  flags: 0 or DG_REDUCE_REFERENCE_SORT.
 *   timings_ms: NULL or 8 doubles = ms of upload + positions + callbacks, then as dg_reduced_function_create (the rows are checked in the
 *       kept-cells stage). */
DG_API int dg_reduce_field_device(const dg_grid_desc* grid, const double* nodes, uint64_t n_nodes, const uint32_t* cells, uint64_t n_cells,
                                  dg_device_node_predicate pred, void* pu, uint64_t chunk_nodes, uint32_t flags, dg_reduced_band** out,
                                  double* timings_ms);

#ifdef __cplusplus
}
#endif
#endif /* DISCREGRID_B200_H */
