// tests/cpp/oracle_from_tree.cpp -- TEST INFRASTRUCTURE: the CPU oracle (oracle/dg_oracle.cpp, included unchanged) plus one entry point that
// installs a given tree and given pseudonormals instead of building them, so that the reference's query rule (_query / signed_distance) and
// every oracle call built on it (orc_mesh_distance, orc_sample_sdf) run over the records a refit exported (dg_mesh_tree,
// dg_mesh_pseudonormals).  Built into build/bin/liborctree.so; the product never loads it.
#include "../../oracle/dg_oracle.cpp"

extern "C" {

// spheres[n][8], kids[n][2] in dg_mesh_tree's pre-order numbering (n = 2T - 1, the oracle's own numbering); pn_tri[T][3], pn_edge[T][3][3],
// pn_vert[nV][3] as dg_mesh_pseudonormals returns them
void* orc_mesh_create_from_tree(const double* V, uint64_t nV, const uint32_t* F, uint64_t nT, const double* spheres, const int32_t* kids,
                                const double* pn_tri, const double* pn_edge, const double* pn_vert)
{
    if (nT == 0) return nullptr;
    Mesh* m = new Mesh();
    m->V.resize(nV);
    for (uint64_t i = 0; i < nV; i++) m->V[i] = {V[3 * i], V[3 * i + 1], V[3 * i + 2]};
    m->T.resize(3 * nT);
    for (uint64_t i = 0; i < 3 * nT; i++) m->T[i] = (int)F[i];
    m->nodes.resize(2 * nT - 1);
    for (uint64_t i = 0; i < 2 * nT - 1; i++) {
        const double* s = spheres + 8 * i;
        Node& n = m->nodes[i];
        n.bl = {{s[0], s[1], s[2]}, s[3]};
        n.br = {{s[4], s[5], s[6]}, s[7]};
        n.left = kids[2 * i]; n.right = kids[2 * i + 1];
    }
    m->pn_tri.resize(nT); m->pn_edge.resize(3 * nT); m->pn_vert.resize(nV);
    memcpy(m->pn_tri.data(), pn_tri, nT * sizeof(V3));
    memcpy(m->pn_edge.data(), pn_edge, 3 * nT * sizeof(V3));
    memcpy(m->pn_vert.data(), pn_vert, nV * sizeof(V3));
    return m;
}

}  // extern "C"
