// DiscreteFieldToMesh -- the level set {phi = iso} of a field in a .cdf/.cdm file as an OBJ mesh (not in the reference; K6, the contract in
// discregrid_b200/csrc/k6_isosurface.cu).  Options follow DiscreteFieldToBitmap.  The OBJ is written with 17 significant digits, so that
// reading it back (dg_obj_read, TriangleMesh(path)) gives the same doubles; TriangleMesh::exportOBJ keeps the reference's default precision.
//   DiscreteFieldToMesh [-f field_id] [-i iso] [-s subdivisions] [-o out.obj] file.cdf|.cdm
#include <Discregrid/All>
#include <cstdio>
#include <iostream>
#include <string>

int main(int argc, char* argv[])
{
    unsigned field_id = 0, subdivisions = 1;
    double iso = 0.0;
    std::string out_file, filename;
    for (int a = 1; a < argc; a++) {
        const std::string s = argv[a];
        auto next = [&]() -> std::string { if (a + 1 >= argc) { std::cerr << "missing value for " << s << std::endl; std::exit(1); } return argv[++a]; };
        if (s == "-f" || s == "--field_id") field_id = (unsigned)std::stoul(next());
        else if (s == "-i" || s == "--iso") iso = std::stod(next());
        else if (s == "-s" || s == "--subdivisions") subdivisions = (unsigned)std::stoul(next());
        else if (s == "-o" || s == "--output") out_file = next();
        else if (s == "-h" || s == "--help") {
            std::cout << "Extracts the level set phi = iso of a discrete field as a triangle mesh (marching tetrahedra).\n"
                         "Example: DiscreteFieldToMesh -s 2 -o surface.obj file.cdf" << std::endl;
            return 0;
        }
        else filename = s;
    }
    if (filename.empty()) { std::cout << "ERROR: No input file given." << std::endl; return 1; }
    try {
        std::cout << "Load SDF...";
        Discregrid::CubicLagrangeDiscreteGrid sdf(filename);
        std::cout << "DONE" << std::endl;
        if (sdf.nFields() <= field_id) { std::cerr << "ERROR: field " << field_id << " does not exist" << std::endl; return 1; }
        std::cout << "Extract level set...";
        const Discregrid::TriangleMesh mesh = sdf.isosurface(field_id, iso, subdivisions);
        std::cout << "DONE" << std::endl;
        if (out_file.empty()) {
            out_file = filename;
            if (out_file.find(".") != std::string::npos) out_file = out_file.substr(0, out_file.find_last_of("."));
            out_file += ".obj";
        }
        std::cout << "Ouput file: " << out_file << std::endl << "Export OBJ...";
        FILE* fp = std::fopen(out_file.c_str(), "w");
        if (!fp) { std::cerr << "ERROR: cannot write " << out_file << std::endl; return 1; }
        bool ok = std::fprintf(fp, "g default\n") > 0;
        for (auto const& p : mesh.vertices()) ok = ok && std::fprintf(fp, "v %.17g %.17g %.17g\n", p[0], p[1], p[2]) > 0;
        for (auto const& f : mesh.faces()) ok = ok && std::fprintf(fp, "f %u %u %u\n", f[0] + 1, f[1] + 1, f[2] + 1) > 0;
        ok = (std::fclose(fp) == 0) && ok;
        if (!ok) { std::cerr << "ERROR: cannot write " << out_file << std::endl; return 1; }
        std::cout << "DONE" << std::endl << std::endl << "Statistics:" << std::endl;
        std::cout << "\tvertices  = " << mesh.nVertices() << std::endl << "\ttriangles = " << mesh.nFaces() << std::endl;
    } catch (std::exception const& e) { std::cerr << "error: " << e.what() << std::endl; return 1; }
    return 0;
}
