// Reference pin for the on-disk map of a model with a skybox.  TEST INFRASTRUCTURE ONLY (built into oracle/_ref/ply_ref_sky).
//
// Drives the reference's OWN PLY writer -- tinyply, compiled from where it lies (/root/reference/src/tinyply.h) -- exactly as
// GaussianModel::saveMap does for a model whose first S rows are the skybox (/root/reference/src/gaussian.cpp:305-397): every
// tensor sliced to rows [S, P) (.index({Slice(skybox_points_num_)})), and the UNSLICED features_dc_.size(0) /
// features_rest_.size(0) = P passed as the row count of the f_dc and f_rest properties, as the reference passes them.
// tinyply keeps the row count of an element's first property (xyz, sliced), so the file holds P - S rows.
// Input: the raw float32 blob of ply_ref.cpp holding all P rows:
//     uint32 P, uint32 M, xyz[P*3], f_dc[P*1*3], f_rest[P*M*3], opacity[P], scale[P*3], rotation[P*4]
// usage: ply_ref_sky <in.blob> <out.ply> <S>
#define TINYPLY_IMPLEMENTATION
#include "tinyply.h"

#include <cstddef>
#include <cstdint>
#include <cstdio>
#include <fstream>
#include <string>
#include <vector>

static std::vector<float> take(std::ifstream& in, size_t n) {
    std::vector<float> v(n);
    in.read(reinterpret_cast<char*>(v.data()), (std::streamsize)(n * sizeof(float)));
    return v;
}

static std::vector<std::string> names(const std::string& prefix, size_t n) {
    std::vector<std::string> v(n);
    for (size_t i = 0; i < n; ++i) v[i] = prefix + std::to_string(i);
    return v;
}

int main(int argc, char** argv) {
    if (argc != 4) { std::fprintf(stderr, "usage: ply_ref_sky in.blob out.ply S\n"); return 2; }
    std::ifstream in(argv[1], std::ios::binary);
    uint32_t P = 0, M = 0;
    in.read(reinterpret_cast<char*>(&P), 4);
    in.read(reinterpret_cast<char*>(&M), 4);
    std::vector<float> xyz = take(in, (size_t)P * 3), dc = take(in, (size_t)P * 3), rest = take(in, (size_t)P * M * 3);
    std::vector<float> opacity = take(in, P), scale = take(in, (size_t)P * 3), rotation = take(in, (size_t)P * 4);
    if (!in) { std::fprintf(stderr, "short blob\n"); return 3; }
    const uint32_t S = (uint32_t)std::stoul(argv[3]);
    if (S > P) { std::fprintf(stderr, "S > P\n"); return 4; }
    const uint32_t F = P - S;                                  // rows after the slice
    auto slice = [&](std::vector<float>& v, size_t k) { v.erase(v.begin(), v.begin() + (std::ptrdiff_t)(S * k)); };
    slice(xyz, 3); slice(dc, 3); slice(rest, (size_t)M * 3); slice(opacity, 1); slice(scale, 3); slice(rotation, 4);
    // features_*.transpose(1, 2).flatten(1): [F, K, 3] -> [F, 3, K]
    std::vector<float> f_dc((size_t)F * 3), f_rest((size_t)F * 3 * M);
    for (uint32_t i = 0; i < F; ++i)
        for (int c = 0; c < 3; ++c) {
            f_dc[(size_t)i * 3 + c] = dc[(size_t)i * 3 + c];
            for (uint32_t k = 0; k < M; ++k) f_rest[((size_t)i * 3 + c) * M + k] = rest[((size_t)i * M + k) * 3 + c];
        }
    std::filebuf fb;
    fb.open(argv[2], std::ios::out | std::ios::binary);
    std::ostream os(&fb);
    tinyply::PlyFile file;
    auto add = [&](const std::vector<std::string>& n, std::vector<float>& data, uint32_t count) {
        file.add_properties_to_element("vertex", n, tinyply::Type::FLOAT32, count, reinterpret_cast<uint8_t*>(data.data()),
                                       tinyply::Type::INVALID, 0);
    };
    add({"x", "y", "z"}, xyz, F);                              // xyz.size(0): sliced
    add(names("f_dc_", 3), f_dc, P);                           // this->features_dc_.size(0): unsliced
    add(names("f_rest_", (size_t)3 * M), f_rest, P);           // this->features_rest_.size(0): unsliced
    add({"opacity"}, opacity, F);
    add(names("scale_", 3), scale, F);
    add(names("rot_", 4), rotation, F);
    file.write(os, true);
    fb.close();
    return 0;
}
