// mesh.cuh -- what mesh.cu shares with the mapper beyond the C ABI (include/glic_b200.h "Meshing").
#pragma once
#include "common.cuh"

namespace glic {
// glic_mesh_count with the number of observed lattice points as well: totals3 = {vertices, faces, observed}; synchronises s
int mesh_count(const glic_tsdf_grid& g, void* scratch, size_t scratch_bytes, uint64_t totals3[3], cudaStream_t s);
}  // namespace glic
