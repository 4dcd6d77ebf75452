// pose_correction.cuh -- the row update of glic_mapper_correct_poses (pose_correction.cu), for mapper.cu
#pragma once
#include "common.cuh"

namespace glic {
// A record whose q[0] is CORRECTION_NONE marks a keyframe that is not corrected (a real record has q[0] >= 0)
constexpr double CORRECTION_NONE = -1.0;
// Rows [0, P) of the arena `params` (capacity Pcap, degree D): each row whose anchor a is in [0, n_table) with table[a] a record
// moves by it (include/glic_b200.h, "Pose corrections"); *moved (zeroed by the caller) gains the number of rows written
int launch_correct_rows(int D, uint32_t P, uint32_t Pcap, float* params, const int32_t* anchor, const glic_rigid_correction* table,
                        int n_table, uint32_t* moved, cudaStream_t s);
// anchor[i] = i < split ? -1 : value for i in [first, end)
int launch_fill_anchors(int32_t* anchor, uint32_t first, uint32_t split, uint32_t end, int32_t value, cudaStream_t s);
}  // namespace glic
