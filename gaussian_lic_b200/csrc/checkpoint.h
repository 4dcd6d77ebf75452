// checkpoint.h -- the mapper checkpoint file (include/glic_b200.h "Checkpoints"): what map_io.cu's host-only reader hands
// mapper_checkpoint.cu, and the writer's framing.  No CUDA here: map_io.cu reads and writes the file, mapper_checkpoint.cu moves
// the bytes between it and the device.
#pragma once

#include "../../include/glic_b200.h"

#include <cstdint>
#include <cstdio>
#include <random>
#include <string>
#include <vector>

namespace glic {
namespace ckpt {

constexpr uint32_t VERSION = 1;
constexpr size_t HEADER_BYTES = 96;
constexpr size_t FRAME_BYTES = 16;             // section frame: tag u32 | reserved u32 (0) | length u64
constexpr size_t KEYFRAME_RECORD_BYTES = 376;  // the fixed part of one keyframe record
constexpr uint32_t FRAME_CHUNK = 8;            // frames per chunk of the 8-bit frame store (mapper.cu)
constexpr uint32_t NO_FRAME = 0xFFFFFFFFu;

constexpr uint32_t fourcc(const char (&s)[5]) {
    return (uint32_t)(uint8_t)s[0] | (uint32_t)(uint8_t)s[1] << 8 | (uint32_t)(uint8_t)s[2] << 16 | (uint32_t)(uint8_t)s[3] << 24;
}
enum Section : int { MAP, COUNTERS, KEYFRAMES, EXPOSURE, POSE, DENSIFICATION, SCHEDULE, FRAMES, N_SECTIONS };
constexpr uint32_t TAGS[N_SECTIONS] = {fourcc("MAP "), fourcc("CNTR"), fourcc("KEYF"), fourcc("EXPO"), fourcc("POSE"), fourcc("DENS"),
                                       fourcc("SCHD"), fourcc("FRMS")};
constexpr uint32_t END_TAG = fourcc("END ");

// CNTR flags
enum : uint32_t { F_INITIALIZED = 1, F_EXPOSURE = 2, F_POSE = 4, F_DENSIFICATION = 8, F_FRAMES = 16, F_ALL = 31 };
enum : uint32_t { IMAGE_BGR8 = 0, IMAGE_HOST = 1, IMAGE_DEVICE = 2 };

// Bytes per row of each array of the per-row sections, in file order.  The mapper's buffer groups (mapper_state.cuh) are sized,
// saved and loaded with these widths, so the mapper and the reader agree on every section's length.
constexpr size_t EXPOSURE_ROW[] = {48, 48, 48, 4};        // E [3x4] f32 | Adam m, v [12] f32 | step i32
constexpr size_t POSE_ROW[] = {96, 48, 24, 24, 4};        // T_cw [12] f64 | R_wc, t_wc [12] f32 | Adam m, v [6] f32 | step i32
constexpr size_t DENSIFICATION_ROW[] = {4, 4, 4};         // gradient-norm sum f32 | view count f32 | largest screen radius i32
constexpr size_t SCAN_ROW[] = {12, 3, 4};                 // pending scan point: xyz [3] f32 | rgb [3] u8 | depth f32
template <size_t N>
constexpr uint64_t row_bytes(const size_t (&widths)[N]) {
    uint64_t sum = 0;
    for (size_t w : widths) sum += w;
    return sum;
}

// the section lengths the counts imply
inline uint64_t map_bytes(uint64_t P, int M) { return 12 + P * (3 * 4 * (14 + 3 * (uint64_t)M) + 4); }
inline uint64_t counters_bytes(uint64_t rng_len) { return 92 + rng_len; }
inline uint64_t keyframe_bytes(uint32_t kind, uint32_t mask_valid, int W, int H) {
    const uint64_t HW = (uint64_t)W * H;
    return KEYFRAME_RECORD_BYTES + (kind == IMAGE_BGR8 ? 3 * HW : 12 * HW) + (mask_valid ? 4 * (uint64_t)H * ((W + 31) / 32) : 0);
}
inline uint64_t exposure_bytes(uint64_t n) { return 8 + row_bytes(EXPOSURE_ROW) * n; }
inline uint64_t pose_bytes(uint64_t n) { return 12 + row_bytes(POSE_ROW) * n; }
inline uint64_t densification_bytes(uint64_t P) { return 12 + row_bytes(DENSIFICATION_ROW) * P; }
constexpr uint64_t SCHEDULE_BYTES = 72;
inline uint64_t frames_bytes(uint64_t pending) { return 36 + row_bytes(SCAN_ROW) * pending; }
inline uint64_t frame_stride(int W, int H) { return (3 * (uint64_t)W * H + 255) & ~(uint64_t)255; }

struct Keyframe {
    float R_wc[9], t_wc[3];
    float cam[42];                    // the host camera block: view16 | proj16 | campos4 | tanfovx | tanfovy | lim4
    float cam_dev[36];                // the device camera block: view16 | proj16 | campos4
    uint32_t kind, frame, mask_valid, mask_valid_left;
    uint64_t image_off, mask_off;     // file offsets of the image and (mask_valid > 0) the mask words
};

// Everything load_checkpoint needs, validated; *_off are file offsets of the first array of a section
struct Info {
    glic_mapper_config cfg{};
    uint32_t P = 0, Pcap = 0, n_sky = 0;
    uint64_t map_off = 0;
    glic_mapper_stats st{};
    uint64_t view_counter = 0;
    int64_t bin_cap = 0;
    uint64_t binning_bytes = 0, sample_bytes = 0;
    uint32_t optimizer = 1, deterministic = 0, flags = 0;
    std::mt19937_64 rng;
    uint32_t n_train = 0, n_test = 0;
    std::vector<Keyframe> kf;         // training then held-out
    float expo_lr = 0.f;
    uint64_t expo_off = 0;
    float pose_lr_rho = 0.f, pose_lr_omega = 0.f;
    uint64_t pose_off = 0;
    uint64_t dens_calls = 0, dens_off = 0;
    uint32_t sched_on = 0;
    glic_density_schedule sched{};
    glic_density_counts sched_totals{};
    uint32_t sched_steps = 0, sched_resets = 0;
    int32_t frame_k = 1, sky_points = 0, sky_radius = 0;
    glic_frame_stats fst{};
    uint64_t frames_off = 0;
};

// Reads and validates a whole checkpoint (section framing, every length against its counts, the counts across sections) without
// reading its arrays; GLIC_ERR_INVALID_ARGUMENT with the reason in glic_last_error on any fault.
int read_info(const char* path, Info& out);

// Writes <path>.tmp section by section and renames it over path on commit; the destructor removes an uncommitted file.
class Writer {
public:
    ~Writer();
    int open(const char* path);
    int header(const glic_mapper_config& cfg);
    int begin(Section s, uint64_t length);   // the previous section must be complete
    int write(const void* p, size_t n);
    int end();                               // the open section has its declared length
    int commit();                            // end marker, fflush, fsync, rename
private:
    FILE* f_ = nullptr;
    std::string path_, tmp_;
    uint64_t left_ = 0;
    bool open_section_ = false;
};

// little-endian serialisation of the fixed fields
struct Bytes {
    std::vector<uint8_t> b;
    template <typename T> Bytes& put(const T& v) {
        const uint8_t* p = reinterpret_cast<const uint8_t*>(&v);
        b.insert(b.end(), p, p + sizeof(T));
        return *this;
    }
    template <typename T> Bytes& put_n(const T* v, size_t n) {
        const uint8_t* p = reinterpret_cast<const uint8_t*>(v);
        b.insert(b.end(), p, p + n * sizeof(T));
        return *this;
    }
};
static_assert(__BYTE_ORDER__ == __ORDER_LITTLE_ENDIAN__, "the checkpoint format is little-endian");

void put_config(Bytes& b, const glic_mapper_config& c);   // the 84 config bytes of the header
void put_stats(Bytes& b, const glic_mapper_stats& s);     // the 44 stats bytes of CNTR
void put_schedule(Bytes& b, uint32_t on, const glic_density_schedule& s, const glic_density_counts& t, uint32_t steps, uint32_t resets);
void put_frame_stats(Bytes& b, const glic_frame_stats& s);

}  // namespace ckpt
}  // namespace glic
