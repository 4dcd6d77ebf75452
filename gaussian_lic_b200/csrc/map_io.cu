// map_io.cu -- on-disk map format of Gaussian-LIC (SURVEY 8f rank 4): binary little-endian PLY, one "vertex" element,
// float properties x y z | f_dc_0..2 | f_rest_0..3M-1 | opacity | scale_0..2 | rot_0..3, exactly the file
// GaussianModel::saveMap produces through tinyply (/root/reference/src/gaussian.cpp:305-397; header text
// tinyply.h:664-703, row-interleaved body tinyply.h:588-623) and that 3DGS viewers read.  Values are the RAW
// parameters (opacity logit, log-scale, un-normalised quaternion); f_rest is stored channel-major
// (features_rest.transpose(1,2).flatten(1): f_rest_{c*M+k} = sh[k][c]).  Host-only code: pointers are HOST pointers.
#include "common.cuh"

#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

namespace glic {
namespace {

std::string ply_header(uint32_t P, uint32_t M) {
    std::string h = "ply\nformat binary_little_endian 1.0\nelement vertex " + std::to_string(P) + "\n";
    auto prop = [&h](const std::string& name) { h += "property float " + name + "\n"; };
    prop("x"); prop("y"); prop("z");
    for (int i = 0; i < 3; ++i) prop("f_dc_" + std::to_string(i));
    for (uint32_t i = 0; i < 3 * M; ++i) prop("f_rest_" + std::to_string(i));
    prop("opacity");
    for (int i = 0; i < 3; ++i) prop("scale_" + std::to_string(i));
    for (int i = 0; i < 4; ++i) prop("rot_" + std::to_string(i));
    h += "end_header\n";
    return h;
}

inline size_t row_floats(uint32_t M) { return 3 + 3 + 3 * (size_t)M + 1 + 3 + 4; }

struct File {
    FILE* f;
    explicit File(const char* path, const char* mode) : f(path ? std::fopen(path, mode) : nullptr) {}
    ~File() { if (f) std::fclose(f); }
};

// one row of the file <-> the six parameter arrays (write = false: file row -> arrays)
template <bool WRITE>
inline void row_xfer(float* row, uint32_t i, uint32_t M, float* xyz, float* f_dc, float* f_rest, float* opacity, float* scale,
                     float* rotation) {
    auto mv = [](float& file_v, float& mem_v) { if (WRITE) file_v = mem_v; else mem_v = file_v; };
    float* r = row;
    for (int c = 0; c < 3; ++c) mv(*r++, xyz[3 * (size_t)i + c]);
    for (int c = 0; c < 3; ++c) mv(*r++, f_dc[3 * (size_t)i + c]);                       // [P,1,3] -> transpose -> same order
    for (int c = 0; c < 3; ++c)
        for (uint32_t k = 0; k < M; ++k) mv(*r++, f_rest[((size_t)i * M + k) * 3 + c]);  // channel-major
    mv(*r++, opacity[i]);
    for (int c = 0; c < 3; ++c) mv(*r++, scale[3 * (size_t)i + c]);
    for (int c = 0; c < 4; ++c) mv(*r++, rotation[4 * (size_t)i + c]);
}

}  // namespace
}  // namespace glic

using namespace glic;

extern "C" {

size_t glic_ply_bytes(uint32_t P, uint32_t M) { return ply_header(P, M).size() + (size_t)P * row_floats(M) * sizeof(float); }

int glic_ply_write(const char* path, uint32_t P, uint32_t M, const float* xyz, const float* f_dc, const float* f_rest,
                   const float* opacity, const float* scale, const float* rotation) {
    if (!path) { set_error("ply_write: null path"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (P > 0 && (!xyz || !f_dc || (M > 0 && !f_rest) || !opacity || !scale || !rotation)) { set_error("ply_write: null array"); return GLIC_ERR_INVALID_ARGUMENT; }
    File out(path, "wb");
    if (!out.f) { set_error(std::string("ply_write: cannot open ") + path); return GLIC_ERR_INVALID_ARGUMENT; }
    const std::string h = ply_header(P, M);
    if (std::fwrite(h.data(), 1, h.size(), out.f) != h.size()) { set_error("ply_write: short write"); return GLIC_ERR_INVALID_ARGUMENT; }
    const size_t rf = row_floats(M);
    const uint32_t CHUNK = 4096;
    std::vector<float> buf((size_t)CHUNK * rf);
    for (uint32_t i0 = 0; i0 < P; i0 += CHUNK) {
        const uint32_t n = std::min(CHUNK, P - i0);
        for (uint32_t i = 0; i < n; ++i)
            row_xfer<true>(buf.data() + (size_t)i * rf, i0 + i, M, const_cast<float*>(xyz), const_cast<float*>(f_dc),
                           const_cast<float*>(f_rest), const_cast<float*>(opacity), const_cast<float*>(scale),
                           const_cast<float*>(rotation));
        if (std::fwrite(buf.data(), sizeof(float), (size_t)n * rf, out.f) != (size_t)n * rf) { set_error("ply_write: short write"); return GLIC_ERR_INVALID_ARGUMENT; }
    }
    return GLIC_OK;
}

// Parses the header of a map file written by glic_ply_write / GaussianModel::saveMap; *data_offset = first body byte.
int glic_ply_read_header(const char* path, uint32_t* P, uint32_t* M, size_t* data_offset) {
    if (!path || !P || !M) { set_error("ply_read_header: null argument"); return GLIC_ERR_INVALID_ARGUMENT; }
    File in(path, "rb");
    if (!in.f) { set_error(std::string("ply_read_header: cannot open ") + path); return GLIC_ERR_INVALID_ARGUMENT; }
    char line[256];
    bool ply = false, fmt = false, end = false;
    long long count = -1;
    std::vector<std::string> props;
    while (std::fgets(line, sizeof(line), in.f)) {
        std::string s(line);
        while (!s.empty() && (s.back() == '\n' || s.back() == '\r')) s.pop_back();
        if (s == "ply") ply = true;
        else if (s == "format binary_little_endian 1.0") fmt = true;
        else if (s.rfind("element vertex ", 0) == 0) count = std::atoll(s.c_str() + 15);
        else if (s.rfind("property float ", 0) == 0) props.push_back(s.substr(15));
        else if (s.rfind("comment", 0) == 0) continue;
        else if (s == "end_header") { end = true; break; }
        else { set_error("ply_read_header: unsupported header line: " + s); return GLIC_ERR_INVALID_ARGUMENT; }
    }
    if (!ply || !fmt || !end || count < 0) { set_error("ply_read_header: not a binary little-endian Gaussian map"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (props.size() < 14 || (props.size() - 14) % 3 != 0) { set_error("ply_read_header: unexpected property count"); return GLIC_ERR_INVALID_ARGUMENT; }
    const uint32_t m = (uint32_t)((props.size() - 14) / 3);
    // the property list must be exactly the one saveMap writes, in its order
    const std::string want = ply_header((uint32_t)count, m);
    std::string got = "ply\nformat binary_little_endian 1.0\nelement vertex " + std::to_string(count) + "\n";
    for (const auto& p : props) got += "property float " + p + "\n";
    got += "end_header\n";
    if (got != want) { set_error("ply_read_header: property names / order differ from the Gaussian-LIC map layout"); return GLIC_ERR_INVALID_ARGUMENT; }
    *P = (uint32_t)count; *M = m;
    if (data_offset) *data_offset = (size_t)std::ftell(in.f);
    return GLIC_OK;
}

int glic_ply_read(const char* path, uint32_t P, uint32_t M, float* xyz, float* f_dc, float* f_rest, float* opacity, float* scale,
                  float* rotation) {
    uint32_t p = 0, m = 0;
    size_t off = 0;
    if (int e = glic_ply_read_header(path, &p, &m, &off)) return e;
    if (p != P || m != M) { set_error("ply_read: P / M do not match the file"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (P > 0 && (!xyz || !f_dc || (M > 0 && !f_rest) || !opacity || !scale || !rotation)) { set_error("ply_read: null array"); return GLIC_ERR_INVALID_ARGUMENT; }
    File in(path, "rb");
    if (!in.f || std::fseek(in.f, (long)off, SEEK_SET) != 0) { set_error("ply_read: cannot seek"); return GLIC_ERR_INVALID_ARGUMENT; }
    const size_t rf = row_floats(M);
    const uint32_t CHUNK = 4096;
    std::vector<float> buf((size_t)CHUNK * rf);
    for (uint32_t i0 = 0; i0 < P; i0 += CHUNK) {
        const uint32_t n = std::min(CHUNK, P - i0);
        if (std::fread(buf.data(), sizeof(float), (size_t)n * rf, in.f) != (size_t)n * rf) { set_error("ply_read: truncated file"); return GLIC_ERR_INVALID_ARGUMENT; }
        for (uint32_t i = 0; i < n; ++i) row_xfer<false>(buf.data() + (size_t)i * rf, i0 + i, M, xyz, f_dc, f_rest, opacity, scale, rotation);
    }
    return GLIC_OK;
}

// Convenience for the packed model (glic_packed_offsets layout), HOST copy of the planar parameter buffer.
int glic_ply_write_packed(const char* path, uint32_t P, uint32_t M, const float* params_host) {
    if (P > 0 && !params_host) { set_error("ply_write_packed: null buffer"); return GLIC_ERR_INVALID_ARGUMENT; }
    const float* rot = params_host;
    const float* xyz = rot + 4 * (size_t)P;
    const float* scl = xyz + 3 * (size_t)P;
    const float* opa = scl + 3 * (size_t)P;
    const float* dc = opa + (size_t)P;
    const float* rest = dc + 3 * (size_t)P;
    return glic_ply_write(path, P, M, xyz, dc, rest, opa, scl, rot);
}

}  // extern "C"

// ---- mapper checkpoints (include/glic_b200.h "Checkpoints"): the file's framing, its fixed fields and their validation.  Host-only
// code: mapper.cu moves the arrays between the file and the device.
#include "checkpoint.h"

#include <cerrno>
#include <sstream>
#include <unistd.h>

namespace glic {
namespace ckpt {

namespace {

constexpr char MAGIC[8] = {'G', 'L', 'I', 'C', 'C', 'K', 'P', 'T'};
constexpr int MAX_SLOTS = 32;                    // mapper.cu: world * views_per_rank
constexpr uint32_t MAX_RNG_TEXT = 1u << 16;

int bad(const std::string& why) { set_error("checkpoint: " + why); return GLIC_ERR_INVALID_ARGUMENT; }

// a cursor over fixed fields read from the file
struct Get {
    const uint8_t* p;
    const uint8_t* end;
    template <typename T> T get() {
        T v;
        std::memcpy(&v, p, sizeof(T));
        p += sizeof(T);
        return v;
    }
    template <typename T> void get_n(T* v, size_t n) { std::memcpy(v, p, n * sizeof(T)); p += n * sizeof(T); }
};

struct Reader {
    FILE* f = nullptr;
    uint64_t size = 0;
    ~Reader() { if (f) std::fclose(f); }
    // n bytes at offset off into out (the caller has checked that they lie in the file)
    int at(uint64_t off, size_t n, std::vector<uint8_t>& out) {
        out.resize(n);
        if (fseeko(f, (off_t)off, SEEK_SET) != 0 || std::fread(out.data(), 1, n, f) != n) return bad("read error");
        return GLIC_OK;
    }
};

bool config_valid(const glic_mapper_config& c) {
    return c.width > 0 && c.height > 0 && c.sh_degree >= 0 && c.sh_degree <= 3 && c.world >= 1 && c.world <= 8 && c.rank >= 0 &&
           c.rank < c.world && c.views_per_rank >= 1 && c.world * c.views_per_rank <= MAX_SLOTS && c.capacity >= 256 &&
           c.capacity % 256 == 0 && c.max_iters > 0;
}

int get_config(const uint8_t* h, glic_mapper_config& c) {
    if (std::memcmp(h, MAGIC, 8) != 0) return bad("not a mapper checkpoint (bad magic)");
    uint32_t version;
    std::memcpy(&version, h + 8, 4);
    if (version != VERSION) return bad("unsupported version " + std::to_string(version));
    Get g{h + 12, h + HEADER_BYTES};
    c.width = g.get<int32_t>(); c.height = g.get<int32_t>();
    c.fx = g.get<float>(); c.fy = g.get<float>(); c.cx = g.get<float>(); c.cy = g.get<float>();
    c.sh_degree = g.get<int32_t>();
    c.position_lr = g.get<float>(); c.feature_lr = g.get<float>(); c.opacity_lr = g.get<float>(); c.scaling_lr = g.get<float>();
    c.rotation_lr = g.get<float>(); c.lambda_dssim = g.get<float>(); c.scaling_scale = g.get<float>();
    c.capacity = g.get<uint32_t>(); c.max_iters = g.get<int32_t>(); c.seed = g.get<uint64_t>();
    c.rank = g.get<int32_t>(); c.world = g.get<int32_t>(); c.views_per_rank = g.get<int32_t>();
    if (!config_valid(c)) return bad("configuration out of range");
    return GLIC_OK;
}

int read_header(Reader& r, const char* path, glic_mapper_config& c) {
    r.f = std::fopen(path, "rb");
    if (!r.f) return bad(std::string("cannot open ") + path);
    if (fseeko(r.f, 0, SEEK_END) != 0) return bad("cannot seek");
    r.size = (uint64_t)ftello(r.f);
    if (r.size < HEADER_BYTES) return bad("truncated header");
    std::vector<uint8_t> h;
    if (int e = r.at(0, HEADER_BYTES, h)) return e;
    return get_config(h.data(), c);
}

}  // namespace

void put_config(Bytes& b, const glic_mapper_config& c) {
    b.put<int32_t>(c.width).put<int32_t>(c.height).put(c.fx).put(c.fy).put(c.cx).put(c.cy).put<int32_t>(c.sh_degree);
    b.put(c.position_lr).put(c.feature_lr).put(c.opacity_lr).put(c.scaling_lr).put(c.rotation_lr).put(c.lambda_dssim).put(c.scaling_scale);
    b.put<uint32_t>(c.capacity).put<int32_t>(c.max_iters).put<uint64_t>(c.seed).put<int32_t>(c.rank).put<int32_t>(c.world)
     .put<int32_t>(c.views_per_rank);
}

void put_stats(Bytes& b, const glic_mapper_stats& s) {
    b.put(s.num_gaussians).put(s.capacity).put(s.iterations).put(s.last_inserted).put(s.last_loss).put(s.mean_visible)
     .put(s.overflow_regrows).put(s.ms_extend).put(s.ms_optimize);
}

void put_schedule(Bytes& b, uint32_t on, const glic_density_schedule& s, const glic_density_counts& t, uint32_t steps, uint32_t resets) {
    b.put(on).put(s.densify_from).put(s.densify_until).put(s.densify_interval).put(s.opacity_reset_interval).put(s.grad_threshold)
     .put(s.percent_dense).put(s.min_opacity).put(s.reset_opacity).put(s.screen_radius).put(s.world_scale_factor).put(s.scene_extent);
    b.put(t.cloned).put(t.split).put(t.pruned).put(t.rows).put(steps).put(resets);
}

void put_frame_stats(Bytes& b, const glic_frame_stats& s) {
    b.put(s.frames).put(s.train).put(s.test).put(s.pending_points).put(s.image_bytes);
}

Writer::~Writer() {
    if (f_) { std::fclose(f_); std::remove(tmp_.c_str()); }
}

int Writer::open(const char* path) {
    path_ = path;
    tmp_ = path_ + ".tmp";
    f_ = std::fopen(tmp_.c_str(), "wb");
    if (!f_) return bad("cannot create " + tmp_);
    return GLIC_OK;
}

int Writer::header(const glic_mapper_config& cfg) {
    Bytes b;
    b.put_n(MAGIC, 8).put(VERSION);
    put_config(b, cfg);
    return write(b.b.data(), b.b.size());
}

int Writer::begin(Section s, uint64_t length) {
    if (open_section_) return bad("internal: a section was left open");
    Bytes b;
    b.put(TAGS[s]).put<uint32_t>(0).put(length);
    if (int e = write(b.b.data(), b.b.size())) return e;
    left_ = length;
    open_section_ = true;
    return GLIC_OK;
}

int Writer::write(const void* p, size_t n) {
    if (open_section_) {
        if (n > left_) return bad("internal: a section is longer than its declared length");
        left_ -= n;
    }
    if (n && std::fwrite(p, 1, n, f_) != n) return bad("short write to " + tmp_ + ": " + std::strerror(errno));
    return GLIC_OK;
}

int Writer::end() {
    if (!open_section_ || left_) return bad("internal: a section is shorter than its declared length");
    open_section_ = false;
    return GLIC_OK;
}

int Writer::commit() {
    if (open_section_) return bad("internal: a section was left open");
    Bytes b;
    b.put(END_TAG).put<uint32_t>(0).put<uint64_t>(0);
    if (int e = write(b.b.data(), b.b.size())) return e;
    if (std::fflush(f_) != 0 || fsync(fileno(f_)) != 0) return bad("cannot flush " + tmp_ + ": " + std::strerror(errno));
    const int closed = std::fclose(f_);
    f_ = nullptr;
    if (closed != 0 || std::rename(tmp_.c_str(), path_.c_str()) != 0) {
        std::remove(tmp_.c_str());
        return bad("cannot replace " + path_ + ": " + std::strerror(errno));
    }
    return GLIC_OK;
}

int read_info(const char* path, Info& o) {
    Reader r;
    if (int e = read_header(r, path, o.cfg)) return e;
    const int W = o.cfg.width, H = o.cfg.height, M = (o.cfg.sh_degree + 1) * (o.cfg.sh_degree + 1) - 1;
    // the section table: every tag known and present once, every length inside the file, the end marker last
    uint64_t off[N_SECTIONS], len[N_SECTIONS];
    bool seen[N_SECTIONS] = {};
    uint64_t pos = HEADER_BYTES;
    std::vector<uint8_t> buf;
    for (;;) {
        if (r.size - pos < FRAME_BYTES) return bad("truncated file (section frame)");
        if (int e = r.at(pos, FRAME_BYTES, buf)) return e;
        Get g{buf.data(), buf.data() + FRAME_BYTES};
        const uint32_t tag = g.get<uint32_t>(), zero = g.get<uint32_t>();
        const uint64_t n = g.get<uint64_t>();
        pos += FRAME_BYTES;
        if (zero != 0) return bad("bad section frame");
        if (tag == END_TAG) {
            if (n != 0) return bad("bad end marker");
            if (pos != r.size) return bad("trailing bytes after the end marker");
            break;
        }
        int s = 0;
        while (s < N_SECTIONS && TAGS[s] != tag) ++s;
        if (s == N_SECTIONS) return bad("unknown section");
        if (seen[s]) return bad("duplicated section");
        if (n > r.size - pos) return bad("truncated file (section longer than the file)");
        seen[s] = true; off[s] = pos; len[s] = n;
        pos += n;
    }
    for (int s : {MAP, COUNTERS, KEYFRAMES, SCHEDULE})
        if (!seen[s]) return bad("missing section");
    auto fixed = [&](Section s, size_t n, std::vector<uint8_t>& b) -> int {
        if (len[s] < n) return bad("section length disagrees with its counts");
        return r.at(off[s], n, b);
    };
    auto length_is = [&](Section s, uint64_t want) { return len[s] == want ? GLIC_OK : bad("section length disagrees with its counts"); };
    // CNTR
    if (int e = fixed(COUNTERS, 92, buf)) return e;
    {
        Get g{buf.data(), buf.data() + buf.size()};
        glic_mapper_stats& s = o.st;
        s.num_gaussians = g.get<uint32_t>(); s.capacity = g.get<uint32_t>(); s.iterations = g.get<uint64_t>();
        s.last_inserted = g.get<uint32_t>(); s.last_loss = g.get<float>(); s.mean_visible = g.get<double>();
        s.overflow_regrows = g.get<uint32_t>(); s.ms_extend = g.get<float>(); s.ms_optimize = g.get<float>();
        o.view_counter = g.get<uint64_t>(); o.bin_cap = g.get<int64_t>(); o.binning_bytes = g.get<uint64_t>(); o.sample_bytes = g.get<uint64_t>();
        o.optimizer = g.get<uint32_t>(); o.deterministic = g.get<uint32_t>(); o.flags = g.get<uint32_t>();
        const uint32_t rng_len = g.get<uint32_t>();
        if (rng_len > MAX_RNG_TEXT) return bad("view sampler state too long");
        if (int e = length_is(COUNTERS, counters_bytes(rng_len))) return e;
        if (o.optimizer > 1 || o.deterministic > 1 || (o.flags & ~F_ALL) || o.bin_cap < 0) return bad("counters out of range");
        std::vector<uint8_t> text;
        if (int e = r.at(off[COUNTERS] + 92, rng_len, text)) return e;
        std::istringstream in(std::string(text.begin(), text.end()));
        in >> o.rng;
        if (in.fail() || (in >> std::ws, !in.eof())) return bad("unreadable view sampler state");
    }
    const bool expo = o.flags & F_EXPOSURE, pose = o.flags & F_POSE, dens = o.flags & F_DENSIFICATION, frames = o.flags & F_FRAMES;
    const bool want[N_SECTIONS] = {true, true, true, expo, pose, dens, true, frames};
    for (int s = 0; s < N_SECTIONS; ++s)
        if (seen[s] != want[s]) return bad(seen[s] ? "section of a feature that is off" : "missing section");
    // MAP
    if (int e = fixed(MAP, 12, buf)) return e;
    {
        Get g{buf.data(), buf.data() + buf.size()};
        o.P = g.get<uint32_t>(); o.Pcap = g.get<uint32_t>(); o.n_sky = g.get<uint32_t>();
        if (o.P > o.Pcap || o.n_sky > o.P) return bad("row counts out of range");
        if (o.Pcap != o.cfg.capacity || o.st.capacity != o.Pcap || o.st.num_gaussians != o.P) return bad("row counts disagree between sections");
        if (int e = length_is(MAP, map_bytes(o.P, M))) return e;
        o.map_off = off[MAP] + 12;
    }
    // FRMS (before the keyframes, which refer to its frame store)
    const uint64_t stride = frame_stride(W, H);
    if (frames) {
        if (int e = fixed(FRAMES, 36, buf)) return e;
        Get g{buf.data(), buf.data() + buf.size()};
        o.frame_k = g.get<int32_t>(); o.sky_points = g.get<int32_t>(); o.sky_radius = g.get<int32_t>();
        glic_frame_stats& s = o.fst;
        s.frames = g.get<uint32_t>(); s.train = g.get<uint32_t>(); s.test = g.get<uint32_t>(); s.pending_points = g.get<uint32_t>();
        s.image_bytes = g.get<uint64_t>();
        if (int e = length_is(FRAMES, frames_bytes(s.pending_points))) return e;
        if (o.frame_k < 1 || o.sky_points < 0 || (o.sky_points > 0 && o.sky_radius <= 0) || (uint64_t)s.train + s.test != s.frames ||
            s.image_bytes != (uint64_t)((s.frames + FRAME_CHUNK - 1) / FRAME_CHUNK) * FRAME_CHUNK * stride ||
            (uint64_t)s.pending_points + (uint64_t)o.sky_points > INT32_MAX / 4)
            return bad("frame settings out of range");
        o.frames_off = off[FRAMES] + 36;
    }
    // KEYF: walk the records
    if (int e = fixed(KEYFRAMES, 8, buf)) return e;
    {
        Get g{buf.data(), buf.data() + buf.size()};
        o.n_train = g.get<uint32_t>(); o.n_test = g.get<uint32_t>();
        uint64_t at = off[KEYFRAMES] + 8, end = off[KEYFRAMES] + len[KEYFRAMES];
        const uint64_t n = (uint64_t)o.n_train + o.n_test;
        if (n > (end - at) / KEYFRAME_RECORD_BYTES) return bad("section length disagrees with its counts");
        o.kf.resize(n);
        std::vector<uint8_t> used(frames ? o.fst.frames : 0, 0);
        uint64_t n_frames = 0;
        for (Keyframe& k : o.kf) {
            if (end - at < KEYFRAME_RECORD_BYTES) return bad("section length disagrees with its counts");
            if (int e = r.at(at, KEYFRAME_RECORD_BYTES, buf)) return e;
            Get q{buf.data(), buf.data() + buf.size()};
            q.get_n(k.R_wc, 9); q.get_n(k.t_wc, 3); q.get_n(k.cam, 42); q.get_n(k.cam_dev, 36);
            k.kind = q.get<uint32_t>(); k.frame = q.get<uint32_t>(); k.mask_valid = q.get<uint32_t>(); k.mask_valid_left = q.get<uint32_t>();
            if (k.kind > IMAGE_DEVICE || k.mask_valid > (uint64_t)W * H || k.mask_valid_left > k.mask_valid) return bad("keyframe record out of range");
            if (k.kind == IMAGE_BGR8) {
                if (!frames || k.frame >= o.fst.frames || used[k.frame]) return bad("keyframe frame index out of range");
                used[k.frame] = 1;
                ++n_frames;
            } else if (k.frame != NO_FRAME) {
                return bad("keyframe record out of range");
            }
            const uint64_t b = keyframe_bytes(k.kind, k.mask_valid, W, H);
            if (end - at < b) return bad("section length disagrees with its counts");
            k.image_off = at + KEYFRAME_RECORD_BYTES;
            k.mask_off = k.image_off + (k.kind == IMAGE_BGR8 ? 3 : 12) * (uint64_t)W * H;
            at += b;
        }
        if (at != end) return bad("section length disagrees with its counts");
        if (frames && n_frames != o.fst.frames) return bad("keyframe counts disagree between sections");
    }
    // EXPO, POSE
    if (expo) {
        if (int e = fixed(EXPOSURE, 8, buf)) return e;
        Get g{buf.data(), buf.data() + buf.size()};
        o.expo_lr = g.get<float>();
        const uint32_t n = g.get<uint32_t>();
        if (n != o.n_train) return bad("keyframe counts disagree between sections");
        if (int e = length_is(EXPOSURE, exposure_bytes(n))) return e;
        o.expo_off = off[EXPOSURE] + 8;
    }
    if (pose) {
        if (int e = fixed(POSE, 12, buf)) return e;
        Get g{buf.data(), buf.data() + buf.size()};
        o.pose_lr_rho = g.get<float>(); o.pose_lr_omega = g.get<float>();
        const uint32_t n = g.get<uint32_t>();
        if (n != o.n_train) return bad("keyframe counts disagree between sections");
        if (int e = length_is(POSE, pose_bytes(n))) return e;
        o.pose_off = off[POSE] + 12;
    }
    // DENS
    if (dens) {
        if (int e = fixed(DENSIFICATION, 12, buf)) return e;
        Get g{buf.data(), buf.data() + buf.size()};
        o.dens_calls = g.get<uint64_t>();
        if (g.get<uint32_t>() != o.P) return bad("row counts disagree between sections");
        if (int e = length_is(DENSIFICATION, densification_bytes(o.P))) return e;
        o.dens_off = off[DENSIFICATION] + 12;
    }
    // SCHD
    if (int e = length_is(SCHEDULE, SCHEDULE_BYTES)) return e;
    if (int e = fixed(SCHEDULE, SCHEDULE_BYTES, buf)) return e;
    {
        Get g{buf.data(), buf.data() + buf.size()};
        glic_density_schedule& s = o.sched;
        o.sched_on = g.get<uint32_t>();
        s.densify_from = g.get<uint32_t>(); s.densify_until = g.get<uint32_t>(); s.densify_interval = g.get<uint32_t>();
        s.opacity_reset_interval = g.get<uint32_t>(); s.grad_threshold = g.get<float>(); s.percent_dense = g.get<float>();
        s.min_opacity = g.get<float>(); s.reset_opacity = g.get<float>(); s.screen_radius = g.get<int32_t>();
        s.world_scale_factor = g.get<float>(); s.scene_extent = g.get<float>();
        glic_density_counts& t = o.sched_totals;
        t.cloned = g.get<uint32_t>(); t.split = g.get<uint32_t>(); t.pruned = g.get<uint32_t>(); t.rows = g.get<uint32_t>();
        o.sched_steps = g.get<uint32_t>(); o.sched_resets = g.get<uint32_t>();
        if (o.sched_on > 1 || (o.sched_on && (!dens || s.densify_interval == 0))) return bad("density schedule out of range");
    }
    return GLIC_OK;
}

}  // namespace ckpt
}  // namespace glic

extern "C" int glic_mapper_checkpoint_config(const char* path, glic_mapper_config* out) {
    if (!path || !out) { set_error("mapper_checkpoint_config: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    glic::ckpt::Reader r;
    glic_mapper_config c{};
    if (int e = glic::ckpt::read_header(r, path, c)) return e;
    *out = c;
    return GLIC_OK;
}
