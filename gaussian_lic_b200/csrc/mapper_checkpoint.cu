// mapper_checkpoint.cu -- the native mapper's checkpoints: the arrays of the file (checkpoint.h, map_io.cu) moved between it
// and the device (glic_mapper_save_checkpoint, glic_mapper_load_checkpoint).
#include "mapper_state.cuh"
#include <cstdio>
#include <cstring>
#include <memory>
#include <sstream>

namespace mapper_impl {

// ---- checkpoints (glic_mapper_save_checkpoint, glic_mapper_load_checkpoint) ------------------------------------------------
// The file's framing, fixed fields and validation are map_io.cu's (checkpoint.h); here the arrays move between it and the device
// through two pinned chunks: while one chunk is written (read), the copy of the other is in flight.
constexpr size_t CKPT_CHUNK = size_t(8) << 20;

int make_events(Event (&ev)[2]) {
    for (Event& e : ev) {
        cudaEvent_t h = nullptr;
        GLIC_CUDA_TRY(cudaEventCreateWithFlags(&h, cudaEventDisableTiming));
        e = Event(h);
    }
    return GLIC_OK;
}

// A section's bytes in file order: device spans are copied on `s` into the current chunk, which is written once full while the
// other chunk fills; host bytes are written in place once every device byte before them is.
class SaveStream {
public:
    SaveStream(ckpt::Writer& w, cudaStream_t s, char* stage, const Event (&ev)[2]) : w_(w), s_(s), ev_{ev[0], ev[1]} {
        buf_[0] = stage; buf_[1] = stage + CKPT_CHUNK;
    }
    int begin(ckpt::Section sec, uint64_t length) { MAP_TRY(flush()); return w_.begin(sec, length); }
    int end() { MAP_TRY(flush()); return w_.end(); }
    int device(const void* src, size_t n) {
        const char* p = static_cast<const char*>(src);
        while (n) {
            const size_t k = std::min(n, CKPT_CHUNK - fill_);
            GLIC_CUDA_TRY(cudaMemcpyAsync(buf_[cur_] + fill_, p, k, cudaMemcpyDeviceToHost, s_));
            fill_ += k; p += k; n -= k;
            if (fill_ == CKPT_CHUNK) MAP_TRY(submit());
        }
        return GLIC_OK;
    }
    int host(const void* p, size_t n) { MAP_TRY(flush()); return w_.write(p, n); }
    int host(const ckpt::Bytes& b) { return host(b.b.data(), b.b.size()); }
    int flush() { MAP_TRY(submit()); return drain(); }
private:
    // the current chunk's copies are enqueued: write the other chunk, then fill that one
    int submit() {
        if (!fill_) return GLIC_OK;
        GLIC_CUDA_TRY(cudaEventRecord(ev_[cur_], s_));
        MAP_TRY(drain());
        pending_ = fill_; cur_ ^= 1; fill_ = 0;
        return GLIC_OK;
    }
    int drain() {                                  // writes the submitted chunk (the one that is not current)
        if (!pending_) return GLIC_OK;
        GLIC_CUDA_TRY(cudaEventSynchronize(ev_[cur_ ^ 1]));
        MAP_TRY(w_.write(buf_[cur_ ^ 1], pending_));
        pending_ = 0;
        return GLIC_OK;
    }
    ckpt::Writer& w_;
    cudaStream_t s_;
    cudaEvent_t ev_[2];
    char* buf_[2];
    int cur_ = 0;
    size_t fill_ = 0, pending_ = 0;
};

// File bytes at given offsets into device memory (read into one chunk while the other's copy on `s` is in flight) or host memory
class LoadStream {
public:
    LoadStream(cudaStream_t s, char* stage, const Event (&ev)[2]) : s_(s), ev_{ev[0], ev[1]} { buf_[0] = stage; buf_[1] = stage + CKPT_CHUNK; }
    ~LoadStream() { if (f_) std::fclose(f_); }
    int open(const char* path) {
        f_ = std::fopen(path, "rb");
        if (!f_) { set_error(std::string("checkpoint: cannot open ") + path); return GLIC_ERR_INVALID_ARGUMENT; }
        return GLIC_OK;
    }
    int device(uint64_t off, void* dst, size_t n) {
        MAP_TRY(seek(off));
        char* d = static_cast<char*>(dst);
        while (n) {
            const size_t k = std::min(n, CKPT_CHUNK);
            if (busy_[cur_]) GLIC_CUDA_TRY(cudaEventSynchronize(ev_[cur_]));
            MAP_TRY(read(buf_[cur_], k));
            GLIC_CUDA_TRY(cudaMemcpyAsync(d, buf_[cur_], k, cudaMemcpyHostToDevice, s_));
            GLIC_CUDA_TRY(cudaEventRecord(ev_[cur_], s_));
            busy_[cur_] = true; cur_ ^= 1; d += k; n -= k;
        }
        return GLIC_OK;
    }
    int host(uint64_t off, void* dst, size_t n) { MAP_TRY(seek(off)); return read(dst, n); }
private:
    int seek(uint64_t off) {
        if (off == pos_) return GLIC_OK;
        if (fseeko(f_, (off_t)off, SEEK_SET) != 0) { set_error("checkpoint: cannot seek"); return GLIC_ERR_INVALID_ARGUMENT; }
        pos_ = off;
        return GLIC_OK;
    }
    int read(void* p, size_t n) {
        if (n && std::fread(p, 1, n, f_) != n) { set_error("checkpoint: truncated file"); return GLIC_ERR_INVALID_ARGUMENT; }
        pos_ += n;
        return GLIC_OK;
    }
    FILE* f_ = nullptr;
    uint64_t pos_ = 0;
    cudaStream_t s_;
    cudaEvent_t ev_[2];
    char* buf_[2];
    bool busy_[2] = {false, false};
    int cur_ = 0;
};

static_assert(sizeof(CamBlock) == 42 * sizeof(float), "the host camera block is 42 floats in the file");

uint32_t image_kind(const Keyframe& kf) { return kf.bgr ? ckpt::IMAGE_BGR8 : kf.image_on_device ? ckpt::IMAGE_DEVICE : ckpt::IMAGE_HOST; }

// the slot of an add_frame keyframe's image in the frame store
uint32_t frame_index(const glic_mapper* m, const uint8_t* bgr) {
    for (size_t c = 0; c < m->frame_chunks.size(); ++c) {
        const uint8_t* base = m->frame_chunks[c];
        if (bgr >= base && bgr < base + FRAME_CHUNK * m->frame_stride) return (uint32_t)(c * FRAME_CHUNK + (size_t)(bgr - base) / m->frame_stride);
    }
    return ckpt::NO_FRAME;
}

uint32_t feature_flags(const glic_mapper* m) {
    return (m->initialized ? ckpt::F_INITIALIZED : 0) | (m->expo_on ? ckpt::F_EXPOSURE : 0) | (m->pose_on ? ckpt::F_POSE : 0) |
           (m->dens_on ? ckpt::F_DENSIFICATION : 0) | (m->frames_on ? ckpt::F_FRAMES : 0);
}

// glic_mapper_save_checkpoint after its checks: the drain, the staging, then every section in file order
int save_checkpoint(glic_mapper* m, const char* path) {
    using namespace ckpt;
    const int W = m->cfg.width, H = m->cfg.height;
    const size_t HW = (size_t)W * H, P = m->P, mask_bytes = sizeof(uint32_t) * (size_t)H * mask_words_per_row(W);
    GLIC_CUDA_TRY(cudaStreamSynchronize(m->stream));
    MAP_TRY(poll_ring(m, true));
    Buf stage;
    MAP_TRY(stage.allocate(2 * CKPT_CHUNK, true));
    Event ev[2];
    MAP_TRY(make_events(ev));
    Writer w;
    MAP_TRY(w.open(path));
    glic_mapper_config cfg = m->cfg;
    cfg.capacity = m->Pcap;                                  // a restored mapper is created at the saved capacity
    MAP_TRY(w.header(cfg));
    SaveStream out(w, m->copy_stream, static_cast<char*>(stage.raw()), ev);
    // the map: the live rows of the six groups of each arena, then the anchors
    MAP_TRY(out.begin(MAP, map_bytes(P, m->M)));
    MAP_TRY(out.host(Bytes().put(m->P).put(m->Pcap).put(m->n_sky)));
    const auto kk = group_widths(m->M);
    for (float* arena : {(float*)m->params, (float*)m->m1, (float*)m->m2}) {
        const auto g = arena_rows(arena, m->Pcap, m->M).groups();
        for (int q = 0; q < 6; ++q) MAP_TRY(out.device(g[q], sizeof(float) * kk[q] * P));
    }
    MAP_TRY(out.device(m->anchor, sizeof(int32_t) * P));
    MAP_TRY(out.end());
    // the counters, the options and the view sampler
    {
        std::ostringstream os;
        os << m->rng;
        const std::string rng = os.str();
        Bytes b;
        put_stats(b, m->st);
        b.put(m->view_counter).put<int64_t>(m->bin_cap).put<uint64_t>(m->binning_ws.bytes()).put<uint64_t>(m->sample_ws.bytes())
         .put<uint32_t>(m->run_optimizer).put<uint32_t>(m->deterministic).put(feature_flags(m)).put<uint32_t>((uint32_t)rng.size())
         .put_n(rng.data(), rng.size());
        MAP_TRY(out.begin(COUNTERS, counters_bytes(rng.size())));
        MAP_TRY(out.host(b));
        MAP_TRY(out.end());
    }
    // the keyframes, training then held-out
    uint64_t kf_bytes = 8;
    for (const auto* list : {&m->train, &m->test})
        for (const Keyframe& kf : *list) kf_bytes += keyframe_bytes(image_kind(kf), kf.mask_valid, W, H);
    MAP_TRY(out.begin(KEYFRAMES, kf_bytes));
    MAP_TRY(out.host(Bytes().put((uint32_t)m->train.size()).put((uint32_t)m->test.size())));
    for (const auto* list : {&m->train, &m->test})
        for (const Keyframe& kf : *list) {
            const uint32_t kind = image_kind(kf);
            MAP_TRY(out.host(Bytes().put_n(kf.R_wc, 9).put_n(kf.t_wc, 3).put_n(reinterpret_cast<const float*>(&kf.cam), 42)));
            MAP_TRY(out.device(kf.cam_dev, 36 * sizeof(float)));   // verbatim: pose refinement and corrections move it on the device
            MAP_TRY(out.host(Bytes().put(kind).put(kind == IMAGE_BGR8 ? frame_index(m, kf.bgr) : NO_FRAME).put(kf.mask_valid)
                                    .put(kf.mask_valid_left)));
            if (kind == IMAGE_BGR8) MAP_TRY(out.device(kf.bgr, 3 * HW));
            else if (kind == IMAGE_DEVICE) MAP_TRY(out.device(kf.image, sizeof(float) * 3 * HW));
            else MAP_TRY(out.host(kf.image, sizeof(float) * 3 * HW));   // read where the caller keeps it
            if (kf.mask_valid) MAP_TRY(out.device(kf.mask, mask_bytes));
        }
    MAP_TRY(out.end());
    // rows [0, n) of each buffer of a group, in the group's order
    auto rows = [&](const std::vector<Rows>& group, size_t n) -> int {
        for (const Rows& r : group) MAP_TRY(out.device(r.buf.raw(), r.bytes * n));
        return GLIC_OK;
    };
    const size_t n = m->train.size();
    if (m->expo_on) {
        MAP_TRY(out.begin(ckpt::EXPOSURE, exposure_bytes(n)));
        MAP_TRY(out.host(Bytes().put(m->expo_lr).put((uint32_t)n)));
        MAP_TRY(rows(exposure_rows(m), n));
        MAP_TRY(out.end());
    }
    if (m->pose_on) {
        MAP_TRY(out.begin(ckpt::POSE, pose_bytes(n)));
        MAP_TRY(out.host(Bytes().put(m->pose_lr_rho).put(m->pose_lr_omega).put((uint32_t)n)));
        MAP_TRY(rows(pose_rows(m), n));
        MAP_TRY(out.end());
    }
    if (m->dens_on) {
        MAP_TRY(out.begin(DENSIFICATION, densification_bytes(P)));
        MAP_TRY(out.host(Bytes().put<uint64_t>(m->dens_calls).put(m->P)));
        MAP_TRY(rows(densification_rows(m), P));
        MAP_TRY(out.end());
    }
    {
        Bytes b;
        put_schedule(b, m->sched_on, m->sched, m->sched_totals, m->sched_steps, m->sched_resets);
        MAP_TRY(out.begin(SCHEDULE, SCHEDULE_BYTES));
        MAP_TRY(out.host(b));
        MAP_TRY(out.end());
    }
    if (m->frames_on) {
        const size_t p = m->fst.pending_points;
        Bytes b;
        b.put<int32_t>(m->frame_k).put<int32_t>(m->frame_sky_points).put<int32_t>(m->frame_sky_radius);
        put_frame_stats(b, m->fst);
        MAP_TRY(out.begin(FRAMES, frames_bytes(p)));
        MAP_TRY(out.host(b));
        MAP_TRY(rows(scan_rows(m), p));
        MAP_TRY(out.end());
    }
    return w.commit();
}

// created, and nothing since that leaves a trace in the state a checkpoint holds (load_lpips and set_option aside)
bool mapper_fresh(const glic_mapper* m) {
    return !m->initialized && m->P == 0 && m->train.empty() && m->test.empty() && !m->expo_on && !m->pose_on && !m->dens_on &&
           !m->frames_on && !m->sched_on && !m->exported && !m->connected;
}

// every field but the capacity, floats by their bits
bool same_config(const glic_mapper_config& a, const glic_mapper_config& b) {
    ckpt::Bytes x, y;
    glic_mapper_config a1 = a, b1 = b;
    a1.capacity = b1.capacity = 0;
    ckpt::put_config(x, a1);
    ckpt::put_config(y, b1);
    return x.b == y.b;
}

// glic_mapper_load_checkpoint after its checks: validate the whole file, allocate everything (keyframes first, then the mapper's
// buffers in one growth whose fill streams the file in), and only then set the scalars
int load_checkpoint(glic_mapper* m, const char* path) {
    using namespace ckpt;
    if (!mapper_fresh(m)) {
        set_error("mapper_load_checkpoint: the mapper is not fresh (load into a mapper that is only created, with no rows, keyframes or "
                  "features, before glic_mapper_export)");
        return GLIC_ERR_INVALID_ARGUMENT;
    }
    auto in = std::make_unique<Info>();
    MAP_TRY(read_info(path, *in));
    if (!same_config(in->cfg, m->cfg)) {
        set_error("mapper_load_checkpoint: the mapper's configuration differs from the checkpoint's (create it from "
                  "glic_mapper_checkpoint_config)");
        return GLIC_ERR_INVALID_ARGUMENT;
    }
    const int W = m->cfg.width, H = m->cfg.height;
    const size_t HW = (size_t)W * H, mask_bytes = sizeof(uint32_t) * (size_t)H * mask_words_per_row(W);
    if (glic_binning_capacity(in->binning_bytes, in->sample_bytes, W, H, 0) != in->bin_cap) {
        set_error("checkpoint: the binning workspaces do not give the saved binning capacity"); return GLIC_ERR_INVALID_ARGUMENT;
    }
    const bool expo = in->flags & F_EXPOSURE, pose = in->flags & F_POSE, dens = in->flags & F_DENSIFICATION, frames = in->flags & F_FRAMES;
    const uint64_t stride = frame_stride(W, H);
    GLIC_CUDA_TRY(cudaStreamSynchronize(m->stream));
    MAP_TRY(poll_ring(m, true));
    // 1. the staging, the frame store and the keyframes, outside the mapper
    Buf stage;
    MAP_TRY(stage.allocate(2 * CKPT_CHUNK, true));
    Event ev[2];
    MAP_TRY(make_events(ev));
    std::vector<Dev<uint8_t>> chunks(frames ? (in->fst.frames + FRAME_CHUNK - 1) / FRAME_CHUNK : 0);
    for (Dev<uint8_t>& c : chunks) MAP_TRY(c.allocate(FRAME_CHUNK * stride));
    std::vector<Keyframe> kfs(in->kf.size());
    for (size_t i = 0; i < kfs.size(); ++i) {
        const ckpt::Keyframe& r = in->kf[i];
        Keyframe& k = kfs[i];
        std::memcpy(k.R_wc, r.R_wc, sizeof(k.R_wc)); std::memcpy(k.t_wc, r.t_wc, sizeof(k.t_wc));
        std::memcpy(&k.cam, r.cam, sizeof(k.cam));
        MAP_TRY(k.cam_dev.allocate(36 * sizeof(float)));
        if (r.kind == IMAGE_BGR8) {
            k.bgr = chunks[r.frame / FRAME_CHUNK] + (r.frame % FRAME_CHUNK) * stride;
        } else {                                             // the image keeps its memory class, now owned by the mapper
            MAP_TRY(k.owned_image.allocate(sizeof(float) * 3 * HW, r.kind == IMAGE_HOST));
            k.image = static_cast<const float*>(k.owned_image.raw());
            k.image_on_device = r.kind == IMAGE_DEVICE;
        }
        if (r.mask_valid) MAP_TRY(k.mask.allocate(mask_bytes));
        k.mask_valid = r.mask_valid;
        k.mask_valid_left = r.mask_valid_left;
        k.view = make_view(k.cam, k.cam_dev, W, H);
    }
    // 2. the mapper's buffers at the saved capacity, as set_capacity, enable_densification, set_option, enable_exposure and
    //    add_frame size them; zeroed where they start zeroed.  The mapper is fresh (P = 0), so capacity_buffers keeps nothing.
    const uint32_t cap = in->Pcap, P = in->P, n = in->n_train, pending = frames ? in->fst.pending_points : 0;
    const XLayout x = xblock_layout(m->S, cap, dens);
    const size_t kf_cap = (expo || pose) ? std::max<size_t>(n, 64) : 0;
    std::vector<Grow> list = capacity_buffers(m, cap, dens);
    list.push_back({m->binning_ws, (size_t)in->binning_bytes});
    list.push_back({m->sample_ws, (size_t)in->sample_bytes});
    if (in->deterministic) {
        list.push_back({m->det_ws, glic_deterministic_bytes(in->bin_cap, W, H)});
        list.push_back({m->det_sums, fixed_order_sums_bytes(H, W)});
    }
    if (expo && glic_loss_exposure_scratch_bytes(H, W) > m->loss_scratch.bytes()) list.push_back({m->loss_scratch, glic_loss_exposure_scratch_bytes(H, W)});
    if (kf_cap) {
        grow_rows(list, exposure_rows(m), kf_cap, 0, true);
        grow_rows(list, pose_rows(m), kf_cap, 0, true);
    }
    if (pending) grow_rows(list, scan_rows(m), pending, 0, false);
    auto fill = [&](Buf* fresh) -> int {
        auto at = [&](const Buf& b) -> char* {
            for (size_t i = 0; i < list.size(); ++i) if (&list[i].buf == &b) return static_cast<char*>(fresh[i].raw());
            return nullptr;
        };
        LoadStream L(m->stream, static_cast<char*>(stage.raw()), ev);
        MAP_TRY(L.open(path));
        const auto kk = group_widths(m->M);
        uint64_t off = in->map_off;
        for (const Buf* a : {(const Buf*)&m->params, (const Buf*)&m->m1, (const Buf*)&m->m2}) {
            const auto g = arena_rows(reinterpret_cast<float*>(at(*a)), cap, m->M).groups();
            for (int q = 0; q < 6; ++q) {
                MAP_TRY(L.device(off, g[q], sizeof(float) * kk[q] * P));
                off += sizeof(float) * kk[q] * P;
            }
        }
        MAP_TRY(L.device(off, at(m->anchor), sizeof(int32_t) * P));
        for (size_t i = 0; i < kfs.size(); ++i) {
            const ckpt::Keyframe& r = in->kf[i];
            Keyframe& k = kfs[i];
            GLIC_CUDA_TRY(cudaMemcpyAsync(k.cam_dev, r.cam_dev, sizeof(r.cam_dev), cudaMemcpyHostToDevice, m->stream));
            if (r.kind == IMAGE_BGR8) MAP_TRY(L.device(r.image_off, const_cast<uint8_t*>(k.bgr), 3 * HW));
            else if (r.kind == IMAGE_DEVICE) MAP_TRY(L.device(r.image_off, k.owned_image.raw(), sizeof(float) * 3 * HW));
            else MAP_TRY(L.host(r.image_off, k.owned_image.raw(), sizeof(float) * 3 * HW));
            if (r.mask_valid) MAP_TRY(L.device(r.mask_off, k.mask, mask_bytes));
        }
        // rows [0, rows) of each buffer of a group: the consecutive arrays of one section from file offset o
        auto arrays = [&](uint64_t o, const std::vector<Rows>& group, size_t rows) -> int {
            for (const Rows& r : group) { MAP_TRY(L.device(o, at(r.buf), r.bytes * rows)); o += r.bytes * rows; }
            return GLIC_OK;
        };
        if (expo) MAP_TRY(arrays(in->expo_off, exposure_rows(m), n));
        if (pose) MAP_TRY(arrays(in->pose_off, pose_rows(m), n));
        if (dens) MAP_TRY(arrays(in->dens_off, densification_rows(m), P));
        if (pending) MAP_TRY(arrays(in->frames_off, scan_rows(m), pending));
        return GLIC_OK;
    };
    // a failed read returns with copies in flight into the new buffers: they finish before the buffers are released
    MAP_TRY(grow(m, list, [&](Buf* fresh) { const int e = fill(fresh); if (e) cudaStreamSynchronize(m->stream); return e; }));
    // 3. the state: nothing below can fail
    for (size_t i = 0; i < kfs.size(); ++i) (i < n ? m->train : m->test).push_back(std::move(kfs[i]));
    m->frame_chunks = std::move(chunks);
    m->cfg.capacity = cap;
    adopt_capacity(m, cap, x);
    m->P = P; m->n_sky = in->n_sky;
    m->st = in->st;
    m->view_counter = in->view_counter;
    m->rng = in->rng;
    m->bin_cap = in->bin_cap;
    m->run_optimizer = in->optimizer != 0;
    m->deterministic = in->deterministic != 0;
    m->initialized = in->flags & F_INITIALIZED;
    m->kf_cap = kf_cap;
    m->expo_on = expo; m->expo_lr = in->expo_lr;
    m->pose_on = pose; m->pose_lr_rho = in->pose_lr_rho; m->pose_lr_omega = in->pose_lr_omega;
    m->dens_on = dens; m->dens_calls = in->dens_calls;
    m->sched_on = in->sched_on != 0; m->sched = in->sched; m->sched_totals = in->sched_totals;
    m->sched_steps = in->sched_steps; m->sched_resets = in->sched_resets;
    m->frames_on = frames;
    if (frames) {
        m->frame_k = in->frame_k; m->frame_sky_points = in->sky_points; m->frame_sky_radius = in->sky_radius;
        m->frame_stride = stride;
        m->fst = in->fst;
        m->scan_cap = pending;
    }
    return GLIC_OK;
}

}  // namespace mapper_impl

extern "C" {

int glic_mapper_save_checkpoint(glic_mapper* m, const char* path) {
    if (!m || !path) { set_error("mapper_save_checkpoint: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    return save_checkpoint(m, path);
}

int glic_mapper_load_checkpoint(glic_mapper* m, const char* path) {
    if (!m || !path) { set_error("mapper_load_checkpoint: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    return load_checkpoint(m, path);
}

}  // extern "C"
