// mapper_density.cu -- the native mapper's density control: the one compaction behind densify, prune and prune_unseen, the
// schedule of optimize(), the statistics and the contribution scores (include/glic_b200.h "Native mapping host").
#include "mapper_state.cuh"
#include <algorithm>
#include <cmath>

namespace mapper_impl {

// The one stable compaction of the arenas (prune.cu), behind glic_mapper_densify_and_prune, glic_mapper_densify (min_opacity 0,
// both size tests off) and glic_mapper_prune (no row selected, both size tests off): select, reserve (capacity, then the
// spares), gather each arena into a spare one of the same capacity and swap, write the children's xyz and log-scale.  The
// spare is allocated once, before anything changes, and rotates: params -> spare, the old params buffer then takes m1, the old
// m1 buffer m2, and the old m2 buffer is freed.  Peak extra memory: one arena (glic_packed_floats(Pcap, M) floats); the
// selection's scratch (12 B per row and five counts per 1024 rows) lives in the extend() staging buffer, which keeps it.  The
// params gather takes every result row, the moments only the kept rows (the new rows' moments are zero), and each writes output
// rows [0, max(rows, P)): rows [P, Pcap) of every arena are zero already (allocation, initialize, append and regrow keep them
// so), so the rows a prune vacates end up zero like them.
// densify: the call densifies, so it selects by the statistics, zeroes them and advances dens_calls even when no row changes.
// Otherwise it only prunes: no statistic is read, the statistics (with densification on) move with their rows, dens_calls
// stays (it keys the children's draws of every later densify), and a call that removes nothing touches nothing.
// The caller has validated p.  reject_empty: a result without rows is an error (densify on an empty map is not).
// unseen (optional, a prune only): the scores in score_ws (contribution below) also remove rows, by glic_mapper_prune_unseen's test.
int density_step(glic_mapper* m, const glic_density_params& p, bool densify, int dry_run, bool reject_empty, glic_density_counts* out,
                 const char* what, const glic_unseen_params* unseen = nullptr) {
    GLIC_CUDA_TRY(cudaStreamSynchronize(m->stream));
    MAP_TRY(poll_ring(m, true));
    const uint32_t P = m->P;
    uint32_t r[6] = {0, 0, 0, 0, 0, 0};                // clones, splits, surviving kept rows, clones, split rows, sky rows
    cudaStream_t s = m->stream;
    if (P) {
        MAP_TRY(reserve(m, m->extend_ws, density_scratch_bytes(P)));   // the selection's scratch: the idle extend() staging
        const ArenaRows g = arena_rows(m->params, m->Pcap, m->M);
        const float* no_stats = nullptr;                   // a prune selects no row, with densification on or off
        DensitySelect a{P, m->n_sky, densify ? m->dens_accum : no_stats, densify ? m->dens_denom : no_stats, g.log_scale, g.opacity,
                        m->dens_maxr, p.grad_threshold, p.percent_dense * p.scene_extent, p.min_opacity, p.max_world_scale,
                        p.max_screen_radius};
        if (unseen) {
            a.score_hits = reinterpret_cast<const uint64_t*>(m->score_ws.raw());
            a.score_ends = a.score_hits + m->Pcap;
            a.score_max = reinterpret_cast<const float*>(a.score_hits + 2 * (size_t)m->Pcap);
            a.min_weight = unseen->min_weight;
            a.min_hits = unseen->min_hits;
            a.score_sky = unseen->sky;
        }
        MAP_TRY(launch_density_select(a, m->extend_ws, r, s));
    }
    const uint32_t n_clone = r[0], n_split = r[1], kept = r[2], cloned = r[3], split = r[4];
    const uint64_t unpruned = (uint64_t)P + n_clone + n_split, rows = (uint64_t)kept + cloned + 2 * (uint64_t)split;
    if (reject_empty && rows == 0) {
        set_error(std::string(what) + ": the result has no rows (an empty map cannot be trained)");
        return GLIC_ERR_INVALID_ARGUMENT;
    }
    if (!dry_run && (n_clone || n_split || rows != P)) {
        if (rows > m->Pcap) {
            if (m->connected) {
                set_error(std::string(what) + ": the result does not fit the capacity, which is fixed once the exchange blocks are connected (world > 1); prune first");
                return GLIC_ERR_WORKSPACE;
            }
            MAP_TRY(set_capacity(m, std::max<uint32_t>((uint32_t)rows, 2 * m->Pcap)));
        }
        Dev<float> spare;
        Dev<int32_t> spare_anchor;
        const bool move_stats = !densify && m->dens_on;
        const std::vector<Rows> stats = densification_rows(m);
        std::vector<Buf> spare_stats(move_stats ? stats.size() : 0);
        const size_t bytes = arena_floats(m, m->Pcap) * sizeof(float);
        MAP_TRY(spare.allocate(bytes));
        MAP_TRY(spare_anchor.allocate((size_t)m->Pcap * 4));
        for (size_t q = 0; q < spare_stats.size(); ++q) MAP_TRY(spare_stats[q].allocate((size_t)m->Pcap * stats[q].bytes));
        GLIC_CUDA_TRY(cudaMemsetAsync(spare, 0, bytes, s));
        const uint32_t* idx = density_index(m->extend_ws, P);
        const uint32_t written = std::max<uint32_t>((uint32_t)rows, P);   // the rows a prune vacates become zero
        for (Dev<float>* arena : {&m->params, &m->m1, &m->m2}) {
            MAP_TRY(launch_gather_rows(*arena, spare, m->Pcap, m->M, written, arena == &m->params ? (uint32_t)rows : kept, idx, s));
            std::swap(*arena, spare);
        }
        // the anchors follow the params gather: every result row, clones and split children from their parents
        MAP_TRY(launch_gather_words(m->anchor, spare_anchor, written, (uint32_t)rows, idx, s));
        std::swap(m->anchor, spare_anchor);
        MAP_TRY(launch_densify_children(m->params, m->Pcap, m->M, kept + cloned, split, m->extend_ws, P, n_split, m->cfg.seed, m->dens_calls, s));
        for (size_t q = 0; q < spare_stats.size(); ++q) {  // the statistics move with their rows (and their spares are zero)
            GLIC_CUDA_TRY(cudaMemsetAsync(spare_stats[q].raw(), 0, (size_t)m->Pcap * stats[q].bytes, s));
            MAP_TRY(launch_gather_words(stats[q].buf.raw(), spare_stats[q].raw(), written, kept, idx, s));
            std::swap(stats[q].buf, spare_stats[q]);
        }
        m->P = (uint32_t)rows;
        m->n_sky = r[5];
        m->st.num_gaussians = m->P;
    }
    if (!dry_run) {
        if (densify) MAP_TRY(dens_reset(m));                       // densification_postfix: the statistics start again
        GLIC_CUDA_TRY(cudaStreamSynchronize(s));
        if (densify) ++m->dens_calls;
    }
    if (out) *out = glic_density_counts{n_clone, n_split, (uint32_t)(unpruned - rows), (uint32_t)rows};
    return GLIC_OK;
}

// getNerfppNorm's radius over the training keyframes' camera centres (their device poses under pose refinement), in double
int scene_extent(glic_mapper* m, float* out) {
    const size_t n = m->train.size();
    *out = 0.0f;
    if (n == 0) return GLIC_OK;
    std::vector<double> c(3 * n);
    if (m->pose_on) {
        std::vector<float> f12(12 * n);
        GLIC_CUDA_TRY(cudaStreamSynchronize(m->stream));
        GLIC_CUDA_TRY(cudaMemcpy(f12.data(), m->pose_f, f12.size() * sizeof(float), cudaMemcpyDeviceToHost));
        for (size_t k = 0; k < n; ++k) for (int i = 0; i < 3; ++i) c[3 * k + i] = f12[12 * k + 9 + i];
    } else {
        for (size_t k = 0; k < n; ++k) for (int i = 0; i < 3; ++i) c[3 * k + i] = m->train[k].t_wc[i];
    }
    double mean[3] = {0.0, 0.0, 0.0}, far = 0.0;
    for (size_t k = 0; k < n; ++k) for (int i = 0; i < 3; ++i) mean[i] += c[3 * k + i];
    for (int i = 0; i < 3; ++i) mean[i] /= (double)n;
    for (size_t k = 0; k < n; ++k) {
        const double dx = c[3 * k] - mean[0], dy = c[3 * k + 1] - mean[1], dz = c[3 * k + 2] - mean[2];
        far = std::max(far, std::sqrt(dx * dx + dy * dy + dz * dz));
    }
    *out = (float)(1.1 * far);
    return GLIC_OK;
}

// the schedule's work after the iteration that made stats.iterations = n (glic_mapper_set_density_schedule)
int scheduled_density_step(glic_mapper* m) {
    const glic_density_schedule& c = m->sched;
    const uint64_t n = m->st.iterations;
    if (c.densify_from < n && n < c.densify_until && n % c.densify_interval == 0) {
        float extent = c.scene_extent;
        if (!(extent > 0.0f)) MAP_TRY(scene_extent(m, &extent));
        if (extent > 0.0f) {                                        // one keyframe, or all at one place: no step
            const bool sizes = c.opacity_reset_interval > 0 && n > c.opacity_reset_interval;
            const glic_density_params p{c.grad_threshold, c.percent_dense, extent, c.min_opacity, sizes ? c.screen_radius : 0,
                                        sizes ? c.world_scale_factor * extent : 0.0f};
            glic_density_counts k{};
            MAP_TRY(glic_mapper_densify_and_prune(m, &p, 0, &k));
            m->sched_totals.cloned += k.cloned;
            m->sched_totals.split += k.split;
            m->sched_totals.pruned += k.pruned;
            m->sched_totals.rows = k.rows;
            ++m->sched_steps;
        }
    }
    if (c.opacity_reset_interval > 0 && n < c.densify_until && n % c.opacity_reset_interval == 0) {
        MAP_TRY(glic_mapper_reset_opacity(m, c.reset_opacity));
        ++m->sched_resets;
    }
    return GLIC_OK;
}

// ---- contribution scores (glic_mapper_contribution, glic_mapper_prune_unseen) ------------------------------------------------
// score_ws: hits [Pcap] u64 | ends [Pcap] u64 | max_weight [Pcap] f32
size_t score_bytes(uint32_t cap) { return (size_t)cap * (2 * sizeof(uint64_t) + sizeof(float)); }

// a NULL view list (every training keyframe), or n >= 0 training keyframe indices
int views_check(const glic_mapper* m, const int* views, int n, const char* what) {
    if (n < 0) { set_error(std::string(what) + ": n_views must be >= 0"); return GLIC_ERR_INVALID_ARGUMENT; }
    for (int q = 0; views && q < n; ++q)
        if (views[q] < 0 || views[q] >= (int)m->train.size()) { set_error(std::string(what) + ": view index out of range"); return GLIC_ERR_INVALID_ARGUMENT; }
    return GLIC_OK;
}

// The scores of every row over training keyframes views[0 .. n) (NULL: all of them) into score_ws, which the caller has
// reserved (score_bytes(Pcap)) after draining the ring.  Every row is drawn at the keyframe's current camera block, as training
// draws it; an overflowed view added nothing, so it is redrawn into the same arrays with a larger binning workspace.
int contribution(glic_mapper* m, const int* views, int n) {
    cudaStream_t s = m->stream;
    uint64_t* hits = reinterpret_cast<uint64_t*>(m->score_ws.raw());
    uint64_t* ends = hits + m->Pcap;
    float* max_weight = reinterpret_cast<float*>(hits + 2 * (size_t)m->Pcap);
    GLIC_CUDA_TRY(cudaMemsetAsync(m->score_ws, 0, score_bytes(m->Pcap), s));
    if (!m->P) return GLIC_OK;
    MAP_TRY(activate(m));
    const ArenaRows a = arena_rows(m->params, m->Pcap, m->M);
    const int count = views ? n : (int)m->train.size();
    for (int q = 0; q < count; ++q) {
        const glic_view& v = m->train[views ? views[q] : q].view;
        MAP_TRY(draw_settled(m, [&](long long* cnt) {
            return glic_contribution((int)m->P, a.xyz, m->act_scales, 1.0f, m->act_rots, m->act_opacity, &v, m->radii, m->geom_ws,
                                     m->geom_ws.bytes(), m->image_ws, m->image_ws.bytes(), m->binning_ws, m->binning_ws.bytes(), max_weight,
                                     hits, ends, nullptr, (int64_t*)cnt, s);
        }, [&](int64_t pairs) { return grow_render_binning(m, pairs); }));
        // draw_settled gives up after four draws: a view still overflowing then was not scored, and its rows must not go
        if (m->counters_host[2]) { set_error("mapper_contribution: a view still overflows the binning workspace after regrowing it"); return GLIC_ERR_WORKSPACE; }
    }
    return GLIC_OK;
}

}  // namespace mapper_impl

extern "C" {

int glic_mapper_contribution(glic_mapper* m, const int* views_host, int n_views, float* max_weight, uint64_t* hits, uint64_t* ends) {
    if (!m || (!max_weight && !hits && !ends)) { set_error("mapper_contribution: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    MAP_TRY(views_check(m, views_host, n_views, "mapper_contribution"));
    MAP_TRY(poll_ring(m, true));
    MAP_TRY(reserve(m, m->score_ws, score_bytes(m->Pcap)));
    MAP_TRY(contribution(m, views_host, n_views));
    const uint64_t* h = reinterpret_cast<const uint64_t*>(m->score_ws.raw());
    if (m->P && hits) GLIC_CUDA_TRY(cudaMemcpyAsync(hits, h, sizeof(uint64_t) * m->P, cudaMemcpyDefault, m->stream));
    if (m->P && ends) GLIC_CUDA_TRY(cudaMemcpyAsync(ends, h + m->Pcap, sizeof(uint64_t) * m->P, cudaMemcpyDefault, m->stream));
    if (m->P && max_weight) GLIC_CUDA_TRY(cudaMemcpyAsync(max_weight, h + 2 * (size_t)m->Pcap, sizeof(float) * m->P, cudaMemcpyDefault, m->stream));
    GLIC_CUDA_TRY(cudaStreamSynchronize(m->stream));
    return GLIC_OK;
}

// the scores, then the compaction with no row selected, both size tests and the opacity test off, and the unseen test on
int glic_mapper_prune_unseen(glic_mapper* m, const glic_unseen_params* p, int dry_run, uint32_t* removed) {
    if (!m || !p) { set_error("mapper_prune_unseen: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (!std::isfinite(p->min_weight) || p->min_weight < 0.0f || p->min_weight > 1.0f) {
        set_error("mapper_prune_unseen: min_weight must be finite and in [0, 1]"); return GLIC_ERR_INVALID_ARGUMENT;
    }
    if (p->sky != 0 && p->sky != 1) { set_error("mapper_prune_unseen: sky must be 0 or 1"); return GLIC_ERR_INVALID_ARGUMENT; }
    MAP_TRY(views_check(m, p->views, p->n_views, "mapper_prune_unseen"));
    if (m->P) {
        MAP_TRY(poll_ring(m, true));
        MAP_TRY(reserve(m, m->score_ws, score_bytes(m->Pcap)));
        MAP_TRY(reserve(m, m->extend_ws, density_scratch_bytes(m->P)));      // the selection's scratch (density_step)
        MAP_TRY(contribution(m, p->views, p->n_views));
    }
    glic_density_counts k{};
    MAP_TRY(density_step(m, glic_density_params{0.0f, 0.0f, 0.0f, 0.0f, 0, 0.0f}, false, dry_run, m->P != 0, &k, "mapper_prune_unseen", p));
    if (removed) *removed = k.pruned;
    return GLIC_OK;
}

// the compaction with no row selected and both size tests off; a mapper with no rows has nothing to remove (0, not an error)
int glic_mapper_prune(glic_mapper* m, float min_opacity, int dry_run, uint32_t* removed) {
    if (!m) { set_error("mapper_prune: null mapper"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (!std::isfinite(min_opacity) || min_opacity < 0.0f || min_opacity > 1.0f) {
        set_error("mapper_prune: min_opacity must be finite and in [0, 1]"); return GLIC_ERR_INVALID_ARGUMENT;
    }
    glic_density_counts k{};
    MAP_TRY(density_step(m, glic_density_params{0.0f, 0.0f, 0.0f, min_opacity, 0, 0.0f}, false, dry_run, m->P != 0, &k, "mapper_prune"));
    if (removed) *removed = k.pruned;
    return GLIC_OK;
}

int glic_mapper_densify(glic_mapper* m, float grad_threshold, float percent_dense, float scene_extent, int dry_run, uint32_t* cloned,
                        uint32_t* split) {
    if (!m) { set_error("mapper_densify: null mapper"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (!m->dens_on) { set_error("mapper_densify: densification is not enabled (glic_mapper_enable_densification)"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (!finite_at_least_zero(grad_threshold) || !finite_at_least_zero(percent_dense) || !std::isfinite(scene_extent) || !(scene_extent > 0.0f)) {
        set_error("mapper_densify: grad_threshold and percent_dense must be finite and >= 0, scene_extent finite and > 0");
        return GLIC_ERR_INVALID_ARGUMENT;
    }
    glic_density_counts k{};
    MAP_TRY(density_step(m, glic_density_params{grad_threshold, percent_dense, scene_extent, 0.0f, 0, 0.0f}, true, dry_run, false, &k, "mapper_densify"));
    if (cloned) *cloned = k.cloned;
    if (split) *split = k.split;
    return GLIC_OK;
}

int glic_mapper_densify_and_prune(glic_mapper* m, const glic_density_params* p, int dry_run, glic_density_counts* out) {
    if (!m || !p) { set_error("mapper_densify_and_prune: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (!m->dens_on) { set_error("mapper_densify_and_prune: densification is not enabled (glic_mapper_enable_densification)"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (!finite_at_least_zero(p->grad_threshold) || !finite_at_least_zero(p->percent_dense) || !std::isfinite(p->scene_extent) ||
        !(p->scene_extent > 0.0f) || !finite_at_least_zero(p->min_opacity) || p->min_opacity > 1.0f || p->max_screen_radius < 0 ||
        !finite_at_least_zero(p->max_world_scale)) {
        set_error("mapper_densify_and_prune: grad_threshold, percent_dense and max_world_scale must be finite and >= 0, scene_extent finite "
                  "and > 0, min_opacity in [0, 1], max_screen_radius >= 0");
        return GLIC_ERR_INVALID_ARGUMENT;
    }
    return density_step(m, *p, true, dry_run, true, out, "mapper_densify_and_prune");
}

int glic_mapper_screen_radii(glic_mapper* m, int32_t* out) {
    if (!m || !out) { set_error("mapper_screen_radii: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (!m->dens_on) { set_error("mapper_screen_radii: densification is not enabled (glic_mapper_enable_densification)"); return GLIC_ERR_INVALID_ARGUMENT; }
    GLIC_CUDA_TRY(cudaStreamSynchronize(m->stream));
    if (m->P) GLIC_CUDA_TRY(cudaMemcpy(out, m->dens_maxr, (size_t)m->P * 4, cudaMemcpyDeviceToHost));
    return GLIC_OK;
}

// Inria's reset_opacity on the non-sky rows: one kernel (prune.cu) after the pipeline drains
int glic_mapper_reset_opacity(glic_mapper* m, float max_opacity) {
    if (!m) { set_error("mapper_reset_opacity: null mapper"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (!std::isfinite(max_opacity) || !(max_opacity > 0.0f) || !(max_opacity < 1.0f)) {
        set_error("mapper_reset_opacity: max_opacity must be finite and in (0, 1)"); return GLIC_ERR_INVALID_ARGUMENT;
    }
    GLIC_CUDA_TRY(cudaStreamSynchronize(m->stream));
    MAP_TRY(poll_ring(m, true));
    const double r = (double)max_opacity;
    MAP_TRY(launch_reset_opacity(m->n_sky, m->P, m->Pcap, m->M, m->params, m->m1, m->m2, max_opacity, (float)std::log(r / (1.0 - r)), m->stream));
    GLIC_CUDA_TRY(cudaStreamSynchronize(m->stream));
    return GLIC_OK;
}

int glic_mapper_set_density_schedule(glic_mapper* m, const glic_density_schedule* c) {
    if (!m) { set_error("mapper_set_density_schedule: null mapper"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (c) {
        if (!m->dens_on) { set_error("mapper_set_density_schedule: densification is not enabled (glic_mapper_enable_densification)"); return GLIC_ERR_INVALID_ARGUMENT; }
        if (c->densify_interval == 0 || !finite_at_least_zero(c->grad_threshold) || !finite_at_least_zero(c->percent_dense) ||
            !finite_at_least_zero(c->min_opacity) || c->min_opacity > 1.0f || !std::isfinite(c->reset_opacity) || !(c->reset_opacity > 0.0f) ||
            !(c->reset_opacity < 1.0f) || c->screen_radius < 0 || !finite_at_least_zero(c->world_scale_factor) || !finite_at_least_zero(c->scene_extent)) {
            set_error("mapper_set_density_schedule: densify_interval must be >= 1, grad_threshold, percent_dense, world_scale_factor and "
                      "scene_extent finite and >= 0, min_opacity in [0, 1], reset_opacity in (0, 1), screen_radius >= 0");
            return GLIC_ERR_INVALID_ARGUMENT;
        }
        m->sched = *c;
    }
    m->sched_on = c != nullptr;
    m->sched_totals = glic_density_counts{};
    m->sched_steps = m->sched_resets = 0;
    return GLIC_OK;
}

int glic_mapper_scene_extent(glic_mapper* m, float* out) {
    if (!m || !out) { set_error("mapper_scene_extent: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    return scene_extent(m, out);
}

int glic_mapper_density_totals(glic_mapper* m, glic_density_counts* out, uint32_t* steps, uint32_t* resets) {
    if (!m) { set_error("mapper_density_totals: null mapper"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (out) *out = m->sched_totals;
    if (steps) *steps = m->sched_steps;
    if (resets) *resets = m->sched_resets;
    return GLIC_OK;
}

int glic_mapper_densify_stats(glic_mapper* m, float* grad_accum, float* denom) {
    if (!m || !grad_accum || !denom) { set_error("mapper_densify_stats: null pointer"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (!m->dens_on) { set_error("mapper_densify_stats: densification is not enabled (glic_mapper_enable_densification)"); return GLIC_ERR_INVALID_ARGUMENT; }
    GLIC_CUDA_TRY(cudaStreamSynchronize(m->stream));
    if (!m->P) return GLIC_OK;
    GLIC_CUDA_TRY(cudaMemcpy(grad_accum, m->dens_accum, (size_t)m->P * 4, cudaMemcpyDeviceToHost));
    GLIC_CUDA_TRY(cudaMemcpy(denom, m->dens_denom, (size_t)m->P * 4, cudaMemcpyDeviceToHost));
    return GLIC_OK;
}

int glic_mapper_enable_densification(glic_mapper* m) {
    if (!m) { set_error("mapper_enable_densification: null mapper"); return GLIC_ERR_INVALID_ARGUMENT; }
    if (m->dens_on) return GLIC_OK;
    if (m->cfg.world > 1 && (m->exported || m->connected)) {
        set_error("mapper_enable_densification: with world > 1 it must come before glic_mapper_export (the exchange block grows)");
        return GLIC_ERR_INVALID_ARGUMENT;
    }
    GLIC_CUDA_TRY(cudaStreamSynchronize(m->stream));
    MAP_TRY(poll_ring(m, true));
    // the exchange block gains the two statistics rows and the radius slots; every new buffer starts zeroed
    const XLayout x = xblock_layout(m->S, m->Pcap, true);
    std::vector<Grow> list = {{m->xblock, x.bytes, 0, true}};
    grow_rows(list, densification_rows(m), m->Pcap, 0, true);
    MAP_TRY(grow(m, list));
    adopt_capacity(m, m->Pcap, x);
    m->dens_on = true;
    return GLIC_OK;
}

}  // extern "C"
