// Host-buffer frame calls of the DiMP hot path (what bench.py's `e2e` leg times) and the per-sequence device
// state they operate on: sample memory, boxes, sample weights, the target filter, staging for crops and scores.
//   localize: DiMP.track lines pytracking/tracker/dimp/dimp.py:103-117 (extract_backbone_features,
//             get_classification_features, classify_target, max2d of localize_target)
//   update:   DiMP.update_classifier pytracking/tracker/dimp/dimp.py:605-648 (update_memory + filter_optimizer)
#include "dimp_state.cuh"


using namespace b200trk;

// The buffers both optimiser kinds share (and the GN LUTs when num_bins > 0); frees `s` on failure.  filter_ext: see dimp_state.cuh.
static int state_alloc(b200trk_dimp_state* s, b200trk_net* net, int memory_size, int filter_size, const float* label_lut,
                       const float* mask_lut, const float* spatial_lut, int num_bins, float* filter_ext) {
    s->net = net; s->memory_size = memory_size; s->ksz = filter_size; s->max_batch = net->max_batch;
    s->Cc = net->dims[6]; s->Hc = net->dims[7]; s->Wc = net->dims[8];
    s->Ho = s->Hc + (filter_size + 1) % 2; s->Wo = s->Wc + (filter_size + 1) % 2;
    s->num_bins = num_bins;
    const size_t plane = (size_t)s->Cc * s->Hc * s->Wc;
    int e = 0;
    if (filter_ext) s->filter = filter_ext;
    else if (!e) e = s->mem.alloc(&s->filter, (size_t)s->Cc * 16, true);
    s->mem_pitch = (s->Hc * s->Wc + 31) / 32 * 32;
    if (!e) e = s->mem.alloc(&s->memory, (size_t)s->Cc * s->mem_pitch * memory_size, true);
    if (!e) e = s->mem.alloc(&s->boxes, (size_t)memory_size * 4, true);
    if (!e) e = s->mem.alloc(&s->sw, (size_t)memory_size, true);
    if (!filter_ext) {
        if (!e) e = s->mem.alloc(&s->clf, plane * s->max_batch, true);
        if (!e) e = s->mem.alloc(&s->scores, (size_t)s->max_batch * s->Ho * s->Wo, true);
        if (!e) e = s->mem.alloc(&s->crop, (size_t)s->max_batch * 3 * net->crop_h * net->crop_w, true);
        if (!e) e = s->mem.alloc(&s->maxval, (size_t)s->max_batch, true);
        if (!e) e = s->mem.alloc(&s->maxidx, (size_t)s->max_batch * 2, true);
    }
    if (!e && num_bins > 0) e = s->mem.alloc(&s->luts, (size_t)3 * num_bins, true);
    if (!e && num_bins > 0) {
        cudaError_t ce = cudaMemcpy(s->luts, label_lut, num_bins * sizeof(float), cudaMemcpyHostToDevice);
        if (ce == cudaSuccess) ce = cudaMemcpy(s->luts + num_bins, mask_lut, num_bins * sizeof(float), cudaMemcpyHostToDevice);
        if (ce == cudaSuccess) ce = cudaMemcpy(s->luts + 2 * num_bins, spatial_lut, num_bins * sizeof(float), cudaMemcpyHostToDevice);
        if (ce != cudaSuccess) { set_error("dimp_state_create: LUT upload failed: %s", cudaGetErrorString(ce)); e = 1; }
    }
    for (int i = 0; i < b200trk_dimp_state::NSTAGE && !e; ++i) {
        e = s->mem.pinned(&s->stage[i], (size_t)4 + memory_size);
        if (!e) e = s->mem.event(&s->stage_ev[i], cudaEventDisableTiming);
    }
    if (e) delete s;
    return e;
}

int b200trk::dimp_state_create_gn(b200trk_dimp_state** out, b200trk_net* net, int memory_size, int filter_size, const float* label_lut,
                                  const float* mask_lut, const float* spatial_lut, int num_bins, float bin_displacement, float feat_stride,
                                  float step_length, float reg_weight, float alpha_eps, float* filter_ext) {
    B200_REQUIRE(out && net && label_lut && mask_lut && spatial_lut, "dimp_state_create: null pointer");
    B200_REQUIRE(memory_size >= 1 && memory_size <= 1024, "dimp_state_create: memory_size=%d", memory_size);
    B200_REQUIRE(filter_size == 4, "dimp_state_create: filter_size=%d not supported (4)", filter_size);
    B200_REQUIRE(num_bins >= 2 && num_bins <= 4096, "dimp_state_create: num_bins=%d", num_bins);
    b200trk_dimp_state* s = new b200trk_dimp_state();
    s->opt_kind = b200trk_dimp_state::OPT_GN;
    s->bin_displacement = bin_displacement; s->feat_stride = feat_stride;
    s->step_length = step_length; s->reg_weight = reg_weight; s->alpha_eps = alpha_eps;
    if (int e = state_alloc(s, net, memory_size, filter_size, label_lut, mask_lut, spatial_lut, num_bins, filter_ext)) return e;
    *out = s;
    return 0;
}

extern "C" int b200trk_dimp_state_create(b200trk_dimp_state_t** out, b200trk_net_t* net, int memory_size, int filter_size,
                                         const float* label_lut, const float* mask_lut, const float* spatial_lut,
                                         int num_bins, float bin_displacement, float feat_stride, float step_length,
                                         float reg_weight, float alpha_eps) {
    return dimp_state_create_gn(out, net, memory_size, filter_size, label_lut, mask_lut, spatial_lut, num_bins, bin_displacement,
                                feat_stride, step_length, reg_weight, alpha_eps, nullptr);
}

int b200trk::dimp_state_create_newton(b200trk_dimp_state** out, b200trk_net* net, int memory_size, int filter_size, float gauss_sigma,
                                      float feat_stride, float step_length, float reg_weight, float alpha_eps, int has_softmax_reg,
                                      float softmax_reg, float label_threshold, int normalize_label, float label_shrink, float uni_weight,
                                      float* filter_ext) {
    B200_REQUIRE(out && net, "prdimp_state_create: null pointer");
    B200_REQUIRE(memory_size >= 1 && memory_size <= 1024, "prdimp_state_create: memory_size=%d", memory_size);
    B200_REQUIRE(filter_size == 4, "prdimp_state_create: filter_size=%d not supported (4)", filter_size);
    B200_REQUIRE(gauss_sigma > 0.f && feat_stride > 0.f, "prdimp_state_create: gauss_sigma=%g and feat_stride=%g must be positive",
                 gauss_sigma, feat_stride);
    b200trk_dimp_state* s = new b200trk_dimp_state();
    s->opt_kind = b200trk_dimp_state::OPT_NEWTON;
    s->feat_stride = feat_stride; s->step_length = step_length; s->reg_weight = reg_weight; s->alpha_eps = alpha_eps;
    s->gauss_sigma = gauss_sigma; s->has_softmax_reg = has_softmax_reg ? 1 : 0; s->softmax_reg = softmax_reg;
    s->label_threshold = label_threshold; s->normalize_label = normalize_label ? 1 : 0; s->label_shrink = label_shrink;
    s->uni_weight = uni_weight;
    if (int e = state_alloc(s, net, memory_size, filter_size, nullptr, nullptr, nullptr, 0, filter_ext)) return e;
    *out = s;
    return 0;
}

extern "C" int b200trk_prdimp_state_create(b200trk_dimp_state_t** out, b200trk_net_t* net, int memory_size, int filter_size,
                                           float gauss_sigma, float feat_stride, float step_length, float reg_weight, float alpha_eps,
                                           int has_softmax_reg, float softmax_reg, float label_threshold, int normalize_label,
                                           float label_shrink, float uni_weight) {
    return dimp_state_create_newton(out, net, memory_size, filter_size, gauss_sigma, feat_stride, step_length, reg_weight, alpha_eps,
                                    has_softmax_reg, softmax_reg, label_threshold, normalize_label, label_shrink, uni_weight, nullptr);
}

extern "C" int b200trk_dimp_state_optimizer_kind(b200trk_dimp_state_t* s) { return s ? s->opt_kind : -1; }

extern "C" int b200trk_dimp_state_destroy(b200trk_dimp_state_t* s) {
    delete s;
    return 0;
}

extern "C" float* b200trk_dimp_state_filter(b200trk_dimp_state_t* s) { return s ? s->filter : nullptr; }
extern "C" float* b200trk_dimp_state_memory(b200trk_dimp_state_t* s) { return s ? s->memory : nullptr; }
extern "C" int b200trk_dimp_state_memory_pitch(b200trk_dimp_state_t* s) { return s ? s->mem_pitch : 0; }
extern "C" float* b200trk_dimp_state_boxes(b200trk_dimp_state_t* s) { return s ? s->boxes : nullptr; }
extern "C" float* b200trk_dimp_state_sample_weights(b200trk_dimp_state_t* s) { return s ? s->sw : nullptr; }
extern "C" float* b200trk_dimp_state_clf(b200trk_dimp_state_t* s) { return s ? s->clf : nullptr; }
extern "C" float* b200trk_dimp_state_scores(b200trk_dimp_state_t* s) { return s ? s->scores : nullptr; }

extern "C" int b200trk_dimp_localize_host(b200trk_dimp_state_t* s, const float* crop_host, int S, float* scores_host,
                                          float* max_val_host, int64_t* max_idx_host, b200trk_stream_t stream) {
    B200_REQUIRE(s && crop_host && scores_host && max_val_host && max_idx_host, "dimp_localize_host: null pointer");
    B200_REQUIRE(S >= 1 && S <= s->max_batch, "dimp_localize_host: S=%d outside [1,%d]", S, s->max_batch);
    cudaStream_t st = (cudaStream_t)stream;
    const size_t crop_bytes = (size_t)S * 3 * s->net->crop_h * s->net->crop_w * sizeof(float);
    B200_CHECK_CUDA(cudaMemcpyAsync(s->crop, crop_host, crop_bytes, cudaMemcpyHostToDevice, st));
    if (int e = b200trk_net_forward(s->net, s->crop, S, nullptr, nullptr, s->clf, stream)) return e;
    if (int e = b200trk_apply_filter(s->clf, s->filter, s->scores, S, s->Cc, s->Hc, s->Wc, s->ksz, s->maxval, s->maxidx, stream)) return e;
    B200_CHECK_CUDA(cudaMemcpyAsync(scores_host, s->scores, (size_t)S * s->Ho * s->Wo * sizeof(float), cudaMemcpyDeviceToHost, st));
    B200_CHECK_CUDA(cudaMemcpyAsync(max_val_host, s->maxval, (size_t)S * sizeof(float), cudaMemcpyDeviceToHost, st));
    B200_CHECK_CUDA(cudaMemcpyAsync(max_idx_host, s->maxidx, (size_t)S * 2 * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    B200_CHECK_CUDA(cudaStreamSynchronize(st));
    return 0;
}

int b200trk::dimp_state_insert(b200trk_dimp_state* s, const float* feat, int replace_ind, const float* target_box_host,
                               const float* sample_weights_host, int n_stored, int num_iter, cudaStream_t st) {
    B200_REQUIRE(s && feat && target_box_host && sample_weights_host, "dimp_update: null pointer");
    B200_REQUIRE(replace_ind >= 0 && replace_ind < s->memory_size, "dimp_update: replace_ind=%d outside memory of %d", replace_ind, s->memory_size);
    B200_REQUIRE(n_stored >= 1 && n_stored <= s->memory_size, "dimp_update: n_stored=%d", n_stored);
    const size_t row = (size_t)s->Hc * s->Wc * sizeof(float);
    // the caller may rewrite its buffers as soon as this returns: stage the 4 + n floats in a pinned slot of our own
    const int slot = s->stage_next;
    s->stage_next = (slot + 1) % b200trk_dimp_state::NSTAGE;
    B200_CHECK_CUDA(cudaEventSynchronize(s->stage_ev[slot]));
    float* h = s->stage[slot];
    for (int i = 0; i < 4; ++i) h[i] = target_box_host[i];
    for (int i = 0; i < n_stored; ++i) h[4 + i] = sample_weights_host[i];
    B200_CHECK_CUDA(cudaMemcpy2DAsync(s->memory + (size_t)s->Cc * s->mem_pitch * replace_ind, (size_t)s->mem_pitch * sizeof(float),
                                      feat, row, row, (size_t)s->Cc, cudaMemcpyDeviceToDevice, st));
    B200_CHECK_CUDA(cudaMemcpyAsync(s->boxes + 4 * replace_ind, h, 4 * sizeof(float), cudaMemcpyHostToDevice, st));
    B200_CHECK_CUDA(cudaMemcpyAsync(s->sw, h + 4, (size_t)n_stored * sizeof(float), cudaMemcpyHostToDevice, st));
    B200_CHECK_CUDA(cudaEventRecord(s->stage_ev[slot], st));
    if (num_iter > 0) return dimp_state_optimize(s, n_stored, num_iter, st);
    return 0;
}

int b200trk::dimp_state_optimize(b200trk_dimp_state* s, int n_stored, int num_iter, cudaStream_t st) {
    if (s->opt_kind == b200trk_dimp_state::OPT_NEWTON)
        return prdimp_sd_newton_pitched(s->filter, s->filter, s->memory, s->mem_pitch, s->boxes, s->sw, n_stored, s->Cc, s->Hc, s->Wc, s->ksz,
                                        num_iter, s->gauss_sigma, s->feat_stride, s->step_length, s->reg_weight, s->alpha_eps,
                                        s->has_softmax_reg, s->softmax_reg, s->label_threshold, s->normalize_label, s->label_shrink,
                                        s->uni_weight, nullptr, nullptr, st);
    return dimp_sd_gn_pitched(s->filter, s->filter, s->memory, s->mem_pitch, s->boxes, s->sw, n_stored, s->Cc, s->Hc, s->Wc, s->ksz,
                              num_iter, s->luts, s->luts + s->num_bins, s->luts + 2 * s->num_bins, s->num_bins,
                              s->bin_displacement, s->feat_stride, s->step_length, s->reg_weight, s->alpha_eps,
                              nullptr, nullptr, st);
}

// Device half of DiMP.update_classifier for the features of crop scale_ind of the last localize call
extern "C" int b200trk_dimp_update_host(b200trk_dimp_state_t* s, int scale_ind, int replace_ind, const float* target_box_host,
                                        const float* sample_weights_host, int n_stored, int num_iter, b200trk_stream_t stream) {
    B200_REQUIRE(s && target_box_host && sample_weights_host, "dimp_update: null pointer");
    B200_REQUIRE(s->clf, "dimp_update: the state is a slot of a batch; its features are in the batch's buffer");
    B200_REQUIRE(scale_ind >= 0 && scale_ind < s->max_batch, "dimp_update: scale_ind=%d", scale_ind);
    return dimp_state_insert(s, s->clf + (size_t)s->Cc * s->Hc * s->Wc * scale_ind, replace_ind, target_box_host, sample_weights_host,
                             n_stored, num_iter, (cudaStream_t)stream);
}
