// Per-sequence device state of the DiMP online model (shared by dimp_state.cu and dimp_tracker.cu).
#pragma once
#include "net.cuh"
#include "sd_common.cuh"
#include <vector>

struct b200trk_dimp_state {
    b200trk_net* net = nullptr;
    int memory_size = 0, ksz = 4, Cc = 0, Hc = 0, Wc = 0, Ho = 0, Wo = 0, num_bins = 0, max_batch = 1;
    int mem_pitch = 0;      // floats between two channel planes of the sample memory: H*W rounded up to 32, so that every 32-pixel
                            // TMA row of the optimiser is one 128-byte L2 line instead of straddling two
    float bin_displacement = 0.1f, feat_stride = 16.f, step_length = 1.f, reg_weight = 0.01f, alpha_eps = 0.f;
    // which online optimiser updates the filter: DiMPSteepestDescentGN over the three LUTs (DiMP) or
    // PrDiMPSteepestDescentNewton with the Gaussian-label hyper-parameters below (PrDiMP; no LUTs)
    enum OptKind { OPT_GN = 0, OPT_NEWTON = 1 };
    int opt_kind = OPT_GN;
    float gauss_sigma = 0.f, softmax_reg = 0.f, label_threshold = 0.f, label_shrink = 0.f, uni_weight = 0.f;
    int has_softmax_reg = 0, normalize_label = 0;
    float *filter = nullptr, *memory = nullptr, *boxes = nullptr, *sw = nullptr, *clf = nullptr, *scores = nullptr;
    float *crop = nullptr, *maxval = nullptr, *luts = nullptr;
    int64_t* maxidx = nullptr;
    std::vector<void*> owned;
    // pinned staging ring for the small per-update H2D payload (box + sample weights): a slot is rewritten only after the copy
    // that read it has completed (its event), so back-to-back asynchronous update calls never race with their own uploads
    static constexpr int NSTAGE = 4;
    float* stage[NSTAGE] = {nullptr, nullptr, nullptr, nullptr};
    cudaEvent_t stage_ev[NSTAGE] = {nullptr, nullptr, nullptr, nullptr};
    int stage_next = 0;
};

namespace b200trk {
// The two state constructors behind b200trk_dimp_state_create / b200trk_prdimp_state_create.  filter_ext = NULL: the state owns its
// filter and the crop / feature / score buffers of net->max_batch samples.  Otherwise it is one sequence of a batch (dimp_tracker.cu):
// the filter lives at filter_ext inside the batch's [S,C,k,k] buffer and the batch owns the per-frame buffers (clf, crop, scores stay NULL).
int dimp_state_create_gn(b200trk_dimp_state** out, b200trk_net* net, int memory_size, int filter_size, const float* label_lut,
                         const float* mask_lut, const float* spatial_lut, int num_bins, float bin_displacement, float feat_stride,
                         float step_length, float reg_weight, float alpha_eps, float* filter_ext);
int dimp_state_create_newton(b200trk_dimp_state** out, b200trk_net* net, int memory_size, int filter_size, float gauss_sigma,
                             float feat_stride, float step_length, float reg_weight, float alpha_eps, int has_softmax_reg,
                             float softmax_reg, float label_threshold, int normalize_label, float label_shrink, float uni_weight,
                             float* filter_ext);
// The memory update of DiMP.update_classifier: the sample `feat` (device [C,H,W]) with its box goes to memory slot replace_ind, the
// first n_stored sample weights are replaced, then num_iter optimiser iterations run (none for num_iter <= 0)
int dimp_state_insert(b200trk_dimp_state* s, const float* feat, int replace_ind, const float* target_box_host,
                      const float* sample_weights_host, int n_stored, int num_iter, cudaStream_t st);
// num_iter iterations of the state's online optimiser over the first n_stored samples of its pitched memory, filter in place
int dimp_state_optimize(b200trk_dimp_state* s, int n_stored, int num_iter, cudaStream_t st);
}
