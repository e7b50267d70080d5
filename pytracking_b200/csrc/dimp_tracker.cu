// Whole-frame DiMP tracking: uint8 frame in, bounding box out (DiMP.track, pytracking/tracker/dimp/dimp.py:94-175).
//
//   host  plan_crop   get_centered_sample_pos (dimp.py:184-188) + the geometry half of sample_patch
//                     (pytracking/features/preprocessing.py:55-148) + get_sample_location (dimp.py:177-182)
//   device            sample_patch_kernel (decimate + replicate pad + bilinear resize, bit-exact with torch-CPU F.interpolate),
//                     backbone + head + classify (net.cu, corr_api.cu), localize_kernel (dimp.py:196-303)
//   host  commit      translation, update_state (dimp.py:486-497), get_iounet_box (:500-507), update_sample_weights (:445-484),
//                     the iteration schedule of update_classifier (:605-625), the output box (:163-171)
//   device            memory insert + steepest-descent update (dimp_state.cu)
//
// The tracker's scalars live on the host as float32 and every expression below performs the float32 operation sequence torch
// executes for the reference's tensor expression (scalars multiplying a float32 tensor are first rounded to float32; `x / tensor`
// is `tensor.reciprocal() * x`, torch/_tensor.py __rdiv__; integer tensors divided by Python ints become float32; torch.round and
// Python round are round-half-even).  The file is compiled with -fmad=false / -ffp-contract=off: no fused multiply-adds except
// the explicit ones of the resampling kernel.
#include "dimp_state.cuh"
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <limits>

using namespace b200trk;

#include "dimp_tracker_kernels.cuh"      // sample_patch_kernel, localize_kernel, LocArgs (anonymous namespace)

namespace {

inline float f32(double x) { return (float)x; }

// Host frames go up on a copy stream of their own: the previous frame's steepest-descent update may still be running on the caller's
// stream (a frame call returns as soon as the box is known).  The device buffer is free to overwrite: the previous crop kernel finished
// before the previous call returned, which synchronised on its localisation result.
struct FrameUpload {
    uint8_t* dev = nullptr; size_t cap = 0;
    cudaStream_t stream = nullptr; cudaEvent_t ev = nullptr;

    ~FrameUpload() {
        if (dev) cudaFree(dev);
        if (stream) cudaStreamDestroy(stream);
        if (ev) cudaEventDestroy(ev);
    }

    // Copies the n uint8 [H[k],W[k],3] host frames im[k] to 256-byte-aligned offsets of `dev`, replaces each im[k] by its device copy
    // and makes `st` wait for the copies.
    int upload(int n, const uint8_t* im[], const int H[], const int W[], cudaStream_t st) {
        size_t off[kBatchMax], total = 0;
        for (int k = 0; k < n; ++k) { off[k] = total; total += ((size_t)H[k] * W[k] * 3 + 255) / 256 * 256; }
        if (total > cap) {
            if (dev) B200_CHECK_CUDA(cudaFree(dev));
            dev = nullptr; cap = 0;
            B200_CHECK_CUDA(cudaMalloc((void**)&dev, total));
            cap = total;
        }
        if (!stream) {
            B200_CHECK_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
            B200_CHECK_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
        }
        for (int k = 0; k < n; ++k) {
            B200_CHECK_CUDA(cudaMemcpyAsync(dev + off[k], im[k], (size_t)H[k] * W[k] * 3, cudaMemcpyHostToDevice, stream));
            im[k] = dev + off[k];
        }
        B200_CHECK_CUDA(cudaEventRecord(ev, stream));
        B200_CHECK_CUDA(cudaStreamWaitEvent(st, ev, 0));
        return 0;
    }
};

}  // namespace

// ---------------------------------------------------------------------------------------------------------------------------
// host state
// ---------------------------------------------------------------------------------------------------------------------------
struct b200trk_dimp_tracker {
    b200trk_dimp_state* st = nullptr;
    b200trk_dimp_params_t p;
    // DiMP scalars (float32 tensors in the reference), [0] = row / height, [1] = column / width
    float pos[2] = {0, 0}, target_sz[2] = {0, 0}, base_target_sz[2] = {0, 0}, image_sz[2] = {0, 0};
    float img_sample_sz[2] = {0, 0}, feature_sz[2] = {18, 18}, kernel_size[2] = {4, 4}, score_sz[2] = {19, 19};
    float target_scale = 1.f, min_scale_factor = 0.f, max_scale_factor = 0.f;
    int frame_num = 0, initialized = 0;
    // memory bookkeeping (dimp.py:410-484)
    std::vector<float> sw;
    long num_stored = 0; int num_init = 0, prev_replace_ind = -1;
    // IoUNet refinement (dimp.py:650-723)
    b200trk_iou_predictor_t* iou_pred = nullptr;
    float *mod3 = nullptr, *mod4 = nullptr, *iou3 = nullptr, *iou4 = nullptr, *boxes_dev = nullptr;   // device
    float* boxes_host = nullptr;                     // pinned: [16][4] boxes + [16] IoUs
    b200trk_iou_modulation_t* mod_head = nullptr;    // get_modulation; with mod_native, initialize computes mod3 / mod4
    int mod_native = 0;
    int iou_dims[6] = {0, 0, 0, 0, 0, 0};
    float pos_iounet[2] = {0, 0}; int has_pos_iounet = 0;
    std::vector<float> noise;                        // uniform numbers for the next frame's random proposals
    uint64_t rng = 0x9E3779B97F4A7C15ull;
    // device side (a batch slot uses the batch's frames and results instead)
    FrameUpload frames;
    b200trk_loc_result_t* loc_dev = nullptr;
    b200trk_loc_result_t* loc_host = nullptr;      // pinned
    // augmented initialisation (allocated by its first call): launch table, dropout multipliers, expanded patch
    void* aug_table = nullptr;
    float *aug_mult = nullptr, *aug_patch = nullptr;
    size_t aug_patch_cap = 0;
};

// torch's floor division of float32 tensors (aten/src/ATen/native/BinaryOps.h div_floor_floating) for a divisor b > 0
static float floor_div_f32(float a, float b) {
    const float mod = std::fmod(a, b);
    float div = (a - mod) / b;
    if (mod != 0.f && (mod < 0.f)) div -= 1.0f;
    if (div == 0.f) return std::copysign(0.f, a / b);
    float fl = std::floor(div);
    if (div - fl > 0.5f) fl += 1.0f;
    return fl;
}

// sample_patch geometry (preprocessing.py:55-148). border_mode 0 'replicate'; 1 'inside' / 2 'inside_major' (preprocessing.py:76-86,
// 112-122): the sample shrinks by the larger / smaller of its two size ratios to the image, clamped to [1, max_scale_change]
// (max_scale_change <= 0: no upper bound), and is shifted inside the image -- or centred on it when it is larger. Padding stays
// 'replicate' in every mode.
static void plan_patch(const float pos[2], const float sample_sz_in[2], const float output_sz[2], int H, int W, int border_mode,
                       double max_scale_change, b200trk_crop_geom_t* g) {
    long posl[2] = {(long)std::trunc(pos[0]), (long)std::trunc(pos[1])};                       // pos.long()
    float sample_sz[2] = {sample_sz_in[0], sample_sz_in[1]};
    const bool inside = border_mode == 1 || border_mode == 2;
    if (inside) {
        const float im_sz[2] = {(float)H, (float)W};                                           // torch.Tensor([H, W]): float32
        const float s0 = sample_sz[0] / im_sz[0], s1 = sample_sz[1] / im_sz[1];
        float shrink = border_mode == 1 ? std::fmax(s0, s1) : std::fmin(s0, s1);               // .max() / .min()
        shrink = std::fmax(shrink, 1.0f);                                                      // clamp_(min=1, max=...)
        if (max_scale_change > 0.0) shrink = std::fmin(shrink, f32(max_scale_change));
        for (int i = 0; i < 2; ++i) sample_sz[i] = (float)(long)std::trunc(sample_sz[i] / shrink);   // (sample_sz / shrink).long()
    }
    const float rf = std::fmin(sample_sz[0] / output_sz[0], sample_sz[1] / output_sz[1]);      // torch.min(sample_sz / output_sz).item()
    int df = (int)std::trunc((double)rf - 0.1);                                                // int(resize_factor - 0.1)
    if (df < 1) df = 1;
    float sz[2] = {sample_sz[0] / (float)df, sample_sz[1] / (float)df};
    float poslf[2];
    int os[2] = {0, 0};
    for (int i = 0; i < 2; ++i) {
        if (df > 1) {
            long m = posl[i] % df; if (m < 0) m += df;                                         // torch remainder: sign of the divisor
            os[i] = (int)m;
            poslf[i] = (float)(posl[i] - m) / (float)df;                                       // (posl - os) / df: float32 tensor
        } else {
            poslf[i] = (float)posl[i];
        }
    }
    float tl[2], br[2]; int tli[2], bri[2];
    for (int i = 0; i < 2; ++i) {
        const long szl = (long)std::fmax(std::nearbyint(sz[i]), 2.0f);                         // torch.max(sz.round(), 2).long()
        tl[i] = poslf[i] - ((float)(szl - 1) / 2.0f);                                          // posl - (szl - 1)/2
        br[i] = (poslf[i] + ((float)szl / 2.0f)) + 1.0f;                                       // posl + szl/2 + 1
    }
    if (inside) {
        // im2_sz = the decimated image's size im[..., os::df, os::df]; tl, br stay float32 tensors throughout
        const float im2[2] = {(float)((H - os[0] + df - 1) / df), (float)((W - os[1] + df - 1) / df)};
        for (int i = 0; i < 2; ++i) {
            const float shift = std::fmax(-tl[i], 0.0f) - std::fmax(br[i] - im2[i], 0.0f);     // (-tl).clamp(0) - (br - im2_sz).clamp(0)
            tl[i] = tl[i] + shift; br[i] = br[i] + shift;
            const float outside = floor_div_f32(std::fmax(-tl[i], 0.0f) + std::fmax(br[i] - im2[i], 0.0f), 2.0f);
            const float shift2 = (-tl[i] - outside) * (outside > 0.0f ? 1.0f : 0.0f);          // (-tl - outside) * (outside > 0).long()
            tl[i] = tl[i] + shift2; br[i] = br[i] + shift2;
        }
    }
    for (int i = 0; i < 2; ++i) { tli[i] = (int)std::trunc(tl[i]); bri[i] = (int)std::trunc(br[i]); }   // .int().item()
    g->df = df; g->os_r = os[0]; g->os_c = os[1]; g->tl_r = tli[0]; g->tl_c = tli[1];
    g->in_h = bri[0] - tli[0]; g->in_w = bri[1] - tli[1];
    g->out_h = (int)output_sz[0]; g->out_w = (int)output_sz[1]; g->win_r = 0; g->win_c = 0;
    g->coord[0] = (float)df * tl[0]; g->coord[1] = (float)df * tl[1]; g->coord[2] = (float)df * br[0]; g->coord[3] = (float)df * br[1];
}

// DiMP.get_sample_location (dimp.py:177-182)
static void sample_location(const b200trk_dimp_tracker* t, b200trk_crop_geom_t* g) {
    for (int i = 0; i < 2; ++i) g->sample_pos[i] = 0.5f * ((g->coord[i] + g->coord[2 + i]) - 1.0f);
    const float a = (g->coord[2] - g->coord[0]) / t->img_sample_sz[0], b = (g->coord[3] - g->coord[1]) / t->img_sample_sz[1];
    g->sample_scale = std::sqrt(a * b);
}

// DiMP.get_iounet_box (dimp.py:500-507) -> (x, y, w, h) in crop pixels
static void iounet_box(const b200trk_dimp_tracker* t, const float pos[2], const float sz[2], const float sample_pos[2], float sample_scale,
                       float box[4]) {
    float ul[2], bs[2];
    for (int i = 0; i < 2; ++i) {
        const float bc = (pos[i] - sample_pos[i]) / sample_scale + (t->img_sample_sz[i] - 1.0f) / 2.0f;
        bs[i] = sz[i] / sample_scale;
        ul[i] = bc - (bs[i] - 1.0f) / 2.0f;
    }
    box[0] = ul[1]; box[1] = ul[0]; box[2] = bs[1]; box[3] = bs[0];
}

extern "C" int b200trk_dimp_tracker_create(b200trk_dimp_tracker_t** out, b200trk_dimp_state_t* state, const b200trk_dimp_params_t* params) {
    B200_REQUIRE(out && params, "dimp_tracker_create: null pointer");
    B200_REQUIRE(params->image_sample_size > 0 && params->sample_memory_size >= 1, "dimp_tracker_create: bad parameters");
    B200_REQUIRE(params->border_mode >= 0 && params->border_mode <= 2, "dimp_tracker_create: border_mode=%d (0 replicate, 1 inside, 2 inside_major)",
                 params->border_mode);
    B200_REQUIRE(params->score_preprocess >= 0 && params->score_preprocess <= 2, "dimp_tracker_create: score_preprocess=%d (0 none, 1 exp, 2 softmax)",
                 params->score_preprocess);
    B200_REQUIRE(!state || state->memory_size == params->sample_memory_size, "dimp_tracker_create: sample_memory_size=%d but the state holds %d",
                 params->sample_memory_size, state ? state->memory_size : 0);
    B200_REQUIRE(!state || (state->net->crop_h == params->image_sample_size && state->net->crop_w == params->image_sample_size),
                 "dimp_tracker_create: the network was built for %dx%d crops, image_sample_size=%d", state ? state->net->crop_h : 0,
                 state ? state->net->crop_w : 0, params->image_sample_size);
    b200trk_dimp_tracker* t = new b200trk_dimp_tracker();
    t->st = state; t->p = *params;
    t->img_sample_sz[0] = t->img_sample_sz[1] = (float)params->image_sample_size;
    if (state) {
        t->feature_sz[0] = (float)state->Hc; t->feature_sz[1] = (float)state->Wc;
        t->kernel_size[0] = t->kernel_size[1] = (float)state->ksz;
        t->score_sz[0] = (float)state->Ho; t->score_sz[1] = (float)state->Wo;
        // a state without per-frame buffers is a batch slot: the batch holds the localisation results of all its slots
        if (state->clf && (cudaMalloc((void**)&t->loc_dev, sizeof(b200trk_loc_result_t)) != cudaSuccess ||
                           cudaMallocHost((void**)&t->loc_host, sizeof(b200trk_loc_result_t)) != cudaSuccess)) {
            set_error("dimp_tracker_create: allocation failed");
            b200trk_dimp_tracker_destroy(t);
            return 1;
        }
    } else {
        t->feature_sz[0] = t->feature_sz[1] = (float)(params->image_sample_size / 16);
        t->score_sz[0] = t->score_sz[1] = t->feature_sz[0] + 1.f;
    }
    t->sw.assign(params->sample_memory_size, 0.f);
    *out = t;
    return 0;
}

extern "C" int b200trk_dimp_tracker_destroy(b200trk_dimp_tracker_t* t) {
    if (!t) return 0;
    if (t->loc_dev) cudaFree(t->loc_dev);
    if (t->loc_host) cudaFreeHost(t->loc_host);
    for (float* q : {t->mod3, t->mod4, t->iou3, t->iou4, t->boxes_dev, t->aug_mult, t->aug_patch}) if (q) cudaFree(q);
    if (t->aug_table) cudaFree(t->aug_table);
    if (t->boxes_host) cudaFreeHost(t->boxes_host);
    delete t;
    return 0;
}

extern "C" int b200trk_dimp_tracker_init_state(b200trk_dimp_tracker_t* t, int H, int W, const double b[4], b200trk_crop_geom_t* init_crop,
                                               float init_target_box[4]) {
    B200_REQUIRE(t && b, "dimp_tracker_init_state: null pointer");
    B200_REQUIRE(H > 0 && W > 0 && b[2] > 0 && b[3] > 0, "dimp_tracker_init_state: bad image / box");
    B200_REQUIRE(t->p.border_mode != 1, "dimp_tracker_init_state: border_mode 'inside' changes the initial sample (dimp.py:333-347), "
                 "which the native initialisation does not implement; initialise with the reference and adopt its state");
    // dimp.py:44-76
    t->frame_num = 1;
    t->pos[0] = f32(b[1] + (b[3] - 1) / 2); t->pos[1] = f32(b[0] + (b[2] - 1) / 2);
    t->target_sz[0] = f32(b[3]); t->target_sz[1] = f32(b[2]);
    t->image_sz[0] = (float)H; t->image_sz[1] = (float)W;
    const float sas = f32(t->p.search_area_scale);
    const double search_area = (double)((t->target_sz[0] * sas) * (t->target_sz[1] * sas));       // torch.prod(target_sz * scale).item()
    const float root = std::sqrt(t->img_sample_sz[0] * t->img_sample_sz[1]);                      // img_sample_sz.prod().sqrt()
    t->target_scale = (1.0f / root) * f32(std::sqrt(search_area));                                // float / tensor = reciprocal * float
    for (int i = 0; i < 2; ++i) t->base_target_sz[i] = t->target_sz[i] / t->target_scale;
    t->min_scale_factor = std::fmax((1.0f / t->base_target_sz[0]) * 10.0f, (1.0f / t->base_target_sz[1]) * 10.0f);
    t->max_scale_factor = std::fmin(t->image_sz[0] / t->base_target_sz[0], t->image_sz[1] / t->base_target_sz[1]);
    // generate_init_samples (dimp.py:331-398), un-augmented: Identity transform on the expanded patch
    const float init_pos[2] = {std::nearbyint(t->pos[0]), std::nearbyint(t->pos[1])};               // self.pos.round()
    const float init_scale = t->target_scale;
    float aug_sz[2] = {t->img_sample_sz[0], t->img_sample_sz[1]};
    const double ef = t->p.augmentation_expansion_factor;
    if (ef != 0.0 && ef != 1.0) {
        for (int i = 0; i < 2; ++i) {
            long a = (long)std::trunc(t->img_sample_sz[i] * f32(ef));
            a += (a - (long)t->img_sample_sz[i]) % 2;
            aug_sz[i] = (float)a;
        }
    }
    const float sample_sz[2] = {init_scale * aug_sz[0], init_scale * aug_sz[1]};
    b200trk_crop_geom_t g;
    // Always border mode 'replicate' here: generate_init_samples (dimp.py:332-350) enters its border-mode block only for
    // mode == 'inside', so 'inside_major' (PrDiMP) leaves the init crop alone, and sample_patch_transformed then samples with the
    // default mode. 'inside' changes the init sample (scale and global shift); that is not implemented and refused above.
    plan_patch(init_pos, sample_sz, aug_sz, H, W, 0, 0.0, &g);
    // Identity.crop_to_output (augmentation.py:20-37): pad by (output - image)/2, floor on the top / left side
    g.win_r = -(int)std::floor(((double)t->img_sample_sz[0] - (double)aug_sz[0]) / 2);
    g.win_c = -(int)std::floor(((double)t->img_sample_sz[1] - (double)aug_sz[1]) / 2);
    sample_location(t, &g);            // informational; the init sample's position is init_sample_pos / init_sample_scale
    g.sample_pos[0] = init_pos[0]; g.sample_pos[1] = init_pos[1]; g.sample_scale = init_scale;
    if (init_crop) *init_crop = g;
    float box[4];
    iounet_box(t, t->pos, t->target_sz, init_pos, init_scale, box);                                 // init_target_boxes, dimp.py:400-408
    if (init_target_box) std::memcpy(init_target_box, box, sizeof(box));
    // init_memory (dimp.py:410-427) with one init sample
    std::fill(t->sw.begin(), t->sw.end(), 0.f);
    t->sw[0] = 1.0f;
    t->num_init = 1; t->num_stored = 1; t->prev_replace_ind = -1;
    t->initialized = 1;
    return 0;
}

// The refusals of an augmented initialisation; checked before anything changes
static int augment_ok(const b200trk_dimp_tracker* t, const b200trk_dimp_augment_t* aug, const char* what) {
    const int T = aug->num_transforms, n = T + aug->num_dropout;
    B200_REQUIRE(T >= 1 && aug->num_dropout >= 0 && n <= B200TRK_AUG_MAX, "%s: %d transforms and %d dropout copies (at most %d samples)",
                 what, T, aug->num_dropout, B200TRK_AUG_MAX);
    B200_REQUIRE(n <= (int)t->sw.size(), "%s: %d first-frame samples, sample_memory_size=%d", what, n, (int)t->sw.size());
    B200_REQUIRE(aug->num_dropout == 0 || aug->dropout_mult, "%s: dropout copies without multipliers", what);
    B200_REQUIRE(aug->transform[0].kind == B200TRK_AUG_IDENTITY && aug->transform[0].shift[0] == 0 && aug->transform[0].shift[1] == 0,
                 "%s: the first transform must be the identity without shift (the un-augmented sample)", what);
    const char* why = b200trk::augment_refusal(aug->transform, T);
    B200_REQUIRE(!why, "%s: %s", what, why);
    if (t->st) {        // (border_mode 'inside' is refused by init_state, before it changes anything)
        B200_REQUIRE(t->st->clf, "%s: the tracker is a slot of a batch, whose forward pass runs one crop per sequence", what);
        B200_REQUIRE(t->st->max_batch >= n, "%s: the network was built for batches of %d, the augmentation has %d samples", what,
                     t->st->max_batch, n);
    }
    return 0;
}

extern "C" int b200trk_dimp_tracker_init_state_augmented(b200trk_dimp_tracker_t* t, int H, int W, const double b[4],
                                                         const b200trk_dimp_augment_t* aug, b200trk_crop_geom_t* init_crop, float* target_boxes) {
    B200_REQUIRE(t && b && aug && target_boxes, "dimp_tracker_init_state_augmented: null pointer");
    if (int e = augment_ok(t, aug, "dimp_tracker_init_state_augmented")) return e;
    float box[4];
    if (int e = b200trk_dimp_tracker_init_state(t, H, W, b, init_crop, box)) return e;
    // init_target_boxes (dimp.py:399-408): classifier_target_box + [shift_x, shift_y, 0, 0]; the dropout copies carry transform 0's
    const int T = aug->num_transforms, n = T + aug->num_dropout;
    for (int k = 0; k < n; ++k) {
        const int* s = aug->transform[k < T ? k : 0].shift;
        float* o = target_boxes + 4 * k;
        o[0] = box[0] + (float)s[1]; o[1] = box[1] + (float)s[0]; o[2] = box[2] + 0.f; o[3] = box[3] + 0.f;
    }
    // init_memory (dimp.py:410-427): n init samples of weight x.new_ones(1) / n
    std::fill(t->sw.begin(), t->sw.end(), 0.f);
    for (int k = 0; k < n; ++k) t->sw[k] = 1.0f / (float)n;
    t->num_init = n; t->num_stored = n;
    return 0;
}

extern "C" int b200trk_dimp_tracker_adopt(b200trk_dimp_tracker_t* t, int H, int W, const float pos[2], const float target_sz[2], float target_scale,
                                          const float base_target_sz[2], float min_scale_factor, float max_scale_factor,
                                          const float* sample_weights, int num_stored, int num_init, int previous_replace_ind, int frame_num) {
    B200_REQUIRE(t && pos && target_sz && base_target_sz && sample_weights, "dimp_tracker_adopt: null pointer");
    B200_REQUIRE(num_init >= 1 && num_stored >= num_init && num_init <= (int)t->sw.size(), "dimp_tracker_adopt: bad sample counts");
    for (int i = 0; i < 2; ++i) { t->pos[i] = pos[i]; t->target_sz[i] = target_sz[i]; t->base_target_sz[i] = base_target_sz[i]; }
    t->image_sz[0] = (float)H; t->image_sz[1] = (float)W;
    t->target_scale = target_scale; t->min_scale_factor = min_scale_factor; t->max_scale_factor = max_scale_factor;
    for (size_t i = 0; i < t->sw.size(); ++i) t->sw[i] = sample_weights[i];
    t->num_stored = num_stored; t->num_init = num_init; t->prev_replace_ind = previous_replace_ind; t->frame_num = frame_num;
    t->initialized = 1;
    return 0;
}

extern "C" int b200trk_dimp_tracker_state(const b200trk_dimp_tracker_t* t, float out[9]) {
    B200_REQUIRE(t && out, "dimp_tracker_state: null pointer");
    out[0] = t->pos[0]; out[1] = t->pos[1]; out[2] = t->target_sz[0]; out[3] = t->target_sz[1]; out[4] = t->target_scale;
    out[5] = t->base_target_sz[0]; out[6] = t->base_target_sz[1]; out[7] = t->min_scale_factor; out[8] = t->max_scale_factor;
    return 0;
}

extern "C" int b200trk_dimp_tracker_plan_crop(b200trk_dimp_tracker_t* t, b200trk_crop_geom_t* g) {
    B200_REQUIRE(t && g, "dimp_tracker_plan_crop: null pointer");
    B200_REQUIRE(t->initialized, "dimp_tracker_plan_crop: tracker not initialised");
    // get_centered_sample_pos (dimp.py:184-188)
    float cpos[2];
    for (int i = 0; i < 2; ++i) {
        const float m = std::fmod(t->feature_sz[i] + t->kernel_size[i], 2.0f);
        cpos[i] = t->pos[i] + ((m * t->target_scale) * t->img_sample_sz[i]) / (2.0f * t->feature_sz[i]);
    }
    const float s = t->target_scale * 1.0f;                                                       // target_scale * scale_factors (ones(1))
    const float sample_sz[2] = {s * t->img_sample_sz[0], s * t->img_sample_sz[1]};
    plan_patch(cpos, sample_sz, t->img_sample_sz, (int)t->image_sz[0], (int)t->image_sz[1], t->p.border_mode, t->p.patch_max_scale_change, g);
    sample_location(t, g);
    return 0;
}

// DiMP.update_sample_weights (dimp.py:445-484), float32 like the reference's tensor; returns the slot to overwrite
static int update_sample_weights(b200trk_dimp_tracker* t, double lr) {
    std::vector<float>& sw = t->sw;
    const int size = (int)sw.size();
    double init_w = t->p.init_samples_minimum_weight;
    const bool has_init_w = init_w != 0.0;
    const int s_ind = has_init_w ? t->num_init : 0;
    int r_ind;
    auto sum = [&](int a, int b) { float s = 0.f; for (int i = a; i < b; ++i) s += sw[i]; return s; };
    if (t->num_stored == 0 || lr == 1.0) {
        std::fill(sw.begin(), sw.end(), 0.f);
        sw[0] = 1.f; r_ind = 0;
    } else {
        if (t->num_stored < size) {
            r_ind = (int)t->num_stored;
        } else {
            r_ind = s_ind;
            for (int i = s_ind + 1; i < size; ++i) if (sw[i] < sw[r_ind]) r_ind = i;                 // torch.min: first minimum
        }
        const float one_minus = f32(1.0 - lr);
        if (t->prev_replace_ind < 0) {
            for (float& v : sw) v = v / one_minus;
            sw[r_ind] = f32(lr);
        } else {
            sw[r_ind] = sw[t->prev_replace_ind] / one_minus;
        }
    }
    const float tot = sum(0, size);
    for (float& v : sw) v = v / tot;
    if (has_init_w && sum(0, t->num_init) < f32(init_w)) {
        const float d = f32(init_w) + sum(t->num_init, size);
        for (float& v : sw) v = v / d;
        const float iw = f32(init_w / t->num_init);
        for (int i = 0; i < t->num_init; ++i) sw[i] = iw;
    }
    return r_ind;
}

// DiMP.update_state (dimp.py:486-497)
static void update_state(b200trk_dimp_tracker* t, const float new_pos[2], const float* new_scale) {
    if (new_scale) {
        t->target_scale = std::fmin(std::fmax(*new_scale, t->min_scale_factor), t->max_scale_factor);
        for (int i = 0; i < 2; ++i) t->target_sz[i] = t->base_target_sz[i] * t->target_scale;
    }
    const float ir = f32(t->p.target_inside_ratio - 0.5);
    for (int i = 0; i < 2; ++i) {
        const float off = ir * t->target_sz[i];
        t->pos[i] = std::fmax(std::fmin(new_pos[i], t->image_sz[i] - off), off);
    }
}

static bool refines(const b200trk_dimp_tracker* t) { return t->p.use_iou_net != 0; }

// Phase 1 of a frame's host work: everything between localize_target and refine_target_box (dimp.py:97-128)
extern "C" int b200trk_dimp_tracker_commit_localize(b200trk_dimp_tracker_t* t, const b200trk_crop_geom_t* g, const b200trk_loc_result_t* loc,
                                                    b200trk_frame_info_t* info) {
    B200_REQUIRE(t && g && loc && info, "dimp_tracker_commit: null pointer");
    B200_REQUIRE(t->initialized, "dimp_tracker_commit: tracker not initialised");
    t->frame_num += 1;                                                                             // dimp.py:97
    std::memset(info, 0, sizeof(*info));
    info->loc = *loc; info->crop = *g; info->flag = loc->flag; info->max_score = loc->max_score; info->replace_ind = -1;
    const float sample_scale = g->sample_scale;
    // translation (dimp.py:243-257)
    float new_pos[2];
    const int rc[2] = {loc->use_second ? loc->r2 : loc->r1, loc->use_second ? loc->c2 : loc->c1};
    for (int i = 0; i < 2; ++i) {
        const float output_sz = t->score_sz[i] - std::fmod(t->kernel_size[i] + 1.0f, 2.0f);
        const float center = (t->score_sz[i] - 1.0f) / 2.0f;
        const float disp = (float)rc[i] - center;
        const float tv = (disp * (t->img_sample_sz[i] / output_sz)) * sample_scale;
        new_pos[i] = g->sample_pos[i] + tv;
    }
    if (loc->flag != 4) {
        if (refines(t)) update_state(t, new_pos, nullptr);          // the IoUNet sets the size (dimp.py:120-124)
        else update_state(t, new_pos, &sample_scale);               // dimp.py:125-126
    }
    return 0;
}

static float next_uniform(b200trk_dimp_tracker* t, size_t i) {
    if (i < t->noise.size()) return t->noise[i];
    t->rng ^= t->rng << 13; t->rng ^= t->rng >> 7; t->rng ^= t->rng << 17;                        // xorshift64: the tracker's own generator
    return (float)((t->rng >> 40) & 0xFFFFFF) * (1.0f / 16777216.0f);
}

// The proposals of refine_target_box (dimp.py:654-674): the classifier's box followed by num_init_random_boxes jittered copies
extern "C" int b200trk_dimp_tracker_proposals(b200trk_dimp_tracker_t* t, const b200trk_crop_geom_t* g, float* boxes_out, int* count) {
    B200_REQUIRE(t && g && boxes_out && count, "dimp_tracker_proposals: null pointer");
    const int nr = t->p.num_init_random_boxes;
    B200_REQUIRE(nr >= 0 && nr + 1 <= 16, "dimp_tracker_proposals: num_init_random_boxes=%d (at most 15)", nr);
    float ib[4];
    iounet_box(t, t->pos, t->target_sz, g->sample_pos, g->sample_scale, ib);
    for (int i = 0; i < 4; ++i) boxes_out[i] = ib[i];
    if (nr > 0) {
        const float square = std::sqrt(ib[2] * ib[3]);
        const float rf[4] = {square * f32(t->p.box_jitter_pos), square * f32(t->p.box_jitter_pos), square * f32(t->p.box_jitter_sz),
                             square * f32(t->p.box_jitter_sz)};
        const float min_edge = std::fmin(ib[2], ib[3]) / 3.0f;
        for (int r = 0; r < nr; ++r) {
            float rb[4];
            for (int i = 0; i < 4; ++i) rb[i] = (next_uniform(t, (size_t)r * 4 + i) - 0.5f) * rf[i];
            float* o = boxes_out + 4 * (r + 1);
            for (int i = 0; i < 2; ++i) {
                const float nsz = std::fmax(ib[2 + i] + rb[2 + i], min_edge);
                const float nc = (ib[i] + ib[2 + i] / 2.0f) + rb[i];
                o[i] = nc - nsz / 2.0f; o[2 + i] = nsz;
            }
        }
    }
    t->noise.clear();
    *count = nr + 1;
    return 0;
}

// Phase 2: after optimize_boxes -- filter, top-k mean, new position / size / scale (dimp.py:679-721)
extern "C" int b200trk_dimp_tracker_commit_refine(b200trk_dimp_tracker_t* t, const b200trk_crop_geom_t* g, const float* boxes, const float* iou,
                                                  int count, b200trk_frame_info_t* info) {
    B200_REQUIRE(t && g && boxes && iou && info && count >= 1 && count <= 16, "dimp_tracker_commit_refine: bad argument");
    float bx[16][4]; float io[16]; int n = 0;
    const float mar = f32(t->p.maximal_aspect_ratio), imar = f32(1.0 / t->p.maximal_aspect_ratio);
    for (int r = 0; r < count; ++r) {
        const float w = std::fmax(boxes[4 * r + 2], 1.0f), h = std::fmax(boxes[4 * r + 3], 1.0f);    // output_boxes[:, 2:].clamp_(1)
        const float ar = w / h;
        if (ar < mar && ar > imar) { bx[n][0] = boxes[4 * r]; bx[n][1] = boxes[4 * r + 1]; bx[n][2] = w; bx[n][3] = h; io[n] = iou[r]; ++n; }
    }
    if (n == 0) return 0;                                                                               // "If no box found"
    const int k = std::min(t->p.iounet_k > 0 ? t->p.iounet_k : 5, n);
    bool used[16] = {false};
    float pb[4] = {0, 0, 0, 0}, piou = 0.f;
    for (int j = 0; j < k; ++j) {                          // torch.topk: largest first
        int best = -1;
        for (int r = 0; r < n; ++r) if (!used[r] && (best < 0 || io[r] > io[best])) best = r;
        used[best] = true;
        for (int i = 0; i < 4; ++i) pb[i] += bx[best][i];
        piou += io[best];
    }
    for (int i = 0; i < 4; ++i) pb[i] = pb[i] / (float)k;
    info->predicted_iou = piou / (float)k; info->refined = 1;
    // new position and size (dimp.py:703-721); predicted_box = (x, y, w, h), tracker vectors are (row, col)
    const float cx = pb[0] + pb[2] / 2.0f, cy = pb[1] + pb[3] / 2.0f;
    const float c[2] = {cy, cx}, sz[2] = {pb[3], pb[2]};
    float new_pos[2], new_sz[2];
    for (int i = 0; i < 2; ++i) {
        new_pos[i] = (c[i] - (t->img_sample_sz[i] - 1.0f) / 2.0f) * g->sample_scale + g->sample_pos[i];
        new_sz[i] = sz[i] * g->sample_scale;
    }
    const float new_scale = std::sqrt((new_sz[0] * new_sz[1]) / (t->base_target_sz[0] * t->base_target_sz[1]));
    t->pos_iounet[0] = new_pos[0]; t->pos_iounet[1] = new_pos[1]; t->has_pos_iounet = 1;
    if (t->p.use_iounet_pos_for_learning) { t->pos[0] = new_pos[0]; t->pos[1] = new_pos[1]; }
    t->target_sz[0] = new_sz[0]; t->target_sz[1] = new_sz[1];
    const bool update_scale = t->p.update_scale_when_uncertain || info->flag != 3;
    if (update_scale) t->target_scale = new_scale;
    return 0;
}

// Phase 3: the update half of the frame and the output box (dimp.py:131-175, 605-625)
extern "C" int b200trk_dimp_tracker_commit_update(b200trk_dimp_tracker_t* t, const b200trk_crop_geom_t* g, b200trk_frame_info_t* info,
                                                  float* sample_weights_out) {
    B200_REQUIRE(t && g && info, "dimp_tracker_commit: null pointer");
    const float sample_scale = g->sample_scale;
    const bool not_found = info->flag == 4, uncertain = info->flag == 3, hard_negative = info->flag == 2;
    const bool update_flag = !not_found && !uncertain;
    if (update_flag && t->p.update_classifier) {
        iounet_box(t, t->pos, t->target_sz, g->sample_pos, sample_scale, info->target_box);
        const bool hn_flag = hard_negative && t->p.hard_negative_learning_rate >= 0.0;
        const double lr = hn_flag ? t->p.hard_negative_learning_rate : t->p.learning_rate;
        const int interval = t->p.train_sample_interval > 0 ? t->p.train_sample_interval : 1;
        if (hn_flag || t->frame_num % interval == 0) {
            info->replace_ind = update_sample_weights(t, lr);
            t->prev_replace_ind = info->replace_ind;
            t->num_stored += 1;
            info->updated = 1;
        }
        int num_iter = 0;
        if (hn_flag) num_iter = t->p.net_opt_hn_iter;
        else if ((t->frame_num - 1) % (t->p.train_skipping > 0 ? t->p.train_skipping : 1) == 0) num_iter = t->p.net_opt_update_iter;
        info->num_iter = num_iter > 0 ? num_iter : 0;
        info->learning_rate = f32(lr);
    }
    info->n_stored = (int)std::min<long>(t->num_stored, (long)t->sw.size());
    // "Set the pos of the tracker to iounet pos" (dimp.py:148-150)
    if (refines(t) && !not_found && t->has_pos_iounet) { t->pos[0] = t->pos_iounet[0]; t->pos[1] = t->pos_iounet[1]; }
    // output box (dimp.py:163-171)
    if (t->p.output_not_found_box && not_found) {
        for (int i = 0; i < 4; ++i) info->bbox[i] = -1.f;
    } else {
        info->bbox[0] = t->pos[1] - (t->target_sz[1] - 1.0f) / 2.0f;
        info->bbox[1] = t->pos[0] - (t->target_sz[0] - 1.0f) / 2.0f;
        info->bbox[2] = t->target_sz[1];
        info->bbox[3] = t->target_sz[0];
    }
    if (sample_weights_out) std::memcpy(sample_weights_out, t->sw.data(), t->sw.size() * sizeof(float));
    return 0;
}

// The whole host half of a frame without IoUNet refinement (use_iou_net = False): phases 1 + 3
extern "C" int b200trk_dimp_tracker_commit(b200trk_dimp_tracker_t* t, const b200trk_crop_geom_t* g, const b200trk_loc_result_t* loc,
                                           b200trk_frame_info_t* info, float* sample_weights_out) {
    B200_REQUIRE(t && !refines(t), "dimp_tracker_commit: use_iou_net is set -- call commit_localize / proposals / commit_refine / commit_update");
    if (int e = b200trk_dimp_tracker_commit_localize(t, g, loc, info)) return e;
    return b200trk_dimp_tracker_commit_update(t, g, info, sample_weights_out);
}

extern "C" int b200trk_dimp_tracker_set_proposal_noise(b200trk_dimp_tracker_t* t, const float* u01, int count) {
    B200_REQUIRE(t && u01 && count >= 0 && count <= 64, "dimp_tracker_set_proposal_noise: bad argument");
    t->noise.assign(u01, u01 + count);
    return 0;
}

extern "C" int b200trk_dimp_tracker_attach_modulation_head(b200trk_dimp_tracker_t* t, b200trk_iou_modulation_t* head) {
    B200_REQUIRE(t && head, "dimp_tracker_attach_modulation_head: null pointer");
    B200_REQUIRE(t->st, "dimp_tracker_attach_modulation_head: host-logic-only tracker");
    B200_REQUIRE(!t->initialized, "dimp_tracker_attach_modulation_head: refused after initialize (the modulation comes from the first frame)");
    B200_REQUIRE(!t->mod_head, "dimp_tracker_attach_modulation_head: already attached");
    B200_REQUIRE(t->st->net->iouref.op[0] >= 0, "dimp_tracker_attach_modulation_head: the network has no conv3_1r / conv4_1r "
                 "(b200trk_net_attach_iou_ref)");
    t->mod_head = head;
    return 0;
}

extern "C" int b200trk_dimp_tracker_attach_iounet(b200trk_dimp_tracker_t* t, b200trk_iou_predictor_t* pred, const float* modulation3,
                                                  const float* modulation4) {
    B200_REQUIRE(t && pred, "dimp_tracker_attach_iounet: null pointer");
    B200_REQUIRE((modulation3 == nullptr) == (modulation4 == nullptr), "dimp_tracker_attach_iounet: give both modulation vectors or neither");
    const bool native = modulation3 == nullptr;
    B200_REQUIRE(t->st, "dimp_tracker_attach_iounet: host-logic-only tracker");
    B200_REQUIRE(!t->iou_pred, "dimp_tracker_attach_iounet: already attached");
    B200_REQUIRE(!native || t->mod_head, "dimp_tracker_attach_iounet: no modulation vectors and no modulation head "
                 "(b200trk_dimp_tracker_attach_modulation_head)");
    B200_REQUIRE(!native || !t->initialized, "dimp_tracker_attach_iounet: native modulation is computed by initialize; attach before it");
    if (int e = b200trk_net_iou_dims(t->st->net, t->iou_dims)) return e;
    B200_REQUIRE(t->iou_dims[0] > 0, "dimp_tracker_attach_iounet: the network has no IoU feature branch (b200trk_net_attach_iou_head)");
    const int C3 = t->iou_dims[0], C4 = t->iou_dims[3];
    if (native) {
        int md[2];
        if (int e = b200trk_iou_modulation_dims(t->mod_head, md)) return e;
        B200_REQUIRE(md[0] == C3 && md[1] == C4, "dimp_tracker_attach_iounet: the modulation head gives %d / %d values, the IoU features have "
                     "%d / %d channels", md[0], md[1], C3, C4);
    }
    B200_CHECK_CUDA(cudaMalloc((void**)&t->mod3, C3 * sizeof(float)));
    B200_CHECK_CUDA(cudaMalloc((void**)&t->mod4, C4 * sizeof(float)));
    if (!native) {
        B200_CHECK_CUDA(cudaMemcpy(t->mod3, modulation3, C3 * sizeof(float), cudaMemcpyHostToDevice));
        B200_CHECK_CUDA(cudaMemcpy(t->mod4, modulation4, C4 * sizeof(float), cudaMemcpyHostToDevice));
    }
    B200_CHECK_CUDA(cudaMalloc((void**)&t->iou3, (size_t)C3 * t->iou_dims[1] * t->iou_dims[2] * sizeof(float)));
    B200_CHECK_CUDA(cudaMalloc((void**)&t->iou4, (size_t)C4 * t->iou_dims[4] * t->iou_dims[5] * sizeof(float)));
    B200_CHECK_CUDA(cudaMalloc((void**)&t->boxes_dev, 16 * 5 * sizeof(float)));
    B200_CHECK_CUDA(cudaMallocHost((void**)&t->boxes_host, 16 * 5 * sizeof(float)));
    t->iou_pred = pred;
    t->mod_native = native ? 1 : 0;
    return 0;
}

extern "C" int b200trk_dimp_tracker_modulation(const b200trk_dimp_tracker_t* t, float* modulation3, float* modulation4) {
    B200_REQUIRE(t && modulation3 && modulation4, "dimp_tracker_modulation: null pointer");
    B200_REQUIRE(t->iou_pred, "dimp_tracker_modulation: no IoUNet attached");
    B200_CHECK_CUDA(cudaDeviceSynchronize());
    B200_CHECK_CUDA(cudaMemcpy(modulation3, t->mod3, t->iou_dims[0] * sizeof(float), cudaMemcpyDeviceToHost));
    B200_CHECK_CUDA(cudaMemcpy(modulation4, t->mod4, t->iou_dims[3] * sizeof(float), cudaMemcpyDeviceToHost));
    return 0;
}

// ---------------------------------------------------------------------------------------------------------------------------
// device launches
// ---------------------------------------------------------------------------------------------------------------------------
// A crop the sampling kernels can read: a decimation factor >= 1, a non-empty patch, and the win_h x win_w window inside the resampled patch
static int crop_ok(const b200trk_crop_geom_t* g, int win_h, int win_w, const char* what) {
    B200_REQUIRE(g->df >= 1 && g->in_h >= 1 && g->in_w >= 1 && g->out_h >= 1 && g->out_w >= 1, "%s: bad geometry", what);
    B200_REQUIRE(g->win_r >= 0 && g->win_c >= 0 && g->win_r + win_h <= g->out_h && g->win_c + win_w <= g->out_w,
                 "%s: window [%d+%d, %d+%d] outside the %dx%d resampled patch", what, g->win_r, win_h, g->win_c, win_w, g->out_h, g->out_w);
    return 0;
}

extern "C" int b200trk_sample_patch(const uint8_t* image_dev, int H, int W, const b200trk_crop_geom_t* g, int win_h, int win_w, float* out,
                                    b200trk_stream_t stream) {
    B200_REQUIRE(image_dev && g && out, "sample_patch: null pointer");
    B200_REQUIRE(H > 0 && W > 0 && win_h > 0 && win_w > 0, "sample_patch: bad geometry");
    if (int e = crop_ok(g, win_h, win_w, "sample_patch")) return e;
    dim3 grid((win_w + 31) / 32, (win_h + 7) / 8);
    sample_patch_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(image_dev, H, W, *g, win_h, win_w, out);
    B200_LAUNCH_CHECK();
    return 0;
}

extern "C" int b200trk_dimp_localize(const float* scores, int S, int Ho, int Wo, const b200trk_dimp_params_t* p, const float* neigh,
                                     const float* prev_vec, b200trk_loc_result_t* result_dev, b200trk_stream_t stream) {
    B200_REQUIRE(scores && p && result_dev, "dimp_localize: null pointer");
    B200_REQUIRE(S >= 1 && S <= 8 && Ho > 0 && Wo > 0, "dimp_localize: S=%d (1..8), map %dx%d", S, Ho, Wo);
    B200_REQUIRE(!p->advanced_localization || (neigh && prev_vec), "dimp_localize: advanced localisation needs neigh / prev_vec");
    B200_REQUIRE(p->score_preprocess >= 0 && p->score_preprocess <= 2, "dimp_localize: score_preprocess=%d (0 none, 1 exp, 2 softmax)",
                 p->score_preprocess);
    const LocArgs a = make_loc_args(S, Ho, Wo, p, neigh, prev_vec);
    const size_t smem = loc_smem_bytes(a);
    B200_REQUIRE(smem <= 48 * 1024, "dimp_localize: score pre-processing holds S*Ho*Wo=%d floats in shared memory (at most 12288)", S * Ho * Wo);
    localize_kernel<<<1, 256, smem, (cudaStream_t)stream>>>(scores, a, result_dev);
    B200_LAUNCH_CHECK();
    return 0;
}

// The device half of initialize (dimp.py:601-602): the first frame's features `feat` become sample 0 with box `box`, and num_iter
// iterations run from the initial filter.  That is FilterInitializerLinear's when the network has one attached -- the caller has run its
// filter_conv on the S feature maps of the arena, of which this sequence's is `image` -- else FilterInitializerZero's zero filter.  The
// reference passes sample_weight = None, which both optimisers read as 1/num_images (optimizer.py:122-123 GN, :387-388 Newton): with one
// sample that is the weight 1 uploaded here.
// A learnt initialiser attached to the state's network must make filters of the state's size
static int filter_init_ok(const b200trk_dimp_state* s, const char* what) {
    B200_REQUIRE(s->net->finit.conv_op < 0 || s->net->finit.ksz == s->ksz, "%s: the network's filter initialiser makes %dx%d filters, the "
                 "tracker's state holds %dx%d", what, s->net->finit.ksz, s->net->finit.ksz, s->ksz, s->ksz);
    return 0;
}

static int first_frame_update(b200trk_dimp_state* s, const float* feat, int S, int image, const float box[4], int num_iter, cudaStream_t st) {
    if (s->net->finit.conv_op >= 0) {
        if (int e = filter_init_pool(s->net, S, 1, &image, box, s->filter, st)) return e;
    } else {
        B200_CHECK_CUDA(cudaMemsetAsync(s->filter, 0, (size_t)s->Cc * s->ksz * s->ksz * sizeof(float), st));
    }
    B200_CHECK_CUDA(cudaMemsetAsync(s->sw, 0, (size_t)s->memory_size * sizeof(float), st));
    const float one = 1.f;
    return dimp_state_insert(s, feat, 0, box, &one, 1, num_iter, st);
}

// The device half of update_classifier (dimp.py:605-625) after a frame's commit: store the sample `feat` and optimise, or only optimise
// (update_classifier can run iterations without storing a sample: train_sample_interval > 1)
static int frame_update(b200trk_dimp_tracker* t, const float* feat, const b200trk_frame_info_t* info, cudaStream_t st) {
    if (info->updated) return dimp_state_insert(t->st, feat, info->replace_ind, info->target_box, t->sw.data(), info->n_stored, info->num_iter, st);
    if (info->num_iter > 0) return dimp_state_optimize(t->st, info->n_stored, info->num_iter, st);
    return 0;
}

extern "C" int b200trk_dimp_tracker_initialize_host(b200trk_dimp_tracker_t* t, const uint8_t* image, int H, int W, const double init_bbox[4],
                                                    b200trk_stream_t stream) {
    B200_REQUIRE(t && image && init_bbox, "dimp_tracker_initialize_host: null pointer");
    B200_REQUIRE(t->st, "dimp_tracker_initialize_host: host-logic-only tracker (created without a device state)");
    if (int e = filter_init_ok(t->st, "dimp_tracker_initialize_host")) return e;
    cudaStream_t st = (cudaStream_t)stream;
    b200trk_dimp_state* s = t->st;
    b200trk_crop_geom_t g; float box[4];
    if (int e = b200trk_dimp_tracker_init_state(t, H, W, init_bbox, &g, box)) return e;
    if (int e = t->frames.upload(1, &image, &H, &W, st)) return e;
    const int iss = t->p.image_sample_size;
    if (int e = b200trk_sample_patch(image, H, W, &g, iss, iss, s->crop, stream)) return e;
    if (int e = b200trk_net_forward(s->net, s->crop, 1, nullptr, nullptr, s->clf, stream)) return e;
    if (s->net->finit.conv_op >= 0)
        if (int e = filter_init_conv(s->net, s->clf, 1, st)) return e;
    if (int e = first_frame_update(s, s->clf, 1, 0, box, t->p.net_opt_iter > 0 ? t->p.net_opt_iter : 0, st)) return e;
    // DiMP.init_iou_net (dimp.py:509-540) without iounet_augmentation: get_modulation of the identity sample at init_target_box, on the
    // layer2 / layer3 activations of this init pass; the mean over that one box is its own vectors
    if (t->mod_native)
        if (int e = b200trk_iou_modulation_get(t->mod_head, s->net, 1, 1, nullptr, box, t->mod3, t->mod4, stream)) return e;
    B200_CHECK_CUDA(cudaStreamSynchronize(st));
    return 0;
}

// DiMP.initialize with use_augmentation (generate_init_samples, init_classifier, init_iou_net; dimp.py:331-408, 509-602)
extern "C" int b200trk_dimp_tracker_initialize_augmented_host(b200trk_dimp_tracker_t* t, const uint8_t* image, int H, int W,
                                                              const double init_bbox[4], const b200trk_dimp_augment_t* aug,
                                                              b200trk_stream_t stream) {
    const char* what = "dimp_tracker_initialize_augmented_host";
    B200_REQUIRE(t && image && init_bbox && aug, "%s: null pointer", what);
    B200_REQUIRE(t->st, "%s: host-logic-only tracker (created without a device state)", what);
    if (int e = filter_init_ok(t->st, what)) return e;
    if (int e = augment_ok(t, aug, what)) return e;
    cudaStream_t st = (cudaStream_t)stream;
    b200trk_dimp_state* s = t->st;
    const int T = aug->num_transforms, nd = aug->num_dropout, n = T + nd;
    b200trk_crop_geom_t g; float boxes[4 * B200TRK_AUG_MAX];
    if (int e = b200trk_dimp_tracker_init_state_augmented(t, H, W, init_bbox, aug, &g, boxes)) return e;
    const size_t patch_floats = (size_t)3 * g.out_h * g.out_w, plane = (size_t)s->Cc * s->Hc * s->Wc;
    if (!t->aug_table) B200_CHECK_CUDA(cudaMalloc(&t->aug_table, b200trk::augment_table_bytes()));
    if (!t->aug_mult) B200_CHECK_CUDA(cudaMalloc((void**)&t->aug_mult, (size_t)B200TRK_AUG_MAX * s->Cc * sizeof(float)));
    if (patch_floats > t->aug_patch_cap) {
        if (t->aug_patch) B200_CHECK_CUDA(cudaFree(t->aug_patch));
        t->aug_patch = nullptr; t->aug_patch_cap = 0;
        B200_CHECK_CUDA(cudaMalloc((void**)&t->aug_patch, patch_floats * sizeof(float)));
        t->aug_patch_cap = patch_floats;
    }
    if (int e = t->frames.upload(1, &image, &H, &W, st)) return e;
    // the whole expanded patch (sample_patch_transformed's sample_patch), then every transform's crop into the state's crop buffer
    g.win_r = g.win_c = 0;
    if (int e = b200trk_sample_patch(image, H, W, &g, g.out_h, g.out_w, t->aug_patch, stream)) return e;
    const int iss = t->p.image_sample_size;
    if (int e = b200trk::augment_crops(aug->transform, T, g.out_h, g.out_w, iss, iss, t->aug_table, t->aug_patch, s->crop, st)) return e;
    if (int e = b200trk_net_forward(s->net, s->crop, T, nullptr, nullptr, s->clf, stream)) return e;
    if (nd > 0) {
        B200_CHECK_CUDA(cudaMemcpyAsync(t->aug_mult, aug->dropout_mult, (size_t)nd * s->Cc * sizeof(float), cudaMemcpyHostToDevice, st));
        if (int e = b200trk::feature_dropout(s->clf, T, nd, s->Cc, s->Hc * s->Wc, t->aug_mult, st)) return e;
    }
    // get_filter on all n samples: FilterInitializerLinear's filter_conv runs on every map, dropout copies included (it has a bias
    // and mixes channels, so it does not commute with the dropout mask), and the mean pools each sample at its own box
    if (s->net->finit.conv_op >= 0) {
        if (int e = filter_init_conv(s->net, s->clf, n, st)) return e;
        if (int e = filter_init_pool(s->net, n, n, nullptr, boxes, s->filter, st)) return e;
    } else {
        B200_CHECK_CUDA(cudaMemsetAsync(s->filter, 0, (size_t)s->Cc * s->ksz * s->ksz * sizeof(float), st));
    }
    // init_memory, then net_opt_iter iterations with sample_weight = None, which both optimisers read as 1/n per sample
    B200_CHECK_CUDA(cudaMemsetAsync(s->sw, 0, (size_t)s->memory_size * sizeof(float), st));
    const int num_iter = t->p.net_opt_iter > 0 ? t->p.net_opt_iter : 0;
    for (int k = 0; k < n; ++k)
        if (int e = dimp_state_insert(s, s->clf + plane * k, k, boxes + 4 * k, t->sw.data(), n, k == n - 1 ? num_iter : 0, st)) return e;
    // init_iou_net without iounet_augmentation: get_modulation of image 0 (the identity sample) at its box, on the layer2 / layer3
    // activations the batch-T pass left in the arena
    if (t->mod_native)
        if (int e = b200trk_iou_modulation_get(t->mod_head, s->net, 1, 1, nullptr, boxes, t->mod3, t->mod4, stream)) return e;
    B200_CHECK_CUDA(cudaStreamSynchronize(st));
    return 0;
}

// target_neigh_sz (dimp.py:265) and prev_target_vec (dimp.py:283) of the single scale, from the state before the frame's commit
static void loc_inputs(const b200trk_dimp_tracker* t, const b200trk_crop_geom_t& g, float neigh[2], float pv[2]) {
    for (int i = 0; i < 2; ++i) {
        const float output_sz = t->score_sz[i] - std::fmod(t->kernel_size[i] + 1.0f, 2.0f);
        neigh[i] = (f32(t->p.target_neighborhood_scale) * (t->target_sz[i] / g.sample_scale)) * (output_sz / t->img_sample_sz[i]);
        pv[i] = (t->pos[i] - g.sample_pos[i]) / ((t->img_sample_sz[i] / output_sz) * g.sample_scale);
    }
}

// The refusals of a frame of a running sequence: the tracker holds one, and the frame has the size of the sequence's first frame
static int tracking_ok(const b200trk_dimp_tracker* t, int H, int W, const char* what) {
    B200_REQUIRE(t->initialized, "%s: not tracking a sequence (never initialised, or released)", what);
    B200_REQUIRE((float)H == t->image_sz[0] && (float)W == t->image_sz[1], "%s: frame is %dx%d, the sequence started with %dx%d", what, H, W,
                 (int)t->image_sz[0], (int)t->image_sz[1]);
    return 0;
}

static int track_frame(b200trk_dimp_tracker* t, const uint8_t* image, bool on_device, int H, int W, b200trk_frame_info_t* info,
                       b200trk_stream_t stream) {
    B200_REQUIRE(t && image && info, "dimp_track_host: null pointer");
    B200_REQUIRE(t->st, "dimp_track_host: host-logic-only tracker (created without a device state)");
    if (int e = tracking_ok(t, H, W, "dimp_track_host")) return e;
    cudaStream_t st = (cudaStream_t)stream;
    b200trk_dimp_state* s = t->st;
    b200trk_crop_geom_t g;
    if (int e = b200trk_dimp_tracker_plan_crop(t, &g)) return e;
    if (!on_device) { if (int e = t->frames.upload(1, &image, &H, &W, st)) return e; }
    const int iss = t->p.image_sample_size;
    if (int e = b200trk_sample_patch(image, H, W, &g, iss, iss, s->crop, stream)) return e;
    if (int e = b200trk_net_forward(s->net, s->crop, 1, nullptr, nullptr, s->clf, stream)) return e;
    if (int e = b200trk_apply_filter(s->clf, s->filter, s->scores, 1, s->Cc, s->Hc, s->Wc, s->ksz, nullptr, nullptr, stream)) return e;
    float neigh[2], pv[2];
    loc_inputs(t, g, neigh, pv);
    if (int e = b200trk_dimp_localize(s->scores, 1, s->Ho, s->Wo, &t->p, neigh, pv, t->loc_dev, stream)) return e;
    B200_CHECK_CUDA(cudaMemcpyAsync(t->loc_host, t->loc_dev, sizeof(b200trk_loc_result_t), cudaMemcpyDeviceToHost, st));
    B200_CHECK_CUDA(cudaStreamSynchronize(st));
    if (int e = b200trk_dimp_tracker_commit_localize(t, &g, t->loc_host, info)) return e;
    if (refines(t) && info->flag != 4) {
        // refine_target_box (dimp.py:650-723): IoU features of this crop, proposals up, box optimisation on the device, 320 bytes back
        B200_REQUIRE(t->iou_pred, "dimp_track_host: use_iou_net is set but no IoU predictor is attached (b200trk_dimp_tracker_attach_iounet)");
        int R = 0;
        if (int e = b200trk_dimp_tracker_proposals(t, &g, t->boxes_host, &R)) return e;
        B200_CHECK_CUDA(cudaMemcpyAsync(t->boxes_dev, t->boxes_host, (size_t)R * 4 * sizeof(float), cudaMemcpyHostToDevice, st));
        if (int e = b200trk_net_iou_from_arena(s->net, 1, t->iou3, t->iou4, stream)) return e;
        if (int e = b200trk_iou_refine(t->iou_pred, t->mod3, t->mod4, t->iou3, t->iou_dims[1], t->iou_dims[2], t->iou4, t->iou_dims[4],
                                       t->iou_dims[5], t->boxes_dev, R, t->p.box_refinement_iter, f32(t->p.box_refinement_step_length),
                                       f32(t->p.box_refinement_step_decay), t->p.box_refinement_relative, t->boxes_dev + 64, stream)) return e;
        B200_CHECK_CUDA(cudaMemcpyAsync(t->boxes_host, t->boxes_dev, 80 * sizeof(float), cudaMemcpyDeviceToHost, st));
        B200_CHECK_CUDA(cudaStreamSynchronize(st));
        if (int e = b200trk_dimp_tracker_commit_refine(t, &g, t->boxes_host, t->boxes_host + 64, R, info)) return e;
    }
    if (int e = b200trk_dimp_tracker_commit_update(t, &g, info, nullptr)) return e;
    return frame_update(t, s->clf, info, st);
}

extern "C" int b200trk_dimp_track_host(b200trk_dimp_tracker_t* t, const uint8_t* image, int H, int W, b200trk_frame_info_t* info,
                                       b200trk_stream_t stream) {
    return track_frame(t, image, false, H, W, info, stream);
}

extern "C" int b200trk_dimp_track_device(b200trk_dimp_tracker_t* t, const uint8_t* image_dev, int H, int W, b200trk_frame_info_t* info,
                                         b200trk_stream_t stream) {
    return track_frame(t, image_dev, true, H, W, info, stream);
}

// ---------------------------------------------------------------------------------------------------------------------------
// batch of sequences: S per-sequence trackers on one network, one crop / forward / classify / localisation launch per step
// ---------------------------------------------------------------------------------------------------------------------------
// The forward always runs at batch S, idle and released slots included: the convolution plans (tile shape, split-K) depend on the batch
// size and every output tile belongs to one sample, so a sequence's bits depend on its own frames and on S only -- never on its
// batch-mates, its slot or when they started -- and the network's cached graph (keyed on pointers and S) is replayed every step.
// The online optimiser stays per sequence (dimp_state_insert / dimp_state_optimize on the slot's state), enqueued back to back.
struct b200trk_dimp_batch {
    b200trk_net* net = nullptr;
    int cap = 0, Cc = 0, Hc = 0, Wc = 0, Ho = 0, Wo = 0, ksz = 4, iss = 0;
    b200trk_dimp_params_t p;
    b200trk_dimp_tracker* t[kBatchMax] = {};                                         // the slots; the batch also owns their states t[i]->st
    float *crop = nullptr, *clf = nullptr, *scores = nullptr, *filters = nullptr;   // device [S,3,iss,iss] [S,C,Hc,Wc] [S,Ho,Wo] [S,C,k,k]
    FrameUpload frames;                                                              // the step's host frames, back to back
    b200trk_loc_result_t* loc_dev = nullptr;                                         // [S]
    b200trk_loc_result_t* loc_host = nullptr;                                        // pinned [S]
};

extern "C" int b200trk_dimp_batch_destroy(b200trk_dimp_batch_t* b) {
    if (!b) return 0;
    for (b200trk_dimp_tracker* t : b->t) {
        if (!t) continue;
        b200trk_dimp_state* s = t->st;
        b200trk_dimp_tracker_destroy(t);
        b200trk_dimp_state_destroy(s);
    }
    for (void* q : {(void*)b->crop, (void*)b->clf, (void*)b->scores, (void*)b->filters, (void*)b->loc_dev}) if (q) cudaFree(q);
    if (b->loc_host) cudaFreeHost(b->loc_host);
    delete b;
    return 0;
}

template <class MakeState>
static int batch_create(b200trk_dimp_batch** out, b200trk_net* net, int capacity, const b200trk_dimp_params_t* params, int filter_size,
                        MakeState make_state) {
    B200_REQUIRE(out && net && params, "dimp_batch_create: null pointer");
    B200_REQUIRE(capacity >= 1 && capacity <= kBatchMax, "dimp_batch_create: capacity=%d outside 1..%d", capacity, kBatchMax);
    B200_REQUIRE(!params->use_iou_net, "dimp_batch_create: use_iou_net is not supported in a batch (the native IoUNet needs each "
                 "sequence's modulation vectors from the reference's initialisation); set use_iou_net = False");
    B200_REQUIRE(params->border_mode != 1, "dimp_batch_create: border_mode 'inside' changes the initial sample, which the native "
                 "initialisation does not implement");
    B200_REQUIRE(filter_size == 4, "dimp_batch_create: filter_size=%d not supported (4)", filter_size);
    B200_REQUIRE(net->max_batch >= capacity, "dimp_batch_create: the network was built for batches of %d, capacity=%d", net->max_batch, capacity);
    b200trk_dimp_batch* b = new b200trk_dimp_batch();
    b->net = net; b->cap = capacity; b->p = *params; b->ksz = filter_size; b->iss = params->image_sample_size;
    b->Cc = net->dims[6]; b->Hc = net->dims[7]; b->Wc = net->dims[8];
    b->Ho = b->Hc + (filter_size + 1) % 2; b->Wo = b->Wc + (filter_size + 1) % 2;
    const size_t S = (size_t)capacity, fsz = (size_t)b->Cc * filter_size * filter_size;
    auto fail = [&](int e) { b200trk_dimp_batch_destroy(b); return e ? e : 1; };
    auto alloc = [&](void** q, size_t bytes) {
        return cudaMalloc(q, bytes) == cudaSuccess && cudaMemset(*q, 0, bytes) == cudaSuccess;
    };
    if (!alloc((void**)&b->crop, S * 3 * net->crop_h * net->crop_w * sizeof(float)) ||
        !alloc((void**)&b->clf, S * b->Cc * b->Hc * b->Wc * sizeof(float)) || !alloc((void**)&b->scores, S * b->Ho * b->Wo * sizeof(float)) ||
        !alloc((void**)&b->filters, S * fsz * sizeof(float)) || !alloc((void**)&b->loc_dev, S * sizeof(b200trk_loc_result_t)) ||
        cudaMallocHost((void**)&b->loc_host, S * sizeof(b200trk_loc_result_t)) != cudaSuccess) {
        set_error("dimp_batch_create: allocation failed");
        return fail(1);
    }
    for (int i = 0; i < capacity; ++i) {
        b200trk_dimp_state* s = nullptr;
        if (int e = make_state(b->filters + i * fsz, &s)) return fail(e);
        if (int e = b200trk_dimp_tracker_create(&b->t[i], s, params)) { b200trk_dimp_state_destroy(s); return fail(e); }
    }
    *out = b;
    return 0;
}

extern "C" int b200trk_dimp_batch_create(b200trk_dimp_batch_t** out, b200trk_net_t* net, int capacity, const b200trk_dimp_params_t* params,
                                         int filter_size, const float* label_lut, const float* mask_lut, const float* spatial_lut, int num_bins,
                                         float bin_displacement, float feat_stride, float step_length, float reg_weight, float alpha_eps) {
    B200_REQUIRE(params, "dimp_batch_create: null pointer");
    return batch_create(out, net, capacity, params, filter_size, [&](float* filter, b200trk_dimp_state** s) {
        return dimp_state_create_gn(s, net, params->sample_memory_size, filter_size, label_lut, mask_lut, spatial_lut, num_bins,
                                    bin_displacement, feat_stride, step_length, reg_weight, alpha_eps, filter);
    });
}

extern "C" int b200trk_prdimp_batch_create(b200trk_dimp_batch_t** out, b200trk_net_t* net, int capacity, const b200trk_dimp_params_t* params,
                                           int filter_size, float gauss_sigma, float feat_stride, float step_length, float reg_weight,
                                           float alpha_eps, int has_softmax_reg, float softmax_reg, float label_threshold, int normalize_label,
                                           float label_shrink, float uni_weight) {
    B200_REQUIRE(params, "prdimp_batch_create: null pointer");
    return batch_create(out, net, capacity, params, filter_size, [&](float* filter, b200trk_dimp_state** s) {
        return dimp_state_create_newton(s, net, params->sample_memory_size, filter_size, gauss_sigma, feat_stride, step_length, reg_weight,
                                        alpha_eps, has_softmax_reg, softmax_reg, label_threshold, normalize_label, label_shrink, uni_weight,
                                        filter);
    });
}

static int batch_slot_ok(const b200trk_dimp_batch* b, int slot, const char* what) {
    B200_REQUIRE(b, "%s: null pointer", what);
    B200_REQUIRE(slot >= 0 && slot < b->cap, "%s: slot %d outside 0..%d", what, slot, b->cap - 1);
    return 0;
}

extern "C" int b200trk_dimp_batch_release(b200trk_dimp_batch_t* b, int slot) {
    if (int e = batch_slot_ok(b, slot, "dimp_batch_release")) return e;
    b->t[slot]->initialized = 0;       // the slot's device state is overwritten by the next sequence's initialisation
    return 0;
}

extern "C" float* b200trk_dimp_batch_filter(b200trk_dimp_batch_t* b, int slot) {
    return batch_slot_ok(b, slot, "dimp_batch_filter") ? nullptr : b->filters + (size_t)slot * b->Cc * b->ksz * b->ksz;
}
extern "C" float* b200trk_dimp_batch_scores(b200trk_dimp_batch_t* b, int slot) {
    return batch_slot_ok(b, slot, "dimp_batch_scores") ? nullptr : b->scores + (size_t)slot * b->Ho * b->Wo;
}
extern "C" float* b200trk_dimp_batch_crop(b200trk_dimp_batch_t* b, int slot) {
    return batch_slot_ok(b, slot, "dimp_batch_crop") ? nullptr : b->crop + (size_t)slot * 3 * b->iss * b->iss;
}
extern "C" int b200trk_dimp_batch_state(const b200trk_dimp_batch_t* b, int slot, float out[9]) {
    if (int e = batch_slot_ok(b, slot, "dimp_batch_state")) return e;
    return b200trk_dimp_tracker_state(b->t[slot], out);
}

static int batch_step(b200trk_dimp_batch* b, const b200trk_batch_item_t* items, int n, bool on_device, b200trk_frame_info_t* infos,
                      b200trk_stream_t stream) {
    B200_REQUIRE(b && items && infos, "dimp_batch_step: null pointer");
    B200_REQUIRE(n >= 1 && n <= b->cap, "dimp_batch_step: %d items for a batch of %d slots", n, b->cap);
    // every refusal before any state changes
    bool seen[kBatchMax] = {};
    char what[kBatchMax][40];                                                        // "dimp_batch_step: slot %d", the refusals' prefix
    for (int k = 0; k < n; ++k) {
        const b200trk_batch_item_t& it = items[k];
        B200_REQUIRE(it.slot >= 0 && it.slot < b->cap, "dimp_batch_step: slot %d outside 0..%d", it.slot, b->cap - 1);
        B200_REQUIRE(!seen[it.slot], "dimp_batch_step: slot %d appears twice in one step", it.slot);
        seen[it.slot] = true;
        std::snprintf(what[k], sizeof(what[k]), "dimp_batch_step: slot %d", it.slot);
        B200_REQUIRE(it.image && it.H > 0 && it.W > 0, "%s: no frame or an empty one (%dx%d)", what[k], it.H, it.W);
        if (it.init) {
            if (int e = filter_init_ok(b->t[it.slot]->st, what[k])) return e;
            B200_REQUIRE(it.init_bbox[2] > 0 && it.init_bbox[3] > 0, "%s: init box of size %gx%g", what[k], it.init_bbox[2], it.init_bbox[3]);
        } else if (int e = tracking_ok(b->t[it.slot], it.H, it.W, what[k])) {
            return e;
        }
    }
    cudaStream_t st = (cudaStream_t)stream;
    const int iss = b->iss;
    // 1. crop plans on the host
    SampleBatchArgs sa;
    float box[kBatchMax][4];
    for (int k = 0; k < n; ++k) {
        const b200trk_batch_item_t& it = items[k];
        if (it.init) { if (int e = b200trk_dimp_tracker_init_state(b->t[it.slot], it.H, it.W, it.init_bbox, &sa.g[k], box[k])) return e; }
        else if (int e = b200trk_dimp_tracker_plan_crop(b->t[it.slot], &sa.g[k])) return e;
        if (int e = crop_ok(&sa.g[k], iss, iss, what[k])) return e;
        sa.im[k] = it.image; sa.H[k] = it.H; sa.W[k] = it.W; sa.dst[k] = it.slot;
    }
    // 2. the frames, on the copy stream behind one event
    if (!on_device) { if (int e = b->frames.upload(n, sa.im, sa.H, sa.W, st)) return e; }
    // 3. one crop launch for every item
    sample_patch_batch_kernel<<<dim3((iss + 31) / 32, (iss + 7) / 8, n), 256, 0, st>>>(sa, iss, b->crop);
    B200_LAUNCH_CHECK();
    // 4. one forward at batch S
    if (int e = b200trk_net_forward(b->net, b->crop, b->cap, nullptr, nullptr, b->clf, stream)) return e;
    // 5. one classify launch, every slot with its own filter
    {
        constexpr int SL18 = CorrSlots<18>::value, SL22 = CorrSlots<22>::value;
        B200_REQUIRE(b->Hc == b->Wc && (b->Hc == 18 || b->Hc == 22), "dimp_batch_step: feature size %dx%d not supported (18x18, 22x22)", b->Hc, b->Wc);
        const int slots = b->Hc == 18 ? SL18 : SL22;
        B200_REQUIRE(b->Cc % slots == 0, "dimp_batch_step: C=%d must be a multiple of %d", b->Cc, slots);
        const int NCH = b->Cc / slots;
        const int npos = b->Ho * b->Wo;
        char* ws = (char*)workspace(4096 + (size_t)b->cap * NCH * npos * sizeof(float), 0);     // as apply_filter: counters, then partial maps
        if (!ws) return 3;
        const size_t fstride = (size_t)b->Cc * b->ksz * b->ksz;
        auto launch = [&](auto kern, int nthreads, size_t smem) -> int {
            B200_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            kern<<<dim3(NCH, b->cap), nthreads, smem, st>>>(b->clf, b->filters, fstride, b->scores, (float*)(ws + 4096), (unsigned*)ws, b->Cc);
            B200_LAUNCH_CHECK();
            return 0;
        };
        if (int e = b->Hc == 18 ? launch(classify_batch_kernel<18, SL18>, CorrCta<18, SL18>::NTHREADS, classify_smem_bytes<18, SL18>())
                                : launch(classify_batch_kernel<22, SL22>, CorrCta<22, SL22>::NTHREADS, classify_smem_bytes<22, SL22>())) return e;
    }
    // 6. one localisation launch, one CTA per tracked item; 7. one D2H and one synchronisation
    LocBatchArgs la;
    la.a = make_loc_args(1, b->Ho, b->Wo, &b->p, nullptr, nullptr);
    int tracked[kBatchMax], nt = 0;
    for (int k = 0; k < n; ++k) {
        if (items[k].init) continue;
        la.slot[nt] = items[k].slot;
        loc_inputs(b->t[items[k].slot], sa.g[k], la.neigh[nt], la.prev_vec[nt]);
        tracked[nt++] = k;
    }
    if (nt > 0) {
        const size_t smem = loc_smem_bytes(la.a);
        B200_REQUIRE(smem <= 48 * 1024, "dimp_batch_step: score pre-processing holds Ho*Wo=%d floats in shared memory", b->Ho * b->Wo);
        localize_batch_kernel<<<nt, 256, smem, st>>>(b->scores, la, b->loc_dev);
        B200_LAUNCH_CHECK();
        B200_CHECK_CUDA(cudaMemcpyAsync(b->loc_host, b->loc_dev, (size_t)nt * sizeof(b200trk_loc_result_t), cudaMemcpyDeviceToHost, st));
    }
    B200_CHECK_CUDA(cudaStreamSynchronize(st));
    // 8. the host half of every tracked frame; 9. each slot's memory insert and optimiser call, back to back on the stream
    const size_t plane = (size_t)b->Cc * b->Hc * b->Wc;
    for (int j = 0; j < nt; ++j) {
        const int k = tracked[j], slot = items[k].slot;
        b200trk_dimp_tracker* t = b->t[slot];
        if (int e = b200trk_dimp_tracker_commit(t, &sa.g[k], &b->loc_host[j], &infos[k], nullptr)) return e;
        if (int e = frame_update(t, b->clf + plane * slot, &infos[k], st)) return e;
    }
    // initialisation, as b200trk_dimp_tracker_initialize_host; a learnt initialiser's convolution runs once, at batch S like the forward
    const bool any_init = std::any_of(items, items + n, [](const b200trk_batch_item_t& it) { return it.init != 0; });
    if (any_init && b->net->finit.conv_op >= 0)
        if (int e = filter_init_conv(b->net, b->clf, b->cap, st)) return e;
    for (int k = 0; k < n; ++k) {
        if (!items[k].init) continue;
        const int slot = items[k].slot;
        b200trk_frame_info_t* info = &infos[k];
        std::memset(info, 0, sizeof(*info));
        info->crop = sa.g[k];
        for (int i = 0; i < 4; ++i) { info->bbox[i] = f32(items[k].init_bbox[i]); info->target_box[i] = box[k][i]; }
        info->updated = 1; info->n_stored = 1; info->num_iter = b->p.net_opt_iter > 0 ? b->p.net_opt_iter : 0;
        if (int e = first_frame_update(b->t[slot]->st, b->clf + plane * slot, b->cap, slot, box[k], info->num_iter, st)) return e;
    }
    return 0;
}

extern "C" int b200trk_dimp_batch_step_host(b200trk_dimp_batch_t* b, const b200trk_batch_item_t* items, int n, b200trk_frame_info_t* infos,
                                            b200trk_stream_t stream) {
    return batch_step(b, items, n, false, infos, stream);
}

extern "C" int b200trk_dimp_batch_step_device(b200trk_dimp_batch_t* b, const b200trk_batch_item_t* items, int n, b200trk_frame_info_t* infos,
                                              b200trk_stream_t stream) {
    return batch_step(b, items, n, true, infos, stream);
}
