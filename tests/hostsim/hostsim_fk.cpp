// Host build of the forward-kinematics walk of fk_serial_kernel and fk_tree_kernel (pvb_device.cuh fk_walk) and of the
// tree plan's check and save slots (fk_tree_slots), behind a small C interface for tests/test_tree_cpu.py.  Test
// infrastructure only.
#include <vector>

#include "cuda_runtime.h"
#include "../../pytorch_volumetric_b200/csrc/pvb_device.cuh"

using namespace pvb;

// fk_tree_slots: -1 and load / save / n_saves for a pre-order, else the first frame that breaks it
extern "C" int simfk_tree_slots(const int32_t *parents, int n_frames, int8_t *load, int8_t *save, int *n_saves) {
    return fk_tree_slots(parents, n_frames, load, save, n_saves);
}

// fk_serial_kernel's walk for every configuration (n_frames <= 32, n_links <= 16; checked by the caller)
extern "C" void simfk_serial(const pvb_fk_frame *frames, int n_frames, const pvb_fk_link *links, int n_links,
                             const float *q, int n_cfg, int n_joints, float *out) {
    FkPlan<PVB_FK_MAX_FRAMES, PVB_FK_MAX_LINKS> plan;
    std::memset(&plan, 0, sizeof(plan));
    plan.n_frames = n_frames;
    plan.n_links = n_links;
    std::memcpy(plan.frame, frames, sizeof(pvb_fk_frame) * n_frames);
    std::memcpy(plan.link, links, sizeof(pvb_fk_link) * n_links);
    for (int a = 0; a < n_cfg; ++a) fk_walk<false>(plan, q, n_joints, n_cfg, a, out, nullptr, 0);
}

// fk_tree_kernel's walk for every configuration, the saved poses in a per-configuration array (stride 1); returns
// fk_tree_slots' result and walks nothing when it is not -1
extern "C" int simfk_tree(const pvb_fk_frame *frames, const int32_t *parents, int n_frames, const pvb_fk_link *links,
                          int n_links, const float *q, int n_cfg, int n_joints, float *out) {
    FkTreePlan<PVB_FK_TREE_MAX_FRAMES, PVB_FK_TREE_MAX_LINKS> plan;
    std::memset(&plan, 0, sizeof(plan));
    plan.n_frames = n_frames;
    plan.n_links = n_links;
    std::memcpy(plan.frame, frames, sizeof(pvb_fk_frame) * n_frames);
    std::memcpy(plan.link, links, sizeof(pvb_fk_link) * n_links);
    const int bad = fk_tree_slots(parents, n_frames, plan.load, plan.save, &plan.n_saves);
    if (bad >= 0) return bad;
    std::vector<float> saves(12 * (size_t)(plan.n_saves > 0 ? plan.n_saves : 1));
    for (int a = 0; a < n_cfg; ++a) fk_walk<true>(plan, q, n_joints, n_cfg, a, out, saves.data(), 1);
    return -1;
}
