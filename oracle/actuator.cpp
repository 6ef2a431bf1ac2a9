// actuator.cpp - TEST INFRASTRUCTURE ONLY.  C export of oracle_actuator.h, the CPU checker of newton_b200.actuators.
#include "oracle_actuator.h"

extern "C" {

void orc_actuator_step(const nb2_actuator_step_desc* desc) { orc::act::step(*desc); }

void orc_actuator_reset(int32_t count, int32_t buf_depth, const uint8_t* mask, float* buf_pos, float* buf_vel, float* buf_act,
                        int32_t* num_pushes, int32_t* write_idx, float* integral) {
    orc::act::reset(count, buf_depth, mask, buf_pos, buf_vel, buf_act, num_pushes, write_idx, integral);
}

void orc_actuator_param_copy(int32_t gather, const int32_t* map, int32_t entries, int32_t dofs_per_world, const uint8_t* world_mask,
                             const void* src, void* dst) {
    orc::act::param_copy(gather != 0, map, entries, dofs_per_world, world_mask, static_cast<const uint32_t*>(src),
                         static_cast<uint32_t*>(dst));
}
}
