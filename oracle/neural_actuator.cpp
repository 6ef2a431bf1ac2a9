// neural_actuator.cpp - TEST INFRASTRUCTURE ONLY.  C export of oracle_neural_actuator.h, the CPU checker of the learned
// actuator networks.
#include "oracle_neural_actuator.h"

extern "C" {

void orc_neural_actuator_step(const nb2_actuator_step_desc* desc) { orc::neural::step(*desc); }

void orc_neural_actuator_reset(int32_t count, int32_t rows, int32_t width, const uint8_t* mask, float* a, float* b) {
    orc::neural::reset(count, rows, width, mask, a, b);
}
}
