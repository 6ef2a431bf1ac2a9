// controller.cpp - TEST INFRASTRUCTURE ONLY.  C export of oracle_controller.h, the CPU checker of newton_b200.controllers.
#include "oracle_controller.h"

extern "C" {

void orc_joint_impedance_gather_state(const nb2_joint_impedance_desc* desc) { orc::ji::gather_state(*desc); }

void orc_joint_impedance_step(const nb2_joint_impedance_desc* desc) { orc::ji::step(*desc); }
}
