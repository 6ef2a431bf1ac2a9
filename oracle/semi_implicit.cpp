// semi_implicit.cpp - TEST INFRASTRUCTURE ONLY.  C export of oracle_semi_implicit.h, the CPU checker of
// newton_b200.solvers.SolverSemiImplicit.
#include "oracle_semi_implicit.h"

extern "C" {

void orc_semi_implicit_step(const nb2_model_desc* m, const nb2_semi_implicit_params* p, const nb2_state_view* state_in,
                            const nb2_state_view* state_out, const nb2_control_view* control, const nb2_contacts_view* contacts, float dt) {
    orc::si::step(*m, *p, *state_in, *state_out, *control, contacts, dt);
}
}
