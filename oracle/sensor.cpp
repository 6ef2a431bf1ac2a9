// sensor.cpp - TEST INFRASTRUCTURE ONLY.  C export of oracle_sensor.h, the CPU checker of newton_b200.sensors.SensorContact.
#include "oracle_sensor.h"

extern "C" {

void orc_sensor_contact_update(const nb2_sensor_contact_view* sensor, const nb2_contacts_view* contacts, const float* body_q) {
    orc::sensor_contact_update(*sensor, *contacts, body_q);
}
}
