// site_sensor.cpp - TEST INFRASTRUCTURE ONLY.  C export of oracle_site_sensor.h, the CPU checker of
// newton_b200.sensors.SensorFrameTransform and SensorIMU.
#include "oracle_site_sensor.h"

extern "C" {

void orc_sensor_frame_transform_update(const nb2_sensor_frame_transform_view* sensor, const float* body_q) {
    orc::sensor_frame_transform_update(*sensor, body_q);
}

void orc_sensor_imu_update(const nb2_sensor_imu_view* sensor, const float* body_q, const float* body_qd, const float* body_qdd) {
    orc::sensor_imu_update(*sensor, body_q, body_qd, body_qdd);
}
}
