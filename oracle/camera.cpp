// camera.cpp - TEST INFRASTRUCTURE ONLY.  C export of oracle_camera.h, the CPU checker of newton_b200.sensors.SensorTiledCamera.
#include "oracle_camera.h"

extern "C" {

void orc_camera_render(const nb2_raycast_view* view, const int* shape_tri_start, const int* shape_tri_count, const float* tris,
                       const nb2_camera_desc* camera, const int64_t* pixels, int64_t pixel_count) {
    orc::cam::render(*view, shape_tri_start, shape_tri_count, tris, *camera, pixels, pixel_count);
}
}
