// k_sensor_collision_large.cu -- the distance / normal / fromto sensor kernel for models whose mesh hulls exceed the fixed multi-contact buffers
// (see k_collision_mesh_large.cu): the CCD_MESH = 2 build of k_sensor_collision.cu.
#define CCD_MESH 2
#include "k_sensor_collision.cu"
