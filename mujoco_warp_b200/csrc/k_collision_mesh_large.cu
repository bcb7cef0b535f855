// k_collision_mesh_large.cu -- the collision kernel for models whose mesh hulls exceed the fixed multi-contact buffers of k_collision_mesh.cu
// (a polygon of more than 32 vertices, or a vertex shared by more than 16 polygons): the CCD_MESH = 2 build of the same source, whose buffers
// are per-lane slices of global scratch sized from the model (MeshClipDev).  Models within those bounds keep k_collision_mesh.cu.
#define CCD_MESH 2
#define MJB_COLLISION_MESH_LARGE_TU
#include "k_collision.cu"
