// developer probe: the quad kernels alone (fast compile for SASS / register inspection).  The quad_loco_kernel and
// quad_rollout_kernel instantiations are the ones quad_loco_kernel_for and b2g_task_rollout launch (b200gym.cu).
#include <cuda_runtime.h>
#include "../isaacgymenvs_b200/csrc/b2g_device.cuh"
#include "../isaacgymenvs_b200/csrc/b2g_tasks.cuh"
#include "../isaacgymenvs_b200/csrc/b2g_common.cuh"
#include "../isaacgymenvs_b200/csrc/b2g_quad_kernels.cuh"
#define QUAD_LOCO(SP, HOSTIO, LEAN) \
    template __global__ void b2g::quad_loco_kernel<2, SP, 64, HOSTIO, LEAN>(const float4 *, Buffers, const __grid_constant__ b2g_task_params, const float *, int, int, TileArgs)
QUAD_LOCO(3, false, true);
QUAD_LOCO(0, false, true);
QUAD_LOCO(3, false, false);
QUAD_LOCO(0, false, false);
QUAD_LOCO(3, true, false);
QUAD_LOCO(0, true, false);
template __global__ void b2g::quad_simulate_kernel<2, false, 3, 128>(const float4 *, const int16_t *, Buffers, int, int);
template __global__ void b2g::quad_anymal_physics_kernel<true, 128, false>(const float4 *, const int16_t *, Buffers, const __grid_constant__ b2g_anymal_params, const float *, int, int, unsigned);
#include "../isaacgymenvs_b200/csrc/b2g_quad_rollout.cuh"
template __global__ void b2g::quad_rollout_kernel<2, 3>(const float4 *, Buffers, const __grid_constant__ b2g_task_params, int, int, const __grid_constant__ b2g::RollArgs);
template __global__ void b2g::quad_rollout_kernel<2, 0>(const float4 *, Buffers, const __grid_constant__ b2g_task_params, int, int, const __grid_constant__ b2g::RollArgs);
