// ref_harness.cu -- extern "C" access to the REFERENCE's own GPU library (TEST INFRASTRUCTURE).
//
// oracle/build_ref.py compiles the reference's elevation_mapping/elevation_mapping/cuda/
// gpu_process.cu unmodified, from where it lies, together with this file into
// oracle/_ref/libgpu_ref*.so (nothing of the reference is copied into the repository).  The
// reference exports nine C++-mangled functions taking Eigen types by value (gpu_process.cu:940,
// 1004, 1085, 1146, 1154, 1215, 1235, 1256, 1304); this harness re-declares them exactly like
// their callers do (ElevationMapping.cpp:44-50, SensorProcessorBase.cpp:34) and forwards plain
// C arrays, so tests can drive the real reference kernels on a GPU and compare them with
// the CPU oracle (tests/golden/make_reference_pin.py, tests/golden/make_golden.py).
#include <cuda_runtime.h>
#include <Eigen/Core>

// --- the reference's entry points, declared as its own callers declare them -----------------
void Move(float *current_Position, float resolution, int length, float *h_central_coordinate, int *h_start_indice, float *position_shift);
void Init_GPU_elevationmap(int length, float resolution, float h_mahalanobisDistanceThreshold_, float h_obstacle_threshold);
void Map_closeloop(float *update_position, float height_update, int length, float resolution);
void Raytracing(int length_);
void Fuse(int length, int point_num, int *point_index, int *point_colorR, int *point_colorG, int *point_colorB, float *point_intensity, float *point_height, float *point_var);
void Map_feature(int length, float *elevation, float *var, int *point_colorR, int *point_colorG, int *point_colorB, float *rough, float *slope, float *traver, float *intensity);
void Map_optmove(float *opt_p, float height_update, float resolution, int length, float *opt_alignedPosition);
void Mapvar_update(int length, float var_update);
int Process_points(int *mapindex, float *point_x, float *point_y, float *point_z, float *point_var, float *point_x_ts, float *point_y_ts, float *point_z_ts, Eigen::Matrix4f Transform, int point_num, double relativeLowerThreshold, double relativeUpperThreshold, float min_r, float beam_a, float beam_c, Eigen::RowVector3f sensorJacobian, Eigen::Matrix3f rotationVariance, Eigen::Matrix3f C_SB_transpose, Eigen::RowVector3f P_mul_C_BM_transpose, Eigen::Matrix3f B_r_BS_skew);

// device-global layer pointers and scroll state of the reference (gpu_process.cu:20-33); needs -rdc=true
extern __device__ float *map_lowest;
extern __device__ float *map_traver;
extern __device__ float *map_elevation;
extern __device__ float *map_variance;
extern __device__ float *map_intensity;
extern __device__ int *map_colorR;
extern __device__ int *map_colorG;
extern __device__ int *map_colorB;
extern __device__ float central_coordinate[2];
extern __device__ int start_indice[2];
extern __device__ float sensorZatLowestScan;

static int g_length = 0;

extern "C" {

void ref_init(int length, float resolution, float mahalanobis, float obstacle_threshold)
{
    g_length = length;
    Init_GPU_elevationmap(length, resolution, mahalanobis, obstacle_threshold);
    cudaDeviceSynchronize();
}
void ref_move(const float pos[3], float centre_out[2], int start_out[2], float shift_out[2], float resolution)
{
    float p[3] = {pos[0], pos[1], pos[2]};
    Move(p, resolution, g_length, centre_out, start_out, shift_out);
    cudaDeviceSynchronize();
}
int ref_process_points(int *key, float *x, float *y, float *z, float *var, float *x_ts, float *y_ts, float *z_ts,
                       const float T[16], int n, double lo, double hi, float min_r, float beam_a, float beam_c,
                       const float sJ[3], const float rotVar[9], const float CSBT[9], const float P[3], const float Bskew[9])
{
    Eigen::Matrix4f Tm;
    Eigen::Matrix3f rv, cs, bs;
    Eigen::RowVector3f sj, pm;
    for (int i = 0; i < 4; i++)
        for (int j = 0; j < 4; j++) Tm(i, j) = T[4 * i + j];
    for (int i = 0; i < 3; i++) {
        sj(0, i) = sJ[i];
        pm(0, i) = P[i];
        for (int j = 0; j < 3; j++) { rv(i, j) = rotVar[3 * i + j]; cs(i, j) = CSBT[3 * i + j]; bs(i, j) = Bskew[3 * i + j]; }
    }
    const int rc = Process_points(key, x, y, z, var, x_ts, y_ts, z_ts, Tm, n, lo, hi, min_r, beam_a, beam_c, sj, rv, cs, pm, bs);
    cudaDeviceSynchronize();
    return rc;
}
void ref_fuse(int n, int *key, int *R, int *G, int *B, float *intensity, float *h, float *var)
{
    Fuse(g_length, n, key, R, G, B, intensity, h, var);
    cudaDeviceSynchronize();
}
void ref_var_update(float dv) { Mapvar_update(g_length, dv); cudaDeviceSynchronize(); }
void ref_map_feature(float *elevation, float *var, int *R, int *G, int *B, float *rough, float *slope, float *traver, float *intensity)
{
    Map_feature(g_length, elevation, var, R, G, B, rough, slope, traver, intensity);
    cudaDeviceSynchronize();
}
void ref_raytracing(void) { Raytracing(g_length); }
void ref_optmove(float opt_p[2], float height_update, float resolution, float aligned_out[2])
{
    Map_optmove(opt_p, height_update, resolution, g_length, aligned_out);
    cudaDeviceSynchronize();
}
void ref_closeloop(float p[2], float height_update, float resolution)
{
    Map_closeloop(p, height_update, g_length, resolution);
    cudaDeviceSynchronize();
}
// read / write one of the reference's device layers (0 lowest, 1 traver, 2 elevation, 3 variance, 4 intensity,
// 5 colorR, 6 colorG, 7 colorB); every layer has 4-byte elements (float or int)
static void *layer_ptr(int which)
{
    void *p = nullptr;
    if (which == 0) cudaMemcpyFromSymbol(&p, map_lowest, sizeof p);
    else if (which == 1) cudaMemcpyFromSymbol(&p, map_traver, sizeof p);
    else if (which == 2) cudaMemcpyFromSymbol(&p, map_elevation, sizeof p);
    else if (which == 3) cudaMemcpyFromSymbol(&p, map_variance, sizeof p);
    else if (which == 4) cudaMemcpyFromSymbol(&p, map_intensity, sizeof p);
    else if (which == 5) cudaMemcpyFromSymbol(&p, map_colorR, sizeof p);
    else if (which == 6) cudaMemcpyFromSymbol(&p, map_colorG, sizeof p);
    else cudaMemcpyFromSymbol(&p, map_colorB, sizeof p);
    return p;
}
void ref_get_layer(int which, void *host_out)
{
    cudaMemcpy(host_out, layer_ptr(which), 4 * (size_t)g_length * g_length, cudaMemcpyDeviceToHost);
}
void ref_set_layer(int which, const void *host_in)
{
    cudaMemcpy(layer_ptr(which), host_in, 4 * (size_t)g_length * g_length, cudaMemcpyHostToDevice);
}
// the scroll state Move, Map_optmove and Map_closeloop keep in device globals (gpu_process.cu:30-33)
void ref_get_state(float centre_out[2], int start_out[2], float *sensor_z_out)
{
    cudaMemcpyFromSymbol(centre_out, central_coordinate, sizeof(float) * 2);
    cudaMemcpyFromSymbol(start_out, start_indice, sizeof(int) * 2);
    cudaMemcpyFromSymbol(sensor_z_out, sensorZatLowestScan, sizeof(float));
}
int ref_last_cuda_error(void) { return (int)cudaGetLastError(); }

} // extern "C"
