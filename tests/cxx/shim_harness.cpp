// shim_harness.cpp -- extern "C" access to the drop-in shim (compat/gpu_process_shim.cpp), for tests/shim_lib.py.
//
// Built into a shared library together with the unmodified shim source (tests/test_cxx_facade.py:compile_with_shim).
// The nine entry points are declared exactly as the node's callers declare them (ElevationMapping.cpp:44-50,
// SensorProcessorBase.cpp:34), and the ref_* functions have the shape of oracle/ref_harness.cu's, so the same Python
// driver runs the reference's kernels and the shim.  The node can only observe the map through Map_feature's outputs,
// so there is no layer access here.
#include <Eigen/Core>

void Move(float *current_Position, float resolution, int length, float *h_central_coordinate, int *h_start_indice, float *position_shift);
void Init_GPU_elevationmap(int length, float resolution, float h_mahalanobisDistanceThreshold_, float h_obstacle_threshold);
void Map_closeloop(float *update_position, float height_update, int length, float resolution);
void Raytracing(int length_);
void Fuse(int length, int point_num, int *point_index, int *point_colorR, int *point_colorG, int *point_colorB, float *point_intensity, float *point_height, float *point_var);
void Map_feature(int length, float *elevation, float *var, int *point_colorR, int *point_colorG, int *point_colorB, float *rough, float *slope, float *traver, float *intensity);
void Map_optmove(float *opt_p, float height_update, float resolution, int length, float *opt_alignedPosition);
void Mapvar_update(int length, float var_update);
int Process_points(int *mapindex, float *point_x, float *point_y, float *point_z, float *point_var, float *point_x_ts, float *point_y_ts, float *point_z_ts, Eigen::Matrix4f Transform, int point_num, double relativeLowerThreshold, double relativeUpperThreshold, float min_r, float beam_a, float beam_c, Eigen::RowVector3f sensorJacobian, Eigen::Matrix3f rotationVariance, Eigen::Matrix3f C_SB_transpose, Eigen::RowVector3f P_mul_C_BM_transpose, Eigen::Matrix3f B_r_BS_skew);

static int g_length = 0;

extern "C" {

void ref_init(int length, float resolution, float mahalanobis, float obstacle_threshold)
{
    g_length = length;
    Init_GPU_elevationmap(length, resolution, mahalanobis, obstacle_threshold);
}
void ref_move(const float pos[3], float centre_out[2], int start_out[2], float shift_out[2], float resolution)
{
    float p[3] = {pos[0], pos[1], pos[2]};
    Move(p, resolution, g_length, centre_out, start_out, shift_out);
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
    return Process_points(key, x, y, z, var, x_ts, y_ts, z_ts, Tm, n, lo, hi, min_r, beam_a, beam_c, sj, rv, cs, pm, bs);
}
void ref_fuse(int n, int *key, int *R, int *G, int *B, float *intensity, float *h, float *var)
{
    Fuse(g_length, n, key, R, G, B, intensity, h, var);
}
void ref_var_update(float dv) { Mapvar_update(g_length, dv); }
void ref_map_feature(float *elevation, float *var, int *R, int *G, int *B, float *rough, float *slope, float *traver, float *intensity)
{
    Map_feature(g_length, elevation, var, R, G, B, rough, slope, traver, intensity);
}
void ref_raytracing(void) { Raytracing(g_length); }
void ref_optmove(float opt_p[2], float height_update, float resolution, float aligned_out[2])
{
    Map_optmove(opt_p, height_update, resolution, g_length, aligned_out);
}
void ref_closeloop(float p[2], float height_update, float resolution)
{
    Map_closeloop(p, height_update, g_length, resolution);
}

} // extern "C"
