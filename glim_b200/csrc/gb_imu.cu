// gb_imu.cu -- gb_imu_preintegrate: GLIM's IMU preintegration (IMUIntegration::integrate_imu over GTSAM's
// PreintegratedImuMeasurements) for many intervals in one launch (sm_90a).  The rule is stated in include/glim_b200.h and its
// arithmetic lives in gb_imu_math.cuh (also compiled for the host by the CPU test).  One fp64 thread per interval: the steps of
// an interval are a sequential recurrence, and a batch holds as many intervals as a global map has submaps or a sub-map
// odometry frames.
#include "gb_imu_math.cuh"
#include "gb_internal.cuh"

namespace {

constexpr int kImuThreads = 64;

__global__ void __launch_bounds__(kImuThreads) k_imu_preintegrate(const double* __restrict__ samples, int S, const double* __restrict__ intervals,
                                                                   const double* __restrict__ biases, int I, gb_imu_params prm, gb_imu_preintegrated* __restrict__ out) {
  const int i = (int)(blockIdx.x * blockDim.x + threadIdx.x);
  if (i >= I) return;
  gb_imu_preintegrated p;
  imu_preintegrate_interval(samples, S, intervals[2 * i], intervals[2 * i + 1], biases + 6 * (size_t)i, prm, p);
  out[i] = p;
}

}  // namespace

extern "C" gb_status gb_imu_default_params(gb_imu_params* p) {
  GB_REQUIRE(p, "null params");
  p->acc_noise = 0.05;  // config_sensors.json
  p->gyro_noise = 0.02;
  p->int_noise = 0.001;
  p->gravity[0] = 0.0;  // PreintegrationParams::MakeSharedU(9.81)
  p->gravity[1] = 0.0;
  p->gravity[2] = -9.81;
  return GB_OK;
}

extern "C" gb_status gb_imu_preintegrate(gb_ctx* ctx, size_t num_samples, const double* samples, size_t num_intervals, const double* intervals,
                                         const double* biases, const gb_imu_params* prm, gb_imu_preintegrated* out) {
  GB_REQUIRE(ctx, "null ctx");
  GB_REQUIRE(prm, "null params");
  GB_REQUIRE(num_intervals == 0 || (intervals && biases && out), "null interval arrays");
  GB_REQUIRE(num_samples == 0 || samples, "null samples");
  GB_REQUIRE(num_samples < ((size_t)1 << 28) && num_intervals < ((size_t)1 << 24), "too many samples or intervals");
  GB_REQUIRE(num_samples == 0 || gb_all_finite(samples, 7 * num_samples), "samples must be finite");
  for (size_t s = 1; s < num_samples; s++) GB_REQUIRE(samples[7 * s] >= samples[7 * (s - 1)], "sample times must not decrease");
  GB_REQUIRE(num_intervals == 0 || (gb_all_finite(intervals, 2 * num_intervals) && gb_all_finite(biases, 6 * num_intervals)),
             "intervals and biases must be finite");
  for (size_t i = 0; i < num_intervals; i++) GB_REQUIRE(intervals[2 * i] <= intervals[2 * i + 1], "an interval must not end before it starts");
  GB_REQUIRE(isfinite(prm->acc_noise) && isfinite(prm->gyro_noise) && isfinite(prm->int_noise) && prm->acc_noise >= 0.0 && prm->gyro_noise >= 0.0 &&
                 prm->int_noise >= 0.0,
             "IMU noises must be finite and >= 0");
  GB_REQUIRE(gb_all_finite(prm->gravity, 3), "gravity must be finite");
  if (num_intervals == 0) return GB_OK;
  const int S = (int)num_samples, I = (int)num_intervals;

  GB_ENTER(ctx);
  double* d_samples = nullptr;
  double* d_intervals = nullptr;
  double* d_biases = nullptr;
  gb_imu_preintegrated* d_out = nullptr;
  GB_CHECK(gb_carve(ctx, ctx->scratch, [&](Carver& cv) {
    d_samples = cv.take<double>(7 * (size_t)S);
    d_intervals = cv.take<double>(2 * (size_t)I);
    d_biases = cv.take<double>(6 * (size_t)I);
    d_out = cv.take<gb_imu_preintegrated>(I);
  }));
  GB_CHECK(gb_upload(ctx, {{d_samples, samples, sizeof(double) * 7 * (size_t)S},
                           {d_intervals, intervals, sizeof(double) * 2 * (size_t)I},
                           {d_biases, biases, sizeof(double) * 6 * (size_t)I}}));
  GB_CHECK(gb_launch(ctx, "k_imu_preintegrate", k_imu_preintegrate, (I + kImuThreads - 1) / kImuThreads, kImuThreads, 0, d_samples, S, d_intervals,
                     d_biases, I, *prm, d_out));
  return gb_download(ctx, {{out, d_out, sizeof(gb_imu_preintegrated) * (size_t)I}});
}
