// ocean_kernels.cuh -- launch interface between the C-ABI layer (ocean_api.cu) and the
// sm_90a kernels (ocean_kernels.cu).  Internal; the public surface is include/ocean.h.
#pragma once
#include <cstdint>
#include <cuda.h>
#include <cuda_runtime.h>

#include "../../include/ocean.h"

namespace ocean {

constexpr int kMaxMapSize = 1024;
constexpr int kTwiddleCount = kMaxMapSize - 1;   // stage s, index j (< 2^s) lives at (1<<s)-1+j

// Push constants of spectrum_compute.glsl:18-30 for one dirty cascade (already binary32).
struct SpectrumDispatch {
    int32_t cascade;
    int32_t seed_x, seed_y;
    float tile_x, tile_y;
    float alpha, peak_frequency, wind_speed, angle, depth, swell, detail, spread;
};

// Push constants of spectrum_modulate.glsl:24-29 and fft_unpack.glsl:20-25 for one cascade update.  tile_length and
// depth do not travel per update: everything spectrum_modulate derives from them (k_vec, k_unit, the dispersion
// relation, :59-61,49) is time-invariant and lives in the dispersion table `table_slot` points at (TableDispatch).
struct CascadeDispatch {
    int32_t cascade;
    int32_t table_slot;
    float time;
    float whitecap, foam_grow_rate, foam_decay_factor;   // factor = DETMATH exp(-foam_decay_rate), fft_unpack.glsl:62 (uniform per dispatch)
    uint32_t done_target;  // persistent kernel: value of done[done_slot] once this update's row pass is complete (wraps)
    uint32_t wait_target;  // multi-frame launches: value of colpass_done[cascade] once the column pass that last READ this update's
                           // half of the scratch (two frames back) is complete -- the row pass may then overwrite it
    uint32_t col_wait_target;  // multi-frame launches: value of colpass_done[cascade] once the PREVIOUS frame's column pass is complete
                               // (it owns the foam plane this update's column pass reads and the maps it overwrites)
    int32_t done_slot;     // row-pass completion counter of this update: cascade (scratch half 0) or 2 * num_cascades + cascade
                           // (half 1) -- one counter per half, because the row pass of frame f+1 runs beside the column pass
                           // of frame f and its items must not be counted towards frame f's row pass
    int32_t scratch_layer; // first of the cascade's two layer pairs in the row-pass scratch: 2 * cascade in half 0,
                           // 2 * (num_cascades + cascade) in half 1 (consecutive frames of a multi-frame launch alternate)
};
constexpr int kScratchHalves = 2;

// One dispersion table to (re)build: spectrum_modulate.glsl:59-61,49 for every wave vector of a tile.
struct TableDispatch {
    int32_t slot;
    float tile_x, tile_y, depth;
};

struct DeviceBuffers {
    int map_size;
    int num_cascades;
    float4* spectrum;      // [C][N][N] (Re h0(k), Im h0(k), Re h0(-k), -Im h0(-k))      RGBA32F
    float4* rowpass;       // [kScratchHalves][C][2][N][N] (re_a, re_b, im_a, im_b), pair p = layers (2p, 2p+1)
    uint2* displacement;   // [C][N][N] 4 x half                                          RGBA16F
    uint2* normal;         // [C][N][N] 4 x half, .a = copy of the foam state               RGBA16F
    uint16_t* foam;        // [C][N][N] half, the foam state (fft_unpack.glsl:61-64): read and written by the column pass
    float4* displacement_f32;  // optional taps (nullptr when disabled)
    float4* normal_f32;
    const float2* twiddles;    // [kTwiddleCount] global copy of the universal twiddle table
    float4* disp_table;        // [slots][N/2+1][N] (omega, k_vec.x, k_unit.y, k_unit.x) of texel (x, y), y <= N/2
    float* disp_kvy;           // [slots][N] k_vec.y of row y (first N/2+1 entries used)
    alignas(64) CUtensorMap rowpass_tmap;   // TMA descriptor of `rowpass` (kernel B panel loads)
};

// Builds the TMA descriptor of the row-pass scratch (driver entry point cuTensorMapEncodeTiled).
cudaError_t make_rowpass_tensor_map(void* rowpass, int map_size, int num_cascades, CUtensorMap* out);

// Opts the kernels of `map_size` into their dynamic shared-memory footprint (once per device).
cudaError_t configure_kernels(int map_size);

// Computes the universal twiddle table (fft_butterfly.glsl:27) into `twiddles_dev` and into the
// module's __constant__ copy used for warp-uniform lookups.
cudaError_t init_twiddles(float2* twiddles_dev, cudaStream_t stream);

// spectrum_compute.glsl for `count` dirty cascades (dispatch records in device memory).
cudaError_t launch_spectrum_compute(const DeviceBuffers& b, const SpectrumDispatch* dispatch_dev, int count,
                                    cudaStream_t stream);

// Dispersion tables (time-invariant part of spectrum_modulate.glsl: k_vec, k_unit, dispersion_relation) for `count`
// (tile_length, depth) keys, IEEE-exact operations in the shader's order.
cudaError_t launch_dispersion_tables(const DeviceBuffers& b, const TableDispatch* jobs_dev, int count, cudaStream_t stream);

// spectrum_modulate + row IFFT (kernel A) and column IFFT + fft_unpack (kernel B) for `count`
// cascades, issued as L2-sized chunks (chunk_cascades) of one launch pair each.
// Returns the number of kernels launched through *launched.  `mid` / `mid2` are recorded after kernel A / kernel B
// of the FIRST chunk: this path serves profiled updates (per-kernel timing for bench.py).
cudaError_t launch_cascade_update(const DeviceBuffers& b, const CascadeDispatch* dispatch_dev, int count,
                                  cudaStream_t stream, int* launched, cudaEvent_t mid, cudaEvent_t mid2);
int chunk_cascades(int map_size);

// Same work as launch_cascade_update in ONE persistent launch (work queue over A and B items, B items
// wait on per-cascade completion counters).  `dispatch_host` (<= kMaxPersistentCascades records) travels by
// value as a kernel parameter (constant bank).  queue_dev: [0] = work counter, [1 + s] = completion counter s (row pass of
// cascade c in scratch half 0: s = c, column pass: C + c, row pass in half 1: 2C + c; monotonic modulo 2^32;
// dispatch[i].done_target is the value of counter done_slot to wait for).  item_table_dev/total_items from
// build_item_table(map_size, count, persistent_group(map_size)); resident_ctas from persistent_grid_size().
constexpr int kMaxPersistentCascades = 256;
// multi_frame: the records describe several consecutive updates of the same cascades (build_item_table_frames): B items then
// publish their completion in queue_dev[1 + num_cascades + c] and A items wait for wait_target there.
// The work counter queue_dev[0] must be 0 at the launch and is 0 again once the launch is complete (no host reset).
// chained: the stream's previous operation is a persistent launch; this one is queued as its programmatic dependent, so its teams
// start their prologue while that launch drains (the kernel waits for the previous grid's completion before its first item).
cudaError_t launch_cascade_update_persistent(const DeviceBuffers& b, const CascadeDispatch* dispatch_host, int count,
                                             cudaStream_t stream, int* queue_dev, const int* item_table_dev, int total_items,
                                             int resident_ctas, bool multi_frame = false, bool chained = false);
int build_item_table(int map_size, int count, int group, int lag, int* out);
// Queue order of `frames` consecutive updates of the same `count` cascades in one launch: A(f0) A(f1) B(f0) A(f2) B(f1) ... with
// A(f) = the row-pass items of every cascade; slot of (frame f, cascade position c) = f * count + c.  Frames alternate between the
// halves of the scratch: A(f, c) waits for B(f-2, c) (CascadeDispatch::wait_target), B(f, c) for A(f, c) and B(f-1, c).
int build_item_table_frames(int map_size, int count, int frames, int* out);
int b_items_per_cascade(int map_size);
int persistent_group(int map_size);
int persistent_lag(int map_size);     // groups between the row pass and the column pass of a group in the queue order
cudaError_t persistent_grid_size(int map_size, int* out);
int a_items_per_cascade(int map_size);

// Compares the branch-free sqrt/div with __fsqrt_rn/__fdiv_rn on the device (debug entry point).
cudaError_t launch_selftest_math(unsigned long long* failures_dev, unsigned long long* tested_dev, cudaStream_t stream);

// Evaluates device math function `fn` (OCEAN_MATH_* of ocean.h) on n elements (debug entry point).
cudaError_t launch_debug_device_math(int fn, int n, const float* a_dev, const float* b_dev, float2* out_dev, cudaStream_t stream);

// De-interleaves one cascade of the row-pass scratch into [4][N][N][2] floats (debug tap).
cudaError_t launch_rowpass_export(const DeviceBuffers& b, int scratch_layer, float2* out_dev, cudaStream_t stream);
// ocean_sample.cu: batched map queries (water.gdshader:27-39,42-84); scales_dev = map_scales[num_cascades] as float4
cudaError_t launch_sample_maps(const DeviceBuffers& b, int num_cascades, const float2* points_dev, int n, const float4* scales_dev,
                               float* disp_out_dev, float* grad_out_dev, cudaStream_t stream);
// ocean_sample.cu: surface query (P + D_xz(P) = Q solved for P, then sampled; oracle/surface.py); out_dev = [n] records,
// scratch_dev = [surface_scratch_ints(num_cascades, n)] ints
size_t surface_scratch_ints(int num_cascades, int n);
cudaError_t launch_query_surface(const DeviceBuffers& b, int num_cascades, const float2* points_dev, int n, const float4* scales_dev,
                                 float tolerance, int max_iterations, ocean_surface_sample* out_dev, int* scratch_dev, cudaStream_t stream);
// A wake field the ray cast, spray, render map or sample reads (ocean_wake_set_readers; oracle/wake_readers.py): field and
// foam are [n][n] binary32 in the window at world corner (x0, z0), sampled as ocean_sample_wake (0 outside).  The ray cast
// reads the coupling's free surface e in `field`; the others read h in `field` and F in `foam` (null while wake foam is off:
// F reads +0).
struct WakeRead {
    const float* field;
    const float* foam;
    int n;
    float cell, x0, z0;
};
// ocean_sample.cu: ray cast against the displaced surface (oracle/raycast.py); rays_dev / out_dev = [n] rays / hits,
// bounds_dev = [3 * num_cascades] unsigned of scratch (the per-layer height and displacement bounds), [3 * num_cascades + 2]
// with a wake (wake not null: the coupled surface, its e bounds after the layers')
cudaError_t launch_raycast(const DeviceBuffers& b, int num_cascades, const ocean_ray* rays_dev, int n, const float4* scales_dev, float step,
                           int max_samples, float tolerance, int max_iterations, unsigned* bounds_dev, ocean_ray_hit* out_dev,
                           const WakeRead* wake, cudaStream_t stream);

// ocean_buoyancy.cu: buoyancy (oracle/buoyancy.py).  bodies_dev = [num_bodies], offsets_dev = the exclusive prefix of their
// num_points (body-major world points), q_dev / samples_dev = [n] world points' (x, z) / surface records, results_dev = [num_bodies]
cudaError_t launch_buoyancy_transform(const ocean_buoyancy_body* bodies_dev, const int* offsets_dev, int num_bodies,
                                      const ocean_buoyancy_point* points_dev, int n, float2* q_dev, cudaStream_t stream);
cudaError_t launch_buoyancy_reduce(const ocean_buoyancy_body* bodies_dev, const int* offsets_dev, int num_bodies,
                                   const ocean_buoyancy_point* points_dev, const ocean_surface_sample* samples_dev, float rho_g,
                                   float tolerance, ocean_buoyancy_result* results_dev, cudaStream_t stream);
// The drag half of the body-forces op (oracle/drag.py), on the same bodies, offsets, points and surface records:
// velocities_dev = [num_bodies], drag_areas_dev = [num_points] C_d A parallel to points_dev, velocity_dev = the velocity maps
// ([num_cascades used][map_size^2] 4 x half), results_dev = [num_bodies]; wake_wv_dev (may be null) = [n] vertical water
// velocities of the wake layer per world point, added to the water velocity's y (ocean_wake_set_coupling)
cudaError_t launch_drag_reduce(const ocean_buoyancy_body* bodies_dev, const ocean_body_velocity* velocities_dev, const int* offsets_dev,
                               int num_bodies, const ocean_buoyancy_point* points_dev, const float* drag_areas_dev,
                               const ocean_surface_sample* samples_dev, const uint2* velocity_dev, int map_size, int num_cascades,
                               const float4* scales_dev, float half_rho, ocean_drag_result* results_dev, const float* wake_wv_dev,
                               cudaStream_t stream);

// ocean_hull.cu: hull-mesh forces (oracle/hull.py).  bodies_dev / velocities_dev = [num_bodies], offsets_dev = the exclusive
// prefix of their meshes' num_vertices (body-major world vertices), meshes / vertices / triangles = the registered set;
// q_dev = [n] query points, corner_r_dev / corner_u_dev = [n] (r, w.y then d) and (u, 0) per world vertex, samples_dev = [n]
// surface records, wake_wv_dev (may be null) = [n] the wake's vertical velocities
cudaError_t launch_hull_transform(const ocean_hull_body* bodies_dev, const int* offsets_dev, int num_bodies, const ocean_hull_mesh* meshes_dev,
                                  const float* vertices_dev, int n, float2* q_dev, float4* corner_r_dev, cudaStream_t stream);
cudaError_t launch_hull_vertex(const ocean_surface_sample* samples_dev, int n, const uint2* velocity_dev, int map_size, int num_cascades,
                               const float4* scales_dev, const float* wake_wv_dev, float4* corner_r_dev, float4* corner_u_dev,
                               cudaStream_t stream);
cudaError_t launch_hull_reduce(const ocean_hull_body* bodies_dev, const ocean_body_velocity* velocities_dev, const int* offsets_dev,
                               int num_bodies, const ocean_hull_mesh* meshes_dev, const int* triangles_dev, const float4* corner_r_dev,
                               const float4* corner_u_dev, const ocean_surface_sample* samples_dev, float rho_g, float half_rho,
                               float tolerance, ocean_buoyancy_result* hydrostatic_dev, ocean_drag_result* drag_dev, cudaStream_t stream);

// ocean_bodies.cu: the floating-body integrator (oracle/bodies.py).  bodies_dev / states_dev = [num_bodies], r2_dev =
// [num_bodies] max |p|^2 over each hull, pose_dev / velocities_dev = the tables the body-forces kernels read.  prepare fills r2
// and the first sub-step's tables; integrate takes one sub-step of h from the records of the tables' pose and writes the next
// sub-step's tables, and the 3 x 4 transforms ([num_bodies][12]) when transforms_dev is not null.
cudaError_t launch_bodies_prepare(const ocean_floating_body* bodies_dev, const ocean_body_state* states_dev, int num_bodies,
                                  const ocean_buoyancy_point* points_dev, float* r2_dev, ocean_buoyancy_body* pose_dev,
                                  ocean_body_velocity* velocities_dev, cudaStream_t stream);
cudaError_t launch_bodies_integrate(const ocean_floating_body* bodies_dev, const float* r2_dev, int num_bodies,
                                    const ocean_buoyancy_result* hydrostatic_dev, const ocean_drag_result* drag_dev, float density, float h,
                                    ocean_body_state* states_dev, ocean_buoyancy_body* pose_dev, ocean_body_velocity* velocities_dev,
                                    float* transforms_dev, cudaStream_t stream);
// prepare for hull meshes (ocean_simulate_hull_bodies): r2 over the mesh's vertices, pose rows of ocean_hull_body, which
// launch_bodies_integrate takes as ocean_buoyancy_body rows (same layout; it writes only the transform), and rows_dev =
// [num_bodies] the ocean_floating_body rows (mass, inertia) launch_bodies_integrate reads
cudaError_t launch_hull_prepare(const ocean_floating_hull* bodies_dev, const ocean_body_state* states_dev, int num_bodies,
                                const ocean_hull_mesh* meshes_dev, const float* vertices_dev, float* r2_dev, ocean_hull_body* pose_dev,
                                ocean_body_velocity* velocities_dev, ocean_floating_body* rows_dev, cudaStream_t stream);
// The driven form of integrate: the forces, torques and step denominators of each body from launch_drive_reduce's sums_dev.
struct DriveSum {
    float force[3], torque[3];      // hyd + drg, then the drive contributions in incidence order
    float den_v, den_w[3];          // mass + h c_v (+ tethers), inertia + h c_w (+ tethers)
};
cudaError_t launch_bodies_integrate_driven(const ocean_floating_body* bodies_dev, int num_bodies, const DriveSum* sums_dev, float h,
                                           ocean_body_state* states_dev, ocean_buoyancy_body* pose_dev, ocean_body_velocity* velocities_dev,
                                           float* transforms_dev, cudaStream_t stream);

// ocean_drive.cu: thrusters, foils, loads and tethers of the driven integrator (oracle/drive.py).  Actuator k (the thrusters,
// then the foils) has world point world + k of the surface query.  One tether record per tether from the sub-step's tables:
struct TetherForce {
    float force[3];                 // T u, on body_a; body_b gets -T u
    float torque_a[3], torque_b[3]; // r_a x (T u), r_b x (-T u)
    float tension;                  // 0: slack, the tether adds nothing
};
struct DriveArgs {
    const ocean_thruster* thrusters;    // [num_thrusters] device
    int num_thrusters;
    const ocean_foil* foils;            // [num_foils] device
    int num_foils;
    const ocean_tether* tethers;        // [num_tethers] device
    int num_tethers;
    const ocean_body_load* loads;       // [num_bodies] device, or null
    const int* incidence_offsets;       // [num_bodies + 1] device: each body's range of incidence
    const int* incidence;               // thruster k -> k, foil k -> T + k, tether k end e -> T + F + 2 k + e
};
cudaError_t launch_actuator_transform(const DriveArgs& d, const ocean_buoyancy_body* pose_dev, float2* q_dev, cudaStream_t stream);
cudaError_t launch_tethers(const DriveArgs& d, const ocean_buoyancy_body* pose_dev, const ocean_body_velocity* velocities_dev,
                           TetherForce* forces_dev, float* tensions_dev, cudaStream_t stream);
cudaError_t launch_drive_reduce(const DriveArgs& d, int num_bodies, const ocean_floating_body* bodies_dev, const float* r2_dev,
                                const ocean_buoyancy_body* pose_dev, const ocean_body_velocity* velocities_dev,
                                const ocean_buoyancy_result* hydrostatic_dev, const ocean_drag_result* drag_dev,
                                const ocean_surface_sample* actuator_samples_dev, const float* actuator_wv_dev, const TetherForce* tether_forces_dev,
                                const uint2* velocity_dev, int map_size, int num_cascades, const float4* scales_dev, float density, float h,
                                DriveSum* sums_dev, ocean_drive_result* drive_dev, cudaStream_t stream);

// ocean_velocity.cu: velocity maps (oracle_velocity_update).  One record per cascade to recompute: the table slot and time of
// the update that built the cascade's current maps.
struct VelocityDispatch {
    int32_t cascade;
    int32_t table_slot;
    float time;
};
constexpr int kMaxVelocityLaunch = 256;   // records per launch pair (they travel by value)
// Copies the twiddle table into ocean_velocity.cu's constant bank (once per device before its first launch).
cudaError_t init_velocity_twiddles(const float2* twiddles_dev, cudaStream_t stream);
// Row pass into scratch_dev ([C][N][N] float4), column pass into velocity_dev ([C][N][N] 4 x half) and, when not null,
// velocity_f32_dev ([C][N][N] float4).  *launched receives the number of kernels launched.
cudaError_t launch_velocity(const DeviceBuffers& b, const VelocityDispatch* jobs_host, int count, float4* scratch_dev, uint2* velocity_dev,
                            float4* velocity_f32_dev, cudaStream_t stream, int* launched);
// ocean_sample.cu: the displacement half of launch_sample_maps on the velocity map: out_dev = [n][3] floats
cudaError_t launch_sample_velocity(const uint2* velocity_dev, int map_size, int num_cascades, const float2* points_dev, int n,
                                   const float4* scales_dev, float* out_dev, cudaStream_t stream);

// ocean_spray.cu: spray candidates (sea_spray_particle.gdshader:80-94) as a stable stream compaction; counts_dev is
// [spray_blocks(n) + 1] ints of scratch whose last element receives the number of active candidates
int spray_blocks(int n);
// wake (may be null): the wake forms of the kernels, which add the layer's h and F to the spawn test (and h to the particle height)
cudaError_t launch_extract_spray(const DeviceBuffers& b, int num_cascades, const float2* points_dev, int n, const float4* scales_dev,
                                 float3 particle_scale, int* counts_dev, ocean_spray_record* records_dev, int max_records,
                                 const WakeRead* wake, cudaStream_t stream);
// ocean_spray.cu: one particle-process frame [t0, t1) of a spray emitter (oracle/spray_particles.py), three launches when
// amount > 0.  states_dev = [amount] (updated in place), counts_dev = [spray_blocks(amount) + 1] ints of scratch whose last
// element receives the number of live particles, instances_dev = [max_instances][16] floats
cudaError_t launch_spray_particles(const DeviceBuffers& b, int num_cascades, const float4* scales_dev, const ocean_spray_emitter& emitter,
                                   double t0, double t1, ocean_spray_particle* states_dev, int* counts_dev, float* instances_dev,
                                   int max_instances, const WakeRead* wake, cudaStream_t stream);

// ocean_drift.cu: the sea state (oracle/sea_state.py).  One job per cascade to recompute: its spectrum layer and the dispersion
// table its updates use.  moments_dev = [num_cascades][kSeaStateMoments] binary64 (m-1, m0, m1, m2, sum E d.x, sum E d.z,
// sum E kx^2, sum E kz^2, u_s.x, u_s.z); partial_dev = [min(count, kMaxSeaStateLaunch)][sea_state_blocks(N)][kSeaStateMoments]
// of scratch.  Two launches per kMaxSeaStateLaunch jobs; *launched receives the number of kernels launched.
struct SeaStateJob {
    int32_t cascade;
    int32_t table_slot;
};
constexpr int kSeaStateMoments = 10;
constexpr int kMaxSeaStateLaunch = 256;
int sea_state_blocks(int map_size);
cudaError_t launch_sea_state(const DeviceBuffers& b, const SeaStateJob* jobs_host, int count, double* partial_dev, double* moments_dev,
                             cudaStream_t stream, int* launched);
// ocean_drift.cu: the drifters (oracle/drifters.py), one launch.  drifters_dev = [n] (advanced in place when dt > 0),
// instances_dev = [n][12] floats or null (no render); wake (may be null) = the layer's h the render reads.
cudaError_t launch_drift(const DeviceBuffers& b, int num_cascades, const float4* scales_dev, const double* moments_dev,
                         const ocean_drift_params& params, double dt, ocean_drifter* drifters_dev, int n, float* instances_dev,
                         const WakeRead* wake, cudaStream_t stream);

// ocean_wake.cu: the wake layer (oracle/wake.py).  One sub-step of the layer: h / h_prev ([n][n], read at (i + di, j + dj),
// 0 outside: the scroll folded into the reads) to out_h, and, when out_h_prev is not null, the scrolled h to out_h_prev.
// a1..a3 are the per-ring coefficients, index min(cells to the window edge, sponge_cells).
constexpr int kWakeMaxSponge = 64;
struct WakeStepArgs {
    const float* h;
    const float* h_prev;
    float* out_h;
    float* out_h_prev;
    const ocean_wake_source* sources;               // [num_sources]
    const ocean_body_state* states;                 // [num_states]
    int num_sources, num_states;
    int n, di, dj, sponge_cells;
    float cell, x0, z0, tau;
    float a1[kWakeMaxSponge + 1], a2[kWakeMaxSponge + 1], a3[kWakeMaxSponge + 1];
};
void wake_kernel_taps(float* out);                  // host: the 28 taps in the specification's order
// The obstacle mask (ocean_wake_set_obstacles; oracle/wake_obstacles.py) in the call's window: window cell (i, j) is blocked
// iff q = qx + i and r = qz + j lie in [0, width) x [0, depth) and mask[r][q] != 0.  qx = origin_x - mask origin x,
// computed exactly and clamped to [-2^30, 2^30] (a clamped offset leaves every cell of the halo outside the mask, as the
// exact one does), so q and r are exact in int.
struct WakeObstacles {
    const uint8_t* mask;                            // [depth][width] bytes, nonzero = blocked
    int width, depth;
    int qx, qz;
};
// The foam sub-step (ocean_wake_set_foam; oracle/wake_foam.py): the sub-step of `step`, and F ([n][n], read at (i + di, j + dj),
// 0 outside) advanced to out_foam (another [n][n] field) with the call's constants.
struct WakeFoamStepArgs {
    WakeStepArgs step;
    const float* foam;
    float* out_foam;
    float whitecap;
    float decay;                                    // d = exp(-decay_rate h)
    float grow, stir;                               // grow_rate h, stir_rate h
};
// One sub-step of args; with foam not null the foam sub-step (foam->step is replaced by args), with obstacles not null the
// obstacle form: blocked cells read s = 0 and are written 0 (h and F; h_prev is written unmasked).
cudaError_t launch_wake_step(const WakeStepArgs& args, const WakeFoamStepArgs* foam, const WakeObstacles* obstacles, cudaStream_t stream);
// map_dev = [n][n][4] half (h, dh/dx, dh/dz, F) of wake.field and wake.foam (F = 0 when it is null); out_dev = [count][3] floats
cudaError_t launch_wake_map(const WakeRead& wake, void* map_dev, cudaStream_t stream);
cudaError_t launch_wake_sample(const WakeRead& wake, const float2* xz_dev, int count, float* out_dev, cudaStream_t stream);
// The coupling (ocean_wake_set_coupling; oracle/wake_coupling.py).  free_surface: e = h + phi of the sources at tau (the end
// of the step call) in the window at corner (x0, z0), into e, and into e_old when it is not null (a priming call).
struct WakeFreeSurfaceArgs {
    const float* h;                                 // [n][n], the layer after the call's sub-steps
    float* e;                                       // [n][n]
    float* e_old;                                   // [n][n] or null
    const ocean_wake_source* sources;               // [num_sources]
    const ocean_body_state* states;                 // [num_states]
    int num_sources, num_states;
    int n;
    float cell, x0, z0, tau;
};
// With obstacles not null, e = 0 on blocked cells.
cudaError_t launch_wake_free_surface(const WakeFreeSurfaceArgs& args, const WakeObstacles* obstacles, cudaStream_t stream);
// The snapshots e and e_old ([n][n]) with their window corners, and the interval T between them.
struct WakeCoupleArgs {
    const float* e;
    const float* e_old;
    int n;
    float cell, x0, z0, x0_old, z0_old, interval;
};
// couple: records_dev[k] += sample(e, q_dev[k]) (height into displacement[1], slopes into gradient_foam[0..1]); wv_dev (may be
// null) = [count] vertical velocities (sample(e) - sample(e_old)) / T
cudaError_t launch_wake_couple(const WakeCoupleArgs& args, const float2* q_dev, int count, ocean_surface_sample* records_dev, float* wv_dev,
                               cudaStream_t stream);

}  // namespace ocean
