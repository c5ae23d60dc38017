/*
 * include/ocean.h -- C ABI of libocean.so, the H100-native drop-in for the wave-generation
 * hot path of 2Retr0/GodotOceanWaves (spectrum -> time propagation -> 4 packed N x N inverse
 * FFTs -> displacement / normal / Jacobian-foam maps).
 *
 * Each entry point names the reference interface it replaces (paths relative to the
 * reference repository).  Everything is plain C: opaque handle, POD structs, raw pointers
 * and sizes.  Every function returns an int status (OCEAN_OK == 0) and never throws or
 * aborts; ocean_last_error() returns a thread-local description of the last failure.
 *
 * Threading: a generator is NOT thread-safe (the reference runs on Godot's main thread,
 * assets/water/wave_generator.gd:19).  All GPU work of a generator is issued on its own
 * CUDA stream; calls are asynchronous w.r.t. the GPU until ocean_synchronize() or a
 * *_to_host call without the _async suffix.
 *
 * Ownership: the library owns all device memory (cf. RenderingContext's DeletionQueue,
 * assets/render_context.gd:4-21,40-46); callers borrow device pointers that stay valid until
 * ocean_destroy().  Changing map_size or the cascade count = destroy + create, as in
 * assets/water/water.gd:22-41,84-91.
 */
#ifndef OCEAN_H
#define OCEAN_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define OCEAN_OK 0
#define OCEAN_ERR_INVALID_ARGUMENT 1
#define OCEAN_ERR_CUDA 2
#define OCEAN_ERR_UNSUPPORTED 3
#define OCEAN_ERR_STATE 4

#define OCEAN_MAX_MAP_SIZE 1024 /* assets/shaders/compute/fft_compute.glsl:9 */
#define OCEAN_MIN_MAP_SIZE 128  /* assets/water/water.gd:38, wave_generator.gd:46 */

typedef struct ocean_generator ocean_generator; /* replaces the WaveGenerator node, wave_generator.gd:2 */

/* POD mirror of the WaveCascadeParameters resource, assets/water/wave_cascade_parameters.gd:2-42.
 * GDScript floats are binary64; Vector2 components are binary32.  The library rounds to
 * binary32 exactly where RenderingContext.create_push_constant does (render_context.gd:122-135). */
typedef struct ocean_cascade_params {
    float tile_length[2];             /* :7   metres */
    double displacement_scale;        /* :9   render-side only (map_scales, water.gd:102-110) */
    double normal_scale;              /* :11  render-side only */
    double wind_speed;                /* :15  m/s, clamped >= 1e-4 by the setter */
    double wind_direction;            /* :17  degrees */
    double fetch_length;              /* :20  kilometres, clamped >= 1e-4 */
    double swell;                     /* :22 */
    double spread;                    /* :25 */
    double detail;                    /* :28 */
    double whitecap;                  /* :32 */
    double foam_amount;               /* :34 */
    int32_t spectrum_seed[2];         /* :37 */
    int32_t should_generate_spectrum; /* :38  dirty flag; cleared by the library when it regenerates */
    double time;                      /* :40  advanced by ocean_update */
    double foam_grow_rate;            /* :41  written by ocean_update */
    double foam_decay_rate;           /* :42  written by ocean_update */
} ocean_cascade_params;

typedef struct ocean_info {
    int32_t device;
    int32_t map_size;
    int32_t num_cascades;
    int32_t pending_cascades;      /* pass_num_cascades_remaining, wave_generator.gd:15 */
    uint64_t kernel_launches;      /* kernels launched by this generator since creation */
    uint64_t cascade_updates;      /* cascade updates executed since creation */
    uint64_t device_bytes;         /* device memory owned by the generator */
} ocean_info;

/* class defaults of wave_cascade_parameters.gd:7-42 */
int ocean_default_cascade_params(ocean_cascade_params* out);

/* WaveGenerator.map_size + WaveGenerator.init_gpu(num_cascades), wave_generator.gd:8,17-54.
 * map_size in {128,256,512,1024} (water.gd:38); num_cascades >= 1 (the reference passes
 * max(2, n), water.gd:91 -- callers may do the same).  Allocates the spectrum (RGBA32F x
 * layers), the row-pass scratch, the two RGBA16F layered maps and the twiddle table. */
int ocean_create(int device, int map_size, int num_cascades, ocean_generator** out);

/* NOTIFICATION_PREDELETE -> context.free(), wave_generator.gd:111-113, render_context.gd:40-46 */
int ocean_destroy(ocean_generator* gen);

/* WaveGenerator.update(delta, parameters), wave_generator.gd:90-109: flushes cascades
 * 0..remaining-1 left from the previous pass, then time += delta and the foam rates for every
 * element of parameters[0..count), then arms `count` pending cascades.  `parameters` is in/out
 * (time, foam rates and the dirty flags of flushed cascades are written back). */
int ocean_update(ocean_generator* gen, double delta, ocean_cascade_params* parameters, int count);

/* WaveGenerator._process, wave_generator.gd:56-63: runs ONE pending cascade (highest index
 * first).  If `parameters` is non-NULL the live values are re-read (the reference dereferences the
 * live Resource objects) and the dirty flag is written back.  No-op when nothing is pending. */
int ocean_process(ocean_generator* gen, ocean_cascade_params* parameters, int count);

/* Batched fast path: ocean_update() followed by all pending cascades in one fused launch pair
 * (what `count` rendered frames of _process produce; cascades are independent,
 * wave_generator.gd:96-97). */
int ocean_update_all(ocean_generator* gen, double delta, ocean_cascade_params* parameters, int count);

/* `frames` consecutive ocean_update_all(delta) calls of the same resident cascades, fused: after the first frame the
 * remaining ones run `256 / count` frames per launch, chained on the device through per-cascade completion counters (consecutive
 * frames use alternate halves of the row-pass scratch: the row pass of frame f+1 runs beside the column pass of frame f and only
 * waits for the column pass of frame f-1, the column pass of frame f+1 for its own row pass and -- foam plane -- for the column
 * pass of frame f; the times are accumulated on the host in binary64, one addition per frame, exactly as wave_generator.gd:103 does).  Results are bit-identical to the frame-by-frame
 * calls; what it removes is the per-frame launch and host latency (SURVEY 8d cfg3: 1000-frame foam accumulate/decay loop). */
int ocean_update_frames(ocean_generator* gen, double delta, ocean_cascade_params* parameters, int count, int frames);

/* ---- the Water node's side of the hand-off (assets/water/water.gd), for hosts that do not bring their own ----
 * ocean_scheduler: the fixed-rate update accumulator of water.gd:51-54,62-63,75-82 as a POD state machine (binary64, the
 * arithmetic of the GDScript).  ocean_scheduler_tick(delta) is Water._process(delta) without the generator call: it returns 1
 * when an update is due and writes the delta to pass to WaveGenerator.update (target period + overshoot, or the frame delta
 * when updates_per_second == 0), then advances the clock.  ocean_scheduler_set_rate is the updates_per_second setter (:52-54).
 * ocean_water_frame is one rendered frame of the node pair: Water._process (tick, ocean_update when due) followed by the child
 * WaveGenerator._process (ocean_process: one pending cascade).  ocean_map_scales fills map_scales[i] = (1 / tile_length.xy,
 * displacement_scale, normal_scale) (water.gd:102-110; the quotients are binary32 as Vector2.ONE / tile_length is).
 * ocean_water_default_time(i) = 120.0 + PI * i, the cascade start time of water.gd:32. */
typedef struct ocean_scheduler {
    double updates_per_second;   /* water.gd:51, default 50 */
    double time;                 /* :62 */
    double next_update_time;     /* :63 */
} ocean_scheduler;
int ocean_scheduler_init(ocean_scheduler* s, double updates_per_second);
int ocean_scheduler_set_rate(ocean_scheduler* s, double updates_per_second);
int ocean_scheduler_tick(ocean_scheduler* s, double delta, double* update_delta);
int ocean_water_frame(ocean_generator* gen, ocean_scheduler* s, double delta, ocean_cascade_params* parameters, int count,
                      int* did_update);
int ocean_map_scales(const ocean_cascade_params* parameters, int count, float* map_scales /* [count][4] */);
double ocean_water_default_time(int cascade);

/* descriptors[&'displacement_map'].rid / descriptors[&'normal_map'].rid, wave_generator.gd:34-35,
 * water.gd:95-96.  Device pointers to [num_cascades][map_size][map_size][4] IEEE half (RGBA16F),
 * layer-major, tightly packed: displacement = (hx,hy,hz,0), normal = (dy/dx/(1+|dxx|),
 * dy/dz/(1+|dzz|), dhx_dx, foam) (fft_unpack.glsl:50,66-67). */
int ocean_get_maps(ocean_generator* gen, void** displacement_dev, void** normal_dev, size_t* layer_bytes);

/* Host hand-off for RenderingDevice.texture_update(rid, layer, bytes) (the maps are created with
 * TEXTURE_USAGE_CAN_UPDATE_BIT, wave_generator.gd:34-35).  Copies layers [first, first+count).
 * Either destination may be NULL.  The _async form returns after enqueueing on the generator's
 * stream (use pinned memory from ocean_host_alloc and ocean_synchronize). */
int ocean_copy_maps_to_host(ocean_generator* gen, int first, int count, void* displacement_host, void* normal_host);
int ocean_copy_maps_to_host_async(ocean_generator* gen, int first, int count, void* displacement_host, void* normal_host);
/* Overlapped hand-off: snapshots the layers on the device (one device-to-device copy on the generator's stream) and moves the
 * snapshot to (pinned) host memory on a second stream, so the NEXT update runs while the maps of this one cross PCIe.
 * ocean_wait_snapshot() returns when the most recent snapshot has arrived; a new snapshot waits for the previous one to have left
 * the device.  Use two host buffers alternately.  ocean_destroy() waits for a snapshot still in flight, so its host buffers
 * are complete when it returns. */
int ocean_snapshot_maps_to_host_async(ocean_generator* gen, int first, int count, void* displacement_host, void* normal_host);
int ocean_wait_snapshot(ocean_generator* gen);
int ocean_synchronize(ocean_generator* gen);
int ocean_host_alloc(void** ptr, size_t bytes); /* pinned host memory */
int ocean_host_free(void* ptr);

/* descriptors[&'spectrum'] (RGBA32F, TEXTURE_USAGE_CAN_COPY_FROM_BIT, wave_generator.gd:31):
 * [map_size][map_size][4] float = (Re h0(k), Im h0(k), Re h0(-k), -Im h0(-k)) for one cascade. */
int ocean_copy_spectrum_to_host(ocean_generator* gen, int cascade, float* host);

/* Injects wave amplitudes in place of spectrum_compute's output (test / authoring tap): amplitudes = [map_size][map_size][2]
 * float, A(id) for every texel id = (x, y) (the value get_spectrum_amplitude(id) would return, spectrum_compute.glsl:103-115).
 * The library stores spectrum[id] = (A(id), conj A(mod(-id, N))) exactly as spectrum_compute.glsl:121-124 does, so the texture stays
 * consistent with what the time-propagation stage assumes.  Pass should_generate_spectrum = 0 for that cascade afterwards, or the
 * next update regenerates the spectrum from the parameters. */
int ocean_set_spectrum_amplitudes(ocean_generator* gen, int cascade, const float* amplitudes);

/* Host evaluation of the DETMATH exp (DESIGN.md): the library computes exp(-foam_decay_rate), uniform per dispatch
 * (fft_unpack.glsl:62), on the host with the same binary64 operation sequence the device functions use.  Exported so
 * that the agreement can be checked without a GPU (tests/test_abi_cpu.py). */
float ocean_detmath_expf(float x);

/* Batched map queries -- the sampling contract of the water shader as an op, at UNDISPLACED points (the surface at a
 * world position, what buoyancy / gameplay code needs, is ocean_query_surface below):
 *   displacement[p]   = sum_i texture(displacements, vec3(xz*scales_i.xy, i)).xyz * scales_i.z         water.gdshader:27-39
 *   gradient_foam[p]  = sum_i mix(texture_bicubic(normals, c_i), texture(normals, c_i), min(1, ppm_i*0.1)).xyw
 *                             * vec3(scales_i.ww, 1),  ppm_i = map_size * min(scales_i.x, scales_i.y)   water.gdshader:42-84
 * over the first num_cascades layers, map_scales[i] = (1/tile_length.x, 1/tile_length.y, displacement_scale,
 * normal_scale) as in assets/water/water.gd:102-110.  points_xz: [num_points][2] world x,z (UV = VERTEX.xz);
 * outputs: [num_points][3] float each.  texture() = exact-weight bilinear filter with REPEAT addressing, binary32,
 * shader operation order (oracle/sampling.py is the specification).  |xz * scale * map_size| must stay below 2^31.
 * ocean_sample_maps takes host buffers (copies inside, synchronous); ocean_sample_maps_device takes device pointers for
 * points and outputs (map_scales stays a host array) and is asynchronous on the generator's stream. */
int ocean_sample_maps(ocean_generator* gen, int num_points, const float* points_xz_host, int num_cascades, const float* map_scales_host,
                      float* displacement_host, float* gradient_foam_host);
int ocean_sample_maps_device(ocean_generator* gen, int num_points, const float* points_xz_dev, int num_cascades, const float* map_scales_host,
                             float* displacement_dev, float* gradient_foam_dev);

/* Surface query -- the water surface at a WORLD position, what a boat, a buoy or a splash test asks.  ocean_sample_maps
 * reads the maps at the undisplaced grid point (UV = VERTEX.xz before VERTEX += displacement, water.gdshader:28,37), so
 * the rendered point it describes sits at P + D_xz(P), not at P.  For each point Q this op solves P + D_xz(P) = Q for P
 * (damped Newton steps on the bilinear displacement sum and its exact Jacobian; where det(I + J) <= 1e-3 a fixed-point
 * step; if the start from Q does not converge, restarts from Q - D_xz(Q) and from Q +- rho along x and z, rho = half the
 * horizontal displacement bound of the maps) and then samples the maps at P as ocean_sample_maps does:
 *   source_x/z     P, the undisplaced point whose rendered surface point is (P.x + dx, dy, P.z + dz)
 *   displacement   D(P); the water height at Q is displacement[1]
 *   gradient_foam  the gradient and foam at P; the normal is normalize(-g.x, 1, -g.y) (water.gdshader:90)
 *   residual       max(|E.x|, |E.z|), E = P + D_xz(P) - Q; the point converged iff residual <= tolerance
 *   iterations     Newton steps taken over all starts
 * The end point with the smallest residual is returned, converged or not.  max_iterations = 0 returns the map query at Q
 * unchanged (source = Q).  oracle/surface.py is the specification (binary32, bit-exact).
 * Limits: the query describes the surface as rendered within 150 m of the camera, where distance_factor is exactly 1
 * (water.gdshader:29); the camera-dependent flattening beyond that is render LOD and is not modelled.  Where the surface
 * folds, several points P may map to Q, and any converged one may be returned.  tolerance (metres) must exceed a few
 * binary32 ulps of |Q|, or points far from the origin cannot converge.  tolerance must be finite and > 0, max_iterations in
 * [0, 64].  ocean_query_surface takes host buffers and is synchronous; ocean_query_surface_device takes device pointers for
 * the points and the records (map_scales stays a host array) and is asynchronous on the generator's stream.  A call with
 * points launches 3 kernels (1 with max_iterations = 0), one more that adds the wake free surface to the records while the
 * wake coupling is live (ocean_wake_set_coupling, "Wake layer"). */
typedef struct ocean_surface_sample {
    float source_x, source_z;
    float displacement[3];
    float gradient_foam[3];
    float residual;
    uint32_t iterations;
} ocean_surface_sample;   /* 40 B */
int ocean_query_surface(ocean_generator* gen, int num_points, const float* points_xz_host, int num_cascades, const float* map_scales_host,
                        float tolerance, int max_iterations, ocean_surface_sample* out_host);
int ocean_query_surface_device(ocean_generator* gen, int num_points, const float* points_xz_dev, int num_cascades, const float* map_scales_host,
                               float tolerance, int max_iterations, ocean_surface_sample* out_dev);

/* Ray cast -- the first crossing of each ray with the displaced water surface: where a projectile enters the water, what
 * the crosshair points at, whether a line of sight crosses a crest, where an underwater camera ray leaves the water.
 * The surface is the one ocean_query_surface describes.  Along the ray r(t) = origin + t * direction the gap is
 * g(t) = r.y - eta(r.x, r.z), eta the water height from the surface query's inversion; a point is above iff g > 0.
 *   slab        the call bounds the heights of the maps per layer (y min and max, scaled and summed over the cascades,
 *               padded by tolerance plus 2^-13 of the summed magnitudes) and clips [0, t_max] to that slab.  A ray that
 *               never enters it is a MISS with 0 evaluations, t = 0 and position = origin (every other field 0).
 *   march       a sample every `step` metres of horizontal travel from the slab entry (ray parameter step / |direction.xz|;
 *               a vertical ray is sampled at entry and exit only), plus one at the slab exit.  Each sample inverts the
 *               horizontal displacement at r.xz, warm-started from the previous sample's source point (the first one from
 *               r.xz, so sample 0 is the surface query at the ray's entry point), with the surface query's restarts.
 *               max_iterations = 0 uses the map height at r.xz: a plain height-field march.
 *   refinement  the first sample on the other side of the surface than sample 0 brackets a crossing with the previous one;
 *               Illinois regula falsi refines it until |g| <= tolerance, the new parameter is not strictly inside the
 *               bracket, or 32 steps have run.  The bracket end with the smaller |g| is reported (the earlier on ties).
 * The record (ocean_ray_hit) describes the reported point: its parameter t, position, source point, the map sample at the
 * source (as ocean_query_surface's displacement and gradient_foam), gap and inversion residual.  status:
 *   OCEAN_RAY_MISS             the segment [0, t_max] ends without a crossing (the last sample's record)
 *   OCEAN_RAY_HIT_FROM_ABOVE   a crossing, sample 0 above the water;  OCEAN_RAY_HIT_FROM_BELOW  sample 0 below it (an
 *                              underwater origin);  |gap| <= tolerance when the refinement converged
 *   OCEAN_RAY_TRUNCATED        max_samples samples without a crossing (the last sample's record): near-horizontal rays in the
 *                              slab, t_max = +inf
 *   OCEAN_RAY_INVALID          a non-finite origin or direction component, a zero direction, or t_max NaN or negative (0
 *                              evaluations, every other field 0); or an evaluation whose gap is NaN (that evaluation's record)
 * evaluations counts march samples plus refinement evaluations, iterations the Newton steps over all of them, unconverged
 * the evaluations whose inversion residual is not <= tolerance.  A bad ray never fails the call nor affects other rays.
 * oracle/raycast.py is the specification (binary32, bit-exact, every operation written out).
 * Limits: the surface as rendered within 150 m of the camera (distance_factor, as for ocean_query_surface); crests thinner
 * than `step` along the ray can be missed; where the surface folds, any crossing may be found; binary32 resolution of the
 * positions falls with distance from the origin (tolerance must exceed a few ulps of the coordinates).
 * direction need not be unit: t is in units of |direction|, and scaling direction by 2^k scales t by 2^-k and changes no
 * other field.  step must be finite and > 0, max_samples in [2, 2^20]; tolerance, max_iterations, num_cascades and
 * map_scales as for ocean_query_surface; an invalid call launches nothing.  map_scales is a host array in both entry points;
 * ocean_raycast takes host rays and records and is synchronous; ocean_raycast_device takes device pointers for them and is
 * asynchronous on the generator's stream.  A call with rays launches 2 kernels, 3 while it reads the wake layer.
 * With OCEAN_WAKE_READ_RAYCAST set (ocean_wake_set_readers) and the wake coupling live, the surface is the coupled one that
 * ocean_query_surface describes: the wake free surface e is added to the height, the slab and the record ("Wake layer",
 * Readers). */
#define OCEAN_RAY_MISS 0
#define OCEAN_RAY_HIT_FROM_ABOVE 1
#define OCEAN_RAY_HIT_FROM_BELOW 2
#define OCEAN_RAY_TRUNCATED 3
#define OCEAN_RAY_INVALID 4
typedef struct ocean_ray {
    float origin[3];
    float direction[3];         /* need not be unit; t is in units of |direction| */
    float t_max;                /* in [0, +inf]; +inf allowed */
} ocean_ray;                    /* 28 B */
typedef struct ocean_ray_hit {
    float t;                    /* ray parameter of the reported point */
    float position[3];          /* origin + t * direction, each component rounded as written */
    float source_x, source_z;   /* undisplaced point P whose surface point is under / over `position` */
    float displacement[3];      /* the map sample at P, as ocean_query_surface's record */
    float gradient_foam[3];
    float gap;                  /* position.y - water height there (|gap| <= tolerance for a resolved hit) */
    float residual;             /* horizontal inversion residual at P */
    uint32_t status;            /* OCEAN_RAY_* */
    uint32_t evaluations;       /* gap evaluations: march samples + refinement */
    uint32_t iterations;        /* Newton steps over all evaluations */
    uint32_t unconverged;       /* evaluations whose inversion residual is not <= tolerance */
} ocean_ray_hit;                /* 72 B */
int ocean_raycast(ocean_generator* gen, int num_rays, const ocean_ray* rays_host, int num_cascades, const float* map_scales_host,
                  float step, int max_samples, float tolerance, int max_iterations, ocean_ray_hit* out_host);
int ocean_raycast_device(ocean_generator* gen, int num_rays, const ocean_ray* rays_dev, int num_cascades, const float* map_scales_host,
                         float step, int max_samples, float tolerance, int max_iterations, ocean_ray_hit* out_dev);

/* Buoyancy -- per-body hydrostatic force and torque for this physics tick, from hull sample points on the displaced surface.
 * A hull point (body-local position, volume in m^3, half_height in m) stands for a vertical column element of that volume,
 * centred on the point and reaching half_height above and below it.  A body is a 3 x 4 row-major body-to-world matrix [R | t]
 * (the layout of ocean_spray_grid's emission_transform) and a range [first_point, first_point + num_points) into the hull
 * points; ranges may overlap, so a thousand identical crates share one hull.  For world point j of a body (p = its hull point):
 *   r = R p (rotated, not translated), w = r + t, eta = the water height over (w.x, w.z) from ocean_query_surface,
 *   f = h > 0 ? min(max((eta - (w.y - h)) / (h + h), 0), 1) : (w.y <= eta),  v = f * volume,
 * with NaN-dropping min/max (a NaN height gives f = 0).  Per body S0 = sum v and S1 = sum v * r, summed in a fixed order
 * (point j in lane j mod 32, lanes in increasing j from +0, then the tree of a warp shuffle reduction), so the results are
 * deterministic and bit-identical to oracle/buoyancy.py, the specification.  With rho_g = density * 9.81f:
 *   submerged_volume  S0
 *   force             (0, rho_g S0, 0)
 *   torque            (-(rho_g S1.z), 0, rho_g S1.x), about the body origin t (the sum of r x F over the points)
 *   center_offset     S1 / S0, or 0 when S0 is not > 0; the centre of buoyancy is t + center_offset, and a Godot host calls
 *                     apply_force(force, center_offset), which gives the same torque
 *   max_residual      NaN-dropping max of the points' surface-query residuals
 *   unconverged       points whose residual is not <= tolerance
 * A body with num_points = 0 gets an all-zero record.  num_cascades, map_scales, tolerance and max_iterations mean what they
 * mean for ocean_query_surface, whose limits carry over (within 150 m of the camera; any converged preimage where the surface
 * folds).  The model is vertical hydrostatics only: no drag (ocean_body_forces below returns this record together with a
 * drag record, from one surface query) and no added mass, the column element stays vertical under rotation, and volumes
 * are not rescaled by a non-rigid transform.
 * density must be finite and > 0, counts non-negative, every body's range inside [0, num_points), and the sum of the bodies'
 * num_points (the world points) at most INT32_MAX.  samples may be NULL, or receives the surface record of every world point
 * ([sum of num_points], body-major, j increasing).  The bodies and map_scales are host arrays in both entry points (the poses
 * come from the host's physics engine every tick); ocean_buoyancy takes host points, results and samples and is synchronous;
 * ocean_buoyancy_device takes device pointers for them and is asynchronous on the generator's stream.  A call with world
 * points launches 5 kernels (3 with max_iterations = 0), one more while the wake coupling is live (ocean_wake_set_coupling). */
typedef struct ocean_buoyancy_point {
    float position[3];
    float volume;
    float half_height;
} ocean_buoyancy_point;    /* 20 B */
typedef struct ocean_buoyancy_body {
    float transform[12];
    int32_t first_point;
    int32_t num_points;
} ocean_buoyancy_body;     /* 56 B */
typedef struct ocean_buoyancy_result {
    float force[3];
    float torque[3];
    float submerged_volume;
    float center_offset[3];
    float max_residual;
    uint32_t unconverged;
} ocean_buoyancy_result;   /* 48 B */
int ocean_buoyancy(ocean_generator* gen, int num_bodies, const ocean_buoyancy_body* bodies_host, int num_points,
                   const ocean_buoyancy_point* points_host, int num_cascades, const float* map_scales_host, float density,
                   float tolerance, int max_iterations, ocean_buoyancy_result* results_host, ocean_surface_sample* samples_host);
int ocean_buoyancy_device(ocean_generator* gen, int num_bodies, const ocean_buoyancy_body* bodies_host, int num_points,
                          const ocean_buoyancy_point* points_dev, int num_cascades, const float* map_scales_host, float density,
                          float tolerance, int max_iterations, ocean_buoyancy_result* results_dev, ocean_surface_sample* samples_dev);

/* Body forces -- buoyancy plus quadratic drag against the water velocity, per body, from one surface query.
 * The bodies, hull points, num_cascades, map_scales, density, tolerance and max_iterations are those of ocean_buoyancy, and
 * `hydrostatic` receives exactly the records ocean_buoyancy returns for them.  Each body also has a velocity (world frame):
 * `linear` is the velocity of the body ORIGIN t, `angular` its angular velocity in rad/s.  Godot's linear_velocity is that
 * of the centre of mass: pass v_com + angular x (t - com).  drag_areas[num_points] runs parallel to the hull points: C_d A in
 * m^2 per hull point, so bodies that share a hull share its areas.  For world point j of a body, with r, w, the surface
 * record and f as in ocean_buoyancy, a point with f > 0 contributes
 *   u  = sum_i texture(velocity, vec3((source_x, source_z) * scales_i.xy, i)).xyz * scales_i.z   (ocean_sample_velocity at
 *        the record's source point: the water velocity at w)
 *   vb = linear + (a.y r.z - a.z r.y, a.z r.x - a.x r.z, a.x r.y - a.y r.x)   (a = angular; each bracket rounded as written)
 *   d  = u - vb,  s = sqrt((d.x d.x + d.y d.y) + d.z d.z),  k = (f * cda) * s,  F = k d,  T = r x F (component order as vb's)
 * and a point with f = 0 contributes nothing.  Per body, in ocean_buoyancy's summation order, with half_rho = 0.5f * density:
 *   force               half_rho * sum F
 *   torque              half_rho * sum T, about the body origin t (like ocean_buoyancy's)
 *   wetted_drag_area    sum f * cda (m^2)
 *   max_relative_speed  NaN-dropping max of s over the points with f > 0, from 0 (0 when there are none)
 * oracle/drag.py is the specification, bit for bit.  A body with num_points = 0 gets an all-zero record.  The model's limits:
 * it uses the SURFACE water velocity at every submerged point, while the orbital velocity of a wave decays as e^(-k z) with
 * depth z (at 1 m of draft this overstates the longest wave of a 16 m tile about 1.5 times, shorter waves more); there is no
 * added mass, radiation or wave-making damping, skin friction, or separate normal and tangential coefficients; nothing is
 * written back into the maps (no foam; wakes are the separate wake layer below, which these ops read only while its coupling is on).  Quadratic drag is stiff for light bodies under explicit integration: the op
 * does not integrate, and max_relative_speed lets a host choose sub-steps (ocean_simulate_bodies below integrates on the
 * device with a step that stays stable under it).
 * The call first brings stale velocity layers up to date (as ocean_sample_velocity does; the velocity buffers are allocated
 * on first use).  Validation is ocean_buoyancy's, plus velocities and drag_areas non-NULL where a count needs them and both
 * outputs non-NULL; an invalid call launches nothing.  samples may be NULL, as for ocean_buoyancy.  The bodies, velocities
 * and map_scales are host arrays in both entry points; ocean_body_forces takes host points, areas and outputs and is
 * synchronous; ocean_body_forces_device takes device pointers for them and is asynchronous on the generator's stream.  With
 * no stale velocity layer, a call with world points launches 6 kernels (4 with max_iterations = 0), one more while the wake
 * coupling is live (ocean_wake_set_coupling). */
typedef struct ocean_body_velocity {
    float linear[3];       /* velocity of the body origin t (m/s) */
    float angular[3];      /* rad/s */
} ocean_body_velocity;     /* 24 B */
typedef struct ocean_drag_result {
    float force[3];
    float torque[3];       /* about the body origin t */
    float wetted_drag_area;
    float max_relative_speed;
} ocean_drag_result;       /* 32 B */
int ocean_body_forces(ocean_generator* gen, int num_bodies, const ocean_buoyancy_body* bodies_host, const ocean_body_velocity* velocities_host,
                      int num_points, const ocean_buoyancy_point* points_host, const float* drag_areas_host, int num_cascades,
                      const float* map_scales_host, float density, float tolerance, int max_iterations, ocean_buoyancy_result* hydrostatic_host,
                      ocean_drag_result* drag_host, ocean_surface_sample* samples_host);
int ocean_body_forces_device(ocean_generator* gen, int num_bodies, const ocean_buoyancy_body* bodies_host,
                             const ocean_body_velocity* velocities_host, int num_points, const ocean_buoyancy_point* points_dev,
                             const float* drag_areas_dev, int num_cascades, const float* map_scales_host, float density, float tolerance,
                             int max_iterations, ocean_buoyancy_result* hydrostatic_dev, ocean_drag_result* drag_dev,
                             ocean_surface_sample* samples_dev);

/* Floating bodies -- advance rigid bodies on the water by `substeps` sub-steps of h = dt / substeps (binary32), with the
 * body state kept in device memory.  A floating body is a mass (kg), principal moments of inertia about its centre of mass
 * (kg m^2, body axes = hull axes) and a range into the hull points and drag areas, as ocean_buoyancy_body's.  The body ORIGIN
 * is its centre of mass and its hull axes are its principal axes: a Godot host whose RigidBody3D has a custom center_of_mass
 * c shifts its hull points by -c once (p - c) and keeps position = global_position + basis * c.  A state is the world
 * position of the origin, a unit quaternion (x, y, z, w) from body to world, and the world-frame linear velocity of the
 * centre of mass and angular velocity (Godot's linear_velocity and angular_velocity).  One sub-step, per body
 * (oracle/bodies.py is the specification, bit for bit):
 *   pose    R = R(q), the standard unit-quaternion rotation (R00 = 1 - 2 (yy + zz), R01 = 2 (xy - wz), R02 = 2 (xz + wy),
 *           R10 = 2 (xy + wz), R11 = 1 - 2 (xx + zz), R12 = 2 (yz - wx), R20 = 2 (xz - wy), R21 = 2 (yz + wx),
 *           R22 = 1 - 2 (xx + yy)); transform = [R | position]; the origin's velocity is (linear, angular).
 *   forces  hyd and drg = ocean_body_forces' two records for that transform and velocity, through the same kernels.
 *   step    c_v = (density * drg.wetted_drag_area) * drg.max_relative_speed   (bounds |dF_drag/dv|)
 *           c_w = c_v * r2, r2 = max |p|^2 over the body's hull points          (bounds |dT_drag/dw|)
 *           F = hyd.force + drg.force, F.y = F.y - mass * 9.81f;   v' = v + (h / (mass + h c_v)) F
 *           tau = hyd.torque + drg.torque; tau_b = R^T tau, w_b = R^T w;  w_b' = w_b + (h tau_b) / (inertia + h c_w) per
 *           axis;  w' = R w_b'
 *           position' = position + h v';   q' = normalize(q + (h / 2) (w' (x) q))
 * A semi-implicit Euler step whose drag Jacobian is bounded by the scalars c_v and c_w: for the linearised drag it never
 * overshoots and is stable at any h, so light bodies with large drag areas do not blow up at 60 Hz; as h -> 0 it is explicit
 * Euler on the true forces.  A body with num_points = 0 is ballistic (all-zero records).  A NaN or infinite state affects
 * only its own body.  hydrostatic and drag (may be NULL) receive the records of the LAST sub-step (the forces at the pose that
 * sub-step started from); transforms (may be NULL) receives the 3 x 4 row-major [R | position] of each final state, the
 * layout of ocean_buoyancy_body.transform and of a Godot 4 MultiMesh transform buffer (RenderingServer.multimesh_set_buffer
 * with TRANSFORM_3D, no colours or custom data: 12 floats per instance).  The model's limits: no added mass (the heave period
 * is shorter than a real body's); no gyroscopic term; no contacts between bodies; the surface water velocity at every depth
 * (ocean_body_forces'); every sub-step of a call sees the same maps; the hydrostatic spring is explicit in position, so h must
 * stay below T_heave / pi with T_heave = 2 pi sqrt(mass / (density * 9.81 * A_waterplane)).
 * The bodies and map_scales are host arrays in both entry points: the call validates the bodies, computes the world-point
 * offsets and uploads both once.  Validation is ocean_body_forces' (without its velocities and outputs), plus mass and every
 * inertia finite and > 0, dt finite and > 0, substeps in [1, 64] and states non-NULL when num_bodies > 0; an invalid call
 * launches nothing and refreshes nothing.  The call brings stale velocity layers up to date once, then launches 1 + 7 S
 * kernels (1 + 5 S with max_iterations = 0, 1 + 3 S when no body has hull points), and S more with world points while the
 * wake coupling is live (ocean_wake_set_coupling; every sub-step reads the same wake snapshots).  ocean_simulate_bodies takes host
 * states, points, areas and outputs and is synchronous; ocean_simulate_bodies_device takes device pointers for them and is
 * asynchronous on the generator's stream. */
typedef struct ocean_floating_body {
    float mass;                 /* kg, finite and > 0 */
    float inertia[3];           /* principal moments about the centre of mass, body axes = hull axes (kg m^2), finite and > 0 */
    int32_t first_point;        /* range into the hull points and drag areas, as ocean_buoyancy_body's */
    int32_t num_points;
} ocean_floating_body;          /* 24 B */
typedef struct ocean_body_state {
    float position[3];          /* world position of the body origin = its centre of mass */
    float orientation[4];       /* unit quaternion (x, y, z, w), body -> world */
    float linear_velocity[3];   /* of the centre of mass, m/s (Godot's linear_velocity) */
    float angular_velocity[3];  /* world frame, rad/s (Godot's angular_velocity) */
} ocean_body_state;             /* 52 B */
int ocean_simulate_bodies(ocean_generator* gen, int num_bodies, const ocean_floating_body* bodies_host, ocean_body_state* states_host,
                          int num_points, const ocean_buoyancy_point* points_host, const float* drag_areas_host, int num_cascades,
                          const float* map_scales_host, float density, float dt, int substeps, float tolerance, int max_iterations,
                          ocean_buoyancy_result* hydrostatic_host, ocean_drag_result* drag_host, float* transforms_host);
int ocean_simulate_bodies_device(ocean_generator* gen, int num_bodies, const ocean_floating_body* bodies_host, ocean_body_state* states_dev,
                                 int num_points, const ocean_buoyancy_point* points_dev, const float* drag_areas_dev, int num_cascades,
                                 const float* map_scales_host, float density, float dt, int substeps, float tolerance, int max_iterations,
                                 ocean_buoyancy_result* hydrostatic_dev, ocean_drag_result* drag_dev, float* transforms_dev);

/* Driven and moored bodies -- ocean_simulate_bodies with thrusters, hull foils, applied loads and tethers (oracle/drive.py is
 * the specification, bit for bit).  A boat is driven by a thruster, steered by a rudder foil, kept on course by a keel foil
 * and moored or towed by a tether; the body state stays on the device as in ocean_simulate_bodies.  Per sub-step, with R, t,
 * v and w the pose and velocity the sub-step starts from, r = R p for a hull-local point p, and f the submerged fraction of
 * ocean_buoyancy at r + t with the actuator's half_height (its world point is queried with the hull's):
 *   thruster  F = (f * thrust) * (R direction), T = r x F; a dry thruster (f = 0) adds nothing, so a propeller that leaves
 *             the water on a crest pushes nothing
 *   foil      d = u - (v + w x r), u the water velocity at the point as ocean_body_forces computes it (plus the wake's
 *             vertical velocity while the coupling is live); n = R normal, dn = (d.x n.x + d.y n.y) + d.z n.z,
 *             F = (((rho/2 * (f * area)) * dn) * |dn|) * n, T = r x F: normal-only drag of a flat plate, area = C_n A; dry adds
 *             nothing
 *   tether    x_a, x_b the end points (x_b = point_b, a world anchor, when body_b = -1), L = |x_b - x_a|, u = (x_b - x_a) / L,
 *             s = k (L - L0) + c ((v_b - v_a) . u) with v_a, v_b the end points' velocities (0 at an anchor); the tension is
 *             s when L > 0 and s > 0, else 0 (slack: the tether adds nothing); +T u acts at x_a and -T u at x_b
 *   load      force and torque added as given (world frame, about the centre of mass)
 *   step      ocean_simulate_bodies' step with the forces added onto F and tau in a fixed order (each body's thrusters,
 *             foils and tether ends in array order, then its load), and the denominators widened by the new Jacobian
 *             bounds: c_v += (density * sum f area) * max |dn| and c_w += that * max |p|^2 over the body's foil points; each
 *             taut tether end adds h c + h^2 k to mass + h c_v and (h c) |p|^2 + (h^2 k) |p|^2 to every inertia + h c_w.
 * For a linear spring this step has determinant 1 and trace in (-2, 2] at any h, for one body on an anchor and for bodies
 * joined by lines: stiff mooring and tow lines do not blow up at 60 Hz.  No floating-point atomics: the result does not
 * depend on the schedule.  A NaN or infinite actuator or load affects only its body, and a tether only the two bodies it
 * joins.  A body with nothing attached and no load row takes ocean_simulate_bodies' step bit for bit, and a call with no
 * thrusters, foils or tethers and loads = NULL is ocean_simulate_bodies (drive, when given, is zeroed).
 * The actuator arrays and loads are host arrays in both entry points (a game changes them every tick).  Validation is
 * ocean_simulate_bodies', plus: counts >= 0 and their arrays non-NULL when positive; every actuator's body and a tether's
 * body_a in [0, num_bodies), body_b -1 or a body other than body_a; foil areas, rest lengths, stiffnesses and dampings finite
 * and >= 0 (they enter the stability bound); world points plus actuators below 2^31.  Positions, directions, thrust and loads
 * are not validated.  An invalid call launches nothing.  drive (may be NULL) receives per body the last sub-step's sum of the
 * forces and torques the drive arguments added, the wetted foil area sum f area and max |dn|; tensions (may be NULL) the last
 * sub-step's tension per tether.  With A = num_thrusters + num_foils, S sub-steps and anything attached, the call launches
 * 1 + S (7 + a + t + 1) kernels, a = 1 when A > 0, t = 1 when num_tethers > 0 (1 + S (5 + a + t + 1) with max_iterations = 0,
 * 1 + S (3 + t + 1) when there are no world points at all), and S more while the wake coupling is live. */
typedef struct ocean_thruster {
    int32_t body;
    float position[3];          /* hull-local point of the propeller */
    float direction[3];         /* hull-local direction of the push (not normalised: thrust scales it) */
    float thrust;               /* N */
    float half_height;          /* of the immersion column, as ocean_buoyancy_point's */
} ocean_thruster;               /* 36 B */
typedef struct ocean_foil {
    int32_t body;
    float position[3];          /* hull-local centre of pressure */
    float normal[3];            /* hull-local unit normal of the plate */
    float area;                 /* C_n A, m^2, finite and >= 0 */
    float half_height;
} ocean_foil;                   /* 36 B */
typedef struct ocean_body_load {
    float force[3];             /* world frame, N */
    float torque[3];            /* world frame, about the centre of mass, N m */
} ocean_body_load;              /* 24 B */
typedef struct ocean_tether {
    int32_t body_a;
    int32_t body_b;             /* -1: point_b is a world anchor */
    float point_a[3];           /* hull-local point of body_a */
    float point_b[3];           /* hull-local point of body_b, or the world anchor */
    float rest_length;          /* m, finite and >= 0 */
    float stiffness;            /* N/m, finite and >= 0 */
    float damping;              /* N s/m, finite and >= 0 */
} ocean_tether;                 /* 44 B */
typedef struct ocean_drive_result {
    float force[3];             /* sum of the forces the thrusters, foils, tethers and load added */
    float torque[3];            /* and of their torques about the centre of mass */
    float wetted_foil_area;     /* sum f * area over the body's foils, m^2 */
    float max_normal_speed;     /* max |dn| over the body's wet foils, m/s */
} ocean_drive_result;           /* 32 B */
int ocean_simulate_driven_bodies(ocean_generator* gen, int num_bodies, const ocean_floating_body* bodies_host, ocean_body_state* states_host,
                                 int num_points, const ocean_buoyancy_point* points_host, const float* drag_areas_host, int num_cascades,
                                 const float* map_scales_host, float density, float dt, int substeps, float tolerance, int max_iterations,
                                 int num_thrusters, const ocean_thruster* thrusters_host, int num_foils, const ocean_foil* foils_host,
                                 const ocean_body_load* loads_host, int num_tethers, const ocean_tether* tethers_host,
                                 ocean_buoyancy_result* hydrostatic_host, ocean_drag_result* drag_host, ocean_drive_result* drive_host,
                                 float* tensions_host, float* transforms_host);
int ocean_simulate_driven_bodies_device(ocean_generator* gen, int num_bodies, const ocean_floating_body* bodies_host,
                                        ocean_body_state* states_dev, int num_points, const ocean_buoyancy_point* points_dev,
                                        const float* drag_areas_dev, int num_cascades, const float* map_scales_host, float density, float dt,
                                        int substeps, float tolerance, int max_iterations, int num_thrusters, const ocean_thruster* thrusters_host,
                                        int num_foils, const ocean_foil* foils_host, const ocean_body_load* loads_host, int num_tethers,
                                        const ocean_tether* tethers_host, ocean_buoyancy_result* hydrostatic_dev, ocean_drag_result* drag_dev,
                                        ocean_drive_result* drive_dev, float* tensions_dev, float* transforms_dev);

/* Hull meshes -- floating bodies whose hull is a closed triangle mesh: hydrostatic pressure and drag integrated over the
 * wetted triangles (oracle/hull.py is the specification, bit for bit).  This is the per-triangle pressure model of game boat
 * physics (Kerner, "Water interaction model for boats in video games"): unlike the point hulls above, the pressure force is
 * normal to the hull, so a hull on a wave slope feels a horizontal force, and on flat water the displaced volume and the
 * centre of buoyancy are exact at any heel.
 * ocean_hull_set_meshes registers the meshes once; the generator keeps them in device memory until the next set, a call with
 * num_meshes = 0 (which releases them) or ocean_destroy.  A mesh is a range of the vertices ([3] float each, hull-local, m) and
 * a range of the triangles ([3] int32 each, indices into the mesh's own vertex range), with its drag coefficients.  Winding is
 * Godot's: front faces are CLOCKWISE seen from outside (Mesh.get_faces(), ArrayMesh triangles), so the outward area vector of
 * triangle (a, b, c) is a = 0.5 (c - a) x (b - a).  Meshes are shared: a thousand crates name one mesh.  The call rejects,
 * with nothing uploaded and the previous set kept: negative counts, NULL arrays where a count needs them, ranges outside the
 * arrays, triangle indices outside their mesh's vertex range, non-finite vertices, negative or non-finite coefficients and
 * more than (2^31 - 1) / 3 vertices or triangles.  The arguments are checked before the generator handle, so they can be
 * validated without a device.  volumes (may be NULL) receives each mesh's enclosed signed volume by the divergence theorem
 * (binary64 on the host, stored as float): negative for a mesh wound the other way, which lets a host catch a wrong winding
 * and derive a mass.
 * ocean_hull_forces: per body (ocean_hull_body: the transform of ocean_buoyancy_body and a mesh index) and its velocity
 * (ocean_body_velocity, as for ocean_body_forces), with rho_g = density * 9.81f and half_rho = 0.5f * density:
 *   vertex    r = R p, w = r + t (k_buoyancy_transform's operations); one surface query at (w.x, w.z) (with the wake coupling
 *             while it is live); depth d = eta - w.y; water velocity u at the record's source point (ocean_body_forces' u,
 *             plus the wake's vertical velocity while the coupling is live)
 *   clip      per triangle, dropped if any corner's d is NaN: corners with d > 0 are wet; 3 wet: the triangle; 1 wet (i, then
 *             j, k in winding order): (P_i, X_ij, X_ik); 2 wet (k dry, i, j after it in winding order): (P_i, P_j, X_jk) and
 *             (P_i, X_jk, X_ki); X_ab = P_a + t (P_b - P_a), t = d_a / (d_a - d_b) from the wet corner a, with d = 0 and
 *             u = u_a + t (u_b - u_a) there
 *   pressure  per wet sub-triangle with area vector a, for data linear over it: force -rho g integral(d n dA) = -rho g a sum(d) / 3,
 *             torque -rho g integral(d r x n dA), V = -integral(d n_y dA), S1 = -integral((d r + y d^2 / 2) n_y dA), from
 *             integral(f n dA) = a sum(f) / 3 and integral(f g n dA) = a (sum(f_i g_i) + sum(f) sum(g)) / 12; no square root
 *   drag      per wet sub-triangle: d_c = the mean of its corners' u - (v + w x r), A = |a|, n = a / A, dn = d_c . n; normal drag
 *             -(rho/2) C_n A dn^2 n on impinging faces (dn < 0) only, tangential (rho/2) C_t A |d_t| d_t, d_t = d_c - dn n,
 *             torque r_c x F about the origin (r_c the sub-triangle's centroid); a zero-area sub-triangle adds nothing
 * The records are ocean_body_forces': hydrostatic.force, torque (about the body origin), submerged_volume = V, center_offset =
 * S1 / V (0 unless V > 0), max_residual and unconverged over the body's world vertices; drag.force and torque, wetted_drag_area
 * = sum (C_n + C_t) A and max_relative_speed = max |d_c| from 0, so c_v = density * wetted_drag_area * max_relative_speed
 * bounds the drag's Jacobian as ocean_simulate_bodies' step assumes.  On flat water, for a closed hull, V and t + S1 / V are
 * exactly the displaced volume and the centre of buoyancy (the waterplane cap has d = 0 and adds nothing), and force =
 * (0, rho g V, 0).  A body whose mesh has no vertices gets all-zero records.  Sums are in the fixed order of ocean_buoyancy
 * (triangle j in lane j mod 32, each triangle's pieces added together first, then the shuffle tree): no atomics, and the result
 * does not depend on the schedule.  A NaN pose affects only its body.  The limits: one warp per body (a 2^16-triangle hull is
 * one warp's loop), the SURFACE water velocity at every depth, no added mass, slamming or wave-making terms, nothing written
 * back into the maps.
 * The bodies, velocities and map_scales are host arrays in both entry points; num_cascades, map_scales, tolerance and
 * max_iterations are ocean_query_surface's.  The call validates every body's mesh index (a call with no meshes registered and
 * bodies is invalid), density, and world vertices (the sum of the bodies' meshes' num_vertices) at most INT32_MAX; an invalid
 * call launches nothing.  It brings stale velocity layers up to date (as ocean_body_forces), then with world vertices launches
 * 6 kernels (4 with max_iterations = 0): the vertex transform, the surface query, a per-vertex pass that writes the depth and
 * the water velocity once per vertex, and one reduce per body that clips and integrates; one more while the wake coupling is
 * live.  With no world vertices only the reduce runs.  samples (may be NULL) receives the surface record of every world
 * vertex, body-major.  ocean_hull_forces takes host outputs and is synchronous; ocean_hull_forces_device takes device outputs
 * and is asynchronous on the generator's stream.
 * ocean_simulate_hull_bodies is ocean_simulate_bodies on hull meshes: per sub-step these kernels on the pose and velocity
 * tables, then the integrator's k_bodies_integrate unchanged, with r2 = max |p|^2 over the mesh's vertices (clip points lie
 * on triangle edges, so c_w = c_v r2 stays a bound).  Its states, dt, substeps and outputs, and its validation beyond the
 * meshes, are ocean_simulate_bodies'.  It launches 1 + 7 S kernels (1 + 5 S with max_iterations = 0, 1 + 2 S with no world
 * vertices) and S more while the wake coupling is live.  Hull bodies keep ocean_body_state, so ocean_wake_step drives wakes
 * from them unchanged. */
typedef struct ocean_hull_mesh {
    int32_t first_vertex;       /* range into the hull vertices ([3] float each, hull-local, m) */
    int32_t num_vertices;
    int32_t first_triangle;     /* range into the triangles ([3] int32 each, indices local to this mesh's vertex range) */
    int32_t num_triangles;
    float normal_drag;          /* C_n, finite and >= 0 */
    float tangential_drag;      /* C_t, finite and >= 0 */
} ocean_hull_mesh;              /* 24 B */
typedef struct ocean_hull_body {
    float transform[12];        /* 3 x 4 row-major [R | t], as ocean_buoyancy_body's */
    int32_t mesh;
    int32_t reserved;
} ocean_hull_body;              /* 56 B, the layout of ocean_buoyancy_body */
typedef struct ocean_floating_hull {
    float mass;                 /* kg, finite and > 0 */
    float inertia[3];           /* principal moments about the centre of mass (the hull origin), kg m^2, finite and > 0 */
    int32_t mesh;
} ocean_floating_hull;          /* 20 B */
int ocean_hull_set_meshes(ocean_generator* gen, int num_meshes, const ocean_hull_mesh* meshes_host, int num_vertices,
                          const float* vertices_host, int num_triangles, const int32_t* triangles_host, float* volumes_host);
int ocean_hull_forces(ocean_generator* gen, int num_bodies, const ocean_hull_body* bodies_host, const ocean_body_velocity* velocities_host,
                      int num_cascades, const float* map_scales_host, float density, float tolerance, int max_iterations,
                      ocean_buoyancy_result* hydrostatic_host, ocean_drag_result* drag_host, ocean_surface_sample* samples_host);
int ocean_hull_forces_device(ocean_generator* gen, int num_bodies, const ocean_hull_body* bodies_host,
                             const ocean_body_velocity* velocities_host, int num_cascades, const float* map_scales_host, float density,
                             float tolerance, int max_iterations, ocean_buoyancy_result* hydrostatic_dev, ocean_drag_result* drag_dev,
                             ocean_surface_sample* samples_dev);
int ocean_simulate_hull_bodies(ocean_generator* gen, int num_bodies, const ocean_floating_hull* bodies_host, ocean_body_state* states_host,
                               int num_cascades, const float* map_scales_host, float density, float dt, int substeps, float tolerance,
                               int max_iterations, ocean_buoyancy_result* hydrostatic_host, ocean_drag_result* drag_host,
                               float* transforms_host);
int ocean_simulate_hull_bodies_device(ocean_generator* gen, int num_bodies, const ocean_floating_hull* bodies_host,
                                      ocean_body_state* states_dev, int num_cascades, const float* map_scales_host, float density, float dt,
                                      int substeps, float tolerance, int max_iterations, ocean_buoyancy_result* hydrostatic_dev,
                                      ocean_drag_result* drag_dev, float* transforms_dev);

/* Velocity maps -- the water velocity: the time derivative of the displacement map, what drag, damping and floating debris
 * need.  A cascade's velocity layer is (vx, vy, vz, 0) = d/dt of its displacement texel (hx, hy, hz, 0): same layout, same
 * orientation (ocean_get_maps), RGBA16F, in m/s before the displacement scale.  It is computed exactly, as one more inverse
 * FFT of the same spectrum (differences of two map sets would not work: the cascades of consecutive map sets are at
 * different times, and the half quantisation swamps the difference).  Per texel, binary32, with every name as in
 * spectrum_modulate.glsl and the update's FMA sites only in mul_complex:
 *   w = sqrt(G * k * tanh(k * depth)) (the dispersion table's omega),  m = (cos(w*time), sin(w*time)),
 *   pa = h0a * m,  pb = h0b * conj(m),  d = (pa.x - pb.x, pa.y - pb.y),  ht = (-(w*d.y), w*d.x),  hti = (-ht.y, ht.x),
 *   vx = hti * k_unit.y,  vy = ht,  vz = hti * k_unit.x  (each product rounded on its own),
 *   layer 0 = (vx.x - vy.y, vx.y + vy.x),  layer 1 = (vz.x, vz.y),
 * then the update's row IFFT, transpose and row IFFT, and texel = (l0.re, l0.im, l1.re, 0) * sign_shift, half RTNE.
 * oracle_velocity_update (oracle/velocity_oracle.c) is the specification, bit for bit.  `time` and the tile are those of the
 * update that built the cascade's CURRENT maps (ocean_update_all, ocean_process, ocean_update_frames: its last frame); the
 * spectrum is the texture as stored when the velocity is computed.
 * Every map write marks the cascade's velocity layer stale.  ocean_update_velocity recomputes the stale layers in one launch
 * sequence (asynchronous on the generator's stream) and reports their number in *recomputed (may be NULL); with one cascade
 * per rendered frame (ocean_water_frame) that is usually one layer per tick.  The sample and copy entry points bring stale
 * layers up to date first.  The buffers are allocated (zeroed) by the first velocity call, so generators that never ask
 * pay no memory; a cascade whose maps were never written has a zero layer.  ocean_get_velocity_map returns the device map
 * ([num_cascades][N][N] 4 x half, layer-major like the displacement map) without refreshing it.
 * ocean_sample_velocity: velocity[p] = sum_i texture(velocity, vec3(xz * scales_i.xy, i)).xyz * scales_i.z, the displacement
 * half of ocean_sample_maps (same filter, wrap and arguments, same validation) at UNDISPLACED points.  The velocity of the
 * water at a world position Q: call ocean_query_surface for Q and pass its source point P (source_x, source_z) to
 * ocean_sample_velocity.  With the binary32 taps on, ocean_copy_f32_velocity_to_host returns one layer before the half
 * conversion ([N][N][4] float). */
int ocean_update_velocity(ocean_generator* gen, int* recomputed);
int ocean_get_velocity_map(ocean_generator* gen, void** velocity_dev, size_t* layer_bytes);
int ocean_copy_velocity_to_host(ocean_generator* gen, int first, int count, void* velocity_host);
int ocean_sample_velocity(ocean_generator* gen, int num_points, const float* points_xz_host, int num_cascades, const float* map_scales_host,
                          float* velocity_host);
int ocean_sample_velocity_device(ocean_generator* gen, int num_points, const float* points_xz_dev, int num_cascades, const float* map_scales_host,
                                 float* velocity_dev);
int ocean_copy_f32_velocity_to_host(ocean_generator* gen, int cascade, float* host);

/* Spray candidates -- the spawn test of the sea-spray particle shader as a stream-compaction op
 * (assets/shaders/spatial/sea_spray_particle.gdshader:80-94; the reference evaluates it for every particle of the emitter and
 * culls the inactive ones, README.md:29).  For each candidate START_POS.xz:
 *   gradient = sum_i texture(normals, vec3(xz * map_scales[i].xy, i)).xyw;  normal = normalize(vec3(-gradient.x, 1, -gradient.y));
 *   foam = gradient.z;  normal_factor = mix(.25, 1, min((normal.y - .92) / (.99 - .92), 1));  foam_factor likewise on [.9, 1];
 *   ACTIVE = normal_factor in [0, 1] && foam > .9;  SCALE_FACTOR = normal_factor * foam_factor;
 *   PARTICLE_SCALE = vec3(foam_factor * (1 + 1e-3)) * vec3(1, normal_factor, 1) * particle_scale
 * Only the ACTIVE candidates are returned, in candidate order (stable compaction, deterministic).  *num_active receives their
 * number even when it exceeds max_records (records beyond max_records are dropped).  oracle/spray.py is the specification.
 * ocean_spray_grid fills the start positions of the emitter's particle grid (sea_spray_particle.gdshader:47,52-54):
 * emission_transform = 3 x 4 row-major (basis columns, origin), NULL = identity; points_xz_host: [num_particles][2].
 * With OCEAN_WAKE_READ_SPRAY set (ocean_wake_set_readers) the gradient and foam also read the wake layer's slopes and foam
 * ("Wake layer", Readers); the launches are the same. */
typedef struct ocean_spray_record {
    uint32_t index;            /* candidate (particle INDEX) */
    float start_x, start_z;    /* START_POS.xz */
    float scale_factor;        /* SCALE_FACTOR (:90) */
    float particle_scale[3];   /* PARTICLE_SCALE (:92-94) */
    float foam;                /* summed normal_map.a at the start position */
} ocean_spray_record;
int ocean_spray_grid(int num_particles, const float* emission_transform, float* points_xz_host);
int ocean_extract_spray(ocean_generator* gen, int num_candidates, const float* points_xz_host, int num_cascades,
                        const float* map_scales_host, const float* particle_scale, int max_records,
                        ocean_spray_record* records_host, int* num_active);
/* device pointers for the candidates, the records and the count (asynchronous on the generator's stream) */
int ocean_extract_spray_device(ocean_generator* gen, int num_candidates, const float* points_xz_dev, int num_cascades,
                               const float* map_scales_host, const float* particle_scale, int max_records,
                               ocean_spray_record* records_dev, int* num_active_dev);

/* Spray particles -- one particle-process frame of a sea-spray emitter: the restarts, start() and process() of
 * sea_spray_particle.gdshader (:45-66, :74-126) on particle states kept in caller-owned memory, and the live particles as
 * render-ready MultiMesh instances, for hosts that do not run Godot's GPUParticles3D (or want only the live particles drawn).
 * The reference does not contain Godot's particle engine: the emitter cycle below is this library's statement of it, for a
 * GPUParticles3D with explosiveness 0, randomness 0, local_coords = false, one_shot = false and disable_velocity
 * (main.tscn:133-140).  oracle/spray_particles.py is the specification, bit for bit.  One call is the frame [t0, t1) of
 * emitter time, with TIME = (float)t1 and L = emitter_lifetime:
 *   restart   particle i (INDEX) restarts when some k >= 0 has t0 <= r_k < t1, r_k = L * ((double)k + (double)i / (double)amount)
 *             in binary64; the largest such k is taken, and NUMBER = k * amount + i (mod 2^32).  A restart sets TRANSFORM to
 *             the identity and CUSTOM to 0, sets ACTIVE and EMITTED, and runs start() literally, including
 *             hash32(uvec2(NUMBER, 1U) + uint(TIME) + RANDOM_SEED) in uint32 arithmetic.
 *   process   process() runs on every ACTIVE particle (an inactive one keeps its state until its next restart), literally:
 *             the spawn test of ocean_extract_spray on the first frame at or after START_TIME, then the displacement
 *             sum texture(displacements, START_POS.xz * map_scales[i].xy, i).xyz * map_scales[i].z, * (0.75, 1, 0.75), the
 *             parabola, the exp_impulse and log(1 + t) scale shaping and set_scale on the previous frame's basis.
 *   live      ACTIVE and HAS_STARTED != 0 after the frame (a restarted particle waiting for its START_TIME sits at
 *             y = -1e10 with scale 1e-3 in Godot; it is not an instance).
 *   instance  16 floats per live particle, in INDEX order: TRANSFORM as basis.x.x, basis.y.x, basis.z.x, origin.x, ... (the
 *             transforms of ocean_simulate_bodies; a MultiMesh TRANSFORM_3D instance with custom data and no colours), then
 *             CUSTOM.xyzw (sea_spray.gdshader reads .z and .w through INSTANCE_CUSTOM).  *num_live receives the number of
 *             live particles even when it exceeds max_instances (instances beyond max_instances are dropped).
 * Numeric policy (as ocean_extract_spray): binary32 in the shader's operation order, no contraction, IEEE division and sqrt;
 * normalize(v) = v / sqrt(dot(v, v)); mat4 products as sums in index order; exp and log are DETMATH's; pow(a, 2.0) is taken
 * as a * a (GLSL leaves pow undefined for a < 0, and 2.5t - 0.45 < 0 for the first 18 % of every particle's life); min(NaN, 1)
 * is 1 (IEEE minNum).
 * ocean_default_spray_emitter fills the reference scene's emitter (32768 particles, 15 * I, particle_scale (20, 8.5, 20),
 * lifetime 3, randomness 0.25, emitter lifetime 6, seed 0).  Validation: amount >= 0, num_particles >= 1, lifetime and
 * emitter_lifetime finite and > 0, lifetime_randomness in [0, 1], 0 <= t0 <= t1 finite with (float)t1 < 2^32 and
 * t1 / emitter_lifetime < 2^32, num_cascades in [1, num_cascades of the generator], max_instances >= 0, and no NULL except
 * states when amount = 0 and instances when max_instances = 0.  An invalid call returns OCEAN_ERR_INVALID_ARGUMENT, launches
 * nothing and leaves the states untouched.  A valid call with amount > 0 launches three kernels (update, scan, write).
 * With OCEAN_WAKE_READ_SPRAY set (ocean_wake_set_readers) the spawn test reads the wake layer as ocean_extract_spray's does,
 * and the height adds the layer's h at START_POS.xz every frame ("Wake layer", Readers).
 * ocean_spray_particles takes host states (updated in place), instances and count and is synchronous;
 * ocean_spray_particles_device takes device pointers for them and is asynchronous on the generator's stream.  A zero-filled
 * state is a particle that was never emitted. */
typedef struct ocean_spray_emitter {
    int32_t amount;                 /* particles of the emitter (GPUParticles3D.amount), >= 0 */
    int32_t num_particles;          /* the shader's num_particles uniform: grid side uint(sqrt(float(num_particles))), >= 1 */
    float emission_transform[12];   /* EMISSION_TRANSFORM, 3 x 4 row-major (basis columns, origin), ocean_spray_grid's layout */
    float particle_scale[3];        /* uniforms of the particle shader */
    float lifetime;
    float lifetime_randomness;
    uint32_t random_seed;           /* RANDOM_SEED */
    double emitter_lifetime;        /* LIFETIME (GPUParticles3D.lifetime), s */
} ocean_spray_emitter;              /* 88 B */
#define OCEAN_SPRAY_ACTIVE 1u
#define OCEAN_SPRAY_EMITTED 2u
typedef struct ocean_spray_particle {
    float transform[12];            /* TRANSFORM, 3 x 4 row-major like the instances */
    float custom[4];                /* CUSTOM */
    float userdata1[4];             /* START_POS, START_TIME */
    float userdata2[4];             /* PARTICLE_SCALE, PARTICLE_LIFETIME */
    float userdata3[4];             /* .z SCALE_FACTOR, .w HAS_STARTED */
    uint32_t number;                /* NUMBER */
    uint32_t flags;                 /* OCEAN_SPRAY_ACTIVE | OCEAN_SPRAY_EMITTED */
} ocean_spray_particle;             /* 120 B */
int ocean_default_spray_emitter(ocean_spray_emitter* out);
int ocean_spray_particles(ocean_generator* gen, const ocean_spray_emitter* emitter, double t0, double t1, int num_cascades,
                          const float* map_scales_host, ocean_spray_particle* states_host, int max_instances, float* instances_host,
                          int* num_live);
int ocean_spray_particles_device(ocean_generator* gen, const ocean_spray_emitter* emitter, double t0, double t1, int num_cascades,
                                 const float* map_scales_host, ocean_spray_particle* states_dev, int max_instances, float* instances_dev,
                                 int* num_live_dev);

/* Wake layer -- interactive wakes: a local, dynamic height field that moving sources (boats, swimmers, splashes) and
 * floating bodies drive, to be added to the spectral ocean.  The FFT cascades are periodic tiles rebuilt from h0 every
 * update and cannot carry a propagating disturbance; this layer has its own state.  oracle/wake.py is the specification,
 * bit for bit.
 *   window    N x N cells of size dx (N a power of two in [128, 2048]) whose corner cell sits at the integer cell origin
 *             (ox, oz): cell (i, j) covers world x in [(ox + i) dx, (ox + i + 1) dx), z likewise; fields are [N][N]
 *             binary32, row j along z.  The world corner is x0 = (float)((double)ox * dx), z0 likewise.
 *   state     h (the current height) and h_prev (the height one sub-step earlier), in metres.
 *   model     iWave (Tessendorf, "Interactive Water Surfaces", 2004) with deep-water dispersion w^2 = g |k|:
 *             one sub-step of h = (float)(dt / S), per cell:
 *               s = h + phi;  c = sum over 28 classes (a, b), 0 <= b <= a <= 6, of G[a][b] * (the sum of the up-to-8 mirrored
 *               neighbours of s), cells outside the window reading 0;  h_new = (a1 h - a2 h_prev) - a3 c
 *             with a1 = (2 - alpha h) / (1 + alpha h), a2 = 1 / (1 + alpha h), a3 = g h^2 / (dx (1 + alpha h)), evaluated in
 *             binary64 and rounded once per ring; alpha is `damping` in the interior and damping + (sponge_damping -
 *             damping) t^2, t = (sponge_cells - r) / sponge_cells, on the ring r < sponge_cells cells from the edge (the
 *             sponge absorbs outgoing waves).
 *   stencil   G (ocean_wake_kernel_taps, fitted by tools/fit_wake_kernel.py) is a radius-6 radial stencil whose symbol
 *             Ghat(k) approximates |k| dx: sum G = 0 exactly, 0 <= Ghat <= 4 over the Brillouin zone, and |Ghat / (|k| dx)
 *             - 1| <= 3.9 % for |k| dx in [0.4, 2.0].  Waves propagate correctly for wavelengths from 3.1 dx to 15.7 dx;
 *             longer ones are too slow (no finite stencil is accurate near k = 0), shorter ones are dispersive.  A source
 *             moving at U leaves a Kelvin wake of wavelength 2 pi U^2 / g: choose dx near 2 pi U^2 / (8 g) = 0.08 U^2
 *             (U = 5 m/s: dx = 2 m, 8 cells per wavelength).  The band holds the Kelvin wavelength while |k| dx = g dx / U^2
 *             lies in [0.4, 2.0], i.e. dx between 0.4 U^2 / g = 0.041 U^2 and 2 U^2 / g = 0.204 U^2.  The source radius
 *             should span a few cells.
 *   stability with alpha = 0 a mode is stable iff 0 <= a3 Ghat(k) <= 4.  A call with g h^2 / dx * 4 > 4 (binary64) is
 *             rejected, so the largest sub-step is h = sqrt(dx / g) (dx = 1 m: 0.319 s; dx = 0.25 m: 0.160 s).
 *   sources   at sub-step k of a call a source sits at c = (x, z) + (vx, vz) tau, tau = (float)k * h, plus, when body >= 0,
 *             states[body].position.xz + states[body].linear_velocity.xz * tau (the device states of
 *             ocean_simulate_bodies_device: a boat's wake follows it with nothing crossing PCIe).  At each cell centre p,
 *             in source index order, phi += head * (1 - q2)^2 with q2 = |p - c|^2 / radius^2 < 1.  A source whose centre,
 *             head or radius is not finite, whose radius is <= 0 or radius^2 not finite, or (device sources) whose body
 *             index is not below num_states contributes nothing.  head is the pressure head p / (rho g); a stationary
 *             source with damping 0 is at rest at h = -phi.  The iWave damping term also pulls h itself towards 0, so with
 *             damping > 0 the rest state is a shallower depression (G(h + phi) = -(2 alpha dx / (g h)) h).
 *   scroll    each step call takes the origin; moving it by (di, dj) is exactly a shift of h and h_prev by those cells with
 *             zero fill (a move of N cells or more clears the layer), folded into the first sub-step's reads.
 * The sponge is sized for waves in the band: with iWave's damping it reflects about 4 % of a pulse in the band through a
 * 48-cell ramp to 1 / s, but much more of waves longer than the band, and a strong sponge_damping (which also acts as a
 * spring of stiffness 2 alpha / h) reflects more than a moderate one.
 * Coupling (ocean_wake_set_coupling, opt-in per generator; off, every op is bit-identical to a generator without a layer):
 * the surface query, buoyancy, body forces and the body integrator then read the wake on top of the maps, so bodies ride
 * each other's wakes.  oracle/wake_coupling.py is the specification, bit for bit.
 *   free surface  what they read is e = h + phi_end, not h: phi_end is the sources rasterised at the end of the step call,
 *             tau_end = (float)S * h (body-attached sources at position.xz + linear_velocity.xz * tau_end of the states the
 *             call was given).  The stencil acts on h + phi, which is 0 at rest under a stationary source, so a body that
 *             carries a source does not feel the depression its own head presses into the layer (that depression is the
 *             hull; reading h would sink it by about the head), while waves from other sources and the body's own radiated
 *             waves pass through e unchanged.  The render map and ocean_sample_wake keep showing h.
 *   snapshots enabling allocates two [N][N] binary32 snapshots e and e_old (counted in device_bytes), each with its own
 *             window origin, and marks them unprimed.  A step call on a coupled layer launches one more kernel after its
 *             sub-steps: the previous e (with its origin) becomes e_old and e = h + phi_end is written in the call's window;
 *             the first call after enabling or after ocean_wake_set_state writes e into both (primed from then on).  The
 *             interval T becomes tau_end of the call.  Disabling releases the snapshots; ocean_wake_init turns the coupling
 *             off.  While the coupling is on but unprimed the ops read nothing of the wake and launch nothing extra.
 *   ops       for each query point Q, after the inversion: (we, gx, gz) = the bilinear sample of e and of its central
 *             differences at Q in e's window (ocean_sample_wake's, 0 outside); displacement[1] += we, gradient_foam[0] += gx,
 *             gradient_foam[1] += gz; source_xz, displacement[0] and [2], foam, residual and iterations are unchanged (the
 *             wake has no horizontal displacement).  ocean_query_surface[_device], and ocean_buoyancy[_device],
 *             ocean_body_forces[_device] and ocean_simulate_bodies[_device] on their world hull points Q = (w.x, w.z), whose
 *             samples outputs carry the coupled records.  Drag adds the wake's vertical water velocity
 *             wv = (sample(e, Q) - sample(e_old, Q)) / T, each snapshot in its own window, to u.y before d = u - vb.
 *             Every sub-step of a simulate call reads the same e and e_old, as it reads the same maps.
 *   launches  while primed, one more kernel per step call, per surface query, per buoyancy or body-forces call with world
 *             points and per simulate sub-step with world points.
 * Foam (ocean_wake_set_foam, opt-in per generator): a foam field F ([N][N] binary32 in window order, values in [0, 1]) of
 * white water where the wake breaks and where sources stir it, advanced by each sub-step in the same kernel as h, for the
 * render map's fourth channel.  oracle/wake_foam.py is the specification, bit for bit.  F feeds nothing back: h, h_prev,
 * the coupling's snapshots and every op are byte-identical with foam on or off.
 *   model     per call the binary32 constants d = ocean_detmath_expf(-(decay_rate * h)) (the cascades' foam decay exp),
 *             gh = grow_rate * h and sh = stir_rate * h; per sub-step at tau_k, per cell, with c the cell's convolution of
 *             s = h + phi above:
 *               beta = c / dx   (at alpha = 0, h_new - 2 h + h_prev = -(g h^2 / dx) c: beta is the cell's downward vertical
 *                               acceleration in units of g, about the steepness kA on a crest of a wave in the stencil's
 *                               band; 0 at rest under a stationary source, so a boat at rest makes no foam)
 *               sigma = sum, in source index order over the sources that add to phi at the cell, of (w w) * |v|^2, with
 *                       w = 1 - q2 the weight above and v the centre velocity (vx, vz), plus linear_velocity.xz of its body
 *                       state when body >= 0; |v|^2 = vx vx + vz vz.  A source of radius r moving straight at U deposits
 *                       stir_rate (16 / 15) r U (1 - y^2 / r^2)^(5/2) at lateral offset y (with no decay)
 *               b = beta - whitecap, 0 unless b > 0;  x = F d + (gh b + sh sigma);  F' = min(x, 1) if x > 0, else 0
 *             (so NaN gives 0).  F scrolls with the window exactly as h does (shift with zero fill).
 *   memory    enabling allocates two [N][N] binary32 fields (counted in device_bytes), F zeroed; disabling releases them.
 *             ocean_wake_init turns foam off; ocean_wake_set_state leaves F as it is.
 *   launches  none extra: while foam is on each sub-step runs the foam form of the same kernel, and the render map the
 *             foam form of its kernel.
 *   limits    foam is not advected (the wake has no horizontal velocity; it stays where it forms, as the cascades' foam
 *             does); ocean_sample_maps and ocean_sample_velocity do not read it (spray does, under
 *             OCEAN_WAKE_READ_SPRAY); there is no per-source foam rate; the cascades' foam is unchanged.
 * Obstacles (ocean_wake_set_obstacles, opt-in per generator; without a mask every kernel and record is as above): a
 * world-fixed binary mask of blocked cells (quays, breakwaters, islands, the shore) that wake waves reflect from and cannot
 * cross.  oracle/wake_obstacles.py is the specification, bit for bit.
 *   grid      the mask lies on the layer's world cell grid: window cell (i, j) at origin (ox, oz) is world cell
 *             (I, J) = (ox + i, oz + j).  Mask bytes [depth][width]: row r is world cell row J = mz + r along z, column q
 *             world cell column I = mx + q along x; nonzero = blocked; every cell outside the rectangle is open.  No
 *             resampling: the window scrolls over the mask in whole cells.
 *   model     B(i, j): whether window cell (i, j) of the step call's window (the origin it is given; on a scrolled first
 *             sub-step the new window, the same world cell h is read at through the scroll) is blocked.  Per sub-step
 *             s = B ? +0 : h + phi;  h_new = B ? +0 : (a1 h - a2 h_prev) - a3 c;  with foam F' = B ? +0 : the update above;
 *             with the coupling e = B ? +0 : h + phi_end.  h_prev is the previous h, unmasked (on a scrolled sub-step the
 *             scrolled h); no open cell reads h_prev at a blocked cell.  The render map, ocean_sample_wake and the coupling's
 *             sampling and wv read h and e unchanged; h is +0 on blocked cells after every sub-step.  Three properties:
 *             1. A blocked cell is exactly a cell outside the window, which the step reads as s = +0: the open cells evolve
 *                bit for bit as in a window whose edge ran along the obstacle, so obstacles reflect as the window's edge
 *                always has (a vertical wall: a shoreline reflects more than a real beach would).
 *             2. Stability is unchanged: on the open cells the operator is P G P, a principal submatrix of the symmetric
 *                stencil G, which is positive semi-definite with 0 <= Ghat <= 4, so every eigenvalue of P G P lies in
 *                [0, 4] and the rule g h^2 / dx * 4 <= 4 above still holds.  The argument needs a 0/1 mask (a fractional
 *                mask multiplying h has none), which is why the mask is binary.
 *             3. Barriers and leaks: two open cells interact only if |di| <= 6 and |dj| <= 6, the stencil's radius.  A
 *                blocked band at least 6 cells thick in that sense (any two open cells on opposite sides more than 6
 *                cells apart along x or along z) is an exact barrier: water that starts at rest on its far side stays
 *                exactly +0, unless a source's own footprint reaches across the band (phi is rasterised at every cell
 *                within a source's radius).  A thinner band transmits part of a wave (a 1-cell wall passes about 6 % of
 *                an in-band pulse, a 5-cell one about 1 %).  In metres the barrier is 6 dx: at dx = 0.5 m a pier must be
 *                at least 3 m of blocked cells to stop waves entirely.
 *   memory    the mask is copied to the device as one byte per cell (width * depth bytes, counted in device_bytes).
 *   lifetime  a mask takes effect at the next step call.  Setting one touches none of h, h_prev, F or the snapshots (a
 *             blocked cell keeps its value until the next sub-step writes +0).  ocean_wake_init (re-create or release)
 *             removes the mask, since the cell size may change; ocean_wake_set_state, ocean_wake_set_foam and
 *             ocean_wake_set_coupling leave it as it is.
 *   launches  none extra: while a mask is set each sub-step and the free surface run the obstacle forms of their kernels.
 * Readers (ocean_wake_set_readers, opt-in per generator; with readers 0 every op is byte-identical to a generator without a
 * layer, whatever the coupling, foam and mask): the ray cast and spray read the layer too, so every op that answers "where is
 * the water" or "where is the white water" reads the same layers.  oracle/wake_readers.py is the specification, bit for bit.
 *   raycast   OCEAN_WAKE_READ_RAYCAST takes effect while the coupling is live (on and primed): ocean_raycast[_device] then
 *             reads what the surface query reads, the free surface e in its own window.  Each evaluation's gap is
 *             g = y - (eta + we), eta the cascades' height at the inverted source point as before and we the sample of e at
 *             the evaluated point's (x, z) (one binary32 add; the wake has no horizontal displacement, so the inversion, warm
 *             starts, restarts, march and refinement are unchanged).  The slab is widened by e's NaN-dropping extrema, taken
 *             per call by one more kernel: y_lo += fminf(e_min, 0), y_hi += fmaxf(e_max, 0) (the sample is 0 outside the
 *             window) and the padding's magnitude sum acc += fmaxf(|e_min|, |e_max|).  The record at the reported point gets
 *             the coupled record's additions at Q = (position.x, position.z): displacement[1] += we, gradient_foam[0] += gx,
 *             gradient_foam[1] += gz, so gap == position.y - displacement[1] holds as without the wake.  While the coupling
 *             is off or unprimed the bit does nothing and launches nothing.
 *   spray     OCEAN_WAKE_READ_SPRAY takes effect whenever a layer exists (no coupling needed: spray follows what the render
 *             map draws).  With (hw, hgx, hgz) = ocean_sample_wake's sample of h and Fw that of F (+0 while foam is off) at
 *             the candidate's START_POS.xz in the current window: the spawn test of ocean_extract_spray[_device] and
 *             ocean_spray_particles[_device] adds, right after the cascade sum and before the normalize, gradient.x += hgx,
 *             gradient.y += hgz, foam += Fw (so ocean_spray_record.foam is the sum); ocean_spray_particles adds hw to the
 *             particle's displacement y right after the cascade sum, every frame, so the spray rises from the wake surface.
 *   order     the ops read the layer as the last step call left it: a ray cast or spray call enqueued after
 *             ocean_wake_step[_device] on the generator's stream sees that tick's wake.
 *   limits    the coupled surface has a step at the edge of e's window (the sample drops to 0 there), as the surface query
 *             and the physics see it: a crossing bracketed across the step ends the refinement without |gap| <= tolerance.
 *             There is no cap on spray candidates per wake, and hull contact makes spray only where it makes wake foam.
 *   launches  one more kernel per ray cast with rays while the ray cast reader is in effect; none extra for spray (its
 *             kernels run their wake forms).
 * Limits: ocean_sample_maps and ocean_sample_velocity read the FFT maps only; the wake has no horizontal water velocity
 * (iWave is vertical only); static obstacles block
 * waves (ocean_wake_set_obstacles) but hulls do not (they are pressure sources); linear deep water only (no breaking,
 * shallow water or nonlinearity); the layer and the cascades interact by superposition only.  Far from the world origin
 * positions are binary32: phi, the cull and the samples use the cell centres x0 + (float)(i + 1/2) * dx, which lie within
 * about ulp(|x0|) of the exact (ox + i + 1/2) dx, i.e. up to 2^-23 |ox| cells (measured: 1.5 cells at |ox| = 2^24, 130 at
 * 2^31).  Keep |ox| and |oz| below about 2^21 cells (at most a quarter of a cell) for sources and samples to land
 * where the integer window says; beyond, the layer stays bit-identical to the specification, and the integer window, the
 * scroll and the mask remain exact.
 * Entry points (an invalid call returns OCEAN_ERR_INVALID_ARGUMENT, launches nothing and leaves the layer untouched; a call
 * on a generator without a layer returns OCEAN_ERR_STATE):
 *   ocean_wake_kernel_taps   the 28 taps G[a][b] in the order (0,0), (1,0), (1,1), (2,0), ... (6,6); host only, no device.
 *   ocean_wake_init          params->size = 0 releases the layer; otherwise (re)creates it zeroed at origin (0, 0).  A
 *                            valid call that fails in CUDA (OCEAN_ERR_CUDA) leaves the generator without a layer.
 *                            size a power of two in [128, 2048], cell_size finite > 0, damping and sponge_damping finite
 *                            >= 0, sponge_cells in [0, 64] and <= size / 2.
 *   ocean_wake_step          dt finite > 0, substeps in [1, 256], the stability rule above, num_sources and num_states
 *                            >= 0 with non-NULL arrays when > 0, and (host form) every source's body < num_states.
 *                            Launches `substeps` kernels, one more while the coupling is on.  The host form takes host sources and states and returns when
 *                            the work is enqueued; the device form takes device pointers; both are asynchronous on the
 *                            generator's stream.
 *   ocean_wake_render_map    writes [N][N][4] half (h, dh/dx, dh/dz, F) in window order into map_dev (device memory), F
 *                            while foam is on and 0 while it is off, each rounded to nearest even from binary32, central
 *                            differences (h[i+1] - h[i-1]) / (2 dx), cells outside reading 0; world_rect (host,
 *                            may be NULL) receives (x0, z0, N dx, N dx).  One kernel, asynchronous.
 *   ocean_sample_wake        bilinear h, dh/dx and dh/dz ([n][3] float) from the binary32 state at world (x, z); 0 outside
 *                            the window.  One kernel; the host form is synchronous, the device form asynchronous.
 *   ocean_wake_get_state / ocean_wake_set_state   host copies of h, h_prev ([N][N] float) and the origin, for tests and
 *                            checkpoints (synchronous).  set_state makes the coupling's snapshots unprimed.
 *   ocean_wake_set_coupling  enable 0 or 1 (anything else: OCEAN_ERR_INVALID_ARGUMENT, nothing changes); enabling a
 *                            coupled layer again changes nothing.  Synchronous on disable.
 *   ocean_wake_get_coupling  host copies of e and e_old ([N][N] float), origins[4] = (e.x, e.z, e_old.x, e_old.z) in cells
 *                            and the interval T; zeros, origins 0 and T = 0 while unprimed.  OCEAN_ERR_STATE while the
 *                            coupling is off; every pointer non-NULL.  Synchronous.
 *   ocean_wake_set_foam      a non-NULL params enables foam (F zeroed) or, when it is on, changes its parameters and keeps
 *                            F; NULL disables it and releases F (synchronous).  Every field finite, grow_rate, stir_rate and
 *                            decay_rate >= 0.
 *   ocean_wake_get_foam_state / ocean_wake_set_foam_state   host copies of F ([N][N] float) in the current window, for
 *                            tests and checkpoints (synchronous).  OCEAN_ERR_STATE while foam is off; non-NULL array.
 *   ocean_wake_set_obstacles mask_host = NULL with width = depth = 0 removes the mask and releases it; otherwise width and
 *                            depth >= 1, width * depth <= 2^28 (a 16384^2 mask: 8 km on a side at dx = 0.5 m), and
 *                            origin + width and origin + depth representable in int64.  An invalid call keeps the previous
 *                            mask.  Synchronous: returns once the mask is on the device.
 *   ocean_wake_set_readers   readers = a combination of OCEAN_WAKE_READ_RAYCAST and OCEAN_WAKE_READ_SPRAY (any other bit:
 *                            OCEAN_ERR_INVALID_ARGUMENT, nothing changes); 0 (the default) reads nothing.  Host only, launches
 *                            nothing.  ocean_wake_init (re-create or release) clears the readers; ocean_wake_set_state,
 *                            ocean_wake_set_foam, ocean_wake_set_coupling and ocean_wake_set_obstacles leave them as they are. */
typedef struct ocean_wake_params {
    int32_t size;               /* N: 0 (release) or a power of two in [128, 2048] */
    int32_t sponge_cells;       /* width of the absorbing ring, [0, 64] and <= size / 2 */
    float cell_size;            /* dx, metres */
    float damping;              /* alpha in the interior, 1/s */
    float sponge_damping;       /* alpha at the window edge, 1/s */
} ocean_wake_params;            /* 20 B */
typedef struct ocean_wake_source {
    float x, z;                 /* world position at the start of the call (offset from the body when body >= 0) */
    float vx, vz;               /* velocity, m/s */
    float radius;               /* m, > 0 */
    float head;                 /* pressure head p / (rho g), m (positive pushes the surface down) */
    int32_t body;               /* index into the body states, or -1 */
} ocean_wake_source;            /* 28 B */
typedef struct ocean_wake_foam_params {
    float whitecap;             /* beta = c / dx above which the wake breaks (units of g) */
    float grow_rate;            /* foam per second per unit of beta above whitecap, >= 0 */
    float stir_rate;            /* foam per second per (m/s)^2 of the sources' weighted squared speed, >= 0 */
    float decay_rate;           /* 1/s, >= 0: F decays as exp(-decay_rate t) */
} ocean_wake_foam_params;       /* 16 B */
int ocean_wake_kernel_taps(float* taps_host);
int ocean_wake_init(ocean_generator* gen, const ocean_wake_params* params);
int ocean_wake_step(ocean_generator* gen, double dt, int substeps, int64_t origin_x, int64_t origin_z, int num_sources,
                    const ocean_wake_source* sources_host, int num_states, const ocean_body_state* states_host);
int ocean_wake_step_device(ocean_generator* gen, double dt, int substeps, int64_t origin_x, int64_t origin_z, int num_sources,
                           const ocean_wake_source* sources_dev, int num_states, const ocean_body_state* states_dev);
int ocean_wake_render_map(ocean_generator* gen, void* map_dev, float* world_rect);
int ocean_sample_wake(ocean_generator* gen, int num_points, const float* points_xz_host, float* out_host);
int ocean_sample_wake_device(ocean_generator* gen, int num_points, const float* points_xz_dev, float* out_dev);
int ocean_wake_get_state(ocean_generator* gen, float* h_host, float* h_prev_host, int64_t* origin_xz);
int ocean_wake_set_state(ocean_generator* gen, const float* h_host, const float* h_prev_host, int64_t origin_x, int64_t origin_z);
int ocean_wake_set_coupling(ocean_generator* gen, int enable);
int ocean_wake_get_coupling(ocean_generator* gen, float* e_host, float* e_old_host, int64_t* origins, float* interval);
int ocean_wake_set_foam(ocean_generator* gen, const ocean_wake_foam_params* params);
int ocean_wake_get_foam_state(ocean_generator* gen, float* foam_host);
int ocean_wake_set_foam_state(ocean_generator* gen, const float* foam_host);
int ocean_wake_set_obstacles(ocean_generator* gen, const uint8_t* mask_host, int32_t width, int32_t depth, int64_t origin_x,
                             int64_t origin_z);
#define OCEAN_WAKE_READ_RAYCAST 1u      /* ocean_raycast[_device] reads the wake free surface e */
#define OCEAN_WAKE_READ_SPRAY 2u        /* ocean_extract_spray[_device], ocean_spray_particles[_device] read h and F */
int ocean_wake_set_readers(ocean_generator* gen, uint32_t readers);

/* Sea state -- the statistics of the sea the cascades' spectra describe: wave height, periods, direction, slope and Stokes
 * drift, for authoring parameters, driving audio and choosing the knobs other ops take (a ray cast's step against crest
 * thickness, the wake layer's cell_size, query tolerances).  oracle/sea_state.py is the specification, bit for bit.
 *   terms     per texel id of a cascade's spectrum texture as stored, A(id) = its .xy (each wave once), with the binary32
 *             k_vec, k_unit and omega of the dispersion table its updates use (rows y > N/2 are the mirror of row N - y:
 *             omega the same, k_vec and k_unit negated except k_vec.x and k_unit.x in column 0) and
 *             k = sqrt(k_vec.x k_vec.x + k_vec.y k_vec.y) + 1e-6 (spectrum_modulate.glsl:60), in binary64:
 *               E = 2 |A|^2 = 2 (A.x A.x + A.y A.y)   the texel's share of the height variance (the transform is
 *                                                      unnormalised: one A of modulus a is a height cosine of amplitude 2a)
 *               d = -(k_unit.y, k_unit.x)            world direction of travel (the maps are the transpose of the
 *                                                      spectrum's field, and h0 e^{+i w t} under e^{+i k.x} travels along -k)
 *               kw = (k_vec.y, k_vec.x)              world wave vector
 *               q = ocean_detmath_expf(-((2 k) * 20)), F = (1 + q q) / ((1 - q)(1 - q)) = cosh 2kD / (2 sinh^2 kD) at the
 *                                                      library's depth D = 20 m
 *             moments (sums over the texels): m_minus1 = E / w, m0 = E, m1 = w E, m2 = (w w) E, direction = E d,
 *             slope = (E kw.x^2, E kw.z^2), stokes = (((2 w) k) E) F d.  The DC texel (N/2, N/2) and texels with E = 0 or
 *             1 - q = 0 contribute nothing.
 *   order     binary64, fixed: thread t of T = N^2 / 16 sums texels t, t + T, ... from +0; a warp shuffle tree (lane l adds
 *             lane l + 16, then + 8, + 4, + 2, + 1); the 8 warps of a 256-thread block in warp order from +0; the N^2 / 4096
 *             blocks in block order from +0.  No floating-point atomics: the moments are a function of the spectrum.
 *   cache     the moments of each cascade are cached on the device (allocated by the first sea-state or drift call, counted
 *             in device_bytes).  A cascade becomes stale when its spectrum is written (regeneration on
 *             should_generate_spectrum, ocean_set_spectrum_amplitudes) or its dispersion table changes (a new tile_length);
 *             a call recomputes the stale cascades in one launch sequence of 2 kernels (none when nothing is stale).  A
 *             cascade that has not been updated yet has zero moments.
 *   total     sum over i in [0, num_cascades) in cascade order of (s_i s_i) moments_i, s_i = (double)map_scales[i].z (the
 *             displacement scale): the statistics of the surface as rendered, the cascades being independent fields whose
 *             variances add.  per_cascade[i] (may be NULL) holds the unscaled moments.
 *   derived   on the host, binary64, every one 0 when m0 = 0:
 *               significant_wave_height  Hs = 4 sqrt(m0)
 *               mean_period              Tm01 = 2 pi m0 / m1
 *               zero_crossing_period     Tm02 = 2 pi sqrt(m0 / m2)
 *               energy_period            Te = 2 pi m_minus1 / m0
 *               mean_direction           degrees(atan2(-direction[1], -direction[0])): the wind_direction whose spectrum
 *                                        peaks there (spectrum_compute.glsl's theta); the waves travel towards it + 180
 *               directional_spread       sqrt(2 max(0, 1 - R)) radians, R = |direction| / m0 (circular spread)
 *               mean_square_slope        slope[0] + slope[1]
 *               stokes_speed             |stokes| (m/s); stokes itself is the surface Stokes drift vector
 *             The peak period is not a moment: 2 pi / ocean_jonswap_peak_angular_frequency is the model's.
 * ocean_get_sea_state is host-only and synchronous (the sea state changes only when a spectrum does); the drifters read the
 * cache on the device.  num_cascades in [1, num_cascades of the generator], map_scales and total non-NULL.  The entry point
 * is ocean_get_sea_state rather than ocean_sea_state because C gives a function and a typedef one namespace, and the record
 * below holds that name. */
typedef struct ocean_sea_state {
    double m_minus1, m0, m1, m2;        /* spectral moments: sum E / w, E, w E, w^2 E (m^2 s, m^2, m^2 / s, m^2 / s^2) */
    double direction[2];                /* sum E d, world (x, z) */
    double slope[2];                    /* sum E kw.x^2, sum E kw.z^2 */
    double stokes[2];                   /* surface Stokes drift, m/s, world (x, z) */
    double significant_wave_height;     /* derived fields (above) */
    double mean_period;
    double zero_crossing_period;
    double energy_period;
    double mean_direction;              /* degrees */
    double directional_spread;          /* radians */
    double mean_square_slope;
    double stokes_speed;                /* m/s */
} ocean_sea_state;                      /* 144 B */
int ocean_get_sea_state(ocean_generator* gen, int num_cascades, const float* map_scales_host, ocean_sea_state* per_cascade_host,
                    ocean_sea_state* total_host);

/* Drifters -- the bulk of what floats in a scene (debris, crates, seaweed, foam patches, buoys used as props): thousands of
 * objects that ride the waves and drift with the sea, one thread each, with render-ready MultiMesh instances.  A drifter is
 * a Lagrangian label: the undisplaced point P whose surface point P + D(P, t) it sits at.  Tessendorf's choppy displacement
 * is the first-order Lagrangian displacement of the surface, so a fixed label moves on a closed orbit (the bodies of
 * ocean_simulate_bodies bob in place); real floating matter drifts with the Stokes drift, the second-order mean of those
 * orbits, which is a label velocity.  oracle/drifters.py is the specification, bit for bit.  One call, per drifter:
 *   drift   (dt > 0 only) u = stokes_scale * us + current + windage * wind, with us = sum over i in cascade order of
 *           (s_i s_i) stokes_i (the sea-state cache under the call's map_scales, s_i = map_scales[i].z), binary64:
 *           u = ((stokes_scale us) + current) + (windage wind);  x += dt u.x, z += dt u.z;
 *           yaw = (float)((double)yaw + dt yaw_rate)
 *   wrap    (dt > 0, OCEAN_DRIFT_WRAP) r = x - x0, x = x0 + (r - W floor(r / W)), z likewise with (z0, D): labels stay in
 *           [x0, x0 + W] x [z0, z0 + D] (the closed box: the last rounding may land on the far edge), the ambient debris
 *           field around a moving camera
 *   render  (instances not NULL) the maps at (float)P with ocean_sample_maps' filter (displacement D, gradient g), then
 *           X = ((float)(x + D.x), (float)((D.y [+ hw]) + offset), (float)(z + D.z)), each sum binary64 and rounded once;
 *           n = normalize(-g.x, 1, -g.y), n_t = normalize(up + tilt (n - up)) (every operation binary32, as written);
 *           basis y = n_t, z = normalize(f - (f . n_t) n_t) with f = (sin yaw, 0, cos yaw) (DETMATH sincos), x = y cross z,
 *           each column times scale -- with tilt = 0 it is Godot's Basis(Vector3.UP, yaw) * scale up to rounding.  12 floats
 *           per drifter in drifter order, the 3 x 4 row-major layout of ocean_simulate_bodies' transforms (a MultiMesh
 *           TRANSFORM_3D buffer).
 *   wake    with OCEAN_DRIFT_READ_WAKE and a wake layer present, ocean_sample_wake's (hw, hgx, hgz) at (X.x, X.z) is added
 *           to the height (in binary64, above) and to g (g.x += hgx, g.y += hgz) before the normal, so drifters sit on the
 *           surface the render maps draw.  The wake has no horizontal velocity: drifters bob on wakes but are not pushed.
 * dt = 0 only renders (the labels are not written).  A drifter is not validated: a NaN or infinite one affects only itself.
 * Limits: the Stokes drift is the surface value of linear theory (no vertical profile, no wave-current interaction); it is
 * uniform in space (the mean of the whole spectrum, not the local wave group's); drifters do not collide with each other or
 * with bodies; the render is the surface within 150 m of the camera (ocean_query_surface's limit).
 * Validation: dt finite and >= 0, params non-NULL with every field finite, box width and depth > 0 with OCEAN_DRIFT_WRAP,
 * no unknown flag, num_cascades in [1, num_cascades of the generator], map_scales non-NULL, num_drifters >= 0 and drifters
 * non-NULL when num_drifters > 0.  An invalid call returns OCEAN_ERR_INVALID_ARGUMENT, launches nothing and leaves the
 * drifters untouched.  A call with drifters and dt > 0 first brings stale sea-state cascades up to date (2 kernels when any
 * is stale), then launches 1 kernel; with dt = 0 only the 1.  ocean_drift takes host drifters (updated in place) and
 * instances and is synchronous; ocean_drift_device takes device pointers for them and is asynchronous on the generator's
 * stream. */
#define OCEAN_DRIFT_WRAP 1u             /* wrap the labels into params.box */
#define OCEAN_DRIFT_READ_WAKE 2u        /* the render reads the wake layer's h and slopes */
typedef struct ocean_drifter {
    double x, z;                /* the label: undisplaced point P, world metres (binary64: mm per frame kilometres out) */
    float yaw, yaw_rate;        /* radians and rad/s, about the surface normal */
    float windage;              /* fraction of the wind vector added to the drift */
    float tilt;                 /* 0 stays upright, 1 follows the surface normal */
    float offset;               /* metres added to the height */
    float scale;                /* uniform instance scale */
} ocean_drifter;                /* 40 B */
typedef struct ocean_drift_params {
    float current[2];           /* m/s, world x and z */
    float wind[2];              /* m/s, world x and z */
    float stokes_scale;         /* 1 is physical, 0 turns the Stokes drift off */
    uint32_t flags;             /* OCEAN_DRIFT_* */
    double box[4];              /* wrap box (x0, z0, width, depth), metres */
} ocean_drift_params;           /* 56 B */
int ocean_drift(ocean_generator* gen, double dt, const ocean_drift_params* params, int num_drifters, ocean_drifter* drifters_host,
                int num_cascades, const float* map_scales_host, float* instances_host);
int ocean_drift_device(ocean_generator* gen, double dt, const ocean_drift_params* params, int num_drifters, ocean_drifter* drifters_dev,
                       int num_cascades, const float* map_scales_host, float* instances_dev);

/* Parity/debug taps (not timed): binary32 maps before the half conversion, the row-pass output
 * ([4][N][N][2] float, == fft_buffer half 1 after the first fft_compute, wave_generator.gd:79) and
 * the twiddle table ([N-1][2] float: stage s, index j at (1<<s)-1+j; fft_butterfly.glsl:27).
 * The row-pass scratch is only preserved while the taps are enabled (otherwise the column pass discards it from
 * L2 as soon as it is consumed): ocean_copy_rowpass_to_host returns OCEAN_ERR_STATE with the taps off. */
int ocean_enable_f32_taps(ocean_generator* gen, int enable);
int ocean_copy_f32_maps_to_host(ocean_generator* gen, int cascade, float* displacement_host, float* normal_host);
int ocean_copy_rowpass_to_host(ocean_generator* gen, int cascade, float* host);
int ocean_copy_twiddles_to_host(ocean_generator* gen, float* host);

/* Checkpoint/resume of the only frame-to-frame state, the foam of fft_unpack.glsl:61-64: [map_size][map_size] IEEE half
 * for one cascade.  The state lives in a plane of its own; every update copies it into normal_map.a, and ocean_set_foam_state
 * writes both.  Writing normal_map.a through ocean_get_maps does not seed the next update's foam. */
int ocean_get_foam_state(ocean_generator* gen, int cascade, uint16_t* host);
int ocean_set_foam_state(ocean_generator* gen, int cascade, const uint16_t* host);

/* static func JONSWAP_alpha / JONSWAP_peak_angular_frequency, wave_generator.gd:116-121
 * (fetch_length in metres, binary64). */
double ocean_jonswap_alpha(double wind_speed, double fetch_length);
double ocean_jonswap_peak_angular_frequency(double wind_speed, double fetch_length);

/* Device-side timing on the generator's stream (CUDA events), used by bench.py. */
int ocean_timer_start(ocean_generator* gen);
int ocean_timer_stop(ocean_generator* gen, float* elapsed_ms); /* synchronizes */

/* Per-kernel device times of the most recent launch sequence (CUDA events between the kernels):
 * spectrum generation, then kernel A (time propagation + row IFFT) and kernel B (column IFFT + maps)
 * of the FIRST L2-sized chunk, whose cascade count is returned through chunk_cascades. */
int ocean_set_profiling(ocean_generator* gen, int enable);
int ocean_get_last_kernel_times(ocean_generator* gen, float* spectrum_ms, float* rowpass_ms, float* colpass_ms,
                                int* chunk_cascades);

/* Device self-test: the kernels' branch-free correctly-rounded sqrt/div against the IEEE intrinsics
 * (every binary32 in [2^-100, 2^100] for sqrt, ~1.2e9 random pairs for div). */
int ocean_selftest_math(ocean_generator* gen, uint64_t* failures, uint64_t* tested);

/* Device math debug entry: evaluates on the device, one element per thread, exactly the device function the kernels use,
 * on n pairs (a[i], b[i]) of host binary32 values, and writes out[2i], out[2i+1] (host, 2n floats).  Slow (staged copies
 * and a synchronise); for comparing the device copy of DETMATH and the branch-free quotients with the CPU oracle.
 *   OCEAN_MATH_SINCOS      sincosf_det(a)                        -> sin, cos
 *   OCEAN_MATH_SINCOS_N4   sincosf_det_n<4>, elements 4t..4t+3 as the four lanes of one call -> sin, cos
 *   OCEAN_MATH_COS         cosf_det(a) (binary64 sincos64)       -> cos, 0
 *   OCEAN_MATH_EXP / LOG / TANH / INVERSESQRT of a               -> f, 0
 *   OCEAN_MATH_POW         powf_det(a, b), a >= 0                -> f, 0
 *   OCEAN_MATH_ATAN2       atan2f_det(a, b) (y = a, x = b)       -> f, 0
 *   OCEAN_MATH_DIV         a / b by the column pass's branch-free quotient (rcp_refined + div_rn_fast); correctly rounded
 *                          for a == +0 or 2^-100 <= |a| <= 2^100 and 1 <= b <= 2^20 + 1  -> q, 0
 *   OCEAN_MATH_SQRT        the branch-free sqrt_rn_fast(a); correctly rounded for a == 0 or 2^-100 <= a <= 2^100  -> r, 0
 *   OCEAN_MATH_HALF        the maps' binary32 -> binary16 conversion (round to nearest even) of a and b, widened back to
 *                          binary32 (exact)                      -> half(a), half(b)
 *   OCEAN_MATH_SIN64 / OCEAN_MATH_COS64  the binary64 kernel sincos64((double)a) before any rounding to binary32: one
 *                          binary64 in the 8 bytes of out[2i], out[2i+1] (shows differences far below a binary32 ulp) */
enum {
    OCEAN_MATH_SINCOS = 0, OCEAN_MATH_SINCOS_N4 = 1, OCEAN_MATH_COS = 2, OCEAN_MATH_EXP = 3, OCEAN_MATH_LOG = 4,
    OCEAN_MATH_POW = 5, OCEAN_MATH_TANH = 6, OCEAN_MATH_ATAN2 = 7, OCEAN_MATH_INVERSESQRT = 8, OCEAN_MATH_DIV = 9,
    OCEAN_MATH_SQRT = 10, OCEAN_MATH_HALF = 11, OCEAN_MATH_SIN64 = 12, OCEAN_MATH_COS64 = 13
};
int ocean_debug_device_math(ocean_generator* gen, int fn, int n, const float* a, const float* b, float* out);

/* Host-side view of the persistent kernel's work queue for `count` cascades of `map_size` (no GPU needed): writes up to `capacity`
 * packed items (bit 31 = column-pass item, bits 16..30 = dispatch slot, bits 0..15 = block) in hand-out order and returns the item
 * count (negative status on error).  frames == 0: the order of a single update for the given group size and lag (0 = the library's
 * defaults for that map size, after OCEAN_QUEUE_GROUP / OCEAN_QUEUE_LAG), slot = cascade position.  frames >= 1: the order of a
 * fused launch of that many consecutive updates (ocean_update_frames), slot = frame * count + cascade position.  Lets the
 * deadlock-freedom invariant -- whatever an item waits for was handed out before it, each item exactly once -- be checked on the
 * CPU (tests/test_abi_cpu.py). */
int ocean_debug_work_queue(int map_size, int count, int group, int lag, int frames, int32_t* items, int capacity);

/* Host-side view of the completion-counter protocol of a fused launch (ocean_update_frames; no GPU needed).  `counters` holds
 * 3 * num_cascades values -- [c] row passes of cascade c in scratch half 0, [num_cascades + c] its column passes,
 * [2 * num_cascades + c] its row passes in half 1 -- as they stand when a launch of `frames` frames (frame indices first_frame,
 * first_frame + 1, ... of the call) over cascades 0..count-1 starts; on return they hold the values after the launch.  `records`
 * receives, per (frame, cascade) in the dispatch-slot order of ocean_debug_work_queue(frames >= 1), six int32:
 * cascade, counter the row pass bumps / the column pass waits on, its target, the column-pass count the row pass waits for, the
 * column-pass count the column pass waits for, first scratch layer pair.  tests/test_queue_protocol_cpu.py runs this protocol on
 * the CPU against random team schedules and checks that no item ever reads unfinished or overwritten data and that nobody waits forever. */
int ocean_debug_frame_protocol(int map_size, int num_cascades, int count, int first_frame, int frames, uint32_t* counters, int32_t* records);

int ocean_get_info(ocean_generator* gen, ocean_info* out);
const char* ocean_last_error(void);
const char* ocean_version(void);

#ifdef __cplusplus
}
#endif
#endif /* OCEAN_H */
