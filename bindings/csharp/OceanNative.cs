// OceanNative.cs -- P/Invoke binding of libocean.so (include/ocean.h) and a WaveGenerator-shaped host class.
//
// NOT COMPILED IN THIS REPOSITORY'S CI: the build image has no dotnet/mono/csc.  The ABI is exercised through
// the Python ctypes mirror (godotoceanwaves_b200/native.py) and tests/test_abi_cpu.py instead; this file shows the
// binding a Godot C# project would add.  Convention follows the one in-tree P/Invoke precedent of the reference,
// addons/imgui-godot/ImGuiGodot/Internal/Viewports.cs:157-165 ([LibraryImport], cdecl, unsafe partial).
//
// Replaces: assets/water/wave_generator.gd (WaveGenerator node) and, below it, every RenderingContext call of
// assets/render_context.gd:35-135 that the generator makes.  The two RGBA16F layered maps are handed to Godot with
// RenderingDevice.TextureUpdate(rid, layer, bytes), which the reference's textures already allow
// (TEXTURE_USAGE_CAN_UPDATE_BIT, wave_generator.gd:34-35).
using System;
using System.Runtime.InteropServices;

namespace OceanB200
{
    [StructLayout(LayoutKind.Sequential)]
    public unsafe struct OceanCascadeParams            // struct ocean_cascade_params <- wave_cascade_parameters.gd:2-42
    {
        public fixed float tile_length[2];
        public double displacement_scale, normal_scale;
        public double wind_speed, wind_direction, fetch_length, swell, spread, detail, whitecap, foam_amount;
        public fixed int spectrum_seed[2];
        public int should_generate_spectrum;
        public double time, foam_grow_rate, foam_decay_rate;
    }

    [StructLayout(LayoutKind.Sequential)]
    public struct OceanScheduler                                    // struct ocean_scheduler <- water.gd:51,62-63
    {
        public double updates_per_second, time, next_update_time;
    }

    [StructLayout(LayoutKind.Sequential)]
    public unsafe struct OceanSprayRecord                           // struct ocean_spray_record <- sea_spray_particle.gdshader:80-94
    {
        public uint index;
        public float start_x, start_z, scale_factor;
        public fixed float particle_scale[3];
        public float foam;
    }

    [StructLayout(LayoutKind.Sequential)]
    public unsafe struct OceanSprayEmitter                          // struct ocean_spray_emitter (88 B) <- main.tscn:133-140
    {
        public int amount;                                          // GPUParticles3D.amount
        public int num_particles;                                   // the shader's num_particles uniform (grid side sqrt)
        public fixed float emission_transform[12];                  // 3 x 4 row-major, basis columns then origin
        public fixed float particle_scale[3];
        public float lifetime, lifetime_randomness;
        public uint random_seed;
        public double emitter_lifetime;                             // GPUParticles3D.lifetime (LIFETIME)
    }

    [StructLayout(LayoutKind.Sequential)]
    public unsafe struct OceanSprayParticle                         // struct ocean_spray_particle (120 B); all zero = never emitted
    {
        public fixed float transform[12];                           // 3 x 4 row-major like the instances
        public fixed float custom[4];
        public fixed float userdata1[4];                            // START_POS, START_TIME
        public fixed float userdata2[4];                            // PARTICLE_SCALE, PARTICLE_LIFETIME
        public fixed float userdata3[4];                            // .z SCALE_FACTOR, .w HAS_STARTED
        public uint number, flags;                                  // flags: 1 ACTIVE, 2 EMITTED
    }

    [StructLayout(LayoutKind.Sequential)]
    public struct OceanWakeParams                                   // struct ocean_wake_params (20 B); size 0 releases the layer
    {
        public int size;                                            // N: a power of two in [128, 2048]
        public int sponge_cells;                                    // [0, 64], <= size / 2
        public float cell_size;                                     // dx, m
        public float damping, sponge_damping;                       // alpha in the interior and at the edge, 1/s
    }

    [StructLayout(LayoutKind.Sequential)]
    public struct OceanWakeSource                                   // struct ocean_wake_source (28 B)
    {
        public float x, z, vx, vz;                                  // position at the start of the call (offset from the body when body >= 0), m/s
        public float radius;                                        // m, > 0
        public float head;                                          // pressure head p / (rho g), m
        public int body;                                            // index into the body states, or -1
    }

    [StructLayout(LayoutKind.Sequential)]
    public struct OceanWakeFoamParams                               // struct ocean_wake_foam_params (16 B)
    {
        public float whitecap;                                      // beta = c / dx above which the wake breaks
        public float grow_rate, stir_rate, decay_rate;              // >= 0; 1/s, 1/s per (m/s)^2, 1/s
    }

    [StructLayout(LayoutKind.Sequential)]
    public unsafe struct OceanSeaState                              // struct ocean_sea_state (144 B)
    {
        public double m_minus1, m0, m1, m2;                         // spectral moments
        public fixed double direction[2];                           // sum E d, world (x, z)
        public fixed double slope[2];                               // sum E kx^2, sum E kz^2
        public fixed double stokes[2];                              // surface Stokes drift, m/s
        public double significant_wave_height, mean_period, zero_crossing_period, energy_period;
        public double mean_direction;                               // degrees, wind_direction's convention
        public double directional_spread;                           // radians
        public double mean_square_slope, stokes_speed;
    }

    [StructLayout(LayoutKind.Sequential)]
    public struct OceanDrifter                                      // struct ocean_drifter (40 B)
    {
        public double x, z;                                         // the label: undisplaced point P
        public float yaw, yaw_rate;                                 // radians, rad/s
        public float windage, tilt, offset, scale;
    }

    [StructLayout(LayoutKind.Sequential)]
    public unsafe struct OceanDriftParams                           // struct ocean_drift_params (56 B)
    {
        public fixed float current[2];                              // m/s, world x and z
        public fixed float wind[2];                                 // m/s, world x and z
        public float stokes_scale;                                  // 1 physical, 0 off
        public uint flags;                                          // OCEAN_DRIFT_WRAP (1) | OCEAN_DRIFT_READ_WAKE (2)
        public fixed double box[4];                                 // wrap box (x0, z0, width, depth)
    }

    [StructLayout(LayoutKind.Sequential)]
    public unsafe struct OceanSurfaceSample                         // struct ocean_surface_sample (40 B) <- water.gdshader:28,37 inverted
    {
        public float source_x, source_z;
        public fixed float displacement[3];                         // displacement[1] = water height at the query point
        public fixed float gradient_foam[3];                        // normal = normalize(-g.x, 1, -g.y), water.gdshader:90
        public float residual;
        public uint iterations;
    }

    [StructLayout(LayoutKind.Sequential)]
    public unsafe struct OceanBuoyancyPoint                         // struct ocean_buoyancy_point (20 B), body-local
    {
        public fixed float position[3];
        public float volume;                                        // m^3 of the vertical column element centred on the point
        public float half_height;                                   // m above and below the point
    }

    [StructLayout(LayoutKind.Sequential)]
    public unsafe struct OceanBuoyancyBody                          // struct ocean_buoyancy_body (56 B)
    {
        public fixed float transform[12];                           // 3 x 4 row-major body-to-world [R | t]
        public int first_point, num_points;                         // hull-point range; bodies may share a hull
    }

    [StructLayout(LayoutKind.Sequential)]
    public unsafe struct OceanBuoyancyResult                        // struct ocean_buoyancy_result (48 B)
    {
        public fixed float force[3];                                // apply_force(force, center_offset) in Godot
        public fixed float torque[3];                               // about the body origin
        public float submerged_volume;
        public fixed float center_offset[3];                        // centre of buoyancy - body origin
        public float max_residual;
        public uint unconverged;
    }

    [StructLayout(LayoutKind.Sequential)]
    public unsafe struct OceanBodyVelocity                          // struct ocean_body_velocity (24 B), world frame
    {
        public fixed float linear[3];                               // of the body ORIGIN: Godot's linear_velocity + angular x (t - com)
        public fixed float angular[3];                              // rad/s
    }

    [StructLayout(LayoutKind.Sequential)]
    public unsafe struct OceanDragResult                            // struct ocean_drag_result (32 B)
    {
        public fixed float force[3];
        public fixed float torque[3];                               // about the body origin
        public float wetted_drag_area;                              // sum of f * C_d A (m^2)
        public float max_relative_speed;                            // over the submerged points: for choosing sub-steps
    }

    [StructLayout(LayoutKind.Sequential)]
    public unsafe struct OceanFloatingBody                          // struct ocean_floating_body (24 B)
    {
        public float mass;                                          // kg, finite and > 0
        public fixed float inertia[3];                              // principal moments about the centre of mass (kg m^2), hull axes
        public int first_point, num_points;                         // range into the hull points and drag areas
    }

    [StructLayout(LayoutKind.Sequential)]
    public unsafe struct OceanBodyState                             // struct ocean_body_state (52 B)
    {
        public fixed float position[3];                             // the centre of mass: global_position + basis * center_of_mass
        public fixed float orientation[4];                          // unit quaternion x, y, z, w (Godot's Quaternion order), body -> world
        public fixed float linear_velocity[3];                      // of the centre of mass (RigidBody3D.LinearVelocity)
        public fixed float angular_velocity[3];                     // world frame, rad/s (RigidBody3D.AngularVelocity)
    }

    [StructLayout(LayoutKind.Sequential)]
    public unsafe struct OceanThruster                              // struct ocean_thruster (36 B): an engine or jet
    {
        public int body;
        public fixed float position[3];                             // hull-local
        public fixed float direction[3];                            // hull-local; rotate it to steer an outboard
        public float thrust;                                        // N, scaled by the point's immersion
        public float half_height;
    }

    [StructLayout(LayoutKind.Sequential)]
    public unsafe struct OceanFoil                                  // struct ocean_foil (36 B): a keel, rudder or fin
    {
        public int body;
        public fixed float position[3];                             // hull-local centre of pressure
        public fixed float normal[3];                               // hull-local plate normal; rotate it to turn a rudder
        public float area;                                          // C_n A, m^2, finite and >= 0
        public float half_height;
    }

    [StructLayout(LayoutKind.Sequential)]
    public unsafe struct OceanBodyLoad                              // struct ocean_body_load (24 B): sails, gusts, impulses
    {
        public fixed float force[3];                                // world frame
        public fixed float torque[3];                               // world frame, about the centre of mass
    }

    [StructLayout(LayoutKind.Sequential)]
    public unsafe struct OceanTether                                // struct ocean_tether (44 B): a mooring or tow line
    {
        public int body_a;
        public int body_b;                                          // -1: point_b is a world anchor
        public fixed float point_a[3];
        public fixed float point_b[3];
        public float rest_length, stiffness, damping;               // finite and >= 0
    }

    [StructLayout(LayoutKind.Sequential)]
    public unsafe struct OceanDriveResult                           // struct ocean_drive_result (32 B)
    {
        public fixed float force[3];                                // what the thrusters, foils, tethers and load added
        public fixed float torque[3];
        public float wetted_foil_area;
        public float max_normal_speed;
    }

    [StructLayout(LayoutKind.Sequential)]
    public struct OceanHullMesh                                     // struct ocean_hull_mesh (24 B): a triangle-mesh hull
    {
        public int first_vertex, num_vertices;                      // range of the vertices ([3] float each, hull-local)
        public int first_triangle, num_triangles;                   // range of the triangles ([3] int each, Godot's clockwise winding)
        public float normal_drag, tangential_drag;                  // C_n, C_t, finite and >= 0
    }

    [StructLayout(LayoutKind.Sequential)]
    public unsafe struct OceanHullBody                              // struct ocean_hull_body (56 B)
    {
        public fixed float transform[12];                           // 3 x 4 row-major [R | t]
        public int mesh;
        public int reserved;
    }

    [StructLayout(LayoutKind.Sequential)]
    public unsafe struct OceanFloatingHull                          // struct ocean_floating_hull (20 B)
    {
        public float mass;
        public fixed float inertia[3];
        public int mesh;
    }

    [StructLayout(LayoutKind.Sequential)]
    public unsafe struct OceanRay                                   // struct ocean_ray (28 B)
    {
        public fixed float origin[3];
        public fixed float direction[3];                            // need not be unit; t is in units of |direction|
        public float t_max;                                         // +inf allowed
    }

    [StructLayout(LayoutKind.Sequential)]
    public unsafe struct OceanRayHit                                // struct ocean_ray_hit (72 B)
    {
        public float t;
        public fixed float position[3];
        public float source_x, source_z;
        public fixed float displacement[3];
        public fixed float gradient_foam[3];
        public float gap;                                           // position.y - water height there
        public float residual;
        public uint status;                                         // OCEAN_RAY_*: 0 miss, 1 hit from above, 2 from below, 3 truncated, 4 invalid
        public uint evaluations, iterations, unconverged;
    }

    [StructLayout(LayoutKind.Sequential)]
    public struct OceanInfo
    {
        public int device, map_size, num_cascades, pending_cascades;
        public ulong kernel_launches, cascade_updates, device_bytes;
    }

    internal static unsafe partial class Native
    {
        private const string Lib = "ocean";           // libocean.so next to the Godot binary / in LD_LIBRARY_PATH

        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_default_cascade_params(OceanCascadeParams* p);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_create(int device, int map_size, int num_cascades, IntPtr* handle);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_destroy(IntPtr handle);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_update(IntPtr handle, double delta, OceanCascadeParams* parameters, int count);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_process(IntPtr handle, OceanCascadeParams* parameters, int count);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_update_all(IntPtr handle, double delta, OceanCascadeParams* parameters, int count);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_get_maps(IntPtr handle, IntPtr* displacement_dev, IntPtr* normal_dev, nuint* layer_bytes);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_copy_maps_to_host(IntPtr handle, int first, int count, void* displacement, void* normal);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_copy_maps_to_host_async(IntPtr handle, int first, int count, void* displacement, void* normal);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_synchronize(IntPtr handle);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_host_alloc(void** ptr, nuint bytes);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_host_free(void* ptr);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_get_foam_state(IntPtr handle, int cascade, ushort* host);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_set_foam_state(IntPtr handle, int cascade, ushort* host);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial double ocean_jonswap_alpha(double wind_speed, double fetch_length);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial double ocean_jonswap_peak_angular_frequency(double wind_speed, double fetch_length);
        // map queries (water.gdshader:27-39,42-84): points [n][2] world x,z; map_scales [c][4]; outputs [n][3]
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_sample_maps(IntPtr handle, int num_points, float* points_xz, int num_cascades, float* map_scales,
                                                      float* displacement, float* gradient_foam);
        // fused frames, overlapped hand-off, Water scheduler, spray candidates (include/ocean.h)
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_update_frames(IntPtr handle, double delta, OceanCascadeParams* parameters, int count, int frames);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_snapshot_maps_to_host_async(IntPtr handle, int first, int count, void* displacement, void* normal);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_wait_snapshot(IntPtr handle);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_scheduler_init(OceanScheduler* s, double updates_per_second);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_scheduler_set_rate(OceanScheduler* s, double updates_per_second);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_scheduler_tick(OceanScheduler* s, double delta, double* update_delta);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_water_frame(IntPtr handle, OceanScheduler* s, double delta, OceanCascadeParams* parameters, int count, int* did_update);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_map_scales(OceanCascadeParams* parameters, int count, float* map_scales);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial double ocean_water_default_time(int cascade);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_spray_grid(int num_particles, float* emission_transform, float* points_xz);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_extract_spray(IntPtr handle, int num_candidates, float* points_xz, int num_cascades, float* map_scales,
                                                        float* particle_scale, int max_records, OceanSprayRecord* records, int* num_active);
        // spray particles: one particle-process frame [t0, t1) of the emitter; instances [num_live][16] for multimesh_set_buffer
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_default_spray_emitter(OceanSprayEmitter* emitter);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_spray_particles(IntPtr handle, OceanSprayEmitter* emitter, double t0, double t1, int num_cascades,
                                                          float* map_scales, OceanSprayParticle* states, int max_instances, float* instances,
                                                          int* num_live);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_spray_particles_device(IntPtr handle, OceanSprayEmitter* emitter, double t0, double t1, int num_cascades,
                                                                 float* map_scales, void* states_dev, int max_instances, void* instances_dev,
                                                                 void* num_live_dev);
        // wake layer: a local height field driven by moving sources and floating bodies (include/ocean.h, "Wake layer")
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_wake_kernel_taps(float* taps);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_wake_init(IntPtr handle, OceanWakeParams* parameters);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_wake_step(IntPtr handle, double dt, int substeps, long origin_x, long origin_z, int num_sources,
                                                    OceanWakeSource* sources, int num_states, OceanBodyState* states);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_wake_step_device(IntPtr handle, double dt, int substeps, long origin_x, long origin_z, int num_sources,
                                                           void* sources_dev, int num_states, void* states_dev);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_wake_render_map(IntPtr handle, void* map_dev, float* world_rect);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_sample_wake(IntPtr handle, int num_points, float* points_xz, float* output);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_sample_wake_device(IntPtr handle, int num_points, void* points_xz_dev, void* output_dev);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_wake_get_state(IntPtr handle, float* h, float* h_prev, long* origin_xz);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_wake_set_state(IntPtr handle, float* h, float* h_prev, long origin_x, long origin_z);
        // wake coupling: the surface query, buoyancy, body forces and the body integrator read the wake free surface (enable 0 or 1)
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_wake_set_coupling(IntPtr handle, int enable);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_wake_get_coupling(IntPtr handle, float* e, float* e_old, long* origins, float* interval);
        // wake foam: the foam field F, advanced with the layer, in the render map's fourth channel (null parameters: off)
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_wake_set_foam(IntPtr handle, OceanWakeFoamParams* parameters);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_wake_get_foam_state(IntPtr handle, float* foam);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_wake_set_foam_state(IntPtr handle, float* foam);
        // wake obstacles: a world-fixed mask [depth][width] of blocked cells (nonzero) at world cell origin (x, z); null, 0, 0: none
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_wake_set_obstacles(IntPtr handle, byte* mask, int width, int depth, long origin_x, long origin_z);
        // wake readers: OCEAN_WAKE_READ_RAYCAST (1) makes the ray cast hit the coupled surface, OCEAN_WAKE_READ_SPRAY (2) lets spray read h and F
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_wake_set_readers(IntPtr handle, uint readers);
        // sea state: per-cascade moments (may be null) and the total under map_scales[num_cascades][4] (synchronous)
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_get_sea_state(IntPtr handle, int num_cascades, float* map_scales, OceanSeaState* per_cascade,
                                                        OceanSeaState* total);
        // drifters: advance by dt (0 only renders) and write 12-float MultiMesh instances (may be null)
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_drift(IntPtr handle, double dt, OceanDriftParams* parameters, int num_drifters, OceanDrifter* drifters,
                                                int num_cascades, float* map_scales, float* instances);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_drift_device(IntPtr handle, double dt, OceanDriftParams* parameters, int num_drifters, IntPtr drifters_dev,
                                                       int num_cascades, float* map_scales, IntPtr instances_dev);
        // surface query: the surface at world positions points [n][2] (P + D_xz(P) = Q solved for P, then the map query at P)
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_query_surface(IntPtr handle, int num_points, float* points_xz, int num_cascades, float* map_scales,
                                                        float tolerance, int max_iterations, OceanSurfaceSample* samples);
        // ray cast: the first crossing of each ray with the displaced surface (step = horizontal sample spacing in metres)
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_raycast(IntPtr handle, int num_rays, OceanRay* rays, int num_cascades, float* map_scales, float step,
                                                  int max_samples, float tolerance, int max_iterations, OceanRayHit* hits);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_raycast_device(IntPtr handle, int num_rays, void* rays_dev, int num_cascades, float* map_scales, float step,
                                                         int max_samples, float tolerance, int max_iterations, void* hits_dev);
        // buoyancy: per-body force and torque from hull points on the surface; samples may be null
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_buoyancy(IntPtr handle, int num_bodies, OceanBuoyancyBody* bodies, int num_points, OceanBuoyancyPoint* points,
                                                   int num_cascades, float* map_scales, float density, float tolerance, int max_iterations,
                                                   OceanBuoyancyResult* results, OceanSurfaceSample* samples);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_buoyancy_device(IntPtr handle, int num_bodies, OceanBuoyancyBody* bodies, int num_points, void* points_dev,
                                                          int num_cascades, float* map_scales, float density, float tolerance, int max_iterations,
                                                          void* results_dev, void* samples_dev);
        // body forces: the buoyancy records plus quadratic drag against the water velocity, from one surface query;
        // drag_areas [num_points] (C_d A per hull point); samples may be null
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_body_forces(IntPtr handle, int num_bodies, OceanBuoyancyBody* bodies, OceanBodyVelocity* velocities,
                                                      int num_points, OceanBuoyancyPoint* points, float* drag_areas, int num_cascades,
                                                      float* map_scales, float density, float tolerance, int max_iterations,
                                                      OceanBuoyancyResult* hydrostatic, OceanDragResult* drag, OceanSurfaceSample* samples);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_body_forces_device(IntPtr handle, int num_bodies, OceanBuoyancyBody* bodies, OceanBodyVelocity* velocities,
                                                             int num_points, void* points_dev, void* drag_areas_dev, int num_cascades,
                                                             float* map_scales, float density, float tolerance, int max_iterations,
                                                             void* hydrostatic_dev, void* drag_dev, void* samples_dev);
        // floating bodies: substeps sub-steps of dt / substeps with the states advanced in place; the records are the last
        // sub-step's and transforms [num_bodies][12] is [R | position] row-major (a MultiMesh TRANSFORM_3D buffer); each may be null
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_simulate_bodies(IntPtr handle, int num_bodies, OceanFloatingBody* bodies, OceanBodyState* states,
                                                          int num_points, OceanBuoyancyPoint* points, float* drag_areas, int num_cascades,
                                                          float* map_scales, float density, float dt, int substeps, float tolerance,
                                                          int max_iterations, OceanBuoyancyResult* hydrostatic, OceanDragResult* drag,
                                                          float* transforms);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_simulate_bodies_device(IntPtr handle, int num_bodies, OceanFloatingBody* bodies, void* states_dev,
                                                                 int num_points, void* points_dev, void* drag_areas_dev, int num_cascades,
                                                                 float* map_scales, float density, float dt, int substeps, float tolerance,
                                                                 int max_iterations, void* hydrostatic_dev, void* drag_dev, void* transforms_dev);
        // driven and moored bodies: ocean_simulate_bodies with thrusters, foils, loads (may be null) and tethers, host arrays in
        // both forms; drive and tensions ([num_tethers], for drawing or snapping ropes) are the last sub-step's and may be null
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_simulate_driven_bodies(IntPtr handle, int num_bodies, OceanFloatingBody* bodies, OceanBodyState* states,
                                                                 int num_points, OceanBuoyancyPoint* points, float* drag_areas, int num_cascades,
                                                                 float* map_scales, float density, float dt, int substeps, float tolerance,
                                                                 int max_iterations, int num_thrusters, OceanThruster* thrusters, int num_foils,
                                                                 OceanFoil* foils, OceanBodyLoad* loads, int num_tethers, OceanTether* tethers,
                                                                 OceanBuoyancyResult* hydrostatic, OceanDragResult* drag, OceanDriveResult* drive,
                                                                 float* tensions, float* transforms);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_simulate_driven_bodies_device(IntPtr handle, int num_bodies, OceanFloatingBody* bodies, void* states_dev,
                                                                        int num_points, void* points_dev, void* drag_areas_dev, int num_cascades,
                                                                        float* map_scales, float density, float dt, int substeps, float tolerance,
                                                                        int max_iterations, int num_thrusters, OceanThruster* thrusters,
                                                                        int num_foils, OceanFoil* foils, OceanBodyLoad* loads, int num_tethers,
                                                                        OceanTether* tethers, void* hydrostatic_dev, void* drag_dev, void* drive_dev,
                                                                        void* tensions_dev, void* transforms_dev);
        // hull meshes: register triangle-mesh hulls once (volumes may be null), then pressure and drag over their wetted triangles
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_hull_set_meshes(IntPtr handle, int num_meshes, OceanHullMesh* meshes, int num_vertices, float* vertices,
                                                          int num_triangles, int* triangles, float* volumes);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_hull_forces(IntPtr handle, int num_bodies, OceanHullBody* bodies, OceanBodyVelocity* velocities,
                                                      int num_cascades, float* map_scales, float density, float tolerance, int max_iterations,
                                                      OceanBuoyancyResult* hydrostatic, OceanDragResult* drag, OceanSurfaceSample* samples);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_hull_forces_device(IntPtr handle, int num_bodies, OceanHullBody* bodies, OceanBodyVelocity* velocities,
                                                             int num_cascades, float* map_scales, float density, float tolerance, int max_iterations,
                                                             void* hydrostatic_dev, void* drag_dev, void* samples_dev);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_simulate_hull_bodies(IntPtr handle, int num_bodies, OceanFloatingHull* bodies, OceanBodyState* states,
                                                               int num_cascades, float* map_scales, float density, float dt, int substeps,
                                                               float tolerance, int max_iterations, OceanBuoyancyResult* hydrostatic,
                                                               OceanDragResult* drag, float* transforms);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_simulate_hull_bodies_device(IntPtr handle, int num_bodies, OceanFloatingHull* bodies, void* states_dev,
                                                                      int num_cascades, float* map_scales, float density, float dt, int substeps,
                                                                      float tolerance, int max_iterations, void* hydrostatic_dev, void* drag_dev,
                                                                      void* transforms_dev);
        // velocity maps: d/dt of the displacement map, recomputed for the cascades whose maps changed; recomputed may be null
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_update_velocity(IntPtr handle, int* recomputed);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_get_velocity_map(IntPtr handle, IntPtr* velocity_dev, nuint* layer_bytes);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_copy_velocity_to_host(IntPtr handle, int first, int count, void* velocity);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_copy_f32_velocity_to_host(IntPtr handle, int cascade, float* velocity);
        // water velocity at undisplaced points [n][2]; output [n][3]
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_sample_velocity(IntPtr handle, int num_points, float* points_xz, int num_cascades, float* map_scales,
                                                          float* velocity);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_sample_velocity_device(IntPtr handle, int num_points, void* points_xz_dev, int num_cascades, float* map_scales,
                                                                 void* velocity_dev);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial int ocean_get_info(IntPtr handle, OceanInfo* info);
        [LibraryImport(Lib)] [UnmanagedCallConv(CallConvs = new[] { typeof(System.Runtime.CompilerServices.CallConvCdecl) })]
        internal static partial IntPtr ocean_last_error();
    }

    public sealed class OceanException : Exception { public OceanException(string m) : base(m) { } }

    /// <summary>Same surface as the reference's WaveGenerator (assets/water/wave_generator.gd): MapSize, InitGpu,
    /// Update, Process, the two maps and the static JONSWAP helpers.</summary>
    public sealed unsafe class WaveGenerator : IDisposable
    {
        public const double G = 9.81, Depth = 20.0;               // wave_generator.gd:5-6
        public int MapSize;                                         // wave_generator.gd:8
        private IntPtr _handle;
        private int _layers;
        private byte* _dispHost, _normHost;                         // pinned staging for texture_update

        private static void Check(int status)
        {
            if (status != 0) throw new OceanException(Marshal.PtrToStringAnsi(Native.ocean_last_error()) ?? "libocean error");
        }

        public void InitGpu(int numCascades, int device = 0)        // wave_generator.gd:17-54
        {
            Dispose();
            IntPtr h;
            Check(Native.ocean_create(device, MapSize, numCascades, &h));
            _handle = h; _layers = numCascades;
            nuint bytes = (nuint)numCascades * (nuint)MapSize * (nuint)MapSize * 8;
            void* d, n;
            Check(Native.ocean_host_alloc(&d, bytes)); Check(Native.ocean_host_alloc(&n, bytes));
            _dispHost = (byte*)d; _normHost = (byte*)n;
        }

        public void Update(double delta, Span<OceanCascadeParams> parameters)   // wave_generator.gd:90-109
        {
            if (parameters.Length == 0) throw new ArgumentException("parameters.size() != 0");
            if (_handle == IntPtr.Zero) InitGpu(Math.Max(2, parameters.Length));
            fixed (OceanCascadeParams* p = parameters) Check(Native.ocean_update(_handle, delta, p, parameters.Length));
        }

        public void Process(Span<OceanCascadeParams> parameters)                 // wave_generator.gd:56-63 (_process)
        {
            fixed (OceanCascadeParams* p = parameters) Check(Native.ocean_process(_handle, p, parameters.Length));
        }

        /// <summary>Copies layer `cascade` of both maps to pinned host memory; the caller passes the spans to
        /// RenderingDevice.TextureUpdate(displacementRid, cascade, bytes) / (normalRid, cascade, bytes).</summary>
        public (IntPtr displacement, IntPtr normal, int bytes) FetchLayer(int cascade)
        {
            int layer = MapSize * MapSize * 8;
            Check(Native.ocean_copy_maps_to_host(_handle, cascade, 1, _dispHost + (long)cascade * layer, _normHost + (long)cascade * layer));
            return ((IntPtr)(_dispHost + (long)cascade * layer), (IntPtr)(_normHost + (long)cascade * layer), layer);
        }

        internal IntPtr Handle => _handle;
        internal byte* DisplacementHost => _dispHost;
        internal byte* NormalHost => _normHost;

        public static double JONSWAPAlpha(double windSpeed = 20.0, double fetchLength = 550e3) => Native.ocean_jonswap_alpha(windSpeed, fetchLength);
        public static double JONSWAPPeakAngularFrequency(double windSpeed = 20.0, double fetchLength = 550e3) => Native.ocean_jonswap_peak_angular_frequency(windSpeed, fetchLength);

        public void Dispose()                                       // NOTIFICATION_PREDELETE, wave_generator.gd:111-113
        {
            if (_handle != IntPtr.Zero) { Native.ocean_destroy(_handle); _handle = IntPtr.Zero; }
            if (_dispHost != null) { Native.ocean_host_free(_dispHost); _dispHost = null; }
            if (_normHost != null) { Native.ocean_host_free(_normHost); _normHost = null; }
        }
    }

    /// <summary>The wave side of the reference's Water node (assets/water/water.gd): owns the generator, runs the fixed-rate
    /// update accumulator (:75-82, in the library: ocean_scheduler_tick), gives every cascade its start time (:32), builds
    /// map_scales (:102-110) and hands finished layers to Godot.  In a Godot C# project this class derives from MeshInstance3D
    /// and _Process(delta) calls Frame(delta); the TextureUpdate calls are the only engine API it needs.</summary>
    public sealed unsafe class Water : IDisposable
    {
        public readonly WaveGenerator Generator = new WaveGenerator();
        private OceanScheduler _sched;
        private OceanCascadeParams[] _parameters = Array.Empty<OceanCascadeParams>();

        public Water(int mapSize = 1024, double updatesPerSecond = 50.0)           // water.gd:38,51
        {
            Generator.MapSize = mapSize;
            fixed (OceanScheduler* s = &_sched) Native.ocean_scheduler_init(s, updatesPerSecond);
        }

        public double UpdatesPerSecond                                             // water.gd:51-54
        {
            get => _sched.updates_per_second;
            set { fixed (OceanScheduler* s = &_sched) Native.ocean_scheduler_set_rate(s, value); }
        }

        public void SetParameters(OceanCascadeParams[] value)                      // water.gd:22-35,84-100
        {
            for (int i = 0; i < value.Length; ++i)
            {
                value[i].time = Native.ocean_water_default_time(i);                // :32
                value[i].should_generate_spectrum = 1;                             // :86-87
            }
            _parameters = value;
            Generator.InitGpu(Math.Max(2, value.Length));                          // :91
        }

        public float[] MapScales()                                                 // water.gd:102-110
        {
            var scales = new float[4 * _parameters.Length];
            fixed (OceanCascadeParams* p = _parameters) fixed (float* o = scales) Native.ocean_map_scales(p, _parameters.Length, o);
            return scales;
        }

        /// <summary>One rendered frame: Water._process (:75-82) + the child generator's _process (wave_generator.gd:56-63).
        /// `upload(rid-selector, layer, pointer, bytes)` is RenderingDevice.TextureUpdate on the displacement / normal array.</summary>
        public bool Frame(double delta, Action<bool, int, IntPtr, int> upload)
        {
            int did = 0;
            fixed (OceanScheduler* s = &_sched) fixed (OceanCascadeParams* p = _parameters)
            {
                int before = PendingCascades();
                int rc = Native.ocean_water_frame(Generator.Handle, s, delta, p, _parameters.Length, &did);
                if (rc != 0) throw new OceanException(Marshal.PtrToStringAnsi(Native.ocean_last_error()) ?? "libocean error");
                // the cascade that was just processed is the one to re-upload (highest pending index first, wave_generator.gd:59)
                int after = PendingCascades();
                if (after < before || did != 0)
                {
                    int layer = after;
                    var (d, n, bytes) = Generator.FetchLayer(layer);
                    upload(true, layer, d, bytes);
                    upload(false, layer, n, bytes);
                }
            }
            return did != 0;
        }

        private int PendingCascades()
        {
            OceanInfo info;
            Native.ocean_get_info(Generator.Handle, &info);
            return info.pending_cascades;
        }

        public void Dispose() => Generator.Dispose();                              // water.gd:116-119
    }
}
