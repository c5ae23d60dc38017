// ocean_api.cu -- the C ABI of libocean.so (include/ocean.h) and the host-side sequencing of
// the reference's WaveGenerator (assets/water/wave_generator.gd:17-121): resource allocation,
// dirty-flag handling, push-constant rounding (assets/render_context.gd:122-135), the
// update / _process pending-cascade state machine, and the hand-off of the finished maps.
// No CPU fallback exists: every compute entry point launches the sm_90a kernels or fails.
#include "../../include/ocean.h"
#include "ocean_kernels.cuh"

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <new>
#include <string>
#include <map>
#include <type_traits>
#include <vector>

namespace {

thread_local std::string g_last_error;

int fail(int code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_last_error = buf;
    return code;
}

#define OCEAN_CUDA(expr)                                                                       \
    do {                                                                                       \
        cudaError_t e__ = (expr);                                                              \
        if (e__ != cudaSuccess)                                                                \
            return fail(OCEAN_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
    } while (0)

constexpr double kG = 9.81;       // wave_generator.gd:5
constexpr double kDepth = 20.0;   // wave_generator.gd:6
constexpr int kRing = 8;          // pinned staging slots for dispatch records

}  // namespace

struct ocean_generator;

namespace {
// A device block of `capacity` elements of T owned by one generator and counted in its device_bytes while it lives.
template <typename T>
struct DeviceArray {
    T* ptr = nullptr;
    size_t capacity = 0;
    ocean_generator* owner = nullptr;                   // whose device_bytes count the block

    DeviceArray() = default;
    DeviceArray(const DeviceArray&) = delete;
    DeviceArray& operator=(const DeviceArray&) = delete;
    ~DeviceArray() { release(); }
    cudaError_t grow(ocean_generator* g, size_t n);
    cudaError_t upload(ocean_generator* g, const void* host, size_t n);
    void release();
};

// The host entry points that stage the caller's arrays, one staging block each (ocean_generator::staging, see Staging).
enum StagedOp {
    kStageSampleMaps, kStageExtractSpray, kStageSprayParticles, kStageQuerySurface, kStageRaycast, kStageBuoyancy,
    kStageSampleVelocity, kStageBodyForces, kStageSimulateBodies, kStageDeviceMath, kStageWakeStep, kStageSampleWake, kStageDrift,
    kStageDrivenBodies, kStageHullForces, kStageSimulateHulls, kNumStagedOps
};

// The parts of the wake layer WakeLayer::off turns off; kWakeLayer is the whole layer.
enum : unsigned { kWakeCoupling = 1, kWakeFoam = 2, kWakeMask = 4, kWakeFields = 8, kWakeLayer = 15 };

// The wake layer (ocean_wake_init) and its parts.  The coupling, foam and mask are on exactly while their buffers are
// allocated: the calls that turn a part on leave it allocated (and cleared where the kernels read it) or off.
struct WakeLayer {
    ocean_wake_params params{};                         // size 0: no layer
    // four [size][size] fields -- h, h_prev and the two a sub-step writes -- and the window's origin in whole cells
    DeviceArray<float> fields;
    int h = 0, hp = 1;                                  // which fields hold h and h_prev
    int64_t origin[2] = {0, 0};
    // coupling (ocean_wake_set_coupling): two [size][size] snapshots of the free surface e = h + phi, each with its window
    // origin, the interval between them, and the drag pass's per-world-point vertical velocity
    DeviceArray<float> snapshots;
    DeviceArray<float> wv;
    bool primed = false;                                // the snapshots describe the layer
    int e = 0;                                          // which snapshot holds e (the other holds e_old)
    int64_t snapshot_origin[2][2] = {};                 // [snapshot][x, z]
    float interval = 0.0f;                              // T
    // foam (ocean_wake_set_foam): two [size][size] foam fields, F and the one a sub-step writes, and the parameters
    DeviceArray<float> foam;
    ocean_wake_foam_params foam_params{};
    int f = 0;                                          // which foam field holds F
    // obstacles (ocean_wake_set_obstacles): the mask's bytes ([depth][width], nonzero = blocked) and its world cell origin
    DeviceArray<uint8_t> mask;
    int32_t mask_size[2] = {0, 0};                      // width, depth
    int64_t mask_origin[2] = {0, 0};
    // readers (ocean_wake_set_readers): OCEAN_WAKE_READ_* bits of the ops that read the layer besides the coupling's
    uint32_t readers = 0;

    bool on() const { return params.size > 0; }
    bool coupled() const { return snapshots.ptr != nullptr; }
    bool foamed() const { return foam.ptr != nullptr; }
    bool masked() const { return mask.ptr != nullptr; }
    // the surface query reads the layer while the coupling is on and primed
    bool coupling_live() const { return on() && coupled() && primed; }
    bool reads(uint32_t reader) const { return on() && (readers & reader); }
    size_t cells() const { return (size_t)params.size * params.size; }
    float* field(int k) const { return fields.ptr + k * cells(); }
    float* foam_field(int k) const { return foam.ptr + k * cells(); }
    float* snapshot(int k) const { return snapshots.ptr + k * cells(); }
    // (float)((double)origin * dx), the world corner of a window at `origin`
    float corner(int64_t o) const { return (float)((double)o * (double)params.cell_size); }

    // h in the current window, with F while foam is on
    ocean::WakeRead read_h() const {
        return {field(h), foamed() ? foam_field(f) : nullptr, params.size, params.cell_size, corner(origin[0]), corner(origin[1])};
    }
    // e in its own window
    ocean::WakeRead read_e() const {
        return {snapshot(e), nullptr, params.size, params.cell_size, corner(snapshot_origin[e][0]), corner(snapshot_origin[e][1])};
    }
    ocean::WakeCoupleArgs couple_args() const {
        const int o = e ^ 1;
        return {snapshot(e), snapshot(o), params.size, params.cell_size, corner(snapshot_origin[e][0]), corner(snapshot_origin[e][1]),
                corner(snapshot_origin[o][0]), corner(snapshot_origin[o][1]), interval};
    }
    // The mask in the window at (origin_x, origin_z): the mask cell of window cell (0, 0), exact in __int128 and clamped to
    // [-2^30, 2^30] per axis.  The halo spans window cells [-6, size + 6) and the mask at most 2^28 cells, so a clamped offset
    // leaves the whole halo outside the mask exactly when the exact one does.
    ocean::WakeObstacles obstacles(int64_t origin_x, int64_t origin_z) const {
        auto offset = [](int64_t window, int64_t m) -> int {
            constexpr __int128 kClamp = (__int128)1 << 30;
            const __int128 d = (__int128)window - (__int128)m;
            return (int)(d > kClamp ? kClamp : d < -kClamp ? -kClamp : d);
        };
        return {mask.ptr, mask_size[0], mask_size[1], offset(origin_x, mask_origin[0]), offset(origin_z, mask_origin[1])};
    }
    int off(ocean_generator* g, unsigned parts);
    // the wake's vertical velocity of each of n query points for the drag passes, allocated while the coupling is live (else
    // *out is null); every sub-step of a call reads the same snapshots
    cudaError_t vertical_velocities(ocean_generator* g, size_t n, float** out) {
        *out = nullptr;
        if (n == 0 || !coupling_live()) return cudaSuccess;
        cudaError_t e = wv.grow(g, n);
        if (e == cudaSuccess) *out = wv.ptr;
        return e;
    }
};

// The scratch of the floating-body ops (buoyancy, body forces, hull forces and the three integrators), grown by the calls
// that use it and kept for the next.  The point and mesh forms keep their own pose and row tables.
struct BodyScratch {
    // per body: the pose tables (ocean_buoyancy_body for point hulls, ocean_hull_body for meshes) and velocities the force
    // passes read and the integrators rewrite each sub-step; the offsets of the bodies' first world points, with their host
    // copy (kept here: the upload is asynchronous); max |p|^2 per hull; the integrators' rows (ocean_floating_body, written by
    // k_hull_prepare for meshes, which are uploaded as ocean_floating_hull); the hydrostatic and drag results of an integrator
    // whose caller passes NULL for them
    DeviceArray<ocean_buoyancy_body> poses;
    DeviceArray<ocean_hull_body> hull_poses;
    DeviceArray<ocean_body_velocity> velocities;
    DeviceArray<int> offsets;
    std::vector<int> offsets_host;
    DeviceArray<float> r2;
    DeviceArray<ocean_floating_body> rows;
    DeviceArray<ocean_floating_hull> hull_rows;
    DeviceArray<ocean_buoyancy_result> hydrostatic;
    DeviceArray<ocean_drag_result> drag;
    // per queried point (the world points, then a driven call's actuators): the query positions, the surface records when
    // the caller wants none, and for meshes the (r, d) and (u, 0) of k_hull_vertex per world vertex
    DeviceArray<float2> q;
    DeviceArray<ocean_surface_sample> samples;
    DeviceArray<float4> corners;
    // drive (ocean_simulate_driven_bodies): the actuator, load and tether arrays, the by-body incidence list (offsets, then
    // entries, in one block) with its host copy, the tether records, the integrator's sums, and the drive and tension outputs
    // when the caller passes NULL for them
    DeviceArray<ocean_thruster> thrusters;
    DeviceArray<ocean_foil> foils;
    DeviceArray<ocean_body_load> loads;
    DeviceArray<ocean_tether> tethers;
    DeviceArray<int> incidence;
    std::vector<int> incidence_host;
    DeviceArray<ocean::TetherForce> tether_forces;
    DeviceArray<ocean::DriveSum> sums;
    DeviceArray<ocean_drive_result> drive;
    DeviceArray<float> tensions;
    // the registered mesh set (ocean_hull_set_meshes) and a host copy of its mesh records: the calls validate the bodies'
    // mesh indices and count their world vertices from it
    DeviceArray<ocean_hull_mesh> meshes;
    DeviceArray<float> vertices;
    DeviceArray<int32_t> triangles;
    std::vector<ocean_hull_mesh> meshes_host;
};
}  // namespace

struct ocean_generator {
    int device = 0;
    int map_size = 0;
    int num_cascades = 0;
    uint64_t device_bytes = 0;                          // declared before the DeviceArrays: their destructors update it
    cudaStream_t stream = nullptr;
    cudaStream_t copy_stream = nullptr;                 // snapshot hand-off: device->host copies that overlap the next update
    cudaEvent_t snap_ready = nullptr, snap_free = nullptr;
    DeviceArray<uint2> snap_disp, snap_normal;          // [num_cascades][N][N] snapshot of the maps (lazy)
    bool snap_busy = false;
    // the maps, scratch and tables of ocean_create; `buf` is the view of them (and of the taps) that the kernels take
    DeviceArray<float4> spectrum, rowpass, disp_table;
    DeviceArray<uint2> displacement, normal;
    DeviceArray<uint16_t> foam;                         // the foam state; normal.a holds a copy of it
    DeviceArray<float4> displacement_f32, normal_f32;   // binary32 taps, while they are on
    DeviceArray<float> disp_kvy;
    DeviceArray<float2> twiddles;
    ocean::DeviceBuffers buf{};
    DeviceArray<float2> export_buf;                     // rowpass export scratch (lazy)
    DeviceArray<unsigned char> staging[kNumStagedOps];  // each host entry point's copies of the caller's arrays (Staging)
    DeviceArray<float4> q_scales;                       // map scales of the query ops
    DeviceArray<int> spray_counts;                      // spray op scratch: block counts / offsets (+ total)
    DeviceArray<int> surf_scratch;                      // surface query scratch: pending count, layer maxima, pending list
    BodyScratch body;                                   // the floating-body ops (BodyScratch)
    // velocity maps, allocated by the first velocity call: row-pass scratch, the map, its binary32 tap while the taps are on
    DeviceArray<float4> vel_scratch;                    // [num_cascades][N][N]
    DeviceArray<uint2> velocity;                        // [num_cascades][N][N] 4 x half
    DeviceArray<float4> velocity_f32;                   // [num_cascades][N][N]
    std::vector<ocean::VelocityDispatch> vel_source;    // [num_cascades] table slot and time of the update that built the current maps
    std::vector<char> vel_has_source;                   // the cascade's maps were written at least once
    std::vector<char> vel_stale;                        // its velocity layer does not describe its current maps yet
    // the sea-state cache, allocated by the first sea-state or drift call: per cascade the moments (zero until computed) and
    // whether they describe its current spectrum and dispersion table; partial = the reduction's block sums
    DeviceArray<double> sea_moments;                    // [num_cascades][kSeaStateMoments]
    DeviceArray<double> sea_partial;
    std::vector<char> sea_stale;
    DeviceArray<ocean::CascadeDispatch> d_cascade;      // [num_cascades] (two-kernel path only)
    DeviceArray<ocean::SpectrumDispatch> d_spectrum;    // [num_cascades]
    DeviceArray<ocean::TableDispatch> d_tables;         // [num_cascades]
    ocean::CascadeDispatch* h_cascade = nullptr;        // pinned [kRing][num_cascades]
    ocean::SpectrumDispatch* h_spectrum = nullptr;      // pinned [kRing][num_cascades]
    ocean::TableDispatch* h_tables = nullptr;           // pinned [kRing][num_cascades]
    // dispersion tables are keyed by (tile_length, depth): cascades with equal keys share a slot
    struct TableKey { float tile_x, tile_y, depth; };
    std::vector<TableKey> slot_key;                     // [num_cascades] key whose table the slot holds (valid if slot_valid)
    std::vector<char> slot_valid;
    std::vector<int> slot_refs;                         // cascades currently pointing at the slot
    std::vector<int> cascade_slot;                      // [num_cascades] slot of each cascade, -1 = none yet
    std::vector<int> scratch_layer_of;                  // [num_cascades] where the last update left the cascade's row pass (debug tap)
    cudaEvent_t ring_done[kRing] = {};
    int ring_next = 0;
    cudaEvent_t timer_start = nullptr, timer_stop = nullptr;
    cudaEvent_t prof[5] = {};                           // gen-start, A-start, after A(chunk 0), end, after B(chunk 0)
    int prof_chunk = 0;                                 // cascades in the profiled first chunk
    bool profiling = false;
    bool prof_valid = false, prof_had_gen = false;
    DeviceArray<int> d_queue;                           // [1 + 3 * num_cascades] work counter + completion counters
    std::vector<uint32_t> done_count;                   // host mirror of the completion counters (modulo 2^32)
    int resident_ctas = 0;
    std::map<int, DeviceArray<int>> item_tables;        // cascades per launch -> item table (capacity = item count)
    std::map<std::pair<int, int>, DeviceArray<int>> frame_tables;   // (cascades, frames per launch) -> same, multi-frame order
    std::vector<ocean_cascade_params> pass_parameters;  // wave_generator.gd:14
    int pass_num_cascades_remaining = 0;                // wave_generator.gd:15
    uint64_t kernel_launches = 0;
    uint64_t cascade_updates = 0;
    // Entry points entered so far, and the value it had when the stream's last operation was a persistent single-update
    // launch (0: it is not).  The next update's launch is queued as that launch's programmatic dependent only if no entry
    // point ran in between (any of them may have put work on the stream), see run_cascades.
    uint64_t entries = 0;
    uint64_t update_tail = 0;
    DeviceArray<unsigned> ray_bounds;                   // ray cast scratch: [3 * num_cascades] per-layer bounds (first use)
    WakeLayer wake;
};

namespace {

// Every entry point runs on the generator's device and hands the caller's current device back on return (a host that
// drives other CUDA work from the same thread -- a torch process, a C# engine host -- must not find its device changed).
struct DeviceScope {
    int prev = -1;
    ~DeviceScope() {
        if (prev >= 0) cudaSetDevice(prev);
    }
    cudaError_t enter(int device) {
        int cur = -1;
        if (cudaGetDevice(&cur) != cudaSuccess) cur = -1;
        if (cur == device) return cudaSuccess;
        cudaError_t e = cudaSetDevice(device);
        if (e == cudaSuccess) prev = cur;
        return e;
    }
};
int enter_gen(ocean_generator* g, DeviceScope& scope) {
    if (!g) return fail(OCEAN_ERR_INVALID_ARGUMENT, "generator handle is NULL");
    cudaError_t e = scope.enter(g->device);
    if (e != cudaSuccess) return fail(OCEAN_ERR_CUDA, "cudaSetDevice(%d) failed: %s", g->device, cudaGetErrorString(e));
    g->entries += 1;
    return OCEAN_OK;
}
#define OCEAN_ENTER(gen)                 \
    DeviceScope device_scope__;          \
    int rc = enter_gen(gen, device_scope__)

// At least n elements; the contents are not kept.
template <typename T>
cudaError_t DeviceArray<T>::grow(ocean_generator* g, size_t n) {
    if (n <= capacity) return cudaSuccess;
    if (ptr) {
        cudaError_t e = cudaStreamSynchronize(g->stream);    // an earlier call may still read the old block
        if (e != cudaSuccess) return e;
        release();
    }
    T* p = nullptr;
    cudaError_t e = cudaMalloc(reinterpret_cast<void**>(&p), n * sizeof(T));
    if (e != cudaSuccess) return e;
    ptr = p;
    capacity = n;
    owner = g;
    g->device_bytes += n * sizeof(T);
    return cudaSuccess;
}

// grow(g, n), then the copy of n elements from host memory, enqueued on the generator's stream.
template <typename T>
cudaError_t DeviceArray<T>::upload(ocean_generator* g, const void* host, size_t n) {
    cudaError_t e = grow(g, n);
    if (e != cudaSuccess) return e;
    return cudaMemcpyAsync(ptr, host, n * sizeof(T), cudaMemcpyHostToDevice, g->stream);
}

template <typename T>
void DeviceArray<T>::release() {
    if (!ptr) return;
    cudaFree(ptr);
    owner->device_bytes -= capacity * sizeof(T);
    ptr = nullptr;
    capacity = 0;
}

// A host entry point's device copies of the caller's arrays: one slice per array in the entry point's own block
// gen->staging[op], each at a 256-byte boundary (the kernels load float4 and record types).  upload() grows the block once and
// copies the `in` and `inout` arrays to it; st[slice] is then the slice's device pointer, NULL when the slice is empty (a count
// of 0 or a NULL host array).  finish() copies the `out` and `inout` arrays back and synchronises; `scratch` is not copied.
struct Staging {
    template <typename T> struct Slice { size_t offset, bytes; };
    struct Copy { size_t offset, bytes; const void* up; void* down; };
    std::vector<Copy> copies;
    size_t total = 0;
    unsigned char* base = nullptr;

    template <typename T> Slice<T> add(const void* up, void* down, size_t bytes) {
        copies.push_back({(total + 255) & ~(size_t)255, bytes, up, down});
        total = copies.back().offset + bytes;
        return {copies.back().offset, bytes};
    }
    template <typename T> Slice<const T> in(const T* host, size_t n) { return add<const T>(host, nullptr, host ? n * sizeof(T) : 0); }
    template <typename T> Slice<T> out(T* host, size_t n) { return add<T>(nullptr, host, host ? n * sizeof(T) : 0); }
    template <typename T> Slice<T> inout(T* host, size_t n) { return add<T>(host, host, host ? n * sizeof(T) : 0); }
    template <typename T> Slice<T> scratch(size_t n) { return add<T>(nullptr, nullptr, n * sizeof(T)); }
    template <typename T> T* operator[](Slice<T> s) const { return s.bytes ? reinterpret_cast<T*>(base + s.offset) : nullptr; }

    int upload(ocean_generator* g, StagedOp op) {
        OCEAN_CUDA(g->staging[op].grow(g, total));
        base = g->staging[op].ptr;
        for (const Copy& c : copies)
            if (c.up && c.bytes) OCEAN_CUDA(cudaMemcpyAsync(base + c.offset, c.up, c.bytes, cudaMemcpyHostToDevice, g->stream));
        return OCEAN_OK;
    }
    int finish(ocean_generator* g, int rc) {            // rc: the status of the device work; nothing is copied after a failure
        if (rc) return rc;
        for (const Copy& c : copies)
            if (c.down && c.bytes) OCEAN_CUDA(cudaMemcpyAsync(c.down, base + c.offset, c.bytes, cudaMemcpyDeviceToHost, g->stream));
        OCEAN_CUDA(cudaStreamSynchronize(g->stream));
        return OCEAN_OK;
    }
};

// Device memory is released by the generator's DeviceArrays; the rest is released here.
void release(ocean_generator* g) {
    if (!g) return;
    DeviceScope scope;
    scope.enter(g->device);
    if (g->stream) cudaStreamSynchronize(g->stream);
    if (g->h_tables) cudaFreeHost(g->h_tables);
    if (g->copy_stream) { cudaStreamSynchronize(g->copy_stream); cudaStreamDestroy(g->copy_stream); }
    if (g->snap_ready) cudaEventDestroy(g->snap_ready);
    if (g->snap_free) cudaEventDestroy(g->snap_free);
    if (g->h_cascade) cudaFreeHost(g->h_cascade);
    if (g->h_spectrum) cudaFreeHost(g->h_spectrum);
    for (auto& ev : g->ring_done)
        if (ev) cudaEventDestroy(ev);
    if (g->timer_start) cudaEventDestroy(g->timer_start);
    if (g->timer_stop) cudaEventDestroy(g->timer_stop);
    for (auto& ev : g->prof)
        if (ev) cudaEventDestroy(ev);
    if (g->stream) cudaStreamDestroy(g->stream);
    delete g;
}

// The persistent kernel's work-item table cached under `key`.  On first use build(out) makes it on the host (it returns
// the item count, and fills `out` unless that is NULL) and it is uploaded; the table's capacity is its item count.
template <typename Key, typename Build>
cudaError_t item_table(ocean_generator* g, std::map<Key, DeviceArray<int>>& cache, const Key& key, Build build,
                       const DeviceArray<int>** table) {
    auto slot = cache.try_emplace(key);
    if (slot.second) {
        std::vector<int> host((size_t)build(nullptr));
        build(host.data());
        cudaError_t e = slot.first->second.upload(g, host.data(), host.size());
        if (e == cudaSuccess) e = cudaStreamSynchronize(g->stream);        // host vector goes out of scope
        if (e != cudaSuccess) {
            cache.erase(slot.first);
            return e;
        }
    }
    *table = &slot.first->second;
    return cudaSuccess;
}

// Push constants of wave_generator.gd:69-71 (spectrum_compute) with the binary64 -> binary32
// rounding of render_context.gd:134.
ocean::SpectrumDispatch make_spectrum_dispatch(const ocean_cascade_params& p, int cascade) {
    ocean::SpectrumDispatch d;
    const double alpha = ocean_jonswap_alpha(p.wind_speed, p.fetch_length * 1e3);
    const double omega = ocean_jonswap_peak_angular_frequency(p.wind_speed, p.fetch_length * 1e3);
    d.cascade = cascade;
    d.seed_x = p.spectrum_seed[0];
    d.seed_y = p.spectrum_seed[1];
    d.tile_x = p.tile_length[0];
    d.tile_y = p.tile_length[1];
    d.alpha = (float)alpha;
    d.peak_frequency = (float)omega;
    d.wind_speed = (float)p.wind_speed;
    d.angle = (float)(p.wind_direction * (M_PI / 180.0));   // deg_to_rad
    d.depth = (float)kDepth;
    d.swell = (float)p.swell;
    d.detail = (float)p.detail;
    d.spread = (float)p.spread;
    return d;
}

// DETMATH exp of a binary32 argument (DESIGN.md "DETMATH", same operation sequence as detmath::exp64 in
// detmath.cuh): clamp to [-110, 90], n = rint(x*log2e), two-term ln2 reduction, Taylor polynomial to r^13 in
// binary64, one rounding to binary32.  Evaluated here because exp(-foam_decay_rate) (fft_unpack.glsl:62) is
// uniform per dispatch; std::fma is the exact fused operation, so host and device agree bit for bit.
float exp_det_host(float xf) {
    double x = (double)xf;
    if (x != x) return xf;
    if (x < -110.0) x = -110.0;
    if (x > 90.0) x = 90.0;
    const double fn = std::nearbyint(x * 0x1.71547652b82fep+0);   // default rounding mode: ties to even, like rint() on the device
    double r = std::fma(-fn, 0x1.62e42ff000000p-1, x);
    r = std::fma(-fn, -0x1.718432a1b0e26p-35, r);
    static const double c[12] = {0x1.1eed8eff8d898p-29, 0x1.ae64567f544e4p-26, 0x1.27e4fb7789f5cp-22, 0x1.71de3a556c734p-19,
                                 0x1.a01a01a01a01ap-16, 0x1.a01a01a01a01ap-13, 0x1.6c16c16c16c17p-10, 0x1.1111111111111p-7,
                                 0x1.5555555555555p-5,  0x1.5555555555555p-3,  0x1.0000000000000p-1,  0.0};
    double p = 0x1.6124613a86d09p-33;
    for (int i = 0; i < 11; ++i) p = std::fma(p, r, c[i]);
    volatile double rr = r * r;                                    // a separately rounded product, never contracted
    const double e = std::fma(rr, p, r) + 1.0;
    const long long sb = ((long long)fn + 1023LL) << 52;
    double scale;
    std::memcpy(&scale, &sb, sizeof scale);
    return (float)(e * scale);
}

// Push constants of wave_generator.gd:73 (spectrum_modulate) and :85 (fft_unpack).  tile_length and DEPTH reach the
// kernels through the dispersion table of `table_slot` (assign_table_slot).
ocean::CascadeDispatch make_cascade_dispatch(const ocean_cascade_params& p, int cascade, int table_slot) {
    ocean::CascadeDispatch d;
    d.cascade = cascade;
    d.table_slot = table_slot;
    d.time = (float)p.time;
    d.whitecap = (float)p.whitecap;
    d.foam_grow_rate = (float)p.foam_grow_rate;
    d.foam_decay_factor = exp_det_host(-(float)p.foam_decay_rate);
    d.done_target = 0;
    d.wait_target = 0;
    d.col_wait_target = 0;
    d.done_slot = cascade;
    d.scratch_layer = 2 * cascade;                    // half 0 of the scratch (single updates always use it)
    return d;
}

// Points cascade `i` at the dispersion table of (tile_length, DEPTH): keeps its slot when the key is unchanged, shares a
// slot that already holds the key, otherwise claims an unreferenced slot and queues its (re)build in jobs[*n_jobs].
// There are as many slots as cascades and a cascade holds one reference, so a free slot always exists.
int assign_table_slot(ocean_generator* g, int i, const ocean_cascade_params& p, ocean::TableDispatch* jobs, int* n_jobs) {
    const ocean_generator::TableKey key{p.tile_length[0], p.tile_length[1], (float)kDepth};
    auto same = [&](const ocean_generator::TableKey& k) {
        return std::memcmp(&k, &key, sizeof key) == 0;       // bit equality: the table is a function of the bits
    };
    int cur = g->cascade_slot[i];
    if (cur >= 0 && g->slot_valid[cur] && same(g->slot_key[cur])) return cur;
    g->sea_stale[i] = 1;                                                    // the sea state reads the cascade's table
    if (cur >= 0) {
        g->slot_refs[cur] -= 1;
        g->cascade_slot[i] = -1;
    }
    const int S = (int)g->slot_key.size();
    int pick = -1;
    for (int s2 = 0; s2 < S && pick < 0; ++s2)
        if (g->slot_valid[s2] && same(g->slot_key[s2])) pick = s2;          // shared (or cached) table
    if (pick < 0) {
        for (int s2 = 0; s2 < S && pick < 0; ++s2)
            if (g->slot_refs[s2] == 0) pick = s2;
        if (pick < 0) return -1;                                            // cannot happen (see above)
        g->slot_key[pick] = key;
        g->slot_valid[pick] = 1;
        ocean::TableDispatch job;
        job.slot = pick;
        job.tile_x = key.tile_x;
        job.tile_y = key.tile_y;
        job.depth = key.depth;
        jobs[(*n_jobs)++] = job;
    }
    g->slot_refs[pick] += 1;
    g->cascade_slot[i] = pick;
    return pick;
}

// Every path that writes a cascade's maps records the dispatch it used: the velocity layer is recomputed from it on demand.
void record_velocity_source(ocean_generator* g, const ocean::CascadeDispatch& d) {
    g->vel_source[d.cascade] = ocean::VelocityDispatch{d.cascade, d.table_slot, d.time};
    g->vel_has_source[d.cascade] = 1;
    g->vel_stale[d.cascade] = 1;
}

// Runs WaveGenerator._update (wave_generator.gd:65-85) for the cascades listed in `indices`
// (all of them in ONE batched launch sequence; cascades are independent).
int run_cascades(ocean_generator* g, const int* indices, int n) {
    if (n <= 0) return OCEAN_OK;
    const int slot = g->ring_next;
    OCEAN_CUDA(cudaEventSynchronize(g->ring_done[slot]));           // staging slot free again?
    ocean::CascadeDispatch* hc = g->h_cascade + (size_t)slot * g->num_cascades;
    ocean::SpectrumDispatch* hs = g->h_spectrum + (size_t)slot * g->num_cascades;
    ocean::TableDispatch* ht = g->h_tables + (size_t)slot * g->num_cascades;
    int n_dirty = 0, n_tables = 0;
    const uint32_t per_update = (uint32_t)ocean::a_items_per_cascade(g->map_size);
    for (int k = 0; k < n; ++k) {
        const int i = indices[k];
        const ocean_cascade_params& p = g->pass_parameters[i];
        if (p.should_generate_spectrum) {
            hs[n_dirty++] = make_spectrum_dispatch(p, i);   // :68-72
            g->sea_stale[i] = 1;
        }
        const int ts = assign_table_slot(g, i, p, ht, &n_tables);
        if (ts < 0) return fail(OCEAN_ERR_STATE, "no free dispersion-table slot (internal error)");
        hc[k] = make_cascade_dispatch(p, i, ts);                     // :73,85
        hc[k].done_target = g->done_count[i] + per_update;           // modulo 2^32
        g->scratch_layer_of[i] = hc[k].scratch_layer;
    }
    // From here on the device is touched.  The host-side state that must agree with it (dirty flags, the mirror of
    // the completion counters, the staging ring) is committed only after everything has been enqueued; on a failure
    // the device counters are re-synchronised from the unchanged mirror so that later launches cannot wait forever.
    bool counters_touched = false;
    auto fail_resync = [&](int code) {
        if (counters_touched) {
            cudaStreamSynchronize(g->stream);
            cudaMemcpy(g->d_queue.ptr + 1, g->done_count.data(), sizeof(uint32_t) * g->done_count.size(), cudaMemcpyHostToDevice);
        }
        return code;
    };
#define RUN_CUDA(expr)                                                                                              \
    do {                                                                                                            \
        cudaError_t e__ = (expr);                                                                                   \
        if (e__ != cudaSuccess)                                                                                     \
            return fail_resync(fail(OCEAN_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__)); \
    } while (0)
    if (g->profiling) RUN_CUDA(cudaEventRecord(g->prof[0], g->stream));
    if (n_dirty) {
        RUN_CUDA(cudaMemcpyAsync(g->d_spectrum.ptr, hs, sizeof(ocean::SpectrumDispatch) * n_dirty, cudaMemcpyHostToDevice, g->stream));
        RUN_CUDA(ocean::launch_spectrum_compute(g->buf, g->d_spectrum.ptr, n_dirty, g->stream));
    }
    if (n_tables) {
        RUN_CUDA(cudaMemcpyAsync(g->d_tables.ptr, ht, sizeof(ocean::TableDispatch) * n_tables, cudaMemcpyHostToDevice, g->stream));
        RUN_CUDA(ocean::launch_dispersion_tables(g->buf, g->d_tables.ptr, n_tables, g->stream));
    }
    const bool two_kernel = g->profiling;              // profiled updates time the row and the column pass apart
    if (two_kernel)   // the persistent launch takes its dispatch records by value
        RUN_CUDA(cudaMemcpyAsync(g->d_cascade.ptr, hc, sizeof(ocean::CascadeDispatch) * n, cudaMemcpyHostToDevice, g->stream));
    // The staging slot is free again once the copies above have read it.  Without them (the persistent path with no spectrum
    // or table to rebuild: every step of a steady simulation) nothing on the device reads the slot, no event is recorded, and
    // the last record of ring_done[slot] -- older work -- is what the next use of the slot waits for.
    const bool staged = n_dirty || n_tables || two_kernel;
    if (staged) RUN_CUDA(cudaEventRecord(g->ring_done[slot], g->stream));
    // The first persistent launch follows the previous update's persistent launch directly when no entry point ran in between
    // and nothing was enqueued above: it is then queued as that launch's programmatic dependent.  Later launches of this call
    // follow one of its own.
    bool chained = !staged && g->update_tail != 0 && g->entries - g->update_tail <= 1;
    g->update_tail = 0;
    int launched = 0;
    if (g->profiling) RUN_CUDA(cudaEventRecord(g->prof[1], g->stream));
    if (!two_kernel) {
        // one persistent launch per <= kMaxPersistentCascades cascades (their dispatch records travel by value)
        for (int first = 0; first < n; first += ocean::kMaxPersistentCascades) {
            const int m = (n - first < ocean::kMaxPersistentCascades) ? n - first : ocean::kMaxPersistentCascades;
            auto build = [&](int* out) {
                return ocean::build_item_table(g->map_size, m, ocean::persistent_group(g->map_size), ocean::persistent_lag(g->map_size), out);
            };
            const DeviceArray<int>* table = nullptr;
            const bool cached = g->item_tables.count(m) != 0;        // a first use uploads the table: a copy on the stream
            RUN_CUDA(item_table(g, g->item_tables, m, build, &table));
            counters_touched = true;
            RUN_CUDA(ocean::launch_cascade_update_persistent(g->buf, hc + first, m, g->stream, g->d_queue.ptr, table->ptr,
                                                             (int)table->capacity, g->resident_ctas, false, chained && cached));
            chained = true;
            launched += 1;
        }
    } else {
        RUN_CUDA(ocean::launch_cascade_update(g->buf, g->d_cascade.ptr, n, g->stream, &launched, g->prof[2], g->prof[4]));
        // (the device-side completion counters are brought in step with the host mirror at the commit below)
    }
    if (g->profiling) {
        RUN_CUDA(cudaEventRecord(g->prof[3], g->stream));
        g->prof_valid = true;
        g->prof_had_gen = n_dirty != 0;
        const int ch = ocean::chunk_cascades(g->map_size);
        g->prof_chunk = n < ch ? n : ch;
    }
    // ---- commit ----
    for (int k = 0; k < n; ++k) {
        const int i = indices[k];
        g->pass_parameters[i].should_generate_spectrum = 0;          // :72
        g->done_count[i] += per_update;
        record_velocity_source(g, hc[k]);
    }
    if (two_kernel)
        RUN_CUDA(cudaMemcpyAsync(g->d_queue.ptr + 1, g->done_count.data(), sizeof(uint32_t) * g->done_count.size(), cudaMemcpyHostToDevice, g->stream));
#undef RUN_CUDA
    if (!two_kernel) g->update_tail = g->entries;
    g->ring_next = (g->ring_next + 1) % kRing;
    g->kernel_launches += (uint64_t)launched + (n_dirty ? 1 : 0) + (n_tables ? 1 : 0);
    g->cascade_updates += (uint64_t)n;
    return OCEAN_OK;
}

int validate_params(ocean_generator* g, const ocean_cascade_params* parameters, int count) {
    if (!parameters) return fail(OCEAN_ERR_INVALID_ARGUMENT, "parameters is NULL");
    if (count <= 0) return fail(OCEAN_ERR_INVALID_ARGUMENT, "parameters.size() must be != 0 (wave_generator.gd:91)");
    if (count > g->num_cascades)
        return fail(OCEAN_ERR_INVALID_ARGUMENT, "%d cascades passed but the generator was created with %d layers", count, g->num_cascades);
    for (int i = 0; i < count; ++i) {
        const ocean_cascade_params& p = parameters[i];
        if (!(p.tile_length[0] > 0.0f) || !(p.tile_length[1] > 0.0f))
            return fail(OCEAN_ERR_INVALID_ARGUMENT, "cascade %d: tile_length must be positive", i);
        if (!(p.wind_speed > 0.0) || !(p.fetch_length > 0.0))
            return fail(OCEAN_ERR_INVALID_ARGUMENT, "cascade %d: wind_speed and fetch_length must be positive (setters clamp to 1e-4)", i);
    }
    return OCEAN_OK;
}

int check_cascade(ocean_generator* g, int cascade) {
    if (cascade < 0 || cascade >= g->num_cascades)
        return fail(OCEAN_ERR_INVALID_ARGUMENT, "cascade index %d out of range [0,%d)", cascade, g->num_cascades);
    return OCEAN_OK;
}

// Layers [first, first + count) inside [0, num_cascades); compared without forming first + count, which can overflow an int.
int check_layer_range(ocean_generator* g, int first, int count) {
    if (first < 0 || count < 0 || count > g->num_cascades - first)
        return fail(OCEAN_ERR_INVALID_ARGUMENT, "layer range [%d,%lld) outside [0,%d)", first, (long long)first + count, g->num_cascades);
    return OCEAN_OK;
}

}  // namespace

extern "C" {

const char* ocean_last_error(void) { return g_last_error.c_str(); }
const char* ocean_version(void) { return "godotoceanwaves_b200 0.1 (sm_90a)"; }

double ocean_jonswap_alpha(double wind_speed, double fetch_length) {             // wave_generator.gd:116-117
    return 0.076 * std::pow(wind_speed * wind_speed / (fetch_length * kG), 0.22);
}
double ocean_jonswap_peak_angular_frequency(double wind_speed, double fetch_length) {   // wave_generator.gd:120-121
    return 22.0 * std::pow(kG * kG / (wind_speed * fetch_length), 1.0 / 3.0);
}

int ocean_default_cascade_params(ocean_cascade_params* out) {                    // wave_cascade_parameters.gd:7-42
    if (!out) return fail(OCEAN_ERR_INVALID_ARGUMENT, "out is NULL");
    std::memset(out, 0, sizeof *out);
    out->tile_length[0] = out->tile_length[1] = 50.0f;
    out->displacement_scale = 1.0;
    out->normal_scale = 1.0;
    out->wind_speed = 20.0;
    out->wind_direction = 0.0;
    out->fetch_length = 550.0;
    out->swell = 0.8;
    out->spread = 0.2;
    out->detail = 1.0;
    out->whitecap = 0.5;
    out->foam_amount = 5.0;
    out->should_generate_spectrum = 1;
    return OCEAN_OK;
}

int ocean_create(int device, int map_size, int num_cascades, ocean_generator** out) {
    if (!out) return fail(OCEAN_ERR_INVALID_ARGUMENT, "out is NULL");
    *out = nullptr;
    if (map_size != 128 && map_size != 256 && map_size != 512 && map_size != 1024)
        return fail(OCEAN_ERR_INVALID_ARGUMENT, "map_size %d not in {128,256,512,1024} (water.gd:38)", map_size);
    if (num_cascades < 1) return fail(OCEAN_ERR_INVALID_ARGUMENT, "num_layers >= 1 required (render_context.gd:77)");
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        return fail(OCEAN_ERR_CUDA, "no CUDA device available (%s); this library has no CPU fallback", cudaGetErrorString(e));
    if (device < 0 || device >= ndev) return fail(OCEAN_ERR_INVALID_ARGUMENT, "device %d out of range [0,%d)", device, ndev);
    DeviceScope device_scope;
    OCEAN_CUDA(device_scope.enter(device));
    cudaDeviceProp prop;
    OCEAN_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0)
        return fail(OCEAN_ERR_UNSUPPORTED, "device %d is sm_%d%d; this library is built for sm_90a only", device, prop.major, prop.minor);

    ocean_generator* g = new (std::nothrow) ocean_generator();
    if (!g) return fail(OCEAN_ERR_STATE, "out of host memory");
    g->device = device;
    g->map_size = map_size;
    g->num_cascades = num_cascades;
    const size_t NN = (size_t)map_size * map_size;
    const size_t C = (size_t)num_cascades;
#define CREATE_CUDA(expr)                                                                                        \
    do {                                                                                                         \
        cudaError_t e__ = (expr);                                                                                \
        if (e__ != cudaSuccess) {                                                                                \
            release(g);                                                                                          \
            return fail(OCEAN_ERR_CUDA, "%s failed: %s", #expr, cudaGetErrorString(e__));                        \
        }                                                                                                        \
    } while (0)
    CREATE_CUDA(cudaStreamCreateWithFlags(&g->stream, cudaStreamNonBlocking));
    CREATE_CUDA(g->spectrum.grow(g, C * NN));                             // wave_generator.gd:31
    CREATE_CUDA(g->rowpass.grow(g, ocean::kScratchHalves * C * 2 * NN));  // replaces fft_buffer, :33
    CREATE_CUDA(g->displacement.grow(g, C * NN));                         // :34
    CREATE_CUDA(g->normal.grow(g, C * NN));                               // :35
    CREATE_CUDA(g->foam.grow(g, C * NN));
    CREATE_CUDA(g->twiddles.grow(g, (size_t)ocean::kTwiddleCount + 1));   // :32
    CREATE_CUDA(g->disp_table.grow(g, C * (size_t)(map_size / 2 + 1) * map_size));   // one slot per cascade at most
    CREATE_CUDA(g->disp_kvy.grow(g, C * (size_t)map_size));
    CREATE_CUDA(g->d_cascade.grow(g, C));
    CREATE_CUDA(g->d_spectrum.grow(g, C));
    CREATE_CUDA(g->d_tables.grow(g, C));
    CREATE_CUDA(g->d_queue.grow(g, 3 * C + 1));
    g->buf.spectrum = g->spectrum.ptr;
    g->buf.rowpass = g->rowpass.ptr;
    g->buf.displacement = g->displacement.ptr;
    g->buf.normal = g->normal.ptr;
    g->buf.foam = g->foam.ptr;
    g->buf.twiddles = g->twiddles.ptr;
    g->buf.disp_table = g->disp_table.ptr;
    g->buf.disp_kvy = g->disp_kvy.ptr;
    CREATE_CUDA(cudaMemsetAsync(g->d_queue.ptr, 0, sizeof(int) * (3 * C + 1), g->stream));
    g->done_count.assign(3 * C, 0u);                  // [0, C): row-pass counters (scratch half 0), [C, 2C): column pass, [2C, 3C): row pass, half 1
    g->slot_key.assign(C, ocean_generator::TableKey{0.f, 0.f, 0.f});
    g->slot_valid.assign(C, 0);
    g->slot_refs.assign(C, 0);
    g->cascade_slot.assign(C, -1);
    g->scratch_layer_of.resize(C);
    g->vel_source.assign(C, ocean::VelocityDispatch{0, 0, 0.0f});
    g->vel_has_source.assign(C, 0);
    g->vel_stale.assign(C, 0);
    g->sea_stale.assign(C, 0);
    for (int i = 0; i < C; ++i) g->scratch_layer_of[i] = 2 * i;
    CREATE_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&g->h_cascade), sizeof(ocean::CascadeDispatch) * kRing * C, cudaHostAllocDefault));
    CREATE_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&g->h_spectrum), sizeof(ocean::SpectrumDispatch) * kRing * C, cudaHostAllocDefault));
    CREATE_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&g->h_tables), sizeof(ocean::TableDispatch) * kRing * C, cudaHostAllocDefault));
    for (auto& ev : g->ring_done) CREATE_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    CREATE_CUDA(cudaEventCreate(&g->timer_start));
    CREATE_CUDA(cudaEventCreate(&g->timer_stop));
    for (auto& ev : g->prof) CREATE_CUDA(cudaEventCreate(&ev));
    // textures start cleared (foam state = 0)
    CREATE_CUDA(cudaMemsetAsync(g->buf.spectrum, 0, sizeof(float4) * C * NN, g->stream));
    CREATE_CUDA(cudaMemsetAsync(g->buf.rowpass, 0, sizeof(float4) * ocean::kScratchHalves * C * 2 * NN, g->stream));
    CREATE_CUDA(cudaMemsetAsync(g->buf.displacement, 0, sizeof(uint2) * C * NN, g->stream));
    CREATE_CUDA(cudaMemsetAsync(g->buf.normal, 0, sizeof(uint2) * C * NN, g->stream));
    CREATE_CUDA(cudaMemsetAsync(g->buf.foam, 0, sizeof(uint16_t) * C * NN, g->stream));
    g->buf.map_size = map_size;
    g->buf.num_cascades = num_cascades;
    CREATE_CUDA(ocean::make_rowpass_tensor_map(g->buf.rowpass, map_size, num_cascades, &g->buf.rowpass_tmap));
    CREATE_CUDA(ocean::configure_kernels(map_size));
    CREATE_CUDA(ocean::persistent_grid_size(map_size, &g->resident_ctas));
    CREATE_CUDA(ocean::init_twiddles(g->twiddles.ptr, g->stream));        // fft_butterfly once, :52-54
    g->kernel_launches += 1;
    CREATE_CUDA(cudaStreamSynchronize(g->stream));
#undef CREATE_CUDA
    *out = g;
    return OCEAN_OK;
}

int ocean_destroy(ocean_generator* gen) {
    if (!gen) return fail(OCEAN_ERR_INVALID_ARGUMENT, "generator handle is NULL");
    release(gen);
    return OCEAN_OK;
}

int ocean_update(ocean_generator* gen, double delta, ocean_cascade_params* parameters, int count) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    rc = validate_params(gen, parameters, count);
    if (rc) return rc;
    // wave_generator.gd:94-98: finish the cascades of the previous pass that were never processed
    if (gen->pass_num_cascades_remaining != 0) {
        std::vector<int> idx(gen->pass_num_cascades_remaining);
        for (int i = 0; i < gen->pass_num_cascades_remaining; ++i) idx[i] = i;
        // the reference dereferences the live Resource objects: refresh from the caller's array where it overlaps
        for (int i = 0; i < gen->pass_num_cascades_remaining && i < count; ++i) gen->pass_parameters[i] = parameters[i];
        rc = run_cascades(gen, idx.data(), (int)idx.size());
        if (rc) return rc;
        for (int i = 0; i < gen->pass_num_cascades_remaining && i < count; ++i)
            parameters[i].should_generate_spectrum = gen->pass_parameters[i].should_generate_spectrum;
        gen->pass_num_cascades_remaining = 0;
    }
    // :100-106
    for (int i = 0; i < count; ++i) {
        ocean_cascade_params& p = parameters[i];
        p.time += delta;
        p.foam_grow_rate = delta * p.foam_amount * 7.5;
        p.foam_decay_rate = delta * std::fmax(0.5, 10.0 - p.foam_amount) * 1.15;
    }
    gen->pass_parameters.assign(parameters, parameters + count);       // :108
    gen->pass_num_cascades_remaining = count;                          // :109
    return OCEAN_OK;
}

int ocean_process(ocean_generator* gen, ocean_cascade_params* parameters, int count) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if (gen->pass_num_cascades_remaining == 0) return OCEAN_OK;        // :58
    if (parameters) {
        if (count != (int)gen->pass_parameters.size())
            return fail(OCEAN_ERR_INVALID_ARGUMENT, "ocean_process: count %d differs from the armed pass (%d)", count, (int)gen->pass_parameters.size());
        rc = validate_params(gen, parameters, count);
        if (rc) return rc;
    }
    gen->pass_num_cascades_remaining -= 1;                             // :59
    const int i = gen->pass_num_cascades_remaining;
    if (parameters) gen->pass_parameters[i] = parameters[i];
    rc = run_cascades(gen, &i, 1);                                     // :61-63
    if (rc) return rc;
    if (parameters) parameters[i].should_generate_spectrum = gen->pass_parameters[i].should_generate_spectrum;
    return OCEAN_OK;
}

int ocean_update_all(ocean_generator* gen, double delta, ocean_cascade_params* parameters, int count) {
    int rc = ocean_update(gen, delta, parameters, count);
    if (rc) return rc;
    std::vector<int> idx(count);
    for (int i = 0; i < count; ++i) idx[i] = i;
    rc = run_cascades(gen, idx.data(), count);
    if (rc) return rc;
    for (int i = 0; i < count; ++i) parameters[i].should_generate_spectrum = gen->pass_parameters[i].should_generate_spectrum;
    gen->pass_num_cascades_remaining = 0;
    return OCEAN_OK;
}

// ---- completion-counter protocol of a fused launch: pure host arithmetic, shared by ocean_update_frames and by
// ocean_debug_frame_protocol (tests/test_queue_protocol_cpu.py runs it against random schedules on the CPU) ----
// counters[0, C): row passes in scratch half 0, [C, 2C): column passes, [2C, 3C): row passes in half 1 -- their values when the
// launch starts (every earlier launch is complete by then).  Frame f of the launch is frame first_frame + f of the call.
// Frame `first_frame + f` runs in half (first_frame + f) & 1 of the scratch, so its row pass only waits for the column pass two
// frames back and runs beside the previous frame's column pass; its column pass waits for its own row pass and -- foam plane,
// maps -- for the previous frame's column pass.  The halves count their row passes separately (frames f, f-2, ... of the launch).
static void frame_protocol_targets(ocean::CascadeDispatch& d, const uint32_t* counters, int C, int i, int first_frame, int f,
                                   uint32_t a_per, uint32_t b_per) {
    const int half = (first_frame + f) & 1;
    d.done_slot = half ? 2 * C + i : i;
    d.done_target = counters[d.done_slot] + (uint32_t)(f / 2 + 1) * a_per;
    d.wait_target = counters[C + i] + (uint32_t)(f > 0 ? f - 1 : 0) * b_per;
    d.col_wait_target = counters[C + i] + (uint32_t)f * b_per;
    d.scratch_layer = 2 * (half * C + i);
}
// the counters once a launch of F frames starting at frame first_frame is complete
static void frame_protocol_commit(uint32_t* counters, int C, int i, int first_frame, int F, uint32_t a_per, uint32_t b_per) {
    const int first_half = first_frame & 1;                        // half of the launch's frame 0; it runs (F + 1) / 2 frames there
    counters[first_half ? 2 * C + i : i] += (uint32_t)((F + 1) / 2) * a_per;
    counters[first_half ? i : 2 * C + i] += (uint32_t)(F / 2) * a_per;
    counters[C + i] += (uint32_t)F * b_per;
}

int ocean_debug_frame_protocol(int map_size, int num_cascades, int count, int first_frame, int frames, uint32_t* counters, int32_t* records) {
    const uint32_t a_per = (uint32_t)ocean::a_items_per_cascade(map_size), b_per = (uint32_t)ocean::b_items_per_cascade(map_size);
    if (a_per == 0 || num_cascades < 1 || count < 1 || count > num_cascades || first_frame < 0 || frames < 1 || !counters || !records)
        return fail(OCEAN_ERR_INVALID_ARGUMENT, "ocean_debug_frame_protocol: bad arguments");
    for (int f = 0; f < frames; ++f)
        for (int i = 0; i < count; ++i) {
            ocean::CascadeDispatch d{};
            d.cascade = i;
            frame_protocol_targets(d, counters, num_cascades, i, first_frame, f, a_per, b_per);
            int32_t* r = records + ((size_t)f * count + i) * 6;
            r[0] = d.cascade; r[1] = d.done_slot; r[2] = (int32_t)d.done_target; r[3] = (int32_t)d.wait_target;
            r[4] = (int32_t)d.col_wait_target; r[5] = d.scratch_layer;
        }
    for (int i = 0; i < count; ++i) frame_protocol_commit(counters, num_cascades, i, first_frame, frames, a_per, b_per);
    return OCEAN_OK;
}

int ocean_update_frames(ocean_generator* gen, double delta, ocean_cascade_params* parameters, int count, int frames) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if (frames < 0) return fail(OCEAN_ERR_INVALID_ARGUMENT, "frames %d is negative", frames);
    if (frames == 0) return OCEAN_OK;
    const int per_launch = count > 0 ? ocean::kMaxPersistentCascades / count : 0;
    if (gen->profiling || per_launch < 2) {                            // two-kernel path / huge sets: frame by frame
        for (int f = 0; f < frames; ++f)
            if ((rc = ocean_update_all(gen, delta, parameters, count))) return rc;
        return OCEAN_OK;
    }
    // frame 0 exactly as ocean_update_all: flush of a pending pass, time/rate advance, spectra and tables where needed
    if ((rc = ocean_update_all(gen, delta, parameters, count))) return rc;
    gen->update_tail = 0;                                              // the fused launches below are not single updates
    const uint32_t a_per = (uint32_t)ocean::a_items_per_cascade(gen->map_size), b_per = (uint32_t)ocean::b_items_per_cascade(gen->map_size);
    const int C = gen->num_cascades;
    std::vector<ocean::CascadeDispatch> rec;
    int done = 1;
    while (done < frames) {
        const int F = (frames - done < per_launch) ? frames - done : per_launch;
        rec.resize((size_t)F * count);
        for (int f = 0; f < F; ++f) {
            for (int i = 0; i < count; ++i) {                              // wave_generator.gd:100-106, once per frame
                ocean_cascade_params& p = parameters[i];
                p.time += delta;
                p.foam_grow_rate = delta * p.foam_amount * 7.5;
                p.foam_decay_rate = delta * std::fmax(0.5, 10.0 - p.foam_amount) * 1.15;
                ocean::CascadeDispatch d = make_cascade_dispatch(p, i, gen->cascade_slot[i]);
                frame_protocol_targets(d, gen->done_count.data(), C, i, done, f, a_per, b_per);
                gen->scratch_layer_of[i] = d.scratch_layer;
                rec[(size_t)f * count + i] = d;
            }
        }
        auto build = [&](int* out) { return ocean::build_item_table_frames(gen->map_size, count, F, out); };
        const DeviceArray<int>* table = nullptr;
        OCEAN_CUDA(item_table(gen, gen->frame_tables, std::make_pair(count, F), build, &table));
        cudaError_t le = ocean::launch_cascade_update_persistent(gen->buf, rec.data(), F * count, gen->stream, gen->d_queue.ptr, table->ptr,
                                                                 (int)table->capacity, gen->resident_ctas, true);
        if (le != cudaSuccess) {
            cudaStreamSynchronize(gen->stream);
            cudaMemcpy(gen->d_queue.ptr + 1, gen->done_count.data(), sizeof(uint32_t) * gen->done_count.size(), cudaMemcpyHostToDevice);
            return fail(OCEAN_ERR_CUDA, "multi-frame launch failed: %s", cudaGetErrorString(le));
        }
        for (int i = 0; i < count; ++i) {
            frame_protocol_commit(gen->done_count.data(), C, i, done, F, a_per, b_per);
            record_velocity_source(gen, rec[(size_t)(F - 1) * count + i]);     // the launch's last frame built the maps
        }
        gen->kernel_launches += 1;
        gen->cascade_updates += (uint64_t)F * count;
        done += F;
    }
    gen->pass_parameters.assign(parameters, parameters + count);
    for (int i = 0; i < count; ++i) gen->pass_parameters[i].should_generate_spectrum = 0;
    gen->pass_num_cascades_remaining = 0;
    return OCEAN_OK;
}

// ---- Water node hand-off (assets/water/water.gd) ----
int ocean_scheduler_init(ocean_scheduler* s, double updates_per_second) {
    if (!s) return fail(OCEAN_ERR_INVALID_ARGUMENT, "scheduler is NULL");
    s->updates_per_second = updates_per_second;       // water.gd:51
    s->time = 0.0;                                    // :62
    s->next_update_time = 0.0;                        // :63
    return OCEAN_OK;
}

int ocean_scheduler_set_rate(ocean_scheduler* s, double value) {                  // water.gd:52-54
    if (!s) return fail(OCEAN_ERR_INVALID_ARGUMENT, "scheduler is NULL");
    s->next_update_time = s->next_update_time - (1.0 / (s->updates_per_second + 1e-10) - 1.0 / (value + 1e-10));
    s->updates_per_second = value;
    return OCEAN_OK;
}

int ocean_scheduler_tick(ocean_scheduler* s, double delta, double* update_delta) {   // water.gd:75-82
    if (!s) {
        fail(OCEAN_ERR_INVALID_ARGUMENT, "scheduler is NULL");
        return 0;
    }
    int due = 0;
    if (s->updates_per_second == 0 || s->time >= s->next_update_time) {              // :77
        const double target_update_delta = 1.0 / (s->updates_per_second + 1e-10);    // :78
        const double ud = (s->updates_per_second == 0) ? delta : target_update_delta + (s->time - s->next_update_time);   // :79
        s->next_update_time = s->time + target_update_delta;                         // :80
        if (update_delta) *update_delta = ud;
        due = 1;                                                                     // :81 _update_water(update_delta)
    }
    s->time += delta;                                                                // :82
    return due;
}

int ocean_water_frame(ocean_generator* gen, ocean_scheduler* s, double delta, ocean_cascade_params* parameters, int count, int* did_update) {
    if (!s) return fail(OCEAN_ERR_INVALID_ARGUMENT, "scheduler is NULL");
    double ud = 0.0;
    const int due = ocean_scheduler_tick(s, delta, &ud);
    if (did_update) *did_update = due;
    if (due) {                                                                       // Water._process -> _update_water, :112-114
        const int rc = ocean_update(gen, ud, parameters, count);
        if (rc) return rc;
    }
    return ocean_process(gen, parameters, count);                                    // the child node's _process, wave_generator.gd:56-63
}

int ocean_map_scales(const ocean_cascade_params* parameters, int count, float* map_scales) {     // water.gd:102-110
    if (!parameters || !map_scales) return fail(OCEAN_ERR_INVALID_ARGUMENT, "NULL argument");
    for (int i = 0; i < count; ++i) {
        map_scales[4 * i + 0] = 1.0f / parameters[i].tile_length[0];     // Vector2.ONE / tile_length (binary32)
        map_scales[4 * i + 1] = 1.0f / parameters[i].tile_length[1];
        map_scales[4 * i + 2] = (float)parameters[i].displacement_scale;
        map_scales[4 * i + 3] = (float)parameters[i].normal_scale;
    }
    return OCEAN_OK;
}

double ocean_water_default_time(int cascade) { return 120.0 + M_PI * cascade; }                   // water.gd:32

int ocean_get_maps(ocean_generator* gen, void** displacement_dev, void** normal_dev, size_t* layer_bytes) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if (displacement_dev) *displacement_dev = gen->buf.displacement;
    if (normal_dev) *normal_dev = gen->buf.normal;
    if (layer_bytes) *layer_bytes = sizeof(uint2) * (size_t)gen->map_size * gen->map_size;
    return OCEAN_OK;
}

int ocean_copy_maps_to_host_async(ocean_generator* gen, int first, int count, void* displacement_host, void* normal_host) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if ((rc = check_layer_range(gen, first, count))) return rc;
    const size_t layer = (size_t)gen->map_size * gen->map_size;
    if (displacement_host)
        OCEAN_CUDA(cudaMemcpyAsync(displacement_host, gen->buf.displacement + first * layer, sizeof(uint2) * layer * count, cudaMemcpyDeviceToHost, gen->stream));
    if (normal_host)
        OCEAN_CUDA(cudaMemcpyAsync(normal_host, gen->buf.normal + first * layer, sizeof(uint2) * layer * count, cudaMemcpyDeviceToHost, gen->stream));
    return OCEAN_OK;
}

int ocean_snapshot_maps_to_host_async(ocean_generator* gen, int first, int count, void* displacement_host, void* normal_host) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if ((rc = check_layer_range(gen, first, count))) return rc;
    if (count == 0) return OCEAN_OK;
    const size_t layer = (size_t)gen->map_size * gen->map_size;
    if (!gen->copy_stream) {
        OCEAN_CUDA(cudaStreamCreateWithFlags(&gen->copy_stream, cudaStreamNonBlocking));
        OCEAN_CUDA(cudaEventCreateWithFlags(&gen->snap_ready, cudaEventDisableTiming));
        OCEAN_CUDA(cudaEventCreateWithFlags(&gen->snap_free, cudaEventDisableTiming));
    }
    OCEAN_CUDA(gen->snap_disp.grow(gen, (size_t)gen->num_cascades * layer));
    OCEAN_CUDA(gen->snap_normal.grow(gen, (size_t)gen->num_cascades * layer));
    // the snapshot buffers are free again once the previous hand-off has left the device
    if (gen->snap_busy) OCEAN_CUDA(cudaStreamWaitEvent(gen->stream, gen->snap_free, 0));
    if (displacement_host)
        OCEAN_CUDA(cudaMemcpyAsync(gen->snap_disp.ptr + first * layer, gen->buf.displacement + first * layer, sizeof(uint2) * layer * count,
                                   cudaMemcpyDeviceToDevice, gen->stream));
    if (normal_host)
        OCEAN_CUDA(cudaMemcpyAsync(gen->snap_normal.ptr + first * layer, gen->buf.normal + first * layer, sizeof(uint2) * layer * count,
                                   cudaMemcpyDeviceToDevice, gen->stream));
    OCEAN_CUDA(cudaEventRecord(gen->snap_ready, gen->stream));
    OCEAN_CUDA(cudaStreamWaitEvent(gen->copy_stream, gen->snap_ready, 0));
    if (displacement_host)
        OCEAN_CUDA(cudaMemcpyAsync(displacement_host, gen->snap_disp.ptr + first * layer, sizeof(uint2) * layer * count, cudaMemcpyDeviceToHost,
                                   gen->copy_stream));
    if (normal_host)
        OCEAN_CUDA(cudaMemcpyAsync(normal_host, gen->snap_normal.ptr + first * layer, sizeof(uint2) * layer * count, cudaMemcpyDeviceToHost,
                                   gen->copy_stream));
    OCEAN_CUDA(cudaEventRecord(gen->snap_free, gen->copy_stream));
    gen->snap_busy = true;
    return OCEAN_OK;
}

int ocean_wait_snapshot(ocean_generator* gen) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if (gen->copy_stream) OCEAN_CUDA(cudaStreamSynchronize(gen->copy_stream));
    return OCEAN_OK;
}

int ocean_copy_maps_to_host(ocean_generator* gen, int first, int count, void* displacement_host, void* normal_host) {
    int rc = ocean_copy_maps_to_host_async(gen, first, count, displacement_host, normal_host);
    if (rc) return rc;
    OCEAN_CUDA(cudaStreamSynchronize(gen->stream));
    return OCEAN_OK;
}

int ocean_synchronize(ocean_generator* gen) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    OCEAN_CUDA(cudaStreamSynchronize(gen->stream));
    return OCEAN_OK;
}

int ocean_host_alloc(void** ptr, size_t bytes) {
    if (!ptr) return fail(OCEAN_ERR_INVALID_ARGUMENT, "ptr is NULL");
    OCEAN_CUDA(cudaHostAlloc(ptr, bytes, cudaHostAllocDefault));
    return OCEAN_OK;
}
int ocean_host_free(void* ptr) {
    OCEAN_CUDA(cudaFreeHost(ptr));
    return OCEAN_OK;
}

int ocean_copy_spectrum_to_host(ocean_generator* gen, int cascade, float* host) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if ((rc = check_cascade(gen, cascade))) return rc;
    if (!host) return fail(OCEAN_ERR_INVALID_ARGUMENT, "host is NULL");
    const size_t layer = (size_t)gen->map_size * gen->map_size;
    OCEAN_CUDA(cudaMemcpyAsync(host, gen->buf.spectrum + cascade * layer, sizeof(float4) * layer, cudaMemcpyDeviceToHost, gen->stream));
    OCEAN_CUDA(cudaStreamSynchronize(gen->stream));
    return OCEAN_OK;
}

int ocean_set_spectrum_amplitudes(ocean_generator* gen, int cascade, const float* amplitudes) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if ((rc = check_cascade(gen, cascade))) return rc;
    if (!amplitudes) return fail(OCEAN_ERR_INVALID_ARGUMENT, "amplitudes is NULL");
    const int N = gen->map_size;
    std::vector<float> tex((size_t)N * N * 4);
    for (int y = 0; y < N; ++y)
        for (int x = 0; x < N; ++x) {
            const int xm = (N - x) % N, ym = (N - y) % N;                          // ivec2(mod(-id0, dims)), spectrum_compute.glsl:121
            const float* a0 = amplitudes + ((size_t)y * N + x) * 2;
            const float* a1 = amplitudes + ((size_t)ym * N + xm) * 2;
            float* t = tex.data() + ((size_t)y * N + x) * 4;
            t[0] = a0[0]; t[1] = a0[1]; t[2] = a1[0]; t[3] = -a1[1];                // (h0(k), conj h0(-k))  :124
        }
    OCEAN_CUDA(cudaStreamSynchronize(gen->stream));
    OCEAN_CUDA(cudaMemcpy(gen->buf.spectrum + (size_t)cascade * N * N, tex.data(), sizeof(float) * tex.size(), cudaMemcpyHostToDevice));
    if (gen->vel_has_source[cascade]) gen->vel_stale[cascade] = 1;       // the velocity layer reads the spectrum as stored
    gen->sea_stale[cascade] = 1;                                         // and so does the sea state
    return OCEAN_OK;
}

int ocean_enable_f32_taps(ocean_generator* gen, int enable) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    OCEAN_CUDA(cudaStreamSynchronize(gen->stream));
    const size_t n = (size_t)gen->num_cascades * gen->map_size * gen->map_size;
    if (enable && !gen->buf.displacement_f32) {
        // both maps exist and are cleared before the kernels see either
        OCEAN_CUDA(gen->displacement_f32.grow(gen, n));
        OCEAN_CUDA(gen->normal_f32.grow(gen, n));
        OCEAN_CUDA(cudaMemset(gen->displacement_f32.ptr, 0, sizeof(float4) * n));
        OCEAN_CUDA(cudaMemset(gen->normal_f32.ptr, 0, sizeof(float4) * n));
        gen->buf.displacement_f32 = gen->displacement_f32.ptr;
        gen->buf.normal_f32 = gen->normal_f32.ptr;
    } else if (!enable && gen->buf.displacement_f32) {
        gen->buf.displacement_f32 = gen->buf.normal_f32 = nullptr;
        gen->displacement_f32.release();
        gen->normal_f32.release();
        gen->velocity_f32.release();
    }
    return OCEAN_OK;
}

int ocean_copy_f32_maps_to_host(ocean_generator* gen, int cascade, float* displacement_host, float* normal_host) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if ((rc = check_cascade(gen, cascade))) return rc;
    if (!gen->buf.displacement_f32) return fail(OCEAN_ERR_STATE, "binary32 taps are disabled; call ocean_enable_f32_taps(gen, 1) first");
    const size_t layer = (size_t)gen->map_size * gen->map_size;
    if (displacement_host)
        OCEAN_CUDA(cudaMemcpyAsync(displacement_host, gen->buf.displacement_f32 + cascade * layer, sizeof(float4) * layer, cudaMemcpyDeviceToHost, gen->stream));
    if (normal_host)
        OCEAN_CUDA(cudaMemcpyAsync(normal_host, gen->buf.normal_f32 + cascade * layer, sizeof(float4) * layer, cudaMemcpyDeviceToHost, gen->stream));
    OCEAN_CUDA(cudaStreamSynchronize(gen->stream));
    return OCEAN_OK;
}

int ocean_copy_rowpass_to_host(ocean_generator* gen, int cascade, float* host) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if ((rc = check_cascade(gen, cascade))) return rc;
    if (!host) return fail(OCEAN_ERR_INVALID_ARGUMENT, "host is NULL");
    // without the taps the column pass drops the scratch lines from L2 once it has consumed them (no DRAM write-back)
    if (!gen->buf.displacement_f32) return fail(OCEAN_ERR_STATE, "the row-pass scratch is only kept while the taps are on; call ocean_enable_f32_taps(gen, 1) before the update");
    const size_t layer = (size_t)gen->map_size * gen->map_size;
    OCEAN_CUDA(gen->export_buf.grow(gen, 4 * layer));
    OCEAN_CUDA(ocean::launch_rowpass_export(gen->buf, gen->scratch_layer_of[cascade], gen->export_buf.ptr, gen->stream));
    gen->kernel_launches += 1;
    OCEAN_CUDA(cudaMemcpyAsync(host, gen->export_buf.ptr, sizeof(float2) * 4 * layer, cudaMemcpyDeviceToHost, gen->stream));
    OCEAN_CUDA(cudaStreamSynchronize(gen->stream));
    return OCEAN_OK;
}

float ocean_detmath_expf(float x) { return exp_det_host(x); }

int ocean_debug_work_queue(int map_size, int count, int group, int lag, int frames, int32_t* items, int capacity) {
    if (ocean::a_items_per_cascade(map_size) == 0 || count < 1 || frames < 0 || (long long)count * (frames > 0 ? frames : 1) > 0x7fff ||
        (items == nullptr && capacity > 0))
        return -fail(OCEAN_ERR_INVALID_ARGUMENT, "ocean_debug_work_queue: map_size must be 128/256/512/1024, 1 <= count * frames <= 32767");
    if (group <= 0) group = ocean::persistent_group(map_size);
    if (lag <= 0) lag = ocean::persistent_lag(map_size);
    auto build = [&](int* out) {
        return frames > 0 ? ocean::build_item_table_frames(map_size, count, frames, out) : ocean::build_item_table(map_size, count, group, lag, out);
    };
    const int total = build(nullptr);
    if (items && capacity > 0) {
        std::vector<int> all((size_t)total);
        build(all.data());
        for (int i = 0; i < total && i < capacity; ++i) items[i] = all[(size_t)i];
    }
    return total;
}

// ---- map queries (SURVEY 8f row f2) ----
namespace {
int upload_scales(ocean_generator* gen, int num_cascades, const float* map_scales_host) {
    if (num_cascades < 1 || num_cascades > gen->num_cascades)
        return fail(OCEAN_ERR_INVALID_ARGUMENT, "num_cascades %d outside [1, %d]", num_cascades, gen->num_cascades);
    if (!map_scales_host) return fail(OCEAN_ERR_INVALID_ARGUMENT, "map_scales is NULL");
    OCEAN_CUDA(gen->q_scales.grow(gen, (size_t)gen->num_cascades));
    OCEAN_CUDA(cudaMemcpyAsync(gen->q_scales.ptr, map_scales_host, sizeof(float4) * (size_t)num_cascades, cudaMemcpyHostToDevice, gen->stream));
    return OCEAN_OK;
}
}  // namespace

int ocean_sample_maps_device(ocean_generator* gen, int num_points, const float* points_xz_dev, int num_cascades, const float* map_scales_host,
                             float* displacement_dev, float* gradient_foam_dev) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if (num_points < 0) return fail(OCEAN_ERR_INVALID_ARGUMENT, "num_points %d is negative", num_points);
    if (num_points == 0) return OCEAN_OK;
    if (!points_xz_dev || !displacement_dev || !gradient_foam_dev) return fail(OCEAN_ERR_INVALID_ARGUMENT, "a device buffer is NULL");
    if ((rc = upload_scales(gen, num_cascades, map_scales_host))) return rc;
    OCEAN_CUDA(ocean::launch_sample_maps(gen->buf, num_cascades, reinterpret_cast<const float2*>(points_xz_dev), num_points, gen->q_scales.ptr,
                                         displacement_dev, gradient_foam_dev, gen->stream));
    gen->kernel_launches += 1;
    return OCEAN_OK;
}

int ocean_sample_maps(ocean_generator* gen, int num_points, const float* points_xz_host, int num_cascades, const float* map_scales_host,
                      float* displacement_host, float* gradient_foam_host) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if (num_points < 0) return fail(OCEAN_ERR_INVALID_ARGUMENT, "num_points %d is negative", num_points);
    if (num_points == 0) return OCEAN_OK;
    if (!points_xz_host || !displacement_host || !gradient_foam_host) return fail(OCEAN_ERR_INVALID_ARGUMENT, "a host buffer is NULL");
    Staging st;
    const auto points = st.in(points_xz_host, 2 * (size_t)num_points);
    const auto disp = st.out(displacement_host, 3 * (size_t)num_points), grad = st.out(gradient_foam_host, 3 * (size_t)num_points);
    if ((rc = st.upload(gen, kStageSampleMaps))) return rc;
    return st.finish(gen, ocean_sample_maps_device(gen, num_points, st[points], num_cascades, map_scales_host, st[disp], st[grad]));
}

// ---- spray candidates (SURVEY 8f row f3) ----
static_assert(sizeof(ocean_spray_record) == 32, "ocean_spray_record layout");

int ocean_spray_grid(int num_particles, const float* emission_transform, float* points_xz_host) {
    if (num_particles < 0) return fail(OCEAN_ERR_INVALID_ARGUMENT, "num_particles %d is negative", num_particles);
    if (num_particles == 0) return OCEAN_OK;
    if (!points_xz_host) return fail(OCEAN_ERR_INVALID_ARGUMENT, "points_xz is NULL");
    static const float identity[12] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0};
    const float* E = emission_transform ? emission_transform : identity;
    // sea_spray_particle.gdshader:47,52-54, binary32 with every operation rounded on its own (volatile defeats contraction)
    const unsigned t = (unsigned)std::sqrt((float)num_particles);
    if (t < 2) return fail(OCEAN_ERR_INVALID_ARGUMENT, "num_particles %d gives a grid side below 2 (division by t - 1)", num_particles);
    const float tm1 = (float)t - 1.0f;
    for (unsigned i = 0; i < (unsigned)num_particles; ++i) {
        volatile float cx = (float)(i / t) / tm1, cz = (float)(i % t) / tm1;
        cx = cx - 0.5f; cz = cz - 0.5f;
        cx = cx * 10.0f; cz = cz * 10.0f;
        for (int k = 0; k < 2; ++k) {
            const float* row = E + 4 * (k == 0 ? 0 : 2);
            volatile float a = row[0] * cx, b0 = row[1] * 0.0f, c = row[2] * cz;
            volatile float sum = a + b0;
            sum = sum + c;
            sum = sum + row[3];
            points_xz_host[2 * (size_t)i + k] = sum;
        }
    }
    return OCEAN_OK;
}

int ocean_extract_spray_device(ocean_generator* gen, int num_candidates, const float* points_xz_dev, int num_cascades,
                               const float* map_scales_host, const float* particle_scale, int max_records,
                               ocean_spray_record* records_dev, int* num_active_dev) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if (num_candidates < 0 || max_records < 0) return fail(OCEAN_ERR_INVALID_ARGUMENT, "negative count");
    if (!num_active_dev) return fail(OCEAN_ERR_INVALID_ARGUMENT, "num_active is NULL");
    if (num_candidates == 0) {
        OCEAN_CUDA(cudaMemsetAsync(num_active_dev, 0, sizeof(int), gen->stream));
        return OCEAN_OK;
    }
    if (!points_xz_dev || !particle_scale || (max_records > 0 && !records_dev)) return fail(OCEAN_ERR_INVALID_ARGUMENT, "a buffer is NULL");
    if ((rc = upload_scales(gen, num_cascades, map_scales_host))) return rc;
    const int blocks = ocean::spray_blocks(num_candidates);
    OCEAN_CUDA(gen->spray_counts.grow(gen, (size_t)blocks + 1));
    const bool wk = gen->wake.reads(OCEAN_WAKE_READ_SPRAY);
    const ocean::WakeRead wake = wk ? gen->wake.read_h() : ocean::WakeRead{};
    OCEAN_CUDA(ocean::launch_extract_spray(gen->buf, num_cascades, reinterpret_cast<const float2*>(points_xz_dev), num_candidates,
                                           gen->q_scales.ptr, make_float3(particle_scale[0], particle_scale[1], particle_scale[2]),
                                           gen->spray_counts.ptr, records_dev, max_records, wk ? &wake : nullptr, gen->stream));
    gen->kernel_launches += 3;
    OCEAN_CUDA(cudaMemcpyAsync(num_active_dev, gen->spray_counts.ptr + blocks, sizeof(int), cudaMemcpyDeviceToDevice, gen->stream));
    return OCEAN_OK;
}

int ocean_extract_spray(ocean_generator* gen, int num_candidates, const float* points_xz_host, int num_cascades,
                        const float* map_scales_host, const float* particle_scale, int max_records,
                        ocean_spray_record* records_host, int* num_active) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if (num_candidates < 0 || max_records < 0) return fail(OCEAN_ERR_INVALID_ARGUMENT, "negative count");
    if (!num_active) return fail(OCEAN_ERR_INVALID_ARGUMENT, "num_active is NULL");
    *num_active = 0;
    if (num_candidates == 0) return OCEAN_OK;
    if (!points_xz_host || (max_records > 0 && !records_host)) return fail(OCEAN_ERR_INVALID_ARGUMENT, "a host buffer is NULL");
    int count = 0;
    Staging st;
    const auto points = st.in(points_xz_host, 2 * (size_t)num_candidates);
    const auto records = st.scratch<ocean_spray_record>((size_t)max_records);         // copied back below: only those kept
    const auto count_dev = st.out(&count, 1);
    if ((rc = st.upload(gen, kStageExtractSpray))) return rc;
    if ((rc = st.finish(gen, ocean_extract_spray_device(gen, num_candidates, st[points], num_cascades, map_scales_host, particle_scale,
                                                        max_records, st[records], st[count_dev]))))
        return rc;
    const int kept = std::min(count, max_records);
    if (kept > 0) OCEAN_CUDA(cudaMemcpy(records_host, st[records], sizeof(ocean_spray_record) * (size_t)kept, cudaMemcpyDeviceToHost));
    *num_active = count;
    return OCEAN_OK;
}

// ---- spray particles: one particle-process frame of a spray emitter ----
static_assert(sizeof(ocean_spray_emitter) == 88, "ocean_spray_emitter layout");
static_assert(sizeof(ocean_spray_particle) == 120, "ocean_spray_particle layout");

int ocean_default_spray_emitter(ocean_spray_emitter* out) {
    if (!out) return fail(OCEAN_ERR_INVALID_ARGUMENT, "out is NULL");
    *out = ocean_spray_emitter{};
    out->amount = 32768;                                // main.tscn:137
    out->num_particles = 32768;
    for (int r = 0; r < 3; ++r) out->emission_transform[5 * r] = 15.0f;     // main.tscn:134
    out->particle_scale[0] = 20.0f;
    out->particle_scale[1] = 8.5f;
    out->particle_scale[2] = 20.0f;
    out->lifetime = 3.0f;                               // sea_spray_particle.gdshader:22-23
    out->lifetime_randomness = 0.25f;
    out->random_seed = 0;
    out->emitter_lifetime = 6.0;                        // main.tscn:138
    return OCEAN_OK;
}

namespace {
int check_spray_particles_args(ocean_generator* gen, const ocean_spray_emitter* e, double t0, double t1, int num_cascades,
                               const float* map_scales, const void* states, int max_instances, const void* instances, const void* num_live) {
    if (!e) return fail(OCEAN_ERR_INVALID_ARGUMENT, "emitter is NULL");
    if (e->amount < 0) return fail(OCEAN_ERR_INVALID_ARGUMENT, "amount %d is negative", e->amount);
    if (e->num_particles < 1) return fail(OCEAN_ERR_INVALID_ARGUMENT, "num_particles %d is below 1", e->num_particles);
    if (!(e->lifetime > 0.0f) || !std::isfinite(e->lifetime))
        return fail(OCEAN_ERR_INVALID_ARGUMENT, "lifetime %g is not finite and > 0", e->lifetime);
    if (!(e->emitter_lifetime > 0.0) || !std::isfinite(e->emitter_lifetime))
        return fail(OCEAN_ERR_INVALID_ARGUMENT, "emitter_lifetime %g is not finite and > 0", e->emitter_lifetime);
    if (!(e->lifetime_randomness >= 0.0f && e->lifetime_randomness <= 1.0f))
        return fail(OCEAN_ERR_INVALID_ARGUMENT, "lifetime_randomness %g outside [0, 1]", e->lifetime_randomness);
    if (!std::isfinite(t0) || !std::isfinite(t1) || !(0.0 <= t0 && t0 <= t1))
        return fail(OCEAN_ERR_INVALID_ARGUMENT, "frame [%g, %g) is not 0 <= t0 <= t1, finite", t0, t1);
    if (!((float)t1 < 4294967296.0f) || !(t1 / e->emitter_lifetime < 4294967296.0))
        return fail(OCEAN_ERR_INVALID_ARGUMENT, "t1 %g: (float)t1 and t1 / emitter_lifetime must be below 2^32", t1);
    if (num_cascades < 1 || num_cascades > gen->num_cascades)
        return fail(OCEAN_ERR_INVALID_ARGUMENT, "num_cascades %d outside [1, %d]", num_cascades, gen->num_cascades);
    if (!map_scales) return fail(OCEAN_ERR_INVALID_ARGUMENT, "map_scales is NULL");
    if (max_instances < 0) return fail(OCEAN_ERR_INVALID_ARGUMENT, "max_instances %d is negative", max_instances);
    if (e->amount > 0 && !states) return fail(OCEAN_ERR_INVALID_ARGUMENT, "states is NULL");
    if (max_instances > 0 && !instances) return fail(OCEAN_ERR_INVALID_ARGUMENT, "instances is NULL");
    if (!num_live) return fail(OCEAN_ERR_INVALID_ARGUMENT, "num_live is NULL");
    return OCEAN_OK;
}
}  // namespace

int ocean_spray_particles_device(ocean_generator* gen, const ocean_spray_emitter* emitter, double t0, double t1, int num_cascades,
                                 const float* map_scales_host, ocean_spray_particle* states_dev, int max_instances, float* instances_dev,
                                 int* num_live_dev) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if ((rc = check_spray_particles_args(gen, emitter, t0, t1, num_cascades, map_scales_host, states_dev, max_instances, instances_dev,
                                         num_live_dev)))
        return rc;
    if (emitter->amount == 0) {
        OCEAN_CUDA(cudaMemsetAsync(num_live_dev, 0, sizeof(int), gen->stream));
        return OCEAN_OK;
    }
    if ((rc = upload_scales(gen, num_cascades, map_scales_host))) return rc;
    const int blocks = ocean::spray_blocks(emitter->amount);
    OCEAN_CUDA(gen->spray_counts.grow(gen, (size_t)blocks + 1));
    const bool wk = gen->wake.reads(OCEAN_WAKE_READ_SPRAY);
    const ocean::WakeRead wake = wk ? gen->wake.read_h() : ocean::WakeRead{};
    OCEAN_CUDA(ocean::launch_spray_particles(gen->buf, num_cascades, gen->q_scales.ptr, *emitter, t0, t1, states_dev, gen->spray_counts.ptr,
                                             instances_dev, max_instances, wk ? &wake : nullptr, gen->stream));
    gen->kernel_launches += 3;
    OCEAN_CUDA(cudaMemcpyAsync(num_live_dev, gen->spray_counts.ptr + blocks, sizeof(int), cudaMemcpyDeviceToDevice, gen->stream));
    return OCEAN_OK;
}

int ocean_spray_particles(ocean_generator* gen, const ocean_spray_emitter* emitter, double t0, double t1, int num_cascades,
                          const float* map_scales_host, ocean_spray_particle* states_host, int max_instances, float* instances_host,
                          int* num_live) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if ((rc = check_spray_particles_args(gen, emitter, t0, t1, num_cascades, map_scales_host, states_host, max_instances, instances_host,
                                         num_live)))
        return rc;
    *num_live = 0;
    if (emitter->amount == 0) return OCEAN_OK;
    int count = 0;
    Staging st;
    const auto states = st.inout(states_host, (size_t)emitter->amount);
    const auto instances = st.scratch<float>(16 * (size_t)max_instances);             // copied back below: only those kept
    const auto count_dev = st.out(&count, 1);
    if ((rc = st.upload(gen, kStageSprayParticles))) return rc;
    if ((rc = st.finish(gen, ocean_spray_particles_device(gen, emitter, t0, t1, num_cascades, map_scales_host, st[states], max_instances,
                                                          st[instances], st[count_dev]))))
        return rc;
    const int kept = std::min(count, max_instances);
    if (kept > 0) OCEAN_CUDA(cudaMemcpy(instances_host, st[instances], sizeof(float) * 16 * (size_t)kept, cudaMemcpyDeviceToHost));
    *num_live = count;
    return OCEAN_OK;
}

// ---- surface query: the surface at a world position (inverse of the horizontal displacement, then the map query) ----
static_assert(sizeof(ocean_surface_sample) == 40, "ocean_surface_sample layout");

namespace {
bool finite_positive(float x) { return x > 0.0f && std::isfinite(x); }
bool finite_nonnegative(float x) { return x >= 0.0f && std::isfinite(x); }

// The surface inversion's tolerance and iteration budget.
int check_solver_args(float tolerance, int max_iterations) {
    if (!finite_positive(tolerance)) return fail(OCEAN_ERR_INVALID_ARGUMENT, "tolerance %g is not finite and > 0", tolerance);
    if (max_iterations < 0 || max_iterations > 64) return fail(OCEAN_ERR_INVALID_ARGUMENT, "max_iterations %d outside [0, 64]", max_iterations);
    return OCEAN_OK;
}

int check_surface_args(int num_points, float tolerance, int max_iterations) {
    if (num_points < 0) return fail(OCEAN_ERR_INVALID_ARGUMENT, "num_points %d is negative", num_points);
    return check_solver_args(tolerance, max_iterations);
}

// The surface query on validated arguments, with the map scales already in gen->q_scales (ocean_query_surface_device and
// ocean_buoyancy_device).  With the wake coupling live, one more kernel adds the wake free surface to the records and, when
// wv_dev is not null (a drag pass follows), writes the wake's vertical velocity of each point there.
int run_query_surface(ocean_generator* gen, int num_points, const float2* points_xz_dev, int num_cascades, float tolerance,
                      int max_iterations, ocean_surface_sample* out_dev, float* wv_dev = nullptr) {
    OCEAN_CUDA(gen->surf_scratch.grow(gen, ocean::surface_scratch_ints(gen->num_cascades, num_points)));
    OCEAN_CUDA(ocean::launch_query_surface(gen->buf, num_cascades, points_xz_dev, num_points, gen->q_scales.ptr, tolerance, max_iterations,
                                           out_dev, gen->surf_scratch.ptr, gen->stream));
    gen->kernel_launches += max_iterations > 0 ? 3 : 1;
    if (gen->wake.coupling_live()) {
        OCEAN_CUDA(ocean::launch_wake_couple(gen->wake.couple_args(), points_xz_dev, num_points, out_dev, wv_dev, gen->stream));
        gen->kernel_launches += 1;
    }
    return OCEAN_OK;
}
}  // namespace

int ocean_query_surface_device(ocean_generator* gen, int num_points, const float* points_xz_dev, int num_cascades, const float* map_scales_host,
                               float tolerance, int max_iterations, ocean_surface_sample* out_dev) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if ((rc = check_surface_args(num_points, tolerance, max_iterations))) return rc;
    if (num_points == 0) return OCEAN_OK;
    if (!points_xz_dev || !out_dev) return fail(OCEAN_ERR_INVALID_ARGUMENT, "a device buffer is NULL");
    if ((rc = upload_scales(gen, num_cascades, map_scales_host))) return rc;
    return run_query_surface(gen, num_points, reinterpret_cast<const float2*>(points_xz_dev), num_cascades, tolerance, max_iterations, out_dev);
}

int ocean_query_surface(ocean_generator* gen, int num_points, const float* points_xz_host, int num_cascades, const float* map_scales_host,
                        float tolerance, int max_iterations, ocean_surface_sample* out_host) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if ((rc = check_surface_args(num_points, tolerance, max_iterations))) return rc;
    if (num_points == 0) return OCEAN_OK;
    if (!points_xz_host || !out_host) return fail(OCEAN_ERR_INVALID_ARGUMENT, "a host buffer is NULL");
    Staging st;
    const auto points = st.in(points_xz_host, 2 * (size_t)num_points);
    const auto out = st.out(out_host, (size_t)num_points);
    if ((rc = st.upload(gen, kStageQuerySurface))) return rc;
    return st.finish(gen, ocean_query_surface_device(gen, num_points, st[points], num_cascades, map_scales_host, tolerance, max_iterations,
                                                     st[out]));
}

// ---- ray cast: the first crossing of each ray with the displaced surface (slab bounds, then one thread per ray) ----
static_assert(sizeof(ocean_ray) == 28, "ocean_ray layout");
static_assert(sizeof(ocean_ray_hit) == 72, "ocean_ray_hit layout");

namespace {
int check_raycast_args(int num_rays, float step, int max_samples, float tolerance, int max_iterations) {
    int rc = check_surface_args(num_rays, tolerance, max_iterations);
    if (rc) return rc;
    if (!(step > 0.0f) || !std::isfinite(step)) return fail(OCEAN_ERR_INVALID_ARGUMENT, "step %g is not finite and > 0", step);
    if (max_samples < 2 || max_samples > (1 << 20)) return fail(OCEAN_ERR_INVALID_ARGUMENT, "max_samples %d outside [2, 2^20]", max_samples);
    return OCEAN_OK;
}
}  // namespace

int ocean_raycast_device(ocean_generator* gen, int num_rays, const ocean_ray* rays_dev, int num_cascades, const float* map_scales_host,
                         float step, int max_samples, float tolerance, int max_iterations, ocean_ray_hit* out_dev) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if ((rc = check_raycast_args(num_rays, step, max_samples, tolerance, max_iterations))) return rc;
    if (num_rays == 0) return OCEAN_OK;
    if (!rays_dev || !out_dev) return fail(OCEAN_ERR_INVALID_ARGUMENT, "a device buffer is NULL");
    if ((rc = upload_scales(gen, num_cascades, map_scales_host))) return rc;
    // with the ray cast reader set and the coupling live, the coupled surface: e in its own window, and one more kernel (its bounds)
    const bool wk = gen->wake.reads(OCEAN_WAKE_READ_RAYCAST) && gen->wake.coupling_live();
    const ocean::WakeRead wake = wk ? gen->wake.read_e() : ocean::WakeRead{};
    OCEAN_CUDA(gen->ray_bounds.grow(gen, 3 * (size_t)gen->num_cascades + (wk ? 2 : 0)));
    OCEAN_CUDA(ocean::launch_raycast(gen->buf, num_cascades, rays_dev, num_rays, gen->q_scales.ptr, step, max_samples, tolerance, max_iterations,
                                     gen->ray_bounds.ptr, out_dev, wk ? &wake : nullptr, gen->stream));
    gen->kernel_launches += wk ? 3 : 2;
    return OCEAN_OK;
}

int ocean_raycast(ocean_generator* gen, int num_rays, const ocean_ray* rays_host, int num_cascades, const float* map_scales_host,
                  float step, int max_samples, float tolerance, int max_iterations, ocean_ray_hit* out_host) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if ((rc = check_raycast_args(num_rays, step, max_samples, tolerance, max_iterations))) return rc;
    if (num_rays == 0) return OCEAN_OK;
    if (!rays_host || !out_host) return fail(OCEAN_ERR_INVALID_ARGUMENT, "a host buffer is NULL");
    Staging st;
    const auto rays = st.in(rays_host, (size_t)num_rays);
    const auto out = st.out(out_host, (size_t)num_rays);
    if ((rc = st.upload(gen, kStageRaycast))) return rc;
    return st.finish(gen, ocean_raycast_device(gen, num_rays, st[rays], num_cascades, map_scales_host, step, max_samples, tolerance,
                                               max_iterations, st[out]));
}

// ---- buoyancy: per-body force and torque from hull points on the surface (the surface query between two buoyancy kernels) ----
static_assert(sizeof(ocean_buoyancy_point) == 20, "ocean_buoyancy_point layout");
static_assert(sizeof(ocean_buoyancy_body) == 56, "ocean_buoyancy_body layout");
static_assert(sizeof(ocean_buoyancy_result) == 48, "ocean_buoyancy_result layout");

namespace {
// The bodies' ranges into the hull points, in 64-bit; *world receives the number of world points, the sum of their num_points.
// (The templates here, over the body row types, need C++ linkage inside this extern "C" block.)
extern "C++" template <typename Body>
int check_point_ranges(int num_bodies, const Body* bodies, int num_points, int* world) {
    long long total = 0;
    for (int b = 0; b < num_bodies; ++b) {
        const long long first = bodies[b].first_point, n = bodies[b].num_points;
        if (n < 0) return fail(OCEAN_ERR_INVALID_ARGUMENT, "body %d: num_points %lld is negative", b, n);
        if (first < 0 || first + n > num_points)
            return fail(OCEAN_ERR_INVALID_ARGUMENT, "body %d: points [%lld, %lld) outside [0, %d)", b, first, first + n, num_points);
        total += n;
    }
    if (total > INT32_MAX) return fail(OCEAN_ERR_INVALID_ARGUMENT, "%lld world points exceed INT32_MAX", total);
    *world = (int)total;
    return OCEAN_OK;
}

// The checks both entry points make; *world receives the number of world points, the sum of the bodies' num_points.
int check_buoyancy_args(int num_bodies, const ocean_buoyancy_body* bodies, int num_points, float density, float tolerance,
                        int max_iterations, int* world) {
    int rc = check_surface_args(num_points, tolerance, max_iterations);
    if (rc) return rc;
    if (num_bodies < 0) return fail(OCEAN_ERR_INVALID_ARGUMENT, "num_bodies %d is negative", num_bodies);
    if (!finite_positive(density)) return fail(OCEAN_ERR_INVALID_ARGUMENT, "density %g is not finite and > 0", density);
    if (num_bodies > 0 && !bodies) return fail(OCEAN_ERR_INVALID_ARGUMENT, "bodies is NULL");
    return check_point_ranges(num_bodies, bodies, num_points, world);
}

// The exclusive prefix of count(b), body b's number of world points (hull points or mesh vertices), into
// gen->body.offsets_host, uploaded to gen->body.offsets.  The counts were validated: their sum fits an int.
extern "C++" template <typename Count>
int upload_offsets(ocean_generator* gen, int num_bodies, Count count) {
    std::vector<int>& offsets = gen->body.offsets_host;
    offsets.resize((size_t)num_bodies);
    for (int b = 0, start = 0; b < num_bodies; start += count(b), ++b) offsets[b] = start;
    OCEAN_CUDA(gen->body.offsets.upload(gen, offsets.data(), (size_t)num_bodies));
    return OCEAN_OK;
}

// The buoyancy launches on a body table and offsets already in device memory (bodies_dev may be written by earlier kernels on
// the stream), with the map scales in gen->q_scales and gen->body.q grown to `world`: samples receives the surface records, and
// wv_dev (may be null) the wake's vertical velocity of each world point while the wake coupling is live.  With queried > world
// the query also takes the points gen->body.q holds after the world points (written earlier on the stream).
int launch_buoyancy_sequence(ocean_generator* gen, const ocean_buoyancy_body* bodies_dev, const int* offsets_dev, int num_bodies, int world,
                             const ocean_buoyancy_point* points_dev, int num_cascades, float density, float tolerance, int max_iterations,
                             ocean_buoyancy_result* results_dev, ocean_surface_sample* samples, float* wv_dev = nullptr, int queried = -1) {
    int rc;
    if (queried < 0) queried = world;                   // more query points than world ones: the driven bodies' actuators
    if (world > 0) {
        OCEAN_CUDA(ocean::launch_buoyancy_transform(bodies_dev, offsets_dev, num_bodies, points_dev, world, gen->body.q.ptr, gen->stream));
        gen->kernel_launches += 1;
    }
    if (queried > 0)
        if ((rc = run_query_surface(gen, queried, gen->body.q.ptr, num_cascades, tolerance, max_iterations, samples, wv_dev))) return rc;
    const float rho_g = density * 9.81f;                                 // G, wave_generator.gd:5, in binary32
    OCEAN_CUDA(ocean::launch_buoyancy_reduce(bodies_dev, offsets_dev, num_bodies, points_dev, samples, rho_g, tolerance, results_dev,
                                             gen->stream));
    gen->kernel_launches += 1;
    return OCEAN_OK;
}

// The buoyancy launch sequence on validated arguments (num_bodies > 0), with the map scales already in gen->q_scales: the body
// table and offsets are uploaded to gen->body.poses / gen->body.offsets, and *samples_used receives the surface records
// (samples_dev, or gen->body.samples when samples_dev is NULL) for a drag pass on the same points.
int run_buoyancy(ocean_generator* gen, int num_bodies, const ocean_buoyancy_body* bodies_host, int world, const ocean_buoyancy_point* points_dev,
                 int num_cascades, float density, float tolerance, int max_iterations, ocean_buoyancy_result* results_dev,
                 ocean_surface_sample* samples_dev, ocean_surface_sample** samples_used, float* wv_dev = nullptr) {
    BodyScratch& sc = gen->body;
    int rc;
    OCEAN_CUDA(sc.q.grow(gen, (size_t)world));
    if (!samples_dev) OCEAN_CUDA(sc.samples.grow(gen, (size_t)world));
    ocean_surface_sample* samples = samples_dev ? samples_dev : sc.samples.ptr;
    OCEAN_CUDA(sc.poses.upload(gen, bodies_host, (size_t)num_bodies));
    if ((rc = upload_offsets(gen, num_bodies, [&](int b) { return bodies_host[b].num_points; }))) return rc;
    if ((rc = launch_buoyancy_sequence(gen, sc.poses.ptr, sc.offsets.ptr, num_bodies, world, points_dev, num_cascades, density, tolerance,
                                       max_iterations, results_dev, samples, wv_dev)))
        return rc;
    if (samples_used) *samples_used = samples;
    return OCEAN_OK;
}
}  // namespace

int ocean_buoyancy_device(ocean_generator* gen, int num_bodies, const ocean_buoyancy_body* bodies_host, int num_points,
                          const ocean_buoyancy_point* points_dev, int num_cascades, const float* map_scales_host, float density,
                          float tolerance, int max_iterations, ocean_buoyancy_result* results_dev, ocean_surface_sample* samples_dev) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    int world = 0;
    if ((rc = check_buoyancy_args(num_bodies, bodies_host, num_points, density, tolerance, max_iterations, &world))) return rc;
    if (num_bodies == 0) return OCEAN_OK;
    if (!results_dev || (world > 0 && !points_dev)) return fail(OCEAN_ERR_INVALID_ARGUMENT, "a device buffer is NULL");
    if ((rc = upload_scales(gen, num_cascades, map_scales_host))) return rc;
    return run_buoyancy(gen, num_bodies, bodies_host, world, points_dev, num_cascades, density, tolerance, max_iterations, results_dev,
                        samples_dev, nullptr);
}

int ocean_buoyancy(ocean_generator* gen, int num_bodies, const ocean_buoyancy_body* bodies_host, int num_points,
                   const ocean_buoyancy_point* points_host, int num_cascades, const float* map_scales_host, float density,
                   float tolerance, int max_iterations, ocean_buoyancy_result* results_host, ocean_surface_sample* samples_host) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    int world = 0;
    if ((rc = check_buoyancy_args(num_bodies, bodies_host, num_points, density, tolerance, max_iterations, &world))) return rc;
    if (num_bodies == 0) return OCEAN_OK;
    if (!results_host || (world > 0 && !points_host)) return fail(OCEAN_ERR_INVALID_ARGUMENT, "a host buffer is NULL");
    Staging st;
    const auto points = st.in(points_host, world > 0 ? (size_t)num_points : 0);
    const auto results = st.out(results_host, (size_t)num_bodies);
    const auto samples = st.out(samples_host, (size_t)world);
    if ((rc = st.upload(gen, kStageBuoyancy))) return rc;
    return st.finish(gen, ocean_buoyancy_device(gen, num_bodies, bodies_host, num_points, st[points], num_cascades, map_scales_host, density,
                                                tolerance, max_iterations, st[results], st[samples]));
}

// ---- velocity maps: the time derivative of the displacement map (ocean_velocity.cu; oracle_velocity_update) ----
namespace {
// Allocates the velocity buffers on first use, zeroed: a cascade whose maps were never written has a zero velocity layer.
// A binary32 tap created while the taps are on is filled by recomputing every layer that has a source.
int ensure_velocity(ocean_generator* gen) {
    const size_t n = (size_t)gen->num_cascades * gen->map_size * gen->map_size;
    if (!gen->vel_scratch.ptr) {
        OCEAN_CUDA(gen->vel_scratch.grow(gen, n));
        OCEAN_CUDA(ocean::init_velocity_twiddles(gen->twiddles.ptr, gen->stream));
    }
    if (!gen->velocity.ptr) {
        OCEAN_CUDA(gen->velocity.grow(gen, n));
        OCEAN_CUDA(cudaMemsetAsync(gen->velocity.ptr, 0, sizeof(uint2) * n, gen->stream));
    }
    if (gen->buf.displacement_f32 && !gen->velocity_f32.ptr) {
        OCEAN_CUDA(gen->velocity_f32.grow(gen, n));
        OCEAN_CUDA(cudaMemsetAsync(gen->velocity_f32.ptr, 0, sizeof(float4) * n, gen->stream));
        for (int i = 0; i < gen->num_cascades; ++i) gen->vel_stale[i] = gen->vel_has_source[i];
    }
    return OCEAN_OK;
}

// Recomputes every stale velocity layer in one launch sequence.
int refresh_velocity(ocean_generator* gen, int* recomputed) {
    int rc = ensure_velocity(gen);
    if (rc) return rc;
    std::vector<ocean::VelocityDispatch> jobs;
    for (int i = 0; i < gen->num_cascades; ++i)
        if (gen->vel_has_source[i] && gen->vel_stale[i]) jobs.push_back(gen->vel_source[i]);
    if (!jobs.empty()) {
        int launched = 0;
        OCEAN_CUDA(ocean::launch_velocity(gen->buf, jobs.data(), (int)jobs.size(), gen->vel_scratch.ptr, gen->velocity.ptr,
                                          gen->velocity_f32.ptr, gen->stream, &launched));
        gen->kernel_launches += (uint64_t)launched;
        for (const auto& j : jobs) gen->vel_stale[j.cascade] = 0;
    }
    if (recomputed) *recomputed = (int)jobs.size();
    return OCEAN_OK;
}
}  // namespace

int ocean_update_velocity(ocean_generator* gen, int* recomputed) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if (recomputed) *recomputed = 0;
    return refresh_velocity(gen, recomputed);
}

int ocean_get_velocity_map(ocean_generator* gen, void** velocity_dev, size_t* layer_bytes) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if ((rc = ensure_velocity(gen))) return rc;
    if (velocity_dev) *velocity_dev = gen->velocity.ptr;
    if (layer_bytes) *layer_bytes = sizeof(uint2) * (size_t)gen->map_size * gen->map_size;
    return OCEAN_OK;
}

int ocean_copy_velocity_to_host(ocean_generator* gen, int first, int count, void* velocity_host) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if ((rc = check_layer_range(gen, first, count))) return rc;
    if (count == 0) return OCEAN_OK;
    if (!velocity_host) return fail(OCEAN_ERR_INVALID_ARGUMENT, "velocity_host is NULL");
    if ((rc = refresh_velocity(gen, nullptr))) return rc;
    const size_t layer = (size_t)gen->map_size * gen->map_size;
    OCEAN_CUDA(cudaMemcpyAsync(velocity_host, gen->velocity.ptr + first * layer, sizeof(uint2) * layer * count, cudaMemcpyDeviceToHost, gen->stream));
    OCEAN_CUDA(cudaStreamSynchronize(gen->stream));
    return OCEAN_OK;
}

int ocean_copy_f32_velocity_to_host(ocean_generator* gen, int cascade, float* host) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if ((rc = check_cascade(gen, cascade))) return rc;
    if (!host) return fail(OCEAN_ERR_INVALID_ARGUMENT, "host is NULL");
    if (!gen->buf.displacement_f32) return fail(OCEAN_ERR_STATE, "binary32 taps are disabled; call ocean_enable_f32_taps(gen, 1) first");
    if ((rc = refresh_velocity(gen, nullptr))) return rc;
    const size_t layer = (size_t)gen->map_size * gen->map_size;
    OCEAN_CUDA(cudaMemcpyAsync(host, gen->velocity_f32.ptr + cascade * layer, sizeof(float4) * layer, cudaMemcpyDeviceToHost, gen->stream));
    OCEAN_CUDA(cudaStreamSynchronize(gen->stream));
    return OCEAN_OK;
}

int ocean_sample_velocity_device(ocean_generator* gen, int num_points, const float* points_xz_dev, int num_cascades, const float* map_scales_host,
                                 float* velocity_dev) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if (num_points < 0) return fail(OCEAN_ERR_INVALID_ARGUMENT, "num_points %d is negative", num_points);
    if (num_points == 0) return OCEAN_OK;
    if (!points_xz_dev || !velocity_dev) return fail(OCEAN_ERR_INVALID_ARGUMENT, "a device buffer is NULL");
    if ((rc = upload_scales(gen, num_cascades, map_scales_host))) return rc;       // validates before anything is launched
    if ((rc = refresh_velocity(gen, nullptr))) return rc;
    OCEAN_CUDA(ocean::launch_sample_velocity(gen->velocity.ptr, gen->map_size, num_cascades, reinterpret_cast<const float2*>(points_xz_dev),
                                             num_points, gen->q_scales.ptr, velocity_dev, gen->stream));
    gen->kernel_launches += 1;
    return OCEAN_OK;
}

int ocean_sample_velocity(ocean_generator* gen, int num_points, const float* points_xz_host, int num_cascades, const float* map_scales_host,
                          float* velocity_host) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if (num_points < 0) return fail(OCEAN_ERR_INVALID_ARGUMENT, "num_points %d is negative", num_points);
    if (num_points == 0) return OCEAN_OK;
    if (!points_xz_host || !velocity_host) return fail(OCEAN_ERR_INVALID_ARGUMENT, "a host buffer is NULL");
    Staging st;
    const auto points = st.in(points_xz_host, 2 * (size_t)num_points);
    const auto velocity = st.out(velocity_host, 3 * (size_t)num_points);
    if ((rc = st.upload(gen, kStageSampleVelocity))) return rc;
    return st.finish(gen, ocean_sample_velocity_device(gen, num_points, st[points], num_cascades, map_scales_host, st[velocity]));
}

// ---- body forces: buoyancy plus quadratic drag against the water velocity, from one surface query (oracle/drag.py) ----
static_assert(sizeof(ocean_body_velocity) == 24, "ocean_body_velocity layout");
static_assert(sizeof(ocean_drag_result) == 32, "ocean_drag_result layout");

namespace {
// ocean_buoyancy's checks plus the body velocities and drag areas; *world as for check_buoyancy_args.
int check_body_forces_args(int num_bodies, const ocean_buoyancy_body* bodies, const ocean_body_velocity* velocities, int num_points,
                           const float* drag_areas, float density, float tolerance, int max_iterations, int* world) {
    int rc = check_buoyancy_args(num_bodies, bodies, num_points, density, tolerance, max_iterations, world);
    if (rc) return rc;
    if (num_bodies > 0 && !velocities) return fail(OCEAN_ERR_INVALID_ARGUMENT, "velocities is NULL");
    if (*world > 0 && !drag_areas) return fail(OCEAN_ERR_INVALID_ARGUMENT, "drag_areas is NULL");
    return OCEAN_OK;
}
}  // namespace

int ocean_body_forces_device(ocean_generator* gen, int num_bodies, const ocean_buoyancy_body* bodies_host,
                             const ocean_body_velocity* velocities_host, int num_points, const ocean_buoyancy_point* points_dev,
                             const float* drag_areas_dev, int num_cascades, const float* map_scales_host, float density, float tolerance,
                             int max_iterations, ocean_buoyancy_result* hydrostatic_dev, ocean_drag_result* drag_dev,
                             ocean_surface_sample* samples_dev) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    int world = 0;
    if ((rc = check_body_forces_args(num_bodies, bodies_host, velocities_host, num_points, drag_areas_dev, density, tolerance, max_iterations,
                                     &world)))
        return rc;
    if (num_bodies == 0) return OCEAN_OK;
    if (!hydrostatic_dev || !drag_dev || (world > 0 && !points_dev)) return fail(OCEAN_ERR_INVALID_ARGUMENT, "a device buffer is NULL");
    if ((rc = upload_scales(gen, num_cascades, map_scales_host))) return rc;       // the last check: nothing is launched before it
    if ((rc = refresh_velocity(gen, nullptr))) return rc;
    BodyScratch& sc = gen->body;
    OCEAN_CUDA(sc.velocities.upload(gen, velocities_host, (size_t)num_bodies));
    float* wv = nullptr;
    OCEAN_CUDA(gen->wake.vertical_velocities(gen, (size_t)world, &wv));
    ocean_surface_sample* samples = nullptr;
    if ((rc = run_buoyancy(gen, num_bodies, bodies_host, world, points_dev, num_cascades, density, tolerance, max_iterations, hydrostatic_dev,
                           samples_dev, &samples, wv)))
        return rc;
    const float half_rho = 0.5f * density;
    OCEAN_CUDA(ocean::launch_drag_reduce(sc.poses.ptr, sc.velocities.ptr, sc.offsets.ptr, num_bodies, points_dev, drag_areas_dev, samples,
                                         gen->velocity.ptr, gen->map_size, num_cascades, gen->q_scales.ptr, half_rho, drag_dev, wv, gen->stream));
    gen->kernel_launches += 1;
    return OCEAN_OK;
}

int ocean_body_forces(ocean_generator* gen, int num_bodies, const ocean_buoyancy_body* bodies_host, const ocean_body_velocity* velocities_host,
                      int num_points, const ocean_buoyancy_point* points_host, const float* drag_areas_host, int num_cascades,
                      const float* map_scales_host, float density, float tolerance, int max_iterations, ocean_buoyancy_result* hydrostatic_host,
                      ocean_drag_result* drag_host, ocean_surface_sample* samples_host) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    int world = 0;
    if ((rc = check_body_forces_args(num_bodies, bodies_host, velocities_host, num_points, drag_areas_host, density, tolerance, max_iterations,
                                     &world)))
        return rc;
    if (num_bodies == 0) return OCEAN_OK;
    if (!hydrostatic_host || !drag_host || (world > 0 && !points_host)) return fail(OCEAN_ERR_INVALID_ARGUMENT, "a host buffer is NULL");
    const size_t P = world > 0 ? (size_t)num_points : 0, B = (size_t)num_bodies;
    Staging st;
    const auto points = st.in(points_host, P);
    const auto areas = st.in(drag_areas_host, P);
    const auto hydrostatic = st.out(hydrostatic_host, B);
    const auto drag = st.out(drag_host, B);
    const auto samples = st.out(samples_host, (size_t)world);
    if ((rc = st.upload(gen, kStageBodyForces))) return rc;
    return st.finish(gen, ocean_body_forces_device(gen, num_bodies, bodies_host, velocities_host, num_points, st[points], st[areas],
                                                   num_cascades, map_scales_host, density, tolerance, max_iterations, st[hydrostatic],
                                                   st[drag], st[samples]));
}

// ---- floating bodies: sub-stepped buoyancy and drag with the body state on the device (ocean_bodies.cu; oracle/bodies.py) ----
static_assert(sizeof(ocean_floating_body) == 24, "ocean_floating_body layout");
static_assert(sizeof(ocean_body_state) == 52, "ocean_body_state layout");

namespace {
// The integrators' density, dt and substeps.
int check_step_args(float density, float dt, int substeps) {
    if (!finite_positive(density)) return fail(OCEAN_ERR_INVALID_ARGUMENT, "density %g is not finite and > 0", density);
    if (!finite_positive(dt)) return fail(OCEAN_ERR_INVALID_ARGUMENT, "dt %g is not finite and > 0", dt);
    if (substeps < 1 || substeps > 64) return fail(OCEAN_ERR_INVALID_ARGUMENT, "substeps %d outside [1, 64]", substeps);
    return OCEAN_OK;
}

// Each body's mass and principal inertia (ocean_floating_body or ocean_floating_hull rows).
extern "C++" template <typename Row>
int check_mass_inertia(int num_bodies, const Row* bodies) {
    for (int b = 0; b < num_bodies; ++b) {
        const Row& fb = bodies[b];
        if (!finite_positive(fb.mass)) return fail(OCEAN_ERR_INVALID_ARGUMENT, "body %d: mass %g is not finite and > 0", b, fb.mass);
        for (int k = 0; k < 3; ++k)
            if (!finite_positive(fb.inertia[k]))
                return fail(OCEAN_ERR_INVALID_ARGUMENT, "body %d: inertia[%d] %g is not finite and > 0", b, k, fb.inertia[k]);
    }
    return OCEAN_OK;
}

// ocean_body_forces' checks on the floating bodies, plus mass, inertia, dt, substeps and the states; *world as for
// check_buoyancy_args.
int check_simulate_args(int num_bodies, const ocean_floating_body* bodies, const ocean_body_state* states, int num_points,
                        const float* drag_areas, float density, float dt, int substeps, float tolerance, int max_iterations, int* world) {
    int rc = check_surface_args(num_points, tolerance, max_iterations);
    if (rc) return rc;
    if (num_bodies < 0) return fail(OCEAN_ERR_INVALID_ARGUMENT, "num_bodies %d is negative", num_bodies);
    if ((rc = check_step_args(density, dt, substeps))) return rc;
    if (num_bodies > 0 && !bodies) return fail(OCEAN_ERR_INVALID_ARGUMENT, "bodies is NULL");
    if (num_bodies > 0 && !states) return fail(OCEAN_ERR_INVALID_ARGUMENT, "states is NULL");
    if ((rc = check_mass_inertia(num_bodies, bodies))) return rc;
    if ((rc = check_point_ranges(num_bodies, bodies, num_points, world))) return rc;
    if (*world > 0 && !drag_areas) return fail(OCEAN_ERR_INVALID_ARGUMENT, "drag_areas is NULL");
    return OCEAN_OK;
}

// The drive arguments of ocean_simulate_driven_bodies[_device] (host arrays), as validated by check_drive_args.
struct DriveHost {
    int num_thrusters = 0;
    const ocean_thruster* thrusters = nullptr;
    int num_foils = 0;
    const ocean_foil* foils = nullptr;
    const ocean_body_load* loads = nullptr;
    int num_tethers = 0;
    const ocean_tether* tethers = nullptr;
    int actuators() const { return num_thrusters + num_foils; }
    bool any() const { return num_thrusters > 0 || num_foils > 0 || num_tethers > 0 || loads; }
};

// The counts and arrays, the body indices, and the foil areas and tether constants that enter the stability bound; the world
// points plus the actuators must stay below 2^31 (one surface query takes them all).
int check_drive_args(int num_bodies, int world, const DriveHost& d) {
    if (d.num_thrusters < 0 || d.num_foils < 0 || d.num_tethers < 0)
        return fail(OCEAN_ERR_INVALID_ARGUMENT, "a count is negative (thrusters %d, foils %d, tethers %d)", d.num_thrusters, d.num_foils,
                    d.num_tethers);
    if ((d.num_thrusters > 0 && !d.thrusters) || (d.num_foils > 0 && !d.foils) || (d.num_tethers > 0 && !d.tethers))
        return fail(OCEAN_ERR_INVALID_ARGUMENT, "an actuator or tether array is NULL");
    if ((long long)world + d.num_thrusters + d.num_foils > 2147483647LL)
        return fail(OCEAN_ERR_INVALID_ARGUMENT, "world points plus actuators exceed 2^31 - 1");
    for (int k = 0; k < d.num_thrusters; ++k)
        if (d.thrusters[k].body < 0 || d.thrusters[k].body >= num_bodies)
            return fail(OCEAN_ERR_INVALID_ARGUMENT, "thruster %d: body %d outside [0, %d)", k, d.thrusters[k].body, num_bodies);
    for (int k = 0; k < d.num_foils; ++k) {
        const ocean_foil& f = d.foils[k];
        if (f.body < 0 || f.body >= num_bodies) return fail(OCEAN_ERR_INVALID_ARGUMENT, "foil %d: body %d outside [0, %d)", k, f.body, num_bodies);
        if (!finite_nonnegative(f.area)) return fail(OCEAN_ERR_INVALID_ARGUMENT, "foil %d: area %g is not finite and >= 0", k, f.area);
    }
    for (int k = 0; k < d.num_tethers; ++k) {
        const ocean_tether& t = d.tethers[k];
        if (t.body_a < 0 || t.body_a >= num_bodies)
            return fail(OCEAN_ERR_INVALID_ARGUMENT, "tether %d: body_a %d outside [0, %d)", k, t.body_a, num_bodies);
        if (t.body_b != -1 && (t.body_b < 0 || t.body_b >= num_bodies || t.body_b == t.body_a))
            return fail(OCEAN_ERR_INVALID_ARGUMENT, "tether %d: body_b %d is not -1 or another body", k, t.body_b);
        if (!finite_nonnegative(t.rest_length) || !finite_nonnegative(t.stiffness) || !finite_nonnegative(t.damping))
            return fail(OCEAN_ERR_INVALID_ARGUMENT, "tether %d: rest_length, stiffness and damping must be finite and >= 0", k);
    }
    return OCEAN_OK;
}

// The by-body incidence list into gen->body.incidence_host: [num_bodies + 1] offsets, then per body its thrusters, foils
// and tether ends in array order (thruster k -> k, foil k -> T + k, end e of tether k -> T + F + 2 k + e).
void build_incidence(ocean_generator* gen, int num_bodies, const DriveHost& d) {
    const size_t B = (size_t)num_bodies;
    std::vector<int>& v = gen->body.incidence_host;
    const size_t entries = (size_t)d.actuators() + 2 * (size_t)d.num_tethers;
    v.assign(B + 1 + entries, 0);
    int* off = v.data();
    int* list = off + B + 1;
    for (int k = 0; k < d.num_thrusters; ++k) off[d.thrusters[k].body + 1] += 1;
    for (int k = 0; k < d.num_foils; ++k) off[d.foils[k].body + 1] += 1;
    for (int k = 0; k < d.num_tethers; ++k) {
        off[d.tethers[k].body_a + 1] += 1;
        if (d.tethers[k].body_b >= 0) off[d.tethers[k].body_b + 1] += 1;
    }
    for (size_t b = 0; b < B; ++b) off[b + 1] += off[b];
    std::vector<int> next(off, off + B);
    const int T = d.num_thrusters, F = d.num_foils;
    for (int k = 0; k < T; ++k) list[next[d.thrusters[k].body]++] = k;
    for (int k = 0; k < F; ++k) list[next[d.foils[k].body]++] = T + k;
    for (int k = 0; k < d.num_tethers; ++k) {
        list[next[d.tethers[k].body_a]++] = T + F + 2 * k;
        if (d.tethers[k].body_b >= 0) list[next[d.tethers[k].body_b]++] = T + F + 2 * k + 1;
    }
    v.resize(B + 1 + (size_t)off[B]);                   // anchored tethers have one end
}

int launch_hull_sequence(ocean_generator* gen, const ocean_hull_body* poses_dev, const ocean_body_velocity* velocities_dev, int num_bodies,
                         int world, int num_cascades, float density, float tolerance, int max_iterations, ocean_buoyancy_result* hydrostatic_dev,
                         ocean_drag_result* drag_dev, ocean_surface_sample* samples, float* wv);      // with the hull meshes, below

// The body integrator after an entry point's checks (num_bodies > 0, scales uploaded).  Row is the hull: ocean_floating_body
// rows on the hull points points_dev with drag_areas_dev, or ocean_floating_hull rows on the registered meshes (points_dev and
// drag_areas_dev unused).  With drive null the plain integrator runs; with drive (drive->any(), its arrays validated) the
// driven one, drive_dev / tensions_dev the outputs or null.  Every sub-step runs the hull's force sequence on the current
// poses, then the integrator, which writes transforms_dev on the last one.
extern "C++" template <typename Row>
int run_simulate(ocean_generator* gen, int num_bodies, const Row* bodies_host, ocean_body_state* states_dev, int world,
                 const ocean_buoyancy_point* points_dev, const float* drag_areas_dev, int num_cascades, float density, float dt, int substeps,
                 float tolerance, int max_iterations, ocean_buoyancy_result* hydrostatic_dev, ocean_drag_result* drag_dev,
                 float* transforms_dev, const DriveHost* drive = nullptr, ocean_drive_result* drive_dev = nullptr, float* tensions_dev = nullptr) {
    constexpr bool kMesh = std::is_same<Row, ocean_floating_hull>::value;
    BodyScratch& sc = gen->body;
    int rc;
    if ((rc = refresh_velocity(gen, nullptr))) return rc;
    const size_t B = (size_t)num_bodies;
    const int actuators = drive ? drive->actuators() : 0;
    const int queried = world + actuators;              // the hull's world points, then the actuators'
    OCEAN_CUDA(sc.r2.grow(gen, B));
    OCEAN_CUDA(sc.velocities.grow(gen, B));
    OCEAN_CUDA(sc.q.grow(gen, (size_t)queried));
    OCEAN_CUDA(sc.samples.grow(gen, (size_t)queried));
    if constexpr (kMesh) {
        OCEAN_CUDA(sc.hull_poses.grow(gen, B));
        OCEAN_CUDA(sc.rows.grow(gen, B));
        OCEAN_CUDA(sc.corners.grow(gen, 2 * (size_t)world));
    } else {
        OCEAN_CUDA(sc.poses.grow(gen, B));
    }
    float* wv = nullptr;                                // every sub-step reads the same snapshots
    OCEAN_CUDA(gen->wake.vertical_velocities(gen, (size_t)queried, &wv));
    ocean::DriveArgs da{};
    if (drive) {
        da.num_thrusters = drive->num_thrusters;
        da.num_foils = drive->num_foils;
        da.num_tethers = drive->num_tethers;
        if (drive->num_thrusters > 0) {
            OCEAN_CUDA(sc.thrusters.upload(gen, drive->thrusters, (size_t)drive->num_thrusters));
            da.thrusters = sc.thrusters.ptr;
        }
        if (drive->num_foils > 0) {
            OCEAN_CUDA(sc.foils.upload(gen, drive->foils, (size_t)drive->num_foils));
            da.foils = sc.foils.ptr;
        }
        if (drive->num_tethers > 0) {
            OCEAN_CUDA(sc.tethers.upload(gen, drive->tethers, (size_t)drive->num_tethers));
            OCEAN_CUDA(sc.tether_forces.grow(gen, (size_t)drive->num_tethers));
            da.tethers = sc.tethers.ptr;
            if (!tensions_dev) {
                OCEAN_CUDA(sc.tensions.grow(gen, (size_t)drive->num_tethers));
                tensions_dev = sc.tensions.ptr;
            }
        }
        if (drive->loads) {
            OCEAN_CUDA(sc.loads.upload(gen, drive->loads, B));
            da.loads = sc.loads.ptr;
        }
        build_incidence(gen, num_bodies, *drive);
        OCEAN_CUDA(sc.incidence.upload(gen, sc.incidence_host.data(), sc.incidence_host.size()));
        da.incidence_offsets = sc.incidence.ptr;
        da.incidence = sc.incidence.ptr + B + 1;
        OCEAN_CUDA(sc.sums.grow(gen, B));
        if (!drive_dev) {
            OCEAN_CUDA(sc.drive.grow(gen, B));
            drive_dev = sc.drive.ptr;
        }
    }
    if (!hydrostatic_dev) {
        OCEAN_CUDA(sc.hydrostatic.grow(gen, B));
        hydrostatic_dev = sc.hydrostatic.ptr;
    }
    if (!drag_dev) {
        OCEAN_CUDA(sc.drag.grow(gen, B));
        drag_dev = sc.drag.ptr;
    }
    if constexpr (kMesh) {
        OCEAN_CUDA(sc.hull_rows.upload(gen, bodies_host, B));
        if ((rc = upload_offsets(gen, num_bodies, [&](int b) { return sc.meshes_host[bodies_host[b].mesh].num_vertices; }))) return rc;
        OCEAN_CUDA(ocean::launch_hull_prepare(sc.hull_rows.ptr, states_dev, num_bodies, sc.meshes.ptr, sc.vertices.ptr, sc.r2.ptr,
                                              sc.hull_poses.ptr, sc.velocities.ptr, sc.rows.ptr, gen->stream));
    } else {
        OCEAN_CUDA(sc.rows.upload(gen, bodies_host, B));
        if ((rc = upload_offsets(gen, num_bodies, [&](int b) { return bodies_host[b].num_points; }))) return rc;
        OCEAN_CUDA(ocean::launch_bodies_prepare(sc.rows.ptr, states_dev, num_bodies, points_dev, sc.r2.ptr, sc.poses.ptr, sc.velocities.ptr,
                                                gen->stream));
    }
    gen->kernel_launches += 1;
    const ocean_floating_body* bodies = sc.rows.ptr;
    ocean_body_velocity* velocities = sc.velocities.ptr;
    // the pose rows the integrators write: k_bodies_integrate writes a mesh hull's rows as ocean_buoyancy_body rows
    ocean_buoyancy_body* poses = kMesh ? reinterpret_cast<ocean_buoyancy_body*>(sc.hull_poses.ptr) : sc.poses.ptr;
    const float h = dt / (float)substeps;
    const float half_rho = 0.5f * density;
    for (int s = 0; s < substeps; ++s) {
        float* transforms = s == substeps - 1 ? transforms_dev : nullptr;
        if constexpr (kMesh) {
            if ((rc = launch_hull_sequence(gen, sc.hull_poses.ptr, velocities, num_bodies, world, num_cascades, density, tolerance,
                                           max_iterations, hydrostatic_dev, drag_dev, sc.samples.ptr, wv)))
                return rc;
        } else {
            if (actuators > 0) {
                OCEAN_CUDA(ocean::launch_actuator_transform(da, poses, sc.q.ptr + world, gen->stream));
                gen->kernel_launches += 1;
            }
            if ((rc = launch_buoyancy_sequence(gen, poses, sc.offsets.ptr, num_bodies, world, points_dev, num_cascades, density, tolerance,
                                               max_iterations, hydrostatic_dev, sc.samples.ptr, wv, queried)))
                return rc;
            OCEAN_CUDA(ocean::launch_drag_reduce(poses, velocities, sc.offsets.ptr, num_bodies, points_dev, drag_areas_dev, sc.samples.ptr,
                                                 gen->velocity.ptr, gen->map_size, num_cascades, gen->q_scales.ptr, half_rho, drag_dev, wv,
                                                 gen->stream));
            gen->kernel_launches += 1;
        }
        if (!drive) {
            OCEAN_CUDA(ocean::launch_bodies_integrate(bodies, sc.r2.ptr, num_bodies, hydrostatic_dev, drag_dev, density, h, states_dev, poses,
                                                      velocities, transforms, gen->stream));
            gen->kernel_launches += 1;
            continue;
        }
        if (da.num_tethers > 0) {
            OCEAN_CUDA(ocean::launch_tethers(da, poses, velocities, sc.tether_forces.ptr, tensions_dev, gen->stream));
            gen->kernel_launches += 1;
        }
        OCEAN_CUDA(ocean::launch_drive_reduce(da, num_bodies, bodies, sc.r2.ptr, poses, velocities, hydrostatic_dev, drag_dev,
                                              sc.samples.ptr + world, wv ? wv + world : nullptr, sc.tether_forces.ptr, gen->velocity.ptr,
                                              gen->map_size, num_cascades, gen->q_scales.ptr, density, h, sc.sums.ptr, drive_dev, gen->stream));
        OCEAN_CUDA(ocean::launch_bodies_integrate_driven(bodies, num_bodies, sc.sums.ptr, h, states_dev, poses, velocities, transforms,
                                                         gen->stream));
        gen->kernel_launches += 2;
    }
    return OCEAN_OK;
}
}  // namespace

int ocean_simulate_bodies_device(ocean_generator* gen, int num_bodies, const ocean_floating_body* bodies_host, ocean_body_state* states_dev,
                                 int num_points, const ocean_buoyancy_point* points_dev, const float* drag_areas_dev, int num_cascades,
                                 const float* map_scales_host, float density, float dt, int substeps, float tolerance, int max_iterations,
                                 ocean_buoyancy_result* hydrostatic_dev, ocean_drag_result* drag_dev, float* transforms_dev) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    int world = 0;
    if ((rc = check_simulate_args(num_bodies, bodies_host, states_dev, num_points, drag_areas_dev, density, dt, substeps, tolerance,
                                  max_iterations, &world)))
        return rc;
    if (num_bodies == 0) return OCEAN_OK;
    if (world > 0 && !points_dev) return fail(OCEAN_ERR_INVALID_ARGUMENT, "a device buffer is NULL");
    if ((rc = upload_scales(gen, num_cascades, map_scales_host))) return rc;       // the last check: nothing is launched before it
    return run_simulate(gen, num_bodies, bodies_host, states_dev, world, points_dev, drag_areas_dev, num_cascades, density, dt, substeps,
                        tolerance, max_iterations, hydrostatic_dev, drag_dev, transforms_dev);
}

int ocean_simulate_bodies(ocean_generator* gen, int num_bodies, const ocean_floating_body* bodies_host, ocean_body_state* states_host,
                          int num_points, const ocean_buoyancy_point* points_host, const float* drag_areas_host, int num_cascades,
                          const float* map_scales_host, float density, float dt, int substeps, float tolerance, int max_iterations,
                          ocean_buoyancy_result* hydrostatic_host, ocean_drag_result* drag_host, float* transforms_host) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    int world = 0;
    if ((rc = check_simulate_args(num_bodies, bodies_host, states_host, num_points, drag_areas_host, density, dt, substeps, tolerance,
                                  max_iterations, &world)))
        return rc;
    if (num_bodies == 0) return OCEAN_OK;
    if (world > 0 && !points_host) return fail(OCEAN_ERR_INVALID_ARGUMENT, "a host buffer is NULL");
    const size_t P = world > 0 ? (size_t)num_points : 0, B = (size_t)num_bodies;
    Staging st;                                         // an output not asked for stays NULL: the twin uses its own
    const auto points = st.in(points_host, P);
    const auto areas = st.in(drag_areas_host, P);
    const auto states = st.inout(states_host, B);
    const auto hydrostatic = st.out(hydrostatic_host, B);
    const auto drag = st.out(drag_host, B);
    const auto transforms = st.out(transforms_host, 12 * B);
    if ((rc = st.upload(gen, kStageSimulateBodies))) return rc;
    return st.finish(gen, ocean_simulate_bodies_device(gen, num_bodies, bodies_host, st[states], num_points, st[points], st[areas],
                                                       num_cascades, map_scales_host, density, dt, substeps, tolerance, max_iterations,
                                                       st[hydrostatic], st[drag], st[transforms]));
}

// ---- driven and moored bodies: thrusters, foils, loads and tethers in the integrator (ocean_drive.cu; oracle/drive.py) ----
static_assert(sizeof(ocean_thruster) == 36 && sizeof(ocean_foil) == 36, "actuator layouts");
static_assert(sizeof(ocean_body_load) == 24 && sizeof(ocean_tether) == 44 && sizeof(ocean_drive_result) == 32, "drive record layouts");

int ocean_simulate_driven_bodies_device(ocean_generator* gen, int num_bodies, const ocean_floating_body* bodies_host,
                                        ocean_body_state* states_dev, int num_points, const ocean_buoyancy_point* points_dev,
                                        const float* drag_areas_dev, int num_cascades, const float* map_scales_host, float density, float dt,
                                        int substeps, float tolerance, int max_iterations, int num_thrusters, const ocean_thruster* thrusters_host,
                                        int num_foils, const ocean_foil* foils_host, const ocean_body_load* loads_host, int num_tethers,
                                        const ocean_tether* tethers_host, ocean_buoyancy_result* hydrostatic_dev, ocean_drag_result* drag_dev,
                                        ocean_drive_result* drive_dev, float* tensions_dev, float* transforms_dev) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    int world = 0;
    if ((rc = check_simulate_args(num_bodies, bodies_host, states_dev, num_points, drag_areas_dev, density, dt, substeps, tolerance,
                                  max_iterations, &world)))
        return rc;
    const DriveHost drive{num_thrusters, thrusters_host, num_foils, foils_host, num_bodies > 0 ? loads_host : nullptr, num_tethers, tethers_host};
    if ((rc = check_drive_args(num_bodies, world, drive))) return rc;
    if (num_bodies == 0) return OCEAN_OK;
    if (world > 0 && !points_dev) return fail(OCEAN_ERR_INVALID_ARGUMENT, "a device buffer is NULL");
    if ((rc = upload_scales(gen, num_cascades, map_scales_host))) return rc;       // the last check: nothing is launched before it
    if (!drive.any() && drive_dev)                      // ocean_simulate_bodies, with a zero drive record
        OCEAN_CUDA(cudaMemsetAsync(drive_dev, 0, sizeof(ocean_drive_result) * (size_t)num_bodies, gen->stream));
    return run_simulate(gen, num_bodies, bodies_host, states_dev, world, points_dev, drag_areas_dev, num_cascades, density, dt, substeps,
                        tolerance, max_iterations, hydrostatic_dev, drag_dev, transforms_dev, drive.any() ? &drive : nullptr, drive_dev,
                        tensions_dev);
}

int ocean_simulate_driven_bodies(ocean_generator* gen, int num_bodies, const ocean_floating_body* bodies_host, ocean_body_state* states_host,
                                 int num_points, const ocean_buoyancy_point* points_host, const float* drag_areas_host, int num_cascades,
                                 const float* map_scales_host, float density, float dt, int substeps, float tolerance, int max_iterations,
                                 int num_thrusters, const ocean_thruster* thrusters_host, int num_foils, const ocean_foil* foils_host,
                                 const ocean_body_load* loads_host, int num_tethers, const ocean_tether* tethers_host,
                                 ocean_buoyancy_result* hydrostatic_host, ocean_drag_result* drag_host, ocean_drive_result* drive_host,
                                 float* tensions_host, float* transforms_host) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    int world = 0;
    if ((rc = check_simulate_args(num_bodies, bodies_host, states_host, num_points, drag_areas_host, density, dt, substeps, tolerance,
                                  max_iterations, &world)))
        return rc;
    const DriveHost drive{num_thrusters, thrusters_host, num_foils, foils_host, num_bodies > 0 ? loads_host : nullptr, num_tethers, tethers_host};
    if ((rc = check_drive_args(num_bodies, world, drive))) return rc;
    if (num_bodies == 0) return OCEAN_OK;
    if (world > 0 && !points_host) return fail(OCEAN_ERR_INVALID_ARGUMENT, "a host buffer is NULL");
    const size_t P = world > 0 ? (size_t)num_points : 0, B = (size_t)num_bodies;
    Staging st;                                         // an output not asked for stays NULL: the twin uses its own
    const auto points = st.in(points_host, P);
    const auto areas = st.in(drag_areas_host, P);
    const auto states = st.inout(states_host, B);
    const auto hydrostatic = st.out(hydrostatic_host, B);
    const auto drag = st.out(drag_host, B);
    const auto drive_out = st.out(drive_host, B);
    const auto tensions = st.out(tensions_host, (size_t)num_tethers);
    const auto transforms = st.out(transforms_host, 12 * B);
    if ((rc = st.upload(gen, kStageDrivenBodies))) return rc;
    return st.finish(gen, ocean_simulate_driven_bodies_device(gen, num_bodies, bodies_host, st[states], num_points, st[points], st[areas],
                                                              num_cascades, map_scales_host, density, dt, substeps, tolerance, max_iterations,
                                                              num_thrusters, thrusters_host, num_foils, foils_host, loads_host, num_tethers,
                                                              tethers_host, st[hydrostatic], st[drag], st[drive_out], st[tensions],
                                                              st[transforms]));
}

// ---- hull meshes: pressure and drag integrated over the wetted triangles (ocean_hull.cu; oracle/hull.py) ----
static_assert(sizeof(ocean_hull_mesh) == 24 && sizeof(ocean_hull_body) == 56 && sizeof(ocean_floating_hull) == 20, "hull record layouts");
static_assert(offsetof(ocean_hull_body, transform) == offsetof(ocean_buoyancy_body, transform) && sizeof(ocean_hull_body) == sizeof(ocean_buoyancy_body),
              "k_bodies_integrate writes hull pose rows as ocean_buoyancy_body rows");

namespace {
// Every check of ocean_hull_set_meshes, on the host, before anything is uploaded; volumes (may be null) receives each mesh's
// signed volume, sum over its triangles of p0 . (p2 x p1) / 6 in binary64 (Godot's clockwise winding: positive when closed
// and wound outward).
int check_hull_meshes(int num_meshes, const ocean_hull_mesh* meshes, int num_vertices, const float* vertices, int num_triangles,
                      const int32_t* triangles, float* volumes) {
    constexpr int kMaxElements = INT32_MAX / 3;         // 3 * index stays an int32
    if (num_meshes < 0 || num_vertices < 0 || num_triangles < 0)
        return fail(OCEAN_ERR_INVALID_ARGUMENT, "a count is negative (meshes %d, vertices %d, triangles %d)", num_meshes, num_vertices,
                    num_triangles);
    if (num_vertices > kMaxElements || num_triangles > kMaxElements)
        return fail(OCEAN_ERR_INVALID_ARGUMENT, "%d vertices or %d triangles above (2^31 - 1) / 3", num_vertices, num_triangles);
    if ((num_meshes > 0 && !meshes) || (num_vertices > 0 && !vertices) || (num_triangles > 0 && !triangles))
        return fail(OCEAN_ERR_INVALID_ARGUMENT, "an array is NULL where its count is positive");
    for (size_t k = 0; k < 3 * (size_t)num_vertices; ++k)
        if (!std::isfinite(vertices[k])) return fail(OCEAN_ERR_INVALID_ARGUMENT, "vertex %zu is not finite", k / 3);
    for (int m = 0; m < num_meshes; ++m) {
        const ocean_hull_mesh& h = meshes[m];
        const long long fv = h.first_vertex, nv = h.num_vertices, ft = h.first_triangle, nt = h.num_triangles;
        if (nv < 0 || fv < 0 || fv + nv > num_vertices)
            return fail(OCEAN_ERR_INVALID_ARGUMENT, "mesh %d: vertices [%lld, %lld) outside [0, %d)", m, fv, fv + nv, num_vertices);
        if (nt < 0 || ft < 0 || ft + nt > num_triangles)
            return fail(OCEAN_ERR_INVALID_ARGUMENT, "mesh %d: triangles [%lld, %lld) outside [0, %d)", m, ft, ft + nt, num_triangles);
        if (!finite_nonnegative(h.normal_drag) || !finite_nonnegative(h.tangential_drag))
            return fail(OCEAN_ERR_INVALID_ARGUMENT, "mesh %d: drag coefficients %g, %g are not finite and >= 0", m, h.normal_drag,
                        h.tangential_drag);
        const int32_t* tri = triangles + 3 * ft;
        for (long long k = 0; k < 3 * nt; ++k)
            if (tri[k] < 0 || tri[k] >= nv)
                return fail(OCEAN_ERR_INVALID_ARGUMENT, "mesh %d: triangle %lld index %d outside [0, %lld)", m, k / 3, tri[k], nv);
    }
    if (!volumes) return OCEAN_OK;
    for (int m = 0; m < num_meshes; ++m) {
        const ocean_hull_mesh& h = meshes[m];
        const float* p = vertices + 3 * (size_t)h.first_vertex;
        const int32_t* tri = triangles + 3 * (size_t)h.first_triangle;
        double v = 0.0;
        for (int j = 0; j < h.num_triangles; ++j) {
            const float* a = p + 3 * (size_t)tri[3 * j];
            const float* b = p + 3 * (size_t)tri[3 * j + 1];
            const float* c = p + 3 * (size_t)tri[3 * j + 2];
            const double cx = (double)c[1] * b[2] - (double)c[2] * b[1];
            const double cy = (double)c[2] * b[0] - (double)c[0] * b[2];
            const double cz = (double)c[0] * b[1] - (double)c[1] * b[0];
            v += (double)a[0] * cx + (double)a[1] * cy + (double)a[2] * cz;
        }
        volumes[m] = (float)(v / 6.0);
    }
    return OCEAN_OK;
}

// The bodies' mesh indices against the registered set; *world receives the number of world vertices.
extern "C++" template <typename Row>
int check_hull_bodies(const ocean_generator* gen, int num_bodies, const Row* bodies, int* world) {
    if (num_bodies < 0) return fail(OCEAN_ERR_INVALID_ARGUMENT, "num_bodies %d is negative", num_bodies);
    if (num_bodies > 0 && !bodies) return fail(OCEAN_ERR_INVALID_ARGUMENT, "bodies is NULL");
    const std::vector<ocean_hull_mesh>& set = gen->body.meshes_host;
    const int meshes = (int)set.size();
    if (num_bodies > 0 && meshes == 0) return fail(OCEAN_ERR_INVALID_ARGUMENT, "no hull meshes are registered (ocean_hull_set_meshes)");
    long long total = 0;
    for (int b = 0; b < num_bodies; ++b) {
        if (bodies[b].mesh < 0 || bodies[b].mesh >= meshes)
            return fail(OCEAN_ERR_INVALID_ARGUMENT, "body %d: mesh %d outside [0, %d)", b, bodies[b].mesh, meshes);
        total += set[bodies[b].mesh].num_vertices;
    }
    if (total > INT32_MAX) return fail(OCEAN_ERR_INVALID_ARGUMENT, "%lld world vertices exceed INT32_MAX", total);
    *world = (int)total;
    return OCEAN_OK;
}

int check_hull_forces_args(const ocean_generator* gen, int num_bodies, const ocean_hull_body* bodies, const ocean_body_velocity* velocities,
                           float density, float tolerance, int max_iterations, int* world) {
    int rc = check_solver_args(tolerance, max_iterations);
    if (rc) return rc;
    if (!finite_positive(density)) return fail(OCEAN_ERR_INVALID_ARGUMENT, "density %g is not finite and > 0", density);
    if ((rc = check_hull_bodies(gen, num_bodies, bodies, world))) return rc;
    if (num_bodies > 0 && !velocities) return fail(OCEAN_ERR_INVALID_ARGUMENT, "velocities is NULL");
    return OCEAN_OK;
}

// The hull-forces launches on a pose table, velocities and offsets already in device memory (the poses may be written by
// earlier kernels on the stream), with the map scales in gen->q_scales, gen->body.q and gen->body.corners grown to `world`, and
// wv the wake's vertical velocities (or null).
int launch_hull_sequence(ocean_generator* gen, const ocean_hull_body* poses_dev, const ocean_body_velocity* velocities_dev, int num_bodies,
                         int world, int num_cascades, float density, float tolerance, int max_iterations, ocean_buoyancy_result* hydrostatic_dev,
                         ocean_drag_result* drag_dev, ocean_surface_sample* samples, float* wv) {
    const BodyScratch& sc = gen->body;
    int rc;
    float4* corner_r = sc.corners.ptr;
    float4* corner_u = corner_r + world;
    if (world > 0) {
        OCEAN_CUDA(ocean::launch_hull_transform(poses_dev, sc.offsets.ptr, num_bodies, sc.meshes.ptr, sc.vertices.ptr, world, sc.q.ptr, corner_r,
                                                gen->stream));
        gen->kernel_launches += 1;
        if ((rc = run_query_surface(gen, world, sc.q.ptr, num_cascades, tolerance, max_iterations, samples, wv))) return rc;
        OCEAN_CUDA(ocean::launch_hull_vertex(samples, world, gen->velocity.ptr, gen->map_size, num_cascades, gen->q_scales.ptr, wv, corner_r,
                                             corner_u, gen->stream));
        gen->kernel_launches += 1;
    }
    const float rho_g = density * 9.81f;                                 // G, wave_generator.gd:5, in binary32
    const float half_rho = 0.5f * density;
    OCEAN_CUDA(ocean::launch_hull_reduce(poses_dev, velocities_dev, sc.offsets.ptr, num_bodies, sc.meshes.ptr, sc.triangles.ptr, corner_r,
                                         corner_u, samples, rho_g, half_rho, tolerance, hydrostatic_dev, drag_dev, gen->stream));
    gen->kernel_launches += 1;
    return OCEAN_OK;
}

// ocean_simulate_bodies' checks on hull bodies; *world as for check_hull_bodies.
int check_simulate_hull_args(const ocean_generator* gen, int num_bodies, const ocean_floating_hull* bodies, const ocean_body_state* states,
                             float density, float dt, int substeps, float tolerance, int max_iterations, int* world) {
    int rc = check_solver_args(tolerance, max_iterations);
    if (rc) return rc;
    if ((rc = check_step_args(density, dt, substeps))) return rc;
    if ((rc = check_hull_bodies(gen, num_bodies, bodies, world))) return rc;
    if (num_bodies > 0 && !states) return fail(OCEAN_ERR_INVALID_ARGUMENT, "states is NULL");
    return check_mass_inertia(num_bodies, bodies);
}
}  // namespace

int ocean_hull_set_meshes(ocean_generator* gen, int num_meshes, const ocean_hull_mesh* meshes_host, int num_vertices,
                          const float* vertices_host, int num_triangles, const int32_t* triangles_host, float* volumes_host) {
    int rc = check_hull_meshes(num_meshes, meshes_host, num_vertices, vertices_host, num_triangles, triangles_host, volumes_host);
    if (rc) return rc;
    DeviceScope device_scope__;
    if ((rc = enter_gen(gen, device_scope__))) return rc;
    BodyScratch& sc = gen->body;
    sc.meshes_host.clear();                             // off until the new set is in place
    if (num_meshes == 0) {
        OCEAN_CUDA(cudaStreamSynchronize(gen->stream));  // an earlier call may still read the set
        sc.meshes.release();
        sc.vertices.release();
        sc.triangles.release();
        return OCEAN_OK;
    }
    // stream order puts the copies after the calls that read the old set; the call returns once they are done
    OCEAN_CUDA(sc.meshes.upload(gen, meshes_host, (size_t)num_meshes));
    if (num_vertices > 0) OCEAN_CUDA(sc.vertices.upload(gen, vertices_host, 3 * (size_t)num_vertices));
    if (num_triangles > 0) OCEAN_CUDA(sc.triangles.upload(gen, triangles_host, 3 * (size_t)num_triangles));
    OCEAN_CUDA(cudaStreamSynchronize(gen->stream));
    sc.meshes_host.assign(meshes_host, meshes_host + num_meshes);
    return OCEAN_OK;
}

int ocean_hull_forces_device(ocean_generator* gen, int num_bodies, const ocean_hull_body* bodies_host,
                             const ocean_body_velocity* velocities_host, int num_cascades, const float* map_scales_host, float density,
                             float tolerance, int max_iterations, ocean_buoyancy_result* hydrostatic_dev, ocean_drag_result* drag_dev,
                             ocean_surface_sample* samples_dev) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    int world = 0;
    if ((rc = check_hull_forces_args(gen, num_bodies, bodies_host, velocities_host, density, tolerance, max_iterations, &world))) return rc;
    if (num_bodies == 0) return OCEAN_OK;
    if (!hydrostatic_dev || !drag_dev) return fail(OCEAN_ERR_INVALID_ARGUMENT, "a device buffer is NULL");
    if ((rc = upload_scales(gen, num_cascades, map_scales_host))) return rc;       // the last check: nothing is launched before it
    if ((rc = refresh_velocity(gen, nullptr))) return rc;
    BodyScratch& sc = gen->body;
    const size_t n = (size_t)world;
    OCEAN_CUDA(sc.q.grow(gen, n));
    OCEAN_CUDA(sc.corners.grow(gen, 2 * n));
    if (!samples_dev) OCEAN_CUDA(sc.samples.grow(gen, n));
    ocean_surface_sample* samples = samples_dev ? samples_dev : sc.samples.ptr;
    float* wv = nullptr;
    OCEAN_CUDA(gen->wake.vertical_velocities(gen, n, &wv));
    OCEAN_CUDA(sc.hull_poses.upload(gen, bodies_host, (size_t)num_bodies));
    OCEAN_CUDA(sc.velocities.upload(gen, velocities_host, (size_t)num_bodies));
    if ((rc = upload_offsets(gen, num_bodies, [&](int b) { return sc.meshes_host[bodies_host[b].mesh].num_vertices; }))) return rc;
    return launch_hull_sequence(gen, sc.hull_poses.ptr, sc.velocities.ptr, num_bodies, world, num_cascades, density, tolerance, max_iterations,
                                hydrostatic_dev, drag_dev, samples, wv);
}

int ocean_hull_forces(ocean_generator* gen, int num_bodies, const ocean_hull_body* bodies_host, const ocean_body_velocity* velocities_host,
                      int num_cascades, const float* map_scales_host, float density, float tolerance, int max_iterations,
                      ocean_buoyancy_result* hydrostatic_host, ocean_drag_result* drag_host, ocean_surface_sample* samples_host) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    int world = 0;
    if ((rc = check_hull_forces_args(gen, num_bodies, bodies_host, velocities_host, density, tolerance, max_iterations, &world))) return rc;
    if (num_bodies == 0) return OCEAN_OK;
    if (!hydrostatic_host || !drag_host) return fail(OCEAN_ERR_INVALID_ARGUMENT, "a host buffer is NULL");
    const size_t B = (size_t)num_bodies;
    Staging st;
    const auto hydrostatic = st.out(hydrostatic_host, B);
    const auto drag = st.out(drag_host, B);
    const auto samples = st.out(samples_host, (size_t)world);
    if ((rc = st.upload(gen, kStageHullForces))) return rc;
    return st.finish(gen, ocean_hull_forces_device(gen, num_bodies, bodies_host, velocities_host, num_cascades, map_scales_host, density,
                                                   tolerance, max_iterations, st[hydrostatic], st[drag], st[samples]));
}

int ocean_simulate_hull_bodies_device(ocean_generator* gen, int num_bodies, const ocean_floating_hull* bodies_host,
                                      ocean_body_state* states_dev, int num_cascades, const float* map_scales_host, float density, float dt,
                                      int substeps, float tolerance, int max_iterations, ocean_buoyancy_result* hydrostatic_dev,
                                      ocean_drag_result* drag_dev, float* transforms_dev) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    int world = 0;
    if ((rc = check_simulate_hull_args(gen, num_bodies, bodies_host, states_dev, density, dt, substeps, tolerance, max_iterations, &world)))
        return rc;
    if (num_bodies == 0) return OCEAN_OK;
    if ((rc = upload_scales(gen, num_cascades, map_scales_host))) return rc;       // the last check: nothing is launched before it
    return run_simulate(gen, num_bodies, bodies_host, states_dev, world, nullptr, nullptr, num_cascades, density, dt, substeps, tolerance,
                        max_iterations, hydrostatic_dev, drag_dev, transforms_dev);
}

int ocean_simulate_hull_bodies(ocean_generator* gen, int num_bodies, const ocean_floating_hull* bodies_host, ocean_body_state* states_host,
                               int num_cascades, const float* map_scales_host, float density, float dt, int substeps, float tolerance,
                               int max_iterations, ocean_buoyancy_result* hydrostatic_host, ocean_drag_result* drag_host,
                               float* transforms_host) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    int world = 0;
    if ((rc = check_simulate_hull_args(gen, num_bodies, bodies_host, states_host, density, dt, substeps, tolerance, max_iterations, &world)))
        return rc;
    if (num_bodies == 0) return OCEAN_OK;
    const size_t B = (size_t)num_bodies;
    Staging st;                                         // an output not asked for stays NULL: the twin uses its own
    const auto states = st.inout(states_host, B);
    const auto hydrostatic = st.out(hydrostatic_host, B);
    const auto drag = st.out(drag_host, B);
    const auto transforms = st.out(transforms_host, 12 * B);
    if ((rc = st.upload(gen, kStageSimulateHulls))) return rc;
    return st.finish(gen, ocean_simulate_hull_bodies_device(gen, num_bodies, bodies_host, st[states], num_cascades, map_scales_host, density,
                                                            dt, substeps, tolerance, max_iterations, st[hydrostatic], st[drag],
                                                            st[transforms]));
}

int ocean_copy_twiddles_to_host(ocean_generator* gen, float* host) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if (!host) return fail(OCEAN_ERR_INVALID_ARGUMENT, "host is NULL");
    OCEAN_CUDA(cudaMemcpyAsync(host, gen->twiddles.ptr, sizeof(float2) * (gen->map_size - 1), cudaMemcpyDeviceToHost, gen->stream));
    OCEAN_CUDA(cudaStreamSynchronize(gen->stream));
    return OCEAN_OK;
}

int ocean_get_foam_state(ocean_generator* gen, int cascade, uint16_t* host) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if ((rc = check_cascade(gen, cascade))) return rc;
    if (!host) return fail(OCEAN_ERR_INVALID_ARGUMENT, "host is NULL");
    const size_t layer = (size_t)gen->map_size * gen->map_size;
    OCEAN_CUDA(cudaMemcpyAsync(host, gen->buf.foam + cascade * layer, sizeof(uint16_t) * layer, cudaMemcpyDeviceToHost, gen->stream));
    OCEAN_CUDA(cudaStreamSynchronize(gen->stream));
    return OCEAN_OK;
}

int ocean_set_foam_state(ocean_generator* gen, int cascade, const uint16_t* host) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if ((rc = check_cascade(gen, cascade))) return rc;
    if (!host) return fail(OCEAN_ERR_INVALID_ARGUMENT, "host is NULL");
    const size_t layer = (size_t)gen->map_size * gen->map_size;
    // the plane is the state the next update reads; normal.a is its copy in the map
    uint16_t* dst = reinterpret_cast<uint16_t*>(gen->buf.normal + cascade * layer) + 3;
    OCEAN_CUDA(cudaMemcpyAsync(gen->buf.foam + cascade * layer, host, sizeof(uint16_t) * layer, cudaMemcpyHostToDevice, gen->stream));
    OCEAN_CUDA(cudaMemcpy2DAsync(dst, sizeof(uint2), host, sizeof(uint16_t), sizeof(uint16_t), layer, cudaMemcpyHostToDevice, gen->stream));
    OCEAN_CUDA(cudaStreamSynchronize(gen->stream));
    return OCEAN_OK;
}

int ocean_timer_start(ocean_generator* gen) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    OCEAN_CUDA(cudaEventRecord(gen->timer_start, gen->stream));
    return OCEAN_OK;
}

int ocean_timer_stop(ocean_generator* gen, float* elapsed_ms) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if (!elapsed_ms) return fail(OCEAN_ERR_INVALID_ARGUMENT, "elapsed_ms is NULL");
    OCEAN_CUDA(cudaEventRecord(gen->timer_stop, gen->stream));
    OCEAN_CUDA(cudaEventSynchronize(gen->timer_stop));
    OCEAN_CUDA(cudaEventElapsedTime(elapsed_ms, gen->timer_start, gen->timer_stop));
    return OCEAN_OK;
}

int ocean_set_profiling(ocean_generator* gen, int enable) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    gen->profiling = enable != 0;
    gen->prof_valid = false;
    return OCEAN_OK;
}

int ocean_get_last_kernel_times(ocean_generator* gen, float* spectrum_ms, float* rowpass_ms, float* colpass_ms, int* chunk_cascades) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if (!gen->prof_valid) return fail(OCEAN_ERR_STATE, "no profiled launch yet; call ocean_set_profiling(gen, 1) and run an update");
    OCEAN_CUDA(cudaEventSynchronize(gen->prof[3]));
    float t = 0.f;
    if (spectrum_ms) { OCEAN_CUDA(cudaEventElapsedTime(&t, gen->prof[0], gen->prof[1])); *spectrum_ms = gen->prof_had_gen ? t : 0.f; }
    if (rowpass_ms) OCEAN_CUDA(cudaEventElapsedTime(rowpass_ms, gen->prof[1], gen->prof[2]));
    if (colpass_ms) OCEAN_CUDA(cudaEventElapsedTime(colpass_ms, gen->prof[2], gen->prof[4]));
    if (chunk_cascades) *chunk_cascades = gen->prof_chunk;
    return OCEAN_OK;
}

int ocean_selftest_math(ocean_generator* gen, uint64_t* failures, uint64_t* tested) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if (!failures || !tested) return fail(OCEAN_ERR_INVALID_ARGUMENT, "NULL argument");
    DeviceArray<unsigned long long> d;                  // freed and uncounted on every return
    OCEAN_CUDA(d.grow(gen, 2));
    OCEAN_CUDA(cudaMemsetAsync(d.ptr, 0, 2 * sizeof(unsigned long long), gen->stream));
    OCEAN_CUDA(ocean::launch_selftest_math(d.ptr, d.ptr + 1, gen->stream));
    gen->kernel_launches += 1;
    unsigned long long h[2] = {0, 0};
    OCEAN_CUDA(cudaMemcpyAsync(h, d.ptr, sizeof h, cudaMemcpyDeviceToHost, gen->stream));
    OCEAN_CUDA(cudaStreamSynchronize(gen->stream));
    *failures = h[0];
    *tested = h[1];
    return OCEAN_OK;
}

int ocean_debug_device_math(ocean_generator* gen, int fn, int n, const float* a_host, const float* b_host, float* out_host) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if (fn < OCEAN_MATH_SINCOS || fn > OCEAN_MATH_COS64) return fail(OCEAN_ERR_INVALID_ARGUMENT, "unknown device math function %d", fn);
    if (n < 0) return fail(OCEAN_ERR_INVALID_ARGUMENT, "n = %d is negative", n);
    if (n == 0) return OCEAN_OK;
    if (!a_host || !b_host || !out_host) return fail(OCEAN_ERR_INVALID_ARGUMENT, "NULL argument");
    Staging st;
    const auto a = st.in(a_host, (size_t)n), b = st.in(b_host, (size_t)n);
    const auto out = st.out(reinterpret_cast<float2*>(out_host), (size_t)n);
    if ((rc = st.upload(gen, kStageDeviceMath))) return rc;
    OCEAN_CUDA(ocean::launch_debug_device_math(fn, n, st[a], st[b], st[out], gen->stream));
    gen->kernel_launches += 1;
    return st.finish(gen, OCEAN_OK);
}

// ---- wake layer: a local height field driven by moving sources (oracle/wake.py) ----
static_assert(sizeof(ocean_wake_params) == 20, "ocean_wake_params layout");
static_assert(sizeof(ocean_wake_source) == 28, "ocean_wake_source layout");
static_assert(sizeof(ocean_wake_foam_params) == 16, "ocean_wake_foam_params layout");

int ocean_wake_kernel_taps(float* taps_host) {
    if (!taps_host) return fail(OCEAN_ERR_INVALID_ARGUMENT, "taps_host is NULL");
    ocean::wake_kernel_taps(taps_host);
    return OCEAN_OK;
}

namespace {
constexpr double kWakeCap = 4.0;                        // max Ghat of the stencil (tools/fit_wake_kernel.py)

int check_wake_layer(ocean_generator* g) {
    if (!g->wake.on()) return fail(OCEAN_ERR_STATE, "the generator has no wake layer (ocean_wake_init)");
    return OCEAN_OK;
}

// The call's sub-step and per-ring coefficients, or an error for an invalid step.
int wake_step_args(ocean_generator* g, double dt, int substeps, int num_sources, const ocean_wake_source* sources, int num_states,
                   const ocean_body_state* states, ocean::WakeStepArgs* a, float* h_sub) {
    if (!(dt > 0.0) || !std::isfinite(dt)) return fail(OCEAN_ERR_INVALID_ARGUMENT, "dt %g is not finite and > 0", dt);
    if (substeps < 1 || substeps > 256) return fail(OCEAN_ERR_INVALID_ARGUMENT, "substeps %d outside [1, 256]", substeps);
    if (num_sources < 0 || num_states < 0) return fail(OCEAN_ERR_INVALID_ARGUMENT, "negative source or state count");
    if ((num_sources > 0 && !sources) || (num_states > 0 && !states)) return fail(OCEAN_ERR_INVALID_ARGUMENT, "sources or states is NULL");
    const ocean_wake_params& p = g->wake.params;
    const float hf = (float)(dt / substeps);
    const double h = hf, dx = p.cell_size;
    if (kG * h * h / dx * kWakeCap > 4.0)
        return fail(OCEAN_ERR_INVALID_ARGUMENT, "sub-step %g s above the stable bound sqrt(dx / g) = %g s", h, std::sqrt(dx / kG));
    *a = ocean::WakeStepArgs{};
    for (int r = 0; r <= p.sponge_cells; ++r) {
        double alpha = p.damping;
        if (r < p.sponge_cells) {
            const double t = (double)(p.sponge_cells - r) / p.sponge_cells;
            alpha = (double)p.damping + ((double)p.sponge_damping - (double)p.damping) * (t * t);
        }
        const double ah = alpha * h;
        a->a1[r] = (float)((2.0 - ah) / (1.0 + ah));
        a->a2[r] = (float)(1.0 / (1.0 + ah));
        a->a3[r] = (float)(kG * h * h / (dx * (1.0 + ah)));
    }
    a->sources = sources;
    a->states = states;
    a->num_sources = num_sources;
    a->num_states = num_states;
    a->n = p.size;
    a->sponge_cells = p.sponge_cells;
    a->cell = p.cell_size;
    *h_sub = hf;
    return OCEAN_OK;
}

// Turns off the chosen parts of the layer (kWake*; kWakeFields removes the layer itself): one synchronise when a buffer of
// theirs is live, since kernels may still read it, then their buffers are released and their state reset.  The caller has
// entered the generator.
int WakeLayer::off(ocean_generator* g, unsigned parts) {
    const bool live = ((parts & kWakeCoupling) && (snapshots.ptr || wv.ptr)) || ((parts & kWakeFoam) && foam.ptr) ||
                      ((parts & kWakeMask) && mask.ptr) || ((parts & kWakeFields) && fields.ptr);
    if (live) OCEAN_CUDA(cudaStreamSynchronize(g->stream));
    if (parts & kWakeCoupling) {
        snapshots.release();
        wv.release();
        primed = false;
        e = 0;
        interval = 0.0f;
        for (auto& o : snapshot_origin) o[0] = o[1] = 0;
    }
    if (parts & kWakeFoam) {
        foam.release();
        foam_params = ocean_wake_foam_params{};
        f = 0;
    }
    if (parts & kWakeMask) {
        mask.release();
        mask_size[0] = mask_size[1] = 0;
        mask_origin[0] = mask_origin[1] = 0;
    }
    if (parts & kWakeFields) {
        fields.release();
        params = ocean_wake_params{};
        h = 0;
        hp = 1;
        origin[0] = origin[1] = 0;
        readers = 0;
    }
    return OCEAN_OK;
}

// The status of the set-up step `what` of a part that has just been allocated; a failed set-up turns the part off.
int wake_part_setup(ocean_generator* g, unsigned part, cudaError_t e, const char* what) {
    if (e == cudaSuccess) return OCEAN_OK;
    g->wake.off(g, part);
    return fail(OCEAN_ERR_CUDA, "%s failed: %s", what, cudaGetErrorString(e));
}

int check_wake_points(int num_points, const void* points, const void* out) {
    if (num_points < 0) return fail(OCEAN_ERR_INVALID_ARGUMENT, "num_points %d is negative", num_points);
    if (num_points > 0 && (!points || !out)) return fail(OCEAN_ERR_INVALID_ARGUMENT, "points or out is NULL");
    return OCEAN_OK;
}
}  // namespace

int ocean_wake_init(ocean_generator* gen, const ocean_wake_params* params) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if (!params) return fail(OCEAN_ERR_INVALID_ARGUMENT, "params is NULL");
    const ocean_wake_params p = *params;
    WakeLayer& w = gen->wake;
    if (p.size == 0) {
        if ((rc = w.off(gen, kWakeLayer))) return rc;
        // only wake kernels read these, and none is queued once the layer's buffers are released
        gen->staging[kStageWakeStep].release();
        gen->staging[kStageSampleWake].release();
        return OCEAN_OK;
    }
    if (p.size < 128 || p.size > 2048 || (p.size & (p.size - 1)))
        return fail(OCEAN_ERR_INVALID_ARGUMENT, "size %d is not 0 or a power of two in [128, 2048]", p.size);
    if (!(p.cell_size > 0.0f) || !std::isfinite(p.cell_size)) return fail(OCEAN_ERR_INVALID_ARGUMENT, "cell_size %g is not finite and > 0", p.cell_size);
    if (!(p.damping >= 0.0f) || !std::isfinite(p.damping) || !(p.sponge_damping >= 0.0f) || !std::isfinite(p.sponge_damping))
        return fail(OCEAN_ERR_INVALID_ARGUMENT, "damping %g / sponge_damping %g not finite and >= 0", p.damping, p.sponge_damping);
    if (p.sponge_cells < 0 || p.sponge_cells > ocean::kWakeMaxSponge || 2 * p.sponge_cells > p.size)
        return fail(OCEAN_ERR_INVALID_ARGUMENT, "sponge_cells %d outside [0, min(64, size / 2)]", p.sponge_cells);
    const size_t cells = 4 * (size_t)p.size * p.size;  // h, h_prev and two fields a scrolled sub-step writes
    // every part goes (the mask's cells are cells of the old cell size); the fields' block stays when its size does
    if ((rc = w.off(gen, w.fields.capacity == cells ? kWakeLayer & ~kWakeFields : kWakeLayer))) return rc;
    w.params = ocean_wake_params{};                     // no layer until the fields below are allocated and cleared
    w.readers = 0;
    OCEAN_CUDA(w.fields.grow(gen, cells));
    OCEAN_CUDA(cudaMemsetAsync(w.fields.ptr, 0, cells * sizeof(float), gen->stream));
    w.params = p;
    w.h = 0;
    w.hp = 1;
    w.origin[0] = w.origin[1] = 0;
    return OCEAN_OK;
}

int ocean_wake_step_device(ocean_generator* gen, double dt, int substeps, int64_t origin_x, int64_t origin_z, int num_sources,
                           const ocean_wake_source* sources_dev, int num_states, const ocean_body_state* states_dev) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if ((rc = check_wake_layer(gen))) return rc;
    ocean::WakeStepArgs a;
    float h = 0.0f;
    if ((rc = wake_step_args(gen, dt, substeps, num_sources, sources_dev, num_states, states_dev, &a, &h))) return rc;
    WakeLayer& w = gen->wake;
    const int n = w.params.size;
    // the scroll, clamped to [-n, n] per axis (a move of n cells or more reads nothing but zeros)
    auto shift = [n](int64_t to, int64_t from) -> int {
        const __int128 d = (__int128)to - (__int128)from;
        return d > n ? n : d < -n ? -n : (int)d;
    };
    a.di = shift(origin_x, w.origin[0]);
    a.dj = shift(origin_z, w.origin[1]);
    a.x0 = w.corner(origin_x);
    a.z0 = w.corner(origin_z);
    ocean::WakeFoamStepArgs f{};
    const ocean::WakeFoamStepArgs* foam = w.foamed() ? &f : nullptr;
    if (foam) {
        const ocean_wake_foam_params& fp = w.foam_params;
        f.whitecap = fp.whitecap;
        f.decay = exp_det_host(-(fp.decay_rate * h));  // binary32 products, the cascades' DETMATH exp
        f.grow = fp.grow_rate * h;
        f.stir = fp.stir_rate * h;
    }
    // while a mask is set every kernel of the call runs its obstacle form, the mask read in the call's window
    const ocean::WakeObstacles ob = w.obstacles(origin_x, origin_z);
    const ocean::WakeObstacles* obstacles = w.masked() ? &ob : nullptr;
    for (int k = 0; k < substeps; ++k) {
        int spare[2], m = 0;
        for (int b = 0; b < 4 && m < 2; ++b)
            if (b != w.h && b != w.hp) spare[m++] = b;
        const bool scrolled = a.di != 0 || a.dj != 0;
        a.h = w.field(w.h);
        a.h_prev = w.field(w.hp);
        a.out_h = w.field(spare[0]);
        a.out_h_prev = scrolled ? w.field(spare[1]) : nullptr;
        a.tau = (float)k * h;
        if (foam) {
            f.foam = w.foam_field(w.f);
            f.out_foam = w.foam_field(w.f ^ 1);
        }
        OCEAN_CUDA(ocean::launch_wake_step(a, foam, obstacles, gen->stream));
        gen->kernel_launches += 1;
        if (foam) w.f ^= 1;
        w.hp = scrolled ? spare[1] : w.h;
        w.h = spare[0];
        // the fields are now those of the new origin: record it at once, so a later failed launch leaves them consistent
        w.origin[0] = origin_x;
        w.origin[1] = origin_z;
        a.di = a.dj = 0;
    }
    if (w.coupled()) {
        // e = h + phi at the end of the call into the snapshot that held e_old (on a priming call into both)
        const int e = w.primed ? w.e ^ 1 : w.e;
        ocean::WakeFreeSurfaceArgs fs{};
        fs.h = w.field(w.h);
        fs.e = w.snapshot(e);
        fs.e_old = w.primed ? nullptr : w.snapshot(e ^ 1);
        fs.sources = a.sources;
        fs.states = a.states;
        fs.num_sources = a.num_sources;
        fs.num_states = a.num_states;
        fs.n = n;
        fs.cell = a.cell;
        fs.x0 = a.x0;
        fs.z0 = a.z0;
        fs.tau = (float)substeps * h;
        OCEAN_CUDA(ocean::launch_wake_free_surface(fs, obstacles, gen->stream));
        gen->kernel_launches += 1;
        for (int k = 0; k < 2; ++k) {
            if (k != e && w.primed) continue;
            w.snapshot_origin[k][0] = origin_x;
            w.snapshot_origin[k][1] = origin_z;
        }
        w.e = e;
        w.interval = fs.tau;
        w.primed = true;
    }
    return OCEAN_OK;
}

int ocean_wake_step(ocean_generator* gen, double dt, int substeps, int64_t origin_x, int64_t origin_z, int num_sources,
                    const ocean_wake_source* sources_host, int num_states, const ocean_body_state* states_host) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if ((rc = check_wake_layer(gen))) return rc;
    ocean::WakeStepArgs a;
    float h = 0.0f;
    if ((rc = wake_step_args(gen, dt, substeps, num_sources, sources_host, num_states, states_host, &a, &h))) return rc;
    for (int k = 0; k < num_sources; ++k)
        if (sources_host[k].body >= num_states)
            return fail(OCEAN_ERR_INVALID_ARGUMENT, "source %d: body %d is not below num_states %d", k, sources_host[k].body, num_states);
    Staging st;
    const auto sources = st.in(sources_host, (size_t)num_sources);
    const auto states = st.in(states_host, (size_t)num_states);
    if ((rc = st.upload(gen, kStageWakeStep))) return rc;  // and no finish(): the call returns once the step is enqueued
    return ocean_wake_step_device(gen, dt, substeps, origin_x, origin_z, num_sources, st[sources], num_states, st[states]);
}

int ocean_wake_render_map(ocean_generator* gen, void* map_dev, float* world_rect) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if ((rc = check_wake_layer(gen))) return rc;
    if (!map_dev) return fail(OCEAN_ERR_INVALID_ARGUMENT, "map_dev is NULL");
    const ocean::WakeRead r = gen->wake.read_h();
    OCEAN_CUDA(ocean::launch_wake_map(r, map_dev, gen->stream));
    gen->kernel_launches += 1;
    if (world_rect) {
        world_rect[0] = r.x0;
        world_rect[1] = r.z0;
        world_rect[2] = world_rect[3] = (float)r.n * r.cell;
    }
    return OCEAN_OK;
}

int ocean_sample_wake_device(ocean_generator* gen, int num_points, const float* points_xz_dev, float* out_dev) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if ((rc = check_wake_layer(gen))) return rc;
    if ((rc = check_wake_points(num_points, points_xz_dev, out_dev))) return rc;
    if (num_points == 0) return OCEAN_OK;
    OCEAN_CUDA(ocean::launch_wake_sample(gen->wake.read_h(), reinterpret_cast<const float2*>(points_xz_dev), num_points, out_dev, gen->stream));
    gen->kernel_launches += 1;
    return OCEAN_OK;
}

int ocean_sample_wake(ocean_generator* gen, int num_points, const float* points_xz_host, float* out_host) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if ((rc = check_wake_layer(gen))) return rc;
    if ((rc = check_wake_points(num_points, points_xz_host, out_host))) return rc;
    if (num_points == 0) return OCEAN_OK;
    Staging st;
    const auto points = st.in(points_xz_host, 2 * (size_t)num_points);
    const auto out = st.out(out_host, 3 * (size_t)num_points);
    if ((rc = st.upload(gen, kStageSampleWake))) return rc;
    return st.finish(gen, ocean_sample_wake_device(gen, num_points, st[points], st[out]));
}

int ocean_wake_get_state(ocean_generator* gen, float* h_host, float* h_prev_host, int64_t* origin_xz) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if ((rc = check_wake_layer(gen))) return rc;
    if (!h_host || !h_prev_host || !origin_xz) return fail(OCEAN_ERR_INVALID_ARGUMENT, "NULL argument");
    const WakeLayer& w = gen->wake;
    OCEAN_CUDA(cudaMemcpyAsync(h_host, w.field(w.h), sizeof(float) * w.cells(), cudaMemcpyDeviceToHost, gen->stream));
    OCEAN_CUDA(cudaMemcpyAsync(h_prev_host, w.field(w.hp), sizeof(float) * w.cells(), cudaMemcpyDeviceToHost, gen->stream));
    OCEAN_CUDA(cudaStreamSynchronize(gen->stream));
    origin_xz[0] = w.origin[0];
    origin_xz[1] = w.origin[1];
    return OCEAN_OK;
}

int ocean_wake_set_state(ocean_generator* gen, const float* h_host, const float* h_prev_host, int64_t origin_x, int64_t origin_z) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if ((rc = check_wake_layer(gen))) return rc;
    if (!h_host || !h_prev_host) return fail(OCEAN_ERR_INVALID_ARGUMENT, "NULL argument");
    WakeLayer& w = gen->wake;
    OCEAN_CUDA(cudaMemcpyAsync(w.field(w.h), h_host, sizeof(float) * w.cells(), cudaMemcpyHostToDevice, gen->stream));
    OCEAN_CUDA(cudaMemcpyAsync(w.field(w.hp), h_prev_host, sizeof(float) * w.cells(), cudaMemcpyHostToDevice, gen->stream));
    OCEAN_CUDA(cudaStreamSynchronize(gen->stream));
    w.origin[0] = origin_x;
    w.origin[1] = origin_z;
    w.primed = false;                                   // the snapshots no longer describe the layer
    return OCEAN_OK;
}

int ocean_wake_set_coupling(ocean_generator* gen, int enable) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if ((rc = check_wake_layer(gen))) return rc;
    if (enable != 0 && enable != 1) return fail(OCEAN_ERR_INVALID_ARGUMENT, "enable %d is not 0 or 1", enable);
    if (!enable) return gen->wake.off(gen, kWakeCoupling);
    if (gen->wake.coupled()) return OCEAN_OK;
    OCEAN_CUDA(gen->wake.snapshots.grow(gen, 2 * gen->wake.cells()));   // unprimed: nothing reads them before a step
    return OCEAN_OK;
}

int ocean_wake_get_coupling(ocean_generator* gen, float* e_host, float* e_old_host, int64_t* origins, float* interval) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if ((rc = check_wake_layer(gen))) return rc;
    const WakeLayer& w = gen->wake;
    if (!w.coupled()) return fail(OCEAN_ERR_STATE, "the wake layer's coupling is off (ocean_wake_set_coupling)");
    if (!e_host || !e_old_host || !origins || !interval) return fail(OCEAN_ERR_INVALID_ARGUMENT, "NULL argument");
    const size_t cells = w.cells();
    if (!w.primed) {
        std::fill(e_host, e_host + cells, 0.0f);
        std::fill(e_old_host, e_old_host + cells, 0.0f);
        std::fill(origins, origins + 4, (int64_t)0);
        *interval = 0.0f;
        return OCEAN_OK;
    }
    const int e = w.e, o = e ^ 1;
    OCEAN_CUDA(cudaMemcpyAsync(e_host, w.snapshot(e), sizeof(float) * cells, cudaMemcpyDeviceToHost, gen->stream));
    OCEAN_CUDA(cudaMemcpyAsync(e_old_host, w.snapshot(o), sizeof(float) * cells, cudaMemcpyDeviceToHost, gen->stream));
    OCEAN_CUDA(cudaStreamSynchronize(gen->stream));
    origins[0] = w.snapshot_origin[e][0];
    origins[1] = w.snapshot_origin[e][1];
    origins[2] = w.snapshot_origin[o][0];
    origins[3] = w.snapshot_origin[o][1];
    *interval = w.interval;
    return OCEAN_OK;
}

int ocean_wake_set_foam(ocean_generator* gen, const ocean_wake_foam_params* params) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if ((rc = check_wake_layer(gen))) return rc;
    WakeLayer& w = gen->wake;
    if (!params) return w.off(gen, kWakeFoam);
    const ocean_wake_foam_params p = *params;
    if (!std::isfinite(p.whitecap) || !std::isfinite(p.grow_rate) || !std::isfinite(p.stir_rate) || !std::isfinite(p.decay_rate))
        return fail(OCEAN_ERR_INVALID_ARGUMENT, "foam parameters not finite");
    if (!(p.grow_rate >= 0.0f) || !(p.stir_rate >= 0.0f) || !(p.decay_rate >= 0.0f))
        return fail(OCEAN_ERR_INVALID_ARGUMENT, "grow_rate %g, stir_rate %g or decay_rate %g is negative", p.grow_rate, p.stir_rate,
                    p.decay_rate);
    if (!w.foamed()) {
        OCEAN_CUDA(w.foam.grow(gen, 2 * w.cells()));
        const cudaError_t e = cudaMemsetAsync(w.foam.ptr, 0, 2 * w.cells() * sizeof(float), gen->stream);
        if ((rc = wake_part_setup(gen, kWakeFoam, e, "clearing the foam"))) return rc;
        w.f = 0;
    }
    w.foam_params = p;
    return OCEAN_OK;
}

int ocean_wake_set_obstacles(ocean_generator* gen, const uint8_t* mask_host, int32_t width, int32_t depth, int64_t origin_x,
                             int64_t origin_z) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if ((rc = check_wake_layer(gen))) return rc;
    WakeLayer& w = gen->wake;
    if (!mask_host && width == 0 && depth == 0) return w.off(gen, kWakeMask);
    if (!mask_host) return fail(OCEAN_ERR_INVALID_ARGUMENT, "mask_host is NULL with width %d, depth %d", width, depth);
    if (width < 1 || depth < 1) return fail(OCEAN_ERR_INVALID_ARGUMENT, "mask size %d x %d is not at least 1 x 1", width, depth);
    if ((int64_t)width * depth > ((int64_t)1 << 28))
        return fail(OCEAN_ERR_INVALID_ARGUMENT, "mask size %d x %d above 2^28 cells", width, depth);
    if (origin_x > INT64_MAX - width || origin_z > INT64_MAX - depth)
        return fail(OCEAN_ERR_INVALID_ARGUMENT, "mask origin + size not representable in int64");
    const size_t cells = (size_t)width * depth;
    if (w.mask.capacity != cells) {
        if ((rc = w.off(gen, kWakeMask))) return rc;
        OCEAN_CUDA(w.mask.grow(gen, cells));
    }
    // stream order puts the copy after the steps that read the old mask; the call returns once the copy is done
    cudaError_t e = cudaMemcpyAsync(w.mask.ptr, mask_host, cells, cudaMemcpyHostToDevice, gen->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(gen->stream);
    if ((rc = wake_part_setup(gen, kWakeMask, e, "copying the mask"))) return rc;
    w.mask_size[0] = width;
    w.mask_size[1] = depth;
    w.mask_origin[0] = origin_x;
    w.mask_origin[1] = origin_z;
    return OCEAN_OK;
}

int ocean_wake_set_readers(ocean_generator* gen, uint32_t readers) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if ((rc = check_wake_layer(gen))) return rc;
    if (readers & ~(OCEAN_WAKE_READ_RAYCAST | OCEAN_WAKE_READ_SPRAY)) return fail(OCEAN_ERR_INVALID_ARGUMENT, "readers 0x%x: unknown bits", readers);
    gen->wake.readers = readers;
    return OCEAN_OK;
}

int ocean_wake_get_foam_state(ocean_generator* gen, float* foam_host) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if ((rc = check_wake_layer(gen))) return rc;
    const WakeLayer& w = gen->wake;
    if (!w.foamed()) return fail(OCEAN_ERR_STATE, "the wake layer's foam is off (ocean_wake_set_foam)");
    if (!foam_host) return fail(OCEAN_ERR_INVALID_ARGUMENT, "foam_host is NULL");
    OCEAN_CUDA(cudaMemcpyAsync(foam_host, w.foam_field(w.f), sizeof(float) * w.cells(), cudaMemcpyDeviceToHost, gen->stream));
    OCEAN_CUDA(cudaStreamSynchronize(gen->stream));
    return OCEAN_OK;
}

int ocean_wake_set_foam_state(ocean_generator* gen, const float* foam_host) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if ((rc = check_wake_layer(gen))) return rc;
    const WakeLayer& w = gen->wake;
    if (!w.foamed()) return fail(OCEAN_ERR_STATE, "the wake layer's foam is off (ocean_wake_set_foam)");
    if (!foam_host) return fail(OCEAN_ERR_INVALID_ARGUMENT, "foam_host is NULL");
    OCEAN_CUDA(cudaMemcpyAsync(w.foam_field(w.f), foam_host, sizeof(float) * w.cells(), cudaMemcpyHostToDevice, gen->stream));
    OCEAN_CUDA(cudaStreamSynchronize(gen->stream));
    return OCEAN_OK;
}

// ---- sea state and drifters (ocean_drift.cu; oracle/sea_state.py, oracle/drifters.py) ----
namespace {
// Allocates the cache on first use, zeroed, then recomputes every stale cascade that has a dispersion table in one launch
// sequence.  A cascade without a table has never been updated: it keeps zero moments and stays stale until it gets one.
// The cache is allocated whole or not at all: a failure releases both buffers, so the next call starts over.
int refresh_sea_state(ocean_generator* gen) {
    if (!gen->sea_moments.ptr || !gen->sea_partial.ptr) {
        const size_t n = (size_t)gen->num_cascades * ocean::kSeaStateMoments;
        const int per_launch = std::min(gen->num_cascades, ocean::kMaxSeaStateLaunch);
        cudaError_t e = gen->sea_moments.grow(gen, n);
        if (e == cudaSuccess) e = cudaMemsetAsync(gen->sea_moments.ptr, 0, sizeof(double) * n, gen->stream);
        if (e == cudaSuccess) e = gen->sea_partial.grow(gen, (size_t)per_launch * ocean::sea_state_blocks(gen->map_size) * ocean::kSeaStateMoments);
        if (e != cudaSuccess) {
            gen->sea_moments.release();
            gen->sea_partial.release();
            return fail(OCEAN_ERR_CUDA, "sea-state cache allocation failed: %s", cudaGetErrorString(e));
        }
    }
    std::vector<ocean::SeaStateJob> jobs;
    for (int i = 0; i < gen->num_cascades; ++i)
        if (gen->sea_stale[i] && gen->cascade_slot[i] >= 0) jobs.push_back(ocean::SeaStateJob{i, gen->cascade_slot[i]});
    if (jobs.empty()) return OCEAN_OK;
    int launched = 0;
    OCEAN_CUDA(ocean::launch_sea_state(gen->buf, jobs.data(), (int)jobs.size(), gen->sea_partial.ptr, gen->sea_moments.ptr, gen->stream,
                                       &launched));
    gen->kernel_launches += (uint64_t)launched;
    for (const auto& j : jobs) gen->sea_stale[j.cascade] = 0;
    return OCEAN_OK;
}

// The record of moments m (ocean::kSeaStateMoments, the device order) with its derived fields (include/ocean.h).
ocean_sea_state sea_state_record(const double* m) {
    ocean_sea_state s;
    std::memset(&s, 0, sizeof s);
    s.m_minus1 = m[0]; s.m0 = m[1]; s.m1 = m[2]; s.m2 = m[3];
    s.direction[0] = m[4]; s.direction[1] = m[5];
    s.slope[0] = m[6]; s.slope[1] = m[7];
    s.stokes[0] = m[8]; s.stokes[1] = m[9];
    if (s.m0 == 0.0) return s;
    const double two_pi = 2.0 * M_PI;
    s.significant_wave_height = 4.0 * std::sqrt(s.m0);
    s.mean_period = two_pi * s.m0 / s.m1;
    s.zero_crossing_period = two_pi * std::sqrt(s.m0 / s.m2);
    s.energy_period = two_pi * s.m_minus1 / s.m0;
    s.mean_direction = std::atan2(-s.direction[1], -s.direction[0]) * (180.0 / M_PI);
    const double R = std::hypot(s.direction[0], s.direction[1]) / s.m0;
    s.directional_spread = std::sqrt(2.0 * std::fmax(0.0, 1.0 - R));
    s.mean_square_slope = s.slope[0] + s.slope[1];
    s.stokes_speed = std::hypot(s.stokes[0], s.stokes[1]);
    return s;
}

int check_drift_args(ocean_generator* gen, double dt, const ocean_drift_params* p, int num_drifters, const void* drifters, int num_cascades,
                     const float* map_scales) {
    if (!std::isfinite(dt) || !(dt >= 0.0)) return fail(OCEAN_ERR_INVALID_ARGUMENT, "dt %g is not finite and >= 0", dt);
    if (!p) return fail(OCEAN_ERR_INVALID_ARGUMENT, "params is NULL");
    const float fs[5] = {p->current[0], p->current[1], p->wind[0], p->wind[1], p->stokes_scale};
    for (float f : fs)
        if (!std::isfinite(f)) return fail(OCEAN_ERR_INVALID_ARGUMENT, "a drift parameter (%g) is not finite", f);
    for (double b : p->box)
        if (!std::isfinite(b)) return fail(OCEAN_ERR_INVALID_ARGUMENT, "a box coordinate (%g) is not finite", b);
    if (p->flags & ~(OCEAN_DRIFT_WRAP | OCEAN_DRIFT_READ_WAKE)) return fail(OCEAN_ERR_INVALID_ARGUMENT, "flags 0x%x: unknown bits", p->flags);
    if ((p->flags & OCEAN_DRIFT_WRAP) && !(p->box[2] > 0.0 && p->box[3] > 0.0))
        return fail(OCEAN_ERR_INVALID_ARGUMENT, "wrap box %g x %g: width and depth must be > 0", p->box[2], p->box[3]);
    if (num_cascades < 1 || num_cascades > gen->num_cascades)
        return fail(OCEAN_ERR_INVALID_ARGUMENT, "num_cascades %d outside [1, %d]", num_cascades, gen->num_cascades);
    if (!map_scales) return fail(OCEAN_ERR_INVALID_ARGUMENT, "map_scales is NULL");
    if (num_drifters < 0) return fail(OCEAN_ERR_INVALID_ARGUMENT, "num_drifters %d is negative", num_drifters);
    if (num_drifters > 0 && !drifters) return fail(OCEAN_ERR_INVALID_ARGUMENT, "drifters is NULL");
    return OCEAN_OK;
}
}  // namespace

int ocean_get_sea_state(ocean_generator* gen, int num_cascades, const float* map_scales_host, ocean_sea_state* per_cascade_host,
                    ocean_sea_state* total_host) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if (num_cascades < 1 || num_cascades > gen->num_cascades)
        return fail(OCEAN_ERR_INVALID_ARGUMENT, "num_cascades %d outside [1, %d]", num_cascades, gen->num_cascades);
    if (!map_scales_host || !total_host) return fail(OCEAN_ERR_INVALID_ARGUMENT, "map_scales or total is NULL");
    if ((rc = refresh_sea_state(gen))) return rc;
    std::vector<double> m((size_t)num_cascades * ocean::kSeaStateMoments);
    OCEAN_CUDA(cudaMemcpyAsync(m.data(), gen->sea_moments.ptr, sizeof(double) * m.size(), cudaMemcpyDeviceToHost, gen->stream));
    OCEAN_CUDA(cudaStreamSynchronize(gen->stream));
    double total[ocean::kSeaStateMoments] = {};
    for (int i = 0; i < num_cascades; ++i) {
        const double* mi = m.data() + (size_t)i * ocean::kSeaStateMoments;
        if (per_cascade_host) per_cascade_host[i] = sea_state_record(mi);
        const double s = (double)map_scales_host[4 * (size_t)i + 2], s2 = s * s;
        for (int k = 0; k < ocean::kSeaStateMoments; ++k) total[k] = total[k] + s2 * mi[k];
    }
    *total_host = sea_state_record(total);
    return OCEAN_OK;
}

int ocean_drift_device(ocean_generator* gen, double dt, const ocean_drift_params* params, int num_drifters, ocean_drifter* drifters_dev,
                       int num_cascades, const float* map_scales_host, float* instances_dev) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if ((rc = check_drift_args(gen, dt, params, num_drifters, drifters_dev, num_cascades, map_scales_host))) return rc;
    if (num_drifters == 0) return OCEAN_OK;
    if ((rc = upload_scales(gen, num_cascades, map_scales_host))) return rc;
    if (dt > 0.0 && (rc = refresh_sea_state(gen))) return rc;
    const bool wk = instances_dev && (params->flags & OCEAN_DRIFT_READ_WAKE) && gen->wake.on();
    const ocean::WakeRead wake = wk ? gen->wake.read_h() : ocean::WakeRead{};
    OCEAN_CUDA(ocean::launch_drift(gen->buf, num_cascades, gen->q_scales.ptr, gen->sea_moments.ptr, *params, dt, drifters_dev, num_drifters,
                                   instances_dev, wk ? &wake : nullptr, gen->stream));
    gen->kernel_launches += 1;
    return OCEAN_OK;
}

int ocean_drift(ocean_generator* gen, double dt, const ocean_drift_params* params, int num_drifters, ocean_drifter* drifters_host,
                int num_cascades, const float* map_scales_host, float* instances_host) {
    OCEAN_ENTER(gen);
    if (rc) return rc;
    if ((rc = check_drift_args(gen, dt, params, num_drifters, drifters_host, num_cascades, map_scales_host))) return rc;
    if (num_drifters == 0) return OCEAN_OK;
    Staging st;
    const auto drifters = st.inout(drifters_host, (size_t)num_drifters);
    const auto instances = st.out(instances_host, 12 * (size_t)num_drifters);
    if ((rc = st.upload(gen, kStageDrift))) return rc;
    return st.finish(gen, ocean_drift_device(gen, dt, params, num_drifters, st[drifters], num_cascades, map_scales_host, st[instances]));
}

int ocean_get_info(ocean_generator* gen, ocean_info* out) {
    if (!gen || !out) return fail(OCEAN_ERR_INVALID_ARGUMENT, "NULL argument");
    out->device = gen->device;
    out->map_size = gen->map_size;
    out->num_cascades = gen->num_cascades;
    out->pending_cascades = gen->pass_num_cascades_remaining;
    out->kernel_launches = gen->kernel_launches;
    out->cascade_updates = gen->cascade_updates;
    out->device_bytes = gen->device_bytes;
    return OCEAN_OK;
}

}  // extern "C"
