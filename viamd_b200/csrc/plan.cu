// plan.cu — host side of libmdgpu: the evaluation plan, the frame loop dispatched onto CUDA streams, the C ABI.
//
// This is the replacement of eval_properties (reference md_script.c:5730-5973): instead of one enkiTS task per frame range
// evaluating one frame at a time on a CPU thread, frames are grouped into batches, each batch is enqueued on one of a small
// ring of CUDA streams (H2D copy of the batch when the frames are on the host, then the property kernels), and integer
// accumulators stay in HBM until mdgpu_plan_sync folds them into the md_script_property_data_t-shaped results.
#include "common.cuh"
#include "kernels.h"
#include "synth.h"

#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <condition_variable>
#include <functional>
#include <chrono>
#include <string>
#include <thread>
#include <type_traits>
#include <utility>
#include <array>
#include <vector>
#include <map>
#include <memory>
#include <algorithm>
#include <sched.h>
#include <dlfcn.h>
#include <ctype.h>

namespace mdg {

static thread_local std::string g_last_error;
static std::atomic<uint64_t> g_launches{0};

static int fail(int code, const char* fmt, ...) {
    char buf[512]; va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof(buf), fmt, ap); va_end(ap);
    g_last_error = buf;
    fprintf(stderr, "[mdgpu] error: %s\n", buf);
    return code;
}
#define CUDA_TRY(expr) do { cudaError_t e_ = (expr); if (e_ != cudaSuccess) return fail(MDGPU_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e_), __FILE__, __LINE__); } while (0)

void note_launch(const char*, cudaStream_t) { g_launches.fetch_add(1, std::memory_order_relaxed); }

// Owner of one allocation of n elements of T, in device memory or (Host) pinned host memory: freed when the owner is destroyed or
// reallocated, so a buffer's lifetime is its owner's and a failed allocation leaves an empty owner. Move-only.
template <typename T, bool Host = false> class Buf {
    T* p_ = nullptr; size_t n_ = 0;
public:
    using value_type = T;
    Buf() = default;
    Buf(const Buf&) = delete; Buf& operator=(const Buf&) = delete;
    Buf(Buf&& o) noexcept { *this = std::move(o); }
    Buf& operator=(Buf&& o) noexcept { std::swap(p_, o.p_); std::swap(n_, o.n_); return *this; }   // o frees what this held
    ~Buf() { reset(); }
    void reset() { if (p_) { if (Host) cudaFreeHost(p_); else cudaFree(p_); } p_ = nullptr; n_ = 0; }
    cudaError_t alloc(size_t n) {   // n == 0 allocates nothing
        reset();
        if (!n) return cudaSuccess;
        void* q = nullptr; const cudaError_t e = Host ? cudaMallocHost(&q, n * sizeof(T)) : cudaMalloc(&q, n * sizeof(T));
        if (e == cudaSuccess) { p_ = (T*)q; n_ = n; }
        return e;
    }
    cudaError_t upload(const T* h, size_t n) {
        static_assert(!Host, "pinned buffers are written directly");
        const cudaError_t e = alloc(n); if (e != cudaSuccess || !n) return e;
        return cudaMemcpy(p_, h, n * sizeof(T), cudaMemcpyHostToDevice);
    }
    T* get() const { return p_; }
    size_t size() const { return n_; }
    size_t bytes() const { return n_ * sizeof(T); }
    T& operator[](size_t i) const { static_assert(Host, "device memory is not addressable from the host"); return p_[i]; }
};
template <typename T> using DevBuf = Buf<T, false>;
template <typename T> using PinnedBuf = Buf<T, true>;

// Owner of a stream or event, destroyed with its owner; it converts to the handle for the runtime calls that use it.
template <typename H, cudaError_t (*Destroy)(H)> class Handle {
    H h_ = nullptr;
public:
    Handle() = default;
    Handle(const Handle&) = delete; Handle& operator=(const Handle&) = delete;
    Handle(Handle&& o) noexcept { std::swap(h_, o.h_); }
    Handle& operator=(Handle&& o) noexcept { std::swap(h_, o.h_); return *this; }
    ~Handle() { if (h_) Destroy(h_); }
    H* out() { if (h_) Destroy(h_); h_ = nullptr; return &h_; }   // where a create call writes the new handle
    operator H() const { return h_; }
};
using Stream = Handle<cudaStream_t, cudaStreamDestroy>;
using Event = Handle<cudaEvent_t, cudaEventDestroy>;

// Owner of the arrays of one CellList; `cl` is the plain struct the kernels receive (empty until alloc succeeds).
struct CellListBuf {
    DevBuf<float4> sorted, scratch; DevBuf<uint32_t> cell_of, rank, cell_cnt;
    CellList cl{};
    cudaError_t alloc(uint32_t B, uint32_t max_points, uint32_t cap) {
        const size_t n = (size_t)B * max_points; cudaError_t e;
        if ((e = sorted.alloc(n)) != cudaSuccess || (e = scratch.alloc(n)) != cudaSuccess || (e = cell_of.alloc(n)) != cudaSuccess ||
            (e = rank.alloc(n)) != cudaSuccess || (e = cell_cnt.alloc((size_t)B * (cap + 1) + B)) != cudaSuccess) return e;
        cl = CellList{ sorted.get(), scratch.get(), cell_of.get(), rank.get(), cell_cnt.get(), cell_cnt.get() + (size_t)B * (cap + 1), max_points, cap };
        return cudaSuccess;
    }
};

struct Prop {
    std::string name; uint32_t op = 0;
    std::vector<int32_t> h_idx[4];
    DevBuf<int32_t> d_idx[2][4];                   // the lists in each atom space: [SPACE_FULL] global indices, [SPACE_COMPACT] remapped (host ingest of selected atoms)
    int32_t first[2][4] = {};                      // index of each list's first atom in each space (single-atom arguments are passed by value)
    size_t n_struct = 0, struct_size = 0;
    uint32_t com_mask = 0;   // distance/angle/dihedral: bit k = argument k is a selection evaluated through md_util_com_compute
    std::vector<uint32_t> h_soff; DevBuf<uint32_t> d_soff;   // rdf with centre-of-mass references: CSR offsets of the groups in idx[0]
    float cutoff_min = 0.f, cutoff_max = 0.f;
    std::vector<uint32_t> h_goff[2]; DevBuf<uint32_t> d_goff[2];   // argument 0 / 1 is an ARRAY of selections, one position per selection: their CSR offsets in idx[k]
    std::vector<uint32_t> h_aoff[4]; DevBuf<uint32_t> d_aoff[4];   // distance / angle / dihedral / com: argument k is an ARRAY of selections (centre of their centres)
    DevBuf<uint8_t> d_and_mask;   // `selection and within(...)`: one byte per atom of the static side (count(within()) / rdf(within()))
    // count(x, 'residue' | 'chain' | 'structure') (com_args bit 1): the group of every atom (-1: none) and the number of groups
    DevBuf<int32_t> d_group_of; uint32_t n_groups = 0; bool count_groups = false;
    // Dynamic arguments: argument k is within([rmin:]rmax, h_idx[k]) [and a static selection], evaluated per frame on the device into an ascending
    // index list (md_script_functions.inl:2485-2720); the consumers read that list instead of the static one. A coordinate range (`range`:
    // within_x / _y / _z / _xyz, coordinate_range :2394) marks the atoms inside [lo, hi] instead, testing only the static side's atoms (d_and_idx)
    // when it has one; count() of a range is dyn[0] of its MDGPU_OP_WITHIN_COUNT property.
    struct DynArg {
        bool on = false; float rmin = 0.f, rmax = 0.f; DevBuf<uint8_t> d_and_mask;
        bool range = false; float lo[3] = {}, hi[3] = {}; DevBuf<int32_t> d_and_idx; bool has_and = false;
    } dyn[4];
    bool any_dyn() const { return dyn[0].on || dyn[1].on || dyn[2].on || dyn[3].on; }
    // device accumulators (the result accumulators are listed once, in for_each_accumulator)
    DevBuf<unsigned long long> d_acc;             // rdf: 1024 bins; density: 1024 fixed-point sums
    DevBuf<uint32_t> d_vol;                       // sdf: 128^3
    DevBuf<float> d_vol_mean; bool values_registered = false;   // sdf: device-side fold target; host values pinned for the D2H
    DevBuf<unsigned long long> d_frame_total;     // rdf / sdf: [num_frames]
    DevBuf<uint32_t> d_frame_min, d_frame_max;                     // rdf
    DevBuf<unsigned long long> d_frame_min64, d_frame_max64;       // density
    DevBuf<uint32_t> d_keep; DevBuf<unsigned long long> d_keep64;
    DevBuf<float> d_temporal;                     // [num_frames][len]
    size_t len = 1;                               // values per frame of a temporal (distance_pair: |a| * |b|)
    std::vector<float> agg_mean, agg_var, agg_ext;   // len > 1: per-frame mean / population variance / (min, max) (md_script_aggregate_t)
    // sdf statics
    DevBuf<int2> d_unwrap; uint32_t n_unwrap = 0;
    DevBuf<uint2> d_group_pairs;   // rmsd in contexts: per group (first pair in d_unwrap, pair count)
    // density statics (from the initial frame's cell)
    float rc = 0, re = 0, inv_ext = 0, min_point = 0; double dens_factor = 0;
    // results: `values` is the default storage; mdgpu_plan_bind_property_storage points vptr (and the aggregate rows) at the caller's arrays
    // (the md_script shim binds md_script_property_data_t::values, so results are written where VIAMD reads them)
    std::vector<float> values; mdgpu_property_data_t data{};
    float* vptr = nullptr; float* amean = nullptr; float* avar = nullptr; float* aext = nullptr;
    uint64_t frames_accumulated = 0;    // may be overridden after a cross-GPU reduction
    bool frames_overridden = false;
    bool is_density() const { return op >= MDGPU_OP_DENSITY_X && op <= MDGPU_OP_DENSITY_Z; }
    bool is_dist() const { return op == MDGPU_OP_RDF || is_density(); }
    bool needs_cells() const { return op == MDGPU_OP_RDF || op == MDGPU_OP_SDF || op == MDGPU_OP_CONTACT_COUNT; }
    DevBuf<uint32_t> d_set_of, d_excl_off;   // contact_count: set of every atom of the concatenated A list; CSR offsets of the sets' exclusion lists in idx[2]
    int share_trg = -1;   // index of an earlier property with the same target selection and cutoff: its target cell list is reused
    size_t trg_groups = 0;   // rdf: the target argument was an ARRAY of selections: one centre of mass per selection is the target point (h_goff[1] = their CSR offsets in idx[1])
    size_t backbone_segments = 0;   // MDGPU_OP_BACKBONE_ANGLES (evaluated as 2 dihedrals in context per segment): the segments of its (phi, psi) rows
    DevBuf<unsigned long long> d_frame_n;   // porosity: voxels of each frame's grid (N); d_frame_total holds the occupied ones
    size_t ss_segments = 0; DevBuf<uint32_t> d_ss_seg;   // MDGPU_OP_SECONDARY_STRUCTURE: segments; per segment its range id, range begin and range end

    // The result accumulators, each once: f(&Prop::member) in turn until one returns non-zero. They are zeroed by mdgpu_plan_clear, and
    // multi_sync sums them onto the root device (rows of frames a device did not evaluate are zero there) and zeroes them on the peers.
    // An accumulator that is missing here keeps its values across a clear and is never merged.
    template <typename F> static int for_each_accumulator(F&& f) {
        int rc = 0;
        auto one = [&](auto member) { if (!rc) rc = f(member); };
        one(&Prop::d_acc); one(&Prop::d_vol); one(&Prop::d_frame_total); one(&Prop::d_frame_n); one(&Prop::d_frame_min); one(&Prop::d_frame_max);
        one(&Prop::d_frame_min64); one(&Prop::d_frame_max64); one(&Prop::d_keep); one(&Prop::d_keep64); one(&Prop::d_temporal);
        return rc;
    }
};

// One within([rmin:]rmax, selection) query per frame of a batch: the system-wide grid and the cell lists of all atoms and of the selection
// (get_spatial_acc :734), the marks [B][num_atoms] and, for a dynamic argument, the per-frame index list (empty for count(within())).
// count over groups of atoms also takes one hit byte per group and frame (d_hits [B][n_groups]).
struct WithinScratch { DevBuf<FrameGeom> d_geom; DevBuf<float> d_aabb; CellListBuf trg, ref; DevBuf<uint8_t> d_flags; DevBuf<int32_t> d_idx; DevBuf<uint32_t> d_n; DevBuf<uint8_t> d_hits; };

struct PropScratch {   // per (stream slot, property)
    DevBuf<FrameGeom> d_geom; DevBuf<float> d_aabb;
    CellListBuf trg, ref;
    DevBuf<uint32_t> d_frame_bins; DevBuf<unsigned long long> d_frame_bins64;
    DevBuf<float4> d_sdf_xyzw; DevBuf<float> d_sdf_ref0, d_sdf_mats;
    DevBuf<float> d_com;       // rdf with centre-of-mass references: [B][n_struct][3]
    DevBuf<float> d_argpos;    // distance/angle/dihedral with selection arguments: [B][4][3]
    DevBuf<float> d_gpos[2];   // arguments that are arrays of selections: [B][n_groups][3] per argument
    DevBuf<float4> d_parts[4];   // array-of-selections arguments: [B][n_parts] centres (xyz, 1)
    WithinScratch within[4];   // the query of dynamic argument k; count(within()) is the query of its argument 0
    // rdf candidate lists (k_rdf_cull): [B][list stride] entries, [B][cap] headers, [B] cursors
    DevBuf<uint32_t> d_pair_list; DevBuf<uint4> d_list_hdr; DevBuf<uint32_t> d_list_cursor;
    mdgpu_unitcell_t nn_cell{}; size_t nn_stride = 0; bool nn_valid = false;   // candidate-list stride of the last cell seen (list sizing)
    // porosity: per sub-batch of PORO_FRAMES frames the spheres, grid headers, bit grids (zero between sub-batches) and occupied-voxel counters
    DevBuf<float4> d_poro_xyzr; DevBuf<PorosityHdr> d_poro_hdr; DevBuf<unsigned long long> d_poro_grid, d_poro_count;
    // secondary structure: per frame of a batch the segments' atoms and CA cells, the two recorded bonds of every donor, turn / bend bits and flags
    DevBuf<float> d_ss_res; DevBuf<float4> d_ss_hb; DevBuf<uint32_t> d_ss_bits;
};

struct Slot {
    Stream stream; Event done; bool busy = false;
    bool owned = false;                        // a caller thread holds the slot (acquire_slot / release_slot); guarded by mdgpu_plan::slot_mutex
    Event copied;                              // recorded after the batch's host->device copy: the caller's source buffer is free again
    PinnedBuf<int> h_err;                      // pinned mirror of d_err, copied at the end of every batch (read when the slot is retired)
    DevBuf<float> d_frames; PinnedBuf<float> h_frames;   // staging for host-resident frames (ingest atom space)
    DevBuf<float> d_xtc_frames;                          // whole decoded frames (XTC input)
    DevBuf<mdgpu_unitcell_t> d_cells; PinnedBuf<mdgpu_unitcell_t> h_cells;
    DevBuf<int> d_err;
    std::vector<PropScratch> ps;
    uint32_t pending_beg = 0, pending_cnt = 0;
};

// XTC input stage: compressed bytes + scan records of XTC_SUPER batches, scanned by ONE launch on the stage's own stream. The walk over a
// frame's stream is a latency-bound serial chain (one warp per frame), so its throughput comes from scanning many frames at once and from
// running two super-batches ahead of the expand + property kernels that consume it.
constexpr uint32_t XTC_SUPER_MAX = 8;
static uint32_t xtc_super() {   // batches per scan stage; MDGPU_XTC_SUPER overrides (tuning)
    static const uint32_t v = []() { const char* e = getenv("MDGPU_XTC_SUPER"); const long n = e ? atol(e) : 2; return (uint32_t)std::min<long>(std::max<long>(n, 1), XTC_SUPER_MAX); }();
    return v;
}
#define XTC_SUPER xtc_super()

constexpr uint32_t XTC_STAGES = 3;   // the scan of super-batch k+2 is in flight while the batches of k are expanded and evaluated
struct XtcStage {
    Stream stream; Event ready; Event consumed[XTC_SUPER_MAX]; uint32_t n_consumed = 0;
    DevBuf<uint8_t> d_blob; DevBuf<unsigned long long> d_off; PinnedBuf<unsigned long long> h_off;
    DevBuf<XtcFrameInfo> d_info; DevBuf<uint2> d_rec; DevBuf<uint16_t> d_state;
};

struct TimedLaunch { cudaEvent_t a, b; int kind; };   // kind: 0 rdf pair kernel, 1 sdf (all three kernels), 2 density (+finalize), 3 rdf cull kernel
constexpr int TIMED_KINDS = 4;

typedef struct ncclComm* nccl_comm_t;
struct NcclApi {
    void* lib = nullptr;
    int (*CommInitAll)(nccl_comm_t*, int, const int*) = nullptr;
    int (*CommDestroy)(nccl_comm_t) = nullptr;
    int (*GroupStart)() = nullptr; int (*GroupEnd)() = nullptr;
    int (*Reduce)(const void*, void*, size_t, int, int, int, nccl_comm_t, cudaStream_t) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
};
enum { NCCL_UINT32 = 3, NCCL_UINT64 = 5, NCCL_FLOAT32 = 7, NCCL_SUM = 0 };   // ncclDataType_t / ncclRedOp_t values (nccl.h)
template <typename T> constexpr int nccl_type() {
    static_assert(std::is_same<T, uint32_t>::value || std::is_same<T, unsigned long long>::value || std::is_same<T, float>::value, "no NCCL type");
    return std::is_same<T, uint32_t>::value ? NCCL_UINT32 : std::is_same<T, float>::value ? NCCL_FLOAT32 : NCCL_UINT64;
}

struct MultiDevice {
    std::vector<mdgpu_plan*> peers;    // devices[1..]; the root plan is devices[0]
    std::vector<int> devices;
    NcclApi nccl; std::vector<nccl_comm_t> comms;
    double last_reduce_ms = 0.0; uint64_t reduces = 0;
};


}  // namespace mdg

using namespace mdg;

struct IngestPool;
// The atoms of a frame as the kernels see them. SPACE_FULL: every atom of the system, global indices. SPACE_COMPACT: the union of the atoms any property reads,
// ascending: when it is well below the system size, host ingest copies only those atoms (gathered into pinned staging by the ingest threads) and the kernels run on index lists remapped into that space.
enum Space { SPACE_FULL = 0, SPACE_COMPACT = 1 };
struct AtomSpace {
    size_t num_atoms = 0, axis_stride = 0;   // staging layout: [frame][3][axis_stride]
    DevBuf<float> d_mass, d_init, d_radius;  // masses, the initial frame, van der Waals radii (porosity plans only)
};
struct mdgpu_plan {
    int device = 0; int sm_count = 132;
    size_t num_atoms = 0, num_frames = 0;    // of the system (= space[SPACE_FULL].num_atoms)
    uint32_t B = 132; uint32_t S = 2; uint32_t cell_cap = 0; bool keep = false; uint32_t rdf_variant = 0;
    std::vector<float> h_mass, h_radius; AtomSpace space[2];   // space[SPACE_FULL] is always filled, space[SPACE_COMPACT] only when `compact`
    bool compact = false; std::vector<int32_t> needed;   // host ingest copies only the `needed` atoms
    Space ingest_space() const { return compact ? SPACE_COMPACT : SPACE_FULL; }
    uint32_t ingest_mode = 0, ingest_threads = 0; IngestPool* pool = nullptr;
    std::vector<uint32_t> conn_off; std::vector<int32_t> conn_idx;
    std::vector<Prop> props;
    std::vector<Slot> slots;
    bool have_init = false; mdgpu_unitcell_t init_cell{};
    std::vector<uint64_t> frame_mask; std::mutex mask_mutex; std::mutex init_mutex;
    std::atomic<bool> interrupt{false};
    uint64_t next_slot = 0;
    // Concurrency (md_script_eval_frame_range is re-entrant on one eval from many threads with disjoint ranges, task_system.cpp:73-87):
    // a caller thread owns a slot (staging buffers + stream) while it holds the lease acquire_slot gave it; enqueue_batch runs under submit_mutex;
    // one fold at a time (sync_mutex).
    std::mutex slot_mutex; std::condition_variable slot_cv; std::mutex submit_mutex; std::mutex sync_mutex;
    mdgpu_progress_fn progress_fn = nullptr; void* progress_user = nullptr; Stream pub_stream;
    std::chrono::steady_clock::time_point last_pub{};
    bool timing = false; std::vector<TimedLaunch> timed; double timed_ms[TIMED_KINDS] = {0, 0, 0, 0}; uint64_t timed_n[TIMED_KINDS] = {0, 0, 0, 0}; DevBuf<unsigned long long> d_counters;
    Event t_begin; std::vector<Event> t_end;
    XtcStage xtc[XTC_STAGES]; uint64_t next_xtc = 0; std::mutex xtc_mutex;
    std::atomic<bool> dirty{true};   // device accumulators changed since the last fold into the host-visible property data
    std::atomic<uint64_t> frames_retired{0};   // frame evaluations of retired batches: the divisor of the running means
    mdg::MultiDevice* multi = nullptr;   // frame blocks on several GPUs from this one process (mdgpu_plan_options_t.num_devices > 1)
    // temporal expressions: their programs in one buffer, ordered by dependency level; level l is d_expr_progs[expr_level[l] .. expr_level[l+1]),
    // whose longest row has expr_level_len[l] values
    DevBuf<ExprNode> d_expr_nodes; DevBuf<ExprProg> d_expr_progs; std::vector<uint32_t> expr_level, expr_level_len;
};

// get_spatial_acc (md_script_functions.inl:734-760): the system-wide grid of within() has cells of ceil(radius / 6) * 6
static double within_cell_ext(float radius) { return ceil((double)radius / 6.0) * 6.0; }

// BFS order in which md_util_unwrap_vec4(xyzw, NULL, count, bond, cell) visits atoms (md_util.c:8738-8819). NB the reference
// walks the bonds of GLOBAL atoms 0..count-1 there (the local index is used as a global atom index); reproduced as is.
static void build_unwrap_pairs(std::vector<int2>& out, size_t count, const std::vector<uint32_t>& off, const std::vector<int32_t>& idx) {
    out.clear();
    if (count == 0 || off.size() < 2) return;
    const size_t atom_count = off.size() - 1;
    std::vector<char> visited(atom_count + 1, 0);
    std::vector<int> queue; queue.reserve(count + 1);
    for (size_t i = 0; i < count; ++i) {
        const int seed = (int)i;
        if ((size_t)seed >= atom_count || visited[seed]) continue;
        visited[seed] = 1; queue.clear(); queue.push_back(seed); size_t qh = 0;
        while (qh < queue.size()) {
            const int cur = queue[qh++];
            for (uint32_t k = off[cur]; k < off[cur + 1]; ++k) {
                const int next = idx[k];
                if (next < 0 || (size_t)next >= count || visited[next]) continue;
                out.push_back(make_int2(next, cur));
                visited[next] = 1; queue.push_back(next);
            }
        }
    }
}

// MIN / MAX of the reference (core/md_common.h:130-134): the second operand unless the first compares below / above it, so a NaN is taken
// (and dropped again by the next comparison)
static inline float ref_min(float a, float b) { return a < b ? a : b; }
static inline float ref_max(float a, float b) { return a > b ? a : b; }

// compute_min_max_mean_variance (md_script.c:5646-5677): min, max, mean and population variance of one frame's values, two passes in float
static void fold_frame_values(const float* v, size_t len, float& mn, float& mx, float& mean, float& var) {
    const float N = (float)len;
    mn = FLT_MAX; mx = -FLT_MAX; float s1 = 0.0f, s2 = 0.0f;
    for (size_t i = 0; i < len; ++i) { s1 += v[i]; mn = ref_min(mn, v[i]); mx = ref_max(mx, v[i]); }
    s1 = s1 / N;
    for (size_t i = 0; i < len; ++i) s2 += (v[i] - s1) * (v[i] - s1);
    s2 = s2 / N;
    mean = s1; var = s2;
}


// Host threads that gather the atoms a plan reads out of whole frames into pinned staging (and, for mdgpu_eval_trajectory, pull frames through
// the frame source). One parallel_for at a time; callers that arrive while it is busy run their items themselves.
struct IngestPool {
    std::vector<std::thread> th; std::mutex m, job_m; std::condition_variable cv, done_cv;
    std::function<void(uint32_t)> fn; uint32_t n = 0; std::atomic<uint32_t> next{0}; uint32_t active = 0, arrived = 0; uint64_t gen = 0; bool stop = false;
    explicit IngestPool(uint32_t threads) {
        for (uint32_t t = 0; t + 1 < threads; ++t) th.emplace_back([this]() {
            uint64_t seen = 0;
            for (;;) {
                { std::unique_lock<std::mutex> lk(m); cv.wait(lk, [&] { return stop || gen != seen; }); if (stop) return; seen = gen; ++active; ++arrived; }
                for (uint32_t i; (i = next.fetch_add(1)) < n; ) fn(i);
                { std::lock_guard<std::mutex> lk(m); --active; done_cv.notify_all(); }
            }
        });
    }
    ~IngestPool() { { std::lock_guard<std::mutex> lk(m); stop = true; } cv.notify_all(); for (auto& t : th) t.join(); }
    // every worker takes part in every job (and has left it before the call returns), so `fn` / `n` are never touched while a worker reads them
    void parallel_for(uint32_t count, const std::function<void(uint32_t)>& f) {
        if (count == 0) return;
        std::unique_lock<std::mutex> job(job_m, std::try_to_lock);
        if (!job.owns_lock() || th.empty() || count == 1) { for (uint32_t i = 0; i < count; ++i) f(i); return; }   // pool busy with another caller: that caller IS a thread
        { std::lock_guard<std::mutex> lk(m); fn = f; n = count; next = 0; arrived = 0; ++gen; }
        cv.notify_all();
        for (uint32_t i; (i = next.fetch_add(1)) < count; ) f(i);
        std::unique_lock<std::mutex> lk(m); done_cv.wait(lk, [&] { return arrived == (uint32_t)th.size() && active == 0; });
    }
};

static IngestPool* ingest_pool(mdgpu_plan* p) {
    std::lock_guard<std::mutex> guard(p->slot_mutex);
    if (!p->pool) {
        uint32_t t = p->ingest_threads;
        if (!t) { const char* e = getenv("MDGPU_INGEST_THREADS"); t = e ? (uint32_t)atoi(e) : 0; }
        if (!t) { const uint32_t hw = std::thread::hardware_concurrency(); t = std::min(16u, std::max(2u, hw / 2)); }
        p->pool = new IngestPool(std::min(t, 64u));
    }
    return p->pool;
}

// dst[j] = src[needed[j]] for one axis of one frame
static inline void gather_axis(float* __restrict__ dst, const float* __restrict__ src, const int32_t* __restrict__ idx, size_t n) {
    for (size_t j = 0; j < n; ++j) dst[j] = src[idx[j]];
}

static void destroy_multi(mdgpu_plan* p);
static void destroy_plan(mdgpu_plan* p) {
    if (!p) return;
    if (p->multi) destroy_multi(p);   // the peers, each with its own device current
    cudaSetDevice(p->device);         // the owners free this plan's buffers, streams and events on its device
    cudaDeviceSynchronize();
    for (auto& pr : p->props) if (pr.values_registered) cudaHostUnregister(pr.values.data());
    for (auto& t : p->timed) { cudaEventDestroy(t.a); cudaEventDestroy(t.b); }
    delete p->pool;
    delete p;
}

// CSR offsets off[0..n] of groups in a list of `size` entries start at 0, end at the list's size and do not decrease: "" or the error message
static std::string check_offsets(const uint32_t* off, size_t n, size_t size, const std::string& who, const char* noun, const char* list) {
    if (!off || off[0] != 0u || off[n] != size) return who + ": " + noun + " do not cover " + list;
    for (size_t g = 0; g < n; ++g) if (off[g] > off[g + 1]) return who + ": " + noun + " must be non-decreasing";
    return std::string();
}

// the num_structures groups of idx[0]: structure_offsets, or runs of structure_size atoms -> pr.h_soff, checked; "" or the error message
static std::string take_structures(Prop& pr, const mdgpu_property_desc_t& d, const std::string& who) {
    if (d.structure_offsets) pr.h_soff.assign(d.structure_offsets, d.structure_offsets + pr.n_struct + 1);
    else if (!pr.struct_size) return who + ": structure_size or structure_offsets required";
    else { pr.h_soff.resize(pr.n_struct + 1); for (size_t k = 0; k <= pr.n_struct; ++k) pr.h_soff[k] = (uint32_t)(k * pr.struct_size); }
    return check_offsets(pr.h_soff.data(), pr.n_struct, pr.h_idx[0].size(), who, "structure offsets", "idx[0]");
}

// count(x, 'residue' | 'chain' | 'structure'): the num_structures groups of idx[1] (structure_offsets, or runs of structure_size atoms) as the
// map atom -> group in pr.d_group_of; every atom in at most one group. "" or the error message (*e: a failed upload)
static std::string take_count_groups(Prop& pr, const mdgpu_property_desc_t& d, size_t num_atoms, cudaError_t* e) {
    const std::string who = "'" + pr.name + "'";
    const size_t n = d.num_structures;
    if (n >= (size_t)INT32_MAX) return who + ": too many groups";
    std::vector<uint32_t> off(n + 1);
    if (d.structure_offsets) off.assign(d.structure_offsets, d.structure_offsets + n + 1);
    else for (size_t k = 0; k <= n; ++k) off[k] = (uint32_t)(k * d.structure_size);
    const std::string er = check_offsets(off.data(), n, pr.h_idx[1].size(), who, "group offsets", "idx[1]"); if (!er.empty()) return er;
    std::vector<int32_t> group_of(num_atoms, -1);
    for (size_t g = 0; g < n; ++g)
        for (uint32_t j = off[g]; j < off[g + 1]; ++j) {
            int32_t& slot = group_of[(size_t)pr.h_idx[1][j]];   // in range: idx lists are checked when they are taken
            if (slot >= 0) return who + ": atom " + std::to_string(pr.h_idx[1][j]) + " is in two groups";
            slot = (int32_t)g;
        }
    pr.n_groups = (uint32_t)n; pr.count_groups = true;
    *e = pr.d_group_of.upload(group_of.data(), group_of.size());
    return std::string();
}

// a temporal of `len` values per frame: device rows, host values and, for len > 1, the per-frame aggregates (allocate_property_data :5618-5640)
static cudaError_t set_temporal(Prop& pr, size_t num_frames, size_t len) {
    pr.len = len;
    pr.values.assign(num_frames * len, 0.0f);
    if (len > 1) { pr.agg_mean.assign(num_frames, 0.0f); pr.agg_var.assign(num_frames, 0.0f); pr.agg_ext.assign(2 * num_frames, 0.0f); }
    pr.data.dim[0] = (int32_t)num_frames; pr.data.dim[1] = (int32_t)len; pr.data.dim[2] = 0; pr.data.dim[3] = 0;
    return pr.d_temporal.alloc(num_frames * len);
}

// a distribution (rdf, density): 1024 values followed by 1024 weights
static void set_distribution(Prop& pr) {
    pr.values.assign(2 * MDGPU_DIST_BINS, 0.0f);
    pr.data.dim[0] = 1; pr.data.dim[1] = 2; pr.data.dim[2] = MDGPU_DIST_BINS; pr.data.dim[3] = 0;
}

extern "C" {

const char* mdgpu_last_error(void) { return g_last_error.c_str(); }

int mdgpu_device_count(void) { int n = 0; if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; } return n; }

uint64_t mdgpu_launch_count(bool reset) { return reset ? g_launches.exchange(0) : g_launches.load(); }

mdgpu_plan* mdgpu_plan_create(const mdgpu_system_desc_t* sys, const mdgpu_property_desc_t* props, size_t num_props, size_t num_frames,
                              const mdgpu_plan_options_t* opts) {
    return mdgpu_plan_create_ex(sys, props, num_props, num_frames, opts, nullptr, 0, nullptr, 0);
}

mdgpu_plan* mdgpu_plan_create_with_ranges(const mdgpu_system_desc_t* sys, const mdgpu_property_desc_t* props, size_t num_props, size_t num_frames,
                                          const mdgpu_plan_options_t* opts, const mdgpu_range_arg_t* ranges, size_t num_ranges) {
    return mdgpu_plan_create_ex(sys, props, num_props, num_frames, opts, ranges, num_ranges, nullptr, 0);
}

}  // extern "C"

// The programs of the temporal expressions of a plan whose other properties are set up: checked (see mdgpu_plan_create_ex), each expression's
// values per frame from its operands, then the programs in dependency levels -> p->d_expr_*. "" or the error message (an invalid argument).
static std::string take_expressions(mdgpu_plan* p, const mdgpu_property_desc_t* props, size_t num_props, const mdgpu_expr_t* exprs, size_t num_exprs, cudaError_t& e) {
    std::vector<const mdgpu_expr_t*> prog(num_props, nullptr);
    for (size_t j = 0; j < num_exprs; ++j) {
        const mdgpu_expr_t& x = exprs[j];
        if (x.prop >= num_props || props[x.prop].op != MDGPU_OP_EXPRESSION) return "expression " + std::to_string(j) + ": property " + std::to_string(x.prop) + " is not an expression property";
        if (prog[x.prop]) return "property '" + p->props[x.prop].name + "' has more than one program";
        if (!x.num_nodes || !x.nodes) return "property '" + p->props[x.prop].name + "': empty program";
        prog[x.prop] = &x;
    }
    for (size_t i = 0; i < num_props; ++i) if (props[i].op == MDGPU_OP_EXPRESSION && !prog[i]) return "property '" + p->props[i].name + "' has no program";
    // operands first: depth-first over the expression operands, in topological order; 1 = on the current path (a cycle), 2 = placed
    std::vector<int> state(num_props, 0), level(num_props, 0); std::vector<uint32_t> order;
    std::string er;
    std::function<bool(uint32_t)> visit = [&](uint32_t i) -> bool {
        if (state[i] == 2) return true;
        if (state[i] == 1) { er = "expressions depend on each other in a cycle (through '" + p->props[i].name + "')"; return false; }
        state[i] = 1;
        const mdgpu_expr_t& x = *prog[i];
        for (size_t k = 0; k < x.num_nodes; ++k) {
            const mdgpu_expr_node_t& n = x.nodes[k];
            if (n.kind > MDGPU_EXPR_MAX) { er = "'" + p->props[i].name + "': unknown expression node kind " + std::to_string(n.kind); return false; }
            if (n.kind != MDGPU_EXPR_PROP) continue;
            if (n.prop >= num_props) { er = "'" + p->props[i].name + "': operand property " + std::to_string(n.prop) + " out of range"; return false; }
            if (n.prop == i) { er = "'" + p->props[i].name + "': an expression cannot name itself"; return false; }
            if (props[n.prop].op == MDGPU_OP_EXPRESSION) { if (!visit(n.prop)) return false; level[i] = std::max(level[i], level[n.prop] + 1); }
            else if (!p->props[n.prop].d_temporal.get()) { er = "'" + p->props[i].name + "': operand '" + p->props[n.prop].name + "' is not a temporal property"; return false; }
        }
        state[i] = 2; order.push_back(i);
        return true;
    };
    for (size_t i = 0; i < num_props; ++i) if (prog[i] && !visit((uint32_t)i)) return er;
    // value counts: a float is 0 on the stack of counts, an array its length (a temporal of one value per frame is a float)
    for (uint32_t i : order) {
        const mdgpu_expr_t& x = *prog[i]; const std::string who = "'" + p->props[i].name + "': ";
        std::vector<size_t> st;
        for (size_t k = 0; k < x.num_nodes; ++k) {
            const uint32_t kind = x.nodes[k].kind;
            if (kind == MDGPU_EXPR_CONST || kind == MDGPU_EXPR_PROP) {
                if (st.size() == MDGPU_EXPR_MAX_DEPTH) return who + "more than " + std::to_string(MDGPU_EXPR_MAX_DEPTH) + " operands on the stack";
                const size_t len = kind == MDGPU_EXPR_CONST ? 1 : p->props[x.nodes[k].prop].len;
                st.push_back(len > 1 ? len : 0);
                continue;
            }
            const bool binary = kind >= MDGPU_EXPR_ATAN2 || (kind >= MDGPU_EXPR_ADD && kind <= MDGPU_EXPR_DIV);
            if (st.size() < (binary ? 2u : 1u)) return who + "the program pops an empty stack";
            const bool elementwise = binary ? kind <= MDGPU_EXPR_DIV : (kind == MDGPU_EXPR_NEG || kind == MDGPU_EXPR_ABS || kind == MDGPU_EXPR_FLOOR || kind == MDGPU_EXPR_CEIL);
            const size_t b = st.back(), a = binary ? st[st.size() - 2] : 0;
            if (!elementwise && (a || b)) return who + "an array given to a function that takes floats only";
            if (a && b && a != b) return who + "arrays of different lengths (" + std::to_string(a) + " and " + std::to_string(b) + ")";
            if (binary) st.pop_back();
            st.back() = std::max(a, b);
        }
        if (st.size() != 1) return who + "the program leaves " + std::to_string(st.size()) + " values instead of one";
        if ((e = set_temporal(p->props[i], p->num_frames, st[0] ? st[0] : 1)) != cudaSuccess) return "";
    }
    std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return level[a] < level[b]; });
    std::vector<ExprNode> nodes; std::vector<ExprProg> progs;
    for (uint32_t i : order) {
        const mdgpu_expr_t& x = *prog[i];
        if (p->expr_level.size() <= (size_t)level[i]) { p->expr_level.push_back((uint32_t)progs.size()); p->expr_level_len.push_back(0); }
        p->expr_level_len[level[i]] = std::max(p->expr_level_len[level[i]], (uint32_t)p->props[i].len);
        progs.push_back(ExprProg{ (uint32_t)nodes.size(), (uint32_t)x.num_nodes, p->props[i].d_temporal.get(), (uint32_t)p->props[i].len });
        for (size_t k = 0; k < x.num_nodes; ++k) {
            const mdgpu_expr_node_t& n = x.nodes[k];
            const Prop* src = n.kind == MDGPU_EXPR_PROP ? &p->props[n.prop] : nullptr;
            nodes.push_back(ExprNode{ n.kind, n.value, src ? src->d_temporal.get() : nullptr, src ? (uint32_t)src->len : 0u });
        }
    }
    p->expr_level.push_back((uint32_t)progs.size());
    if ((e = p->d_expr_nodes.upload(nodes.data(), nodes.size())) != cudaSuccess) return "";
    e = p->d_expr_progs.upload(progs.data(), progs.size());
    return "";
}

extern "C" {

mdgpu_plan* mdgpu_plan_create_ex(const mdgpu_system_desc_t* sys, const mdgpu_property_desc_t* props, size_t num_props, size_t num_frames,
                                 const mdgpu_plan_options_t* opts, const mdgpu_range_arg_t* ranges, size_t num_ranges, const mdgpu_expr_t* exprs, size_t num_exprs) {
    if (!sys || !props || !num_props || !num_frames || !sys->num_atoms || (num_ranges && !ranges) || (num_exprs && !exprs)) { fail(MDGPU_ERR_INVALID_ARG, "mdgpu_plan_create: invalid arguments"); return nullptr; }
    // the coordinate range of each (property, argument), if any
    std::vector<std::array<const mdgpu_range_arg_t*, 4>> range_of(num_props, std::array<const mdgpu_range_arg_t*, 4>{});
    for (size_t r = 0; r < num_ranges; ++r) {
        const mdgpu_range_arg_t& ra = ranges[r];
        if (ra.prop >= num_props || ra.arg >= 4) { fail(MDGPU_ERR_INVALID_ARG, "coordinate range %zu: property %u / argument %u out of range", r, ra.prop, ra.arg); return nullptr; }
        if (range_of[ra.prop][ra.arg]) { fail(MDGPU_ERR_INVALID_ARG, "coordinate range %zu: argument %u of property %u has two ranges", r, ra.arg, ra.prop); return nullptr; }
        range_of[ra.prop][ra.arg] = &ra;
    }
    mdgpu_plan_options_t o{}; if (opts) o = *opts;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { fail(MDGPU_ERR_CUDA, "no CUDA device available (libmdgpu has no CPU fallback)"); return nullptr; }
    if (o.num_devices > 1) {   // one process, several GPUs: the root plan on devices[0] + one peer plan per further device
        if (o.num_devices > 16) { fail(MDGPU_ERR_INVALID_ARG, "at most 16 devices per plan"); return nullptr; }
        for (uint32_t g = 0; g < o.num_devices; ++g) {
            if (o.devices[g] < 0 || o.devices[g] >= ndev) { fail(MDGPU_ERR_INVALID_ARG, "device %d out of range (%d devices)", o.devices[g], ndev); return nullptr; }
            // (NCCL refuses two ranks on one device; MDGPU_ALLOW_DUPLICATE_DEVICES is for the loopback exchange of the test suite on a one-GPU machine)
            if (!getenv("MDGPU_ALLOW_DUPLICATE_DEVICES")) for (uint32_t h = 0; h < g; ++h) if (o.devices[h] == o.devices[g]) { fail(MDGPU_ERR_INVALID_ARG, "device %d listed twice", o.devices[g]); return nullptr; }
        }
        mdgpu_plan_options_t one = o; one.num_devices = 0; one.device = o.devices[0];
        mdgpu_plan* root = mdgpu_plan_create_ex(sys, props, num_props, num_frames, &one, ranges, num_ranges, exprs, num_exprs);
        if (!root) return nullptr;
        root->multi = new MultiDevice(); root->multi->devices.assign(o.devices, o.devices + o.num_devices);
        for (uint32_t g = 1; g < o.num_devices; ++g) {
            one.device = o.devices[g];
            mdgpu_plan* q = mdgpu_plan_create_ex(sys, props, num_props, num_frames, &one, ranges, num_ranges, exprs, num_exprs);
            if (!q) { destroy_plan(root); return nullptr; }
            root->multi->peers.push_back(q);
        }
        return root;
    }
    if (o.device < 0 || o.device >= ndev) { fail(MDGPU_ERR_INVALID_ARG, "device %d out of range (%d devices)", o.device, ndev); return nullptr; }
    if (cudaSetDevice(o.device) != cudaSuccess) { fail(MDGPU_ERR_CUDA, "cudaSetDevice(%d) failed", o.device); return nullptr; }
    mdgpu_plan* p = new mdgpu_plan();
    p->device = o.device;
    cudaDeviceGetAttribute(&p->sm_count, cudaDevAttrMultiProcessorCount, o.device);
    p->num_atoms = sys->num_atoms; p->num_frames = num_frames;
    AtomSpace& full = p->space[SPACE_FULL];
    full.num_atoms = sys->num_atoms; full.axis_stride = (sys->num_atoms + 3) & ~(size_t)3;
    p->B = o.batch_frames ? o.batch_frames : (uint32_t)p->sm_count;
    if (p->B > 4096) p->B = 4096;
    // 6 slots: the gather + H2D of the batches ahead overlap the kernels of the ones in flight; 2 leave the copy engine idle
    p->S = o.num_streams ? o.num_streams : 6; if (p->S > 8) p->S = 8;
    p->keep = o.keep_frame_results != 0; p->cell_cap = o.cell_capacity; p->rdf_variant = o.rdf_variant;
    p->ingest_mode = o.ingest_mode; p->ingest_threads = o.ingest_threads;
    p->h_mass.assign(sys->num_atoms, 1.0f);
    if (sys->atom_mass) memcpy(p->h_mass.data(), sys->atom_mass, sizeof(float) * sys->num_atoms);
    if (sys->bond_conn_offset && sys->bond_conn_offset_count) {
        p->conn_off.assign(sys->bond_conn_offset, sys->bond_conn_offset + sys->bond_conn_offset_count);
        const size_t nconn = p->conn_off.back();
        if (sys->bond_conn_atom_idx) p->conn_idx.assign(sys->bond_conn_atom_idx, sys->bond_conn_atom_idx + nconn);
    }
    auto bail = [&](int code, const std::string& msg) -> mdgpu_plan* { fail(code, "%s", msg.c_str()); destroy_plan(p); return nullptr; };
    // argument k given as an ARRAY of n selections, one position (centre of mass) per selection: their CSR offsets in idx[k] -> h_goff[k] / d_goff[k].
    // `who`, `role`, `noun` and `list` word the messages for the site; 0 and "", or the error code and its message
    auto take_group = [&](Prop& pr, int k, const uint32_t* off, size_t n, const std::string& who, const char* role, const char* noun, const char* list, std::string& er) -> int {
        if (pr.dyn[k].on) { er = who + ": an array of selections cannot be a dynamic " + role; return MDGPU_ERR_INVALID_ARG; }
        er = check_offsets(off, n, pr.h_idx[k].size(), who, noun, list); if (!er.empty()) return MDGPU_ERR_INVALID_ARG;
        pr.h_goff[k].assign(off, off + n + 1);
        if (pr.d_goff[k].upload(pr.h_goff[k].data(), pr.h_goff[k].size()) != cudaSuccess) { er = std::string("device allocation failed (") + noun + ")"; return MDGPU_ERR_CUDA; }
        return 0;
    };
    // arguments 0 / 1 of distance_pair / distance_min / _max and argument 0 of coord_* / plane given as arrays of selections: CSR offsets in structure_offsets
    // (argument 0, num_structures groups) / structure_offsets_b (argument 1); cnt[k] = positions of argument k. "" or the message (their callers report every failure as an invalid argument)
    auto take_groups = [&](Prop& pr, const mdgpu_property_desc_t& d, size_t cnt[2]) -> std::string {
        const uint32_t* goff[2] = { d.structure_offsets, d.structure_offsets_b }; const size_t gn[2] = { d.num_structures, d.num_structures_b };
        for (int k = 0; k < 2; ++k) {
            cnt[k] = gn[k] ? gn[k] : pr.h_idx[k].size();
            std::string er; if (gn[k] && take_group(pr, k, goff[k], gn[k], "'" + pr.name + "'", "argument", "group offsets", "the index list", er)) return er;
        }
        pr.n_struct = 0;   // num_structures described argument 0's groups here, not structures
        return std::string();
    };
    // `selection and within(...)`: one byte per atom, 1 for the n atoms of the static side -> d_mask; false after bail()
    auto take_and_mask = [&](Prop& pr, DevBuf<uint8_t>& d_mask, const int32_t* idx, size_t n) -> bool {
        std::vector<uint8_t> m(sys->num_atoms, 0);
        for (size_t j = 0; j < n; ++j) { const int32_t a = idx[j]; if (a < 0 || (size_t)a >= sys->num_atoms) { bail(MDGPU_ERR_INVALID_ARG, "property '" + pr.name + "': atom index out of range"); return false; } m[(size_t)a] = 1; }
        if (d_mask.upload(m.data(), m.size()) != cudaSuccess) { bail(MDGPU_ERR_CUDA, "device allocation failed (selection mask)"); return false; }
        return true;
    };
    // argument k of distance / angle / dihedral / com given as an ARRAY of selections (arg_parts[k] >= 2): idx[k] holds them back to back
    auto take_arg_parts = [&](Prop& pr, const mdgpu_property_desc_t& d, int k) -> std::string {
        const uint32_t n = d.arg_parts[k]; const uint32_t* off = d.arg_offsets[k];
        if (pr.dyn[k].on) return "'" + pr.name + "': an array of selections cannot be a dynamic argument";
        const std::string er = check_offsets(off, n, pr.h_idx[k].size(), "'" + pr.name + "'", "argument offsets", "the index list"); if (!er.empty()) return er;
        pr.h_aoff[k].assign(off, off + n + 1);
        if (pr.d_aoff[k].upload(pr.h_aoff[k].data(), pr.h_aoff[k].size()) != cudaSuccess) return "device allocation failed (argument offsets)";
        pr.com_mask |= 1u << k;
        return std::string();
    };
    if (full.d_mass.upload(p->h_mass.data(), p->h_mass.size()) != cudaSuccess) return bail(MDGPU_ERR_CUDA, "device allocation failed (masses)");
    for (size_t i = 0; i < num_props; ++i) if (props[i].op == MDGPU_OP_POROSITY) {   // porosity voxelises van der Waals spheres: the radii are required
        if (!sys->atom_radius) return bail(MDGPU_ERR_INVALID_ARG, "porosity: the system description has no atom radii (mdgpu_system_desc_t.atom_radius)");
        p->h_radius.assign(sys->atom_radius, sys->atom_radius + sys->num_atoms);
        for (size_t a = 0; a < sys->num_atoms; ++a) if (!(p->h_radius[a] >= 0.0f && p->h_radius[a] <= FLT_MAX)) return bail(MDGPU_ERR_INVALID_ARG, "porosity: atom radius " + std::to_string(a) + " is negative or not finite");
        if (full.d_radius.upload(p->h_radius.data(), p->h_radius.size()) != cudaSuccess) return bail(MDGPU_ERR_CUDA, "device allocation failed (radii)");
        break;
    }

    p->props.resize(num_props);
    for (size_t i = 0; i < num_props; ++i) {
        Prop& pr = p->props[i]; const mdgpu_property_desc_t& d = props[i];
        pr.name = d.name ? d.name : ("prop" + std::to_string(i)); pr.op = d.op;
        pr.n_struct = d.num_structures; pr.struct_size = d.structure_size; pr.cutoff_min = d.cutoff_min; pr.cutoff_max = d.cutoff_max;
        for (int k = 0; k < 4; ++k) {
            if (d.idx[k] && d.idx_count[k]) {
                pr.h_idx[k].assign(d.idx[k], d.idx[k] + d.idx_count[k]);
                for (int32_t a : pr.h_idx[k]) if ((a < 0 && !((pr.op == MDGPU_OP_BACKBONE_ANGLES || pr.op == MDGPU_OP_SECONDARY_STRUCTURE) && a == -1)) || (a >= 0 && (size_t)a >= sys->num_atoms)) return bail(MDGPU_ERR_INVALID_ARG, "property '" + pr.name + "': atom index out of range");
                if (pr.d_idx[SPACE_FULL][k].upload(pr.h_idx[k].data(), pr.h_idx[k].size()) != cudaSuccess) return bail(MDGPU_ERR_CUDA, "device allocation failed (indices)");
            }
        }
        {   // dynamic arguments (dyn[k]); rdf's round-1 spelling ref_within_radius + com_args bit 0 + idx[2] becomes dyn[0]
            mdgpu_dynamic_arg_t da[4]; for (int k = 0; k < 4; ++k) da[k] = d.dyn[k];
            if (pr.op == MDGPU_OP_RDF && d.ref_within_radius > 0.0f && !(da[0].radius_max > 0.0f)) {
                da[0].radius_min = d.ref_within_min; da[0].radius_max = d.ref_within_radius; da[0].has_and = d.com_args & 1u;
                da[0].and_idx = d.idx[2]; da[0].and_count = d.idx_count[2];
            }
            for (int k = 0; k < 4; ++k) {
                const mdgpu_range_arg_t* rng = range_of[i][k];
                const bool range = rng != nullptr;
                if (!range && !(da[k].radius_max > 0.0f && pr.op != MDGPU_OP_WITHIN_COUNT)) continue;
                const bool ok_op = (pr.op == MDGPU_OP_RDF && k < 2) || (pr.op == MDGPU_OP_SDF && k == 1) || (pr.is_density() && k == 0) ||
                                   ((pr.op == MDGPU_OP_DISTANCE || pr.op == MDGPU_OP_ANGLE || pr.op == MDGPU_OP_DIHEDRAL) && !d.num_structures) || (pr.op == MDGPU_OP_COM && k == 0) ||
                                   ((pr.op == MDGPU_OP_DISTANCE_MIN || pr.op == MDGPU_OP_DISTANCE_MAX) && k < 2) || (range && pr.op == MDGPU_OP_WITHIN_COUNT && k == 0);
                if (!ok_op) return bail(MDGPU_ERR_UNSUPPORTED, "property '" + pr.name + "': a dynamic selection is not lowered as argument " + std::to_string(k) + " of this procedure");
                if (range) {
                    if (da[k].radius_min != 0.0f || da[k].radius_max != 0.0f || (pr.op == MDGPU_OP_WITHIN_COUNT && (pr.cutoff_min != 0.0f || pr.cutoff_max != 0.0f)))
                        return bail(MDGPU_ERR_INVALID_ARG, "'" + pr.name + "': argument " + std::to_string(k) + " has both a radius and a coordinate range");
                    if (!pr.h_idx[k].empty()) return bail(MDGPU_ERR_INVALID_ARG, "'" + pr.name + "': a coordinate range takes no selection in idx[" + std::to_string(k) + "]");
                    for (int c = 0; c < 3; ++c)
                        if (!(rng->lo[c] <= rng->hi[c])) return bail(MDGPU_ERR_INVALID_ARG, "'" + pr.name + "': invalid coordinate range (lower bound above the upper one, or NaN)");
                    Prop::DynArg& dy = pr.dyn[k];
                    dy.on = true; dy.range = true; dy.has_and = da[k].has_and != 0;
                    for (int c = 0; c < 3; ++c) { dy.lo[c] = rng->lo[c]; dy.hi[c] = rng->hi[c]; }
                    if (dy.has_and) {   // the static side as an index list: the mark kernel tests only these atoms
                        for (size_t j = 0; j < da[k].and_count; ++j) if (da[k].and_idx[j] < 0 || (size_t)da[k].and_idx[j] >= sys->num_atoms) return bail(MDGPU_ERR_INVALID_ARG, "property '" + pr.name + "': atom index out of range");
                        if (da[k].and_count && dy.d_and_idx.upload(da[k].and_idx, da[k].and_count) != cudaSuccess) return bail(MDGPU_ERR_CUDA, "device allocation failed (selection list)");
                    }
                    continue;
                }
                if (da[k].radius_min < 0.0f || da[k].radius_max < da[k].radius_min) return bail(MDGPU_ERR_INVALID_ARG, "'" + pr.name + "': The supplied radius range is invalid");   // :2654
                pr.dyn[k].on = true; pr.dyn[k].rmin = da[k].radius_min; pr.dyn[k].rmax = da[k].radius_max;
                if (da[k].has_and && !take_and_mask(pr, pr.dyn[k].d_and_mask, da[k].and_idx, da[k].and_count)) return nullptr;
            }
        }
        if (pr.op == MDGPU_OP_WITHIN_COUNT && (d.com_args & 1u) && !take_and_mask(pr, pr.d_and_mask, pr.h_idx[2].data(), pr.h_idx[2].size())) return nullptr;   // idx[2] = static side of `sel and within(...)`
        cudaError_t e = cudaSuccess;
        switch (pr.op) {
        case MDGPU_OP_RDF:
            if (pr.h_idx[0].empty() && !pr.dyn[0].on) return bail(MDGPU_ERR_INVALID_ARG, "rdf '" + pr.name + "': empty reference positions");   // internal_rdf :5396-5403
            if (pr.h_idx[1].empty() && !pr.dyn[1].on) return bail(MDGPU_ERR_INVALID_ARG, "rdf '" + pr.name + "': empty target positions");
            if (pr.cutoff_min < 0.0f || pr.cutoff_max <= pr.cutoff_min) return bail(MDGPU_ERR_INVALID_ARG, "rdf '" + pr.name + "': Invalid cutoff");
            if (d.ref_within_radius < 0.0f || (pr.dyn[0].on && pr.n_struct) || d.ref_within_min < 0.0f) return bail(MDGPU_ERR_INVALID_ARG, "rdf '" + pr.name + "': invalid within() reference");
            if (pr.n_struct) {   // references = centres of mass of atom groups, a group's own atoms excluded (compute_rdf :5274-5275)
                const std::string er = take_structures(pr, d, "rdf '" + pr.name + "'"); if (!er.empty()) return bail(MDGPU_ERR_INVALID_ARG, er);
                if (pr.d_soff.upload(pr.h_soff.data(), pr.h_soff.size()) != cudaSuccess) return bail(MDGPU_ERR_CUDA, "device allocation failed (structure offsets)");
            }
            if (d.num_structures_b) {   // targets = centres of mass of atom groups (coordinate_extract :1503 -> extract_com :857 on an array of selections, compute_rdf :5293-5302)
                std::string er; const int code = take_group(pr, 1, d.structure_offsets_b, d.num_structures_b, "rdf '" + pr.name + "'", "target", "target group offsets", "idx[1]", er);
                if (code) return bail(code, er);
                pr.trg_groups = d.num_structures_b;
            }
            e = pr.d_acc.alloc(MDGPU_DIST_BINS);
            if (e == cudaSuccess) e = pr.d_frame_total.alloc(num_frames);
            if (e == cudaSuccess) e = pr.d_frame_min.alloc(num_frames);
            if (e == cudaSuccess) e = pr.d_frame_max.alloc(num_frames);
            if (e == cudaSuccess && p->keep) e = pr.d_keep.alloc(num_frames * MDGPU_DIST_BINS);
            set_distribution(pr);
            break;
        case MDGPU_OP_SDF: {
            if (!pr.n_struct || !pr.struct_size || pr.h_idx[0].size() != pr.n_struct * pr.struct_size)
                return bail(MDGPU_ERR_INVALID_ARG, "sdf '" + pr.name + "': reference structures must be num_structures x structure_size atoms");
            // a structure is an atom set (the reference passes bitfields): k_sdf_scatter excludes its atoms as one run when the first and last
            // index span exactly structure_size atoms, which holds for contiguous rows only if they are strictly ascending
            for (size_t s = 0; s < pr.n_struct; ++s) {
                const int32_t* row = pr.h_idx[0].data() + s * pr.struct_size;
                for (size_t k = 1; k < pr.struct_size; ++k)
                    if (row[k] <= row[k - 1])
                        return bail(MDGPU_ERR_INVALID_ARG, "sdf '" + pr.name + "': the atoms of reference structure " + std::to_string(s) + " are not strictly ascending");
            }
            if (pr.h_idx[1].empty() && !pr.dyn[1].on) return bail(MDGPU_ERR_INVALID_ARG, "sdf '" + pr.name + "': The supplied target bitfield is empty");
            if (p->conn_off.empty()) return bail(MDGPU_ERR_INVALID_ARG, "sdf '" + pr.name + "': Missing bond connectivity");   // md_util.c:8746
            std::vector<int2> pairs; build_unwrap_pairs(pairs, pr.struct_size, p->conn_off, p->conn_idx);
            pr.n_unwrap = (uint32_t)pairs.size();
            e = pr.d_unwrap.upload(pairs.data(), pairs.size());
            if (e == cudaSuccess) e = pr.d_vol.alloc((size_t)MDGPU_VOL_DIM * MDGPU_VOL_DIM * MDGPU_VOL_DIM);
            if (e == cudaSuccess) e = pr.d_vol_mean.alloc((size_t)MDGPU_VOL_DIM * MDGPU_VOL_DIM * MDGPU_VOL_DIM);
            if (e == cudaSuccess) e = pr.d_frame_total.alloc(num_frames);
            pr.values.assign((size_t)MDGPU_VOL_DIM * MDGPU_VOL_DIM * MDGPU_VOL_DIM, 0.0f);
            if (cudaHostRegister(pr.values.data(), pr.values.size() * sizeof(float), cudaHostRegisterDefault) == cudaSuccess) pr.values_registered = true; else cudaGetLastError();
            pr.data.dim[0] = 1; pr.data.dim[1] = MDGPU_VOL_DIM; pr.data.dim[2] = MDGPU_VOL_DIM; pr.data.dim[3] = MDGPU_VOL_DIM;
            break; }
        case MDGPU_OP_DENSITY_X: case MDGPU_OP_DENSITY_Y: case MDGPU_OP_DENSITY_Z:
            if (pr.h_idx[0].empty() && !pr.dyn[0].on) return bail(MDGPU_ERR_INVALID_ARG, "density '" + pr.name + "': empty selection");
            e = pr.d_acc.alloc(MDGPU_DIST_BINS);
            if (e == cudaSuccess) e = pr.d_frame_min64.alloc(num_frames);
            if (e == cudaSuccess) e = pr.d_frame_max64.alloc(num_frames);
            if (e == cudaSuccess && p->keep) e = pr.d_keep64.alloc(num_frames * MDGPU_DIST_BINS);
            set_distribution(pr);
            break;
        case MDGPU_OP_DISTANCE_MIN: case MDGPU_OP_DISTANCE_MAX:
            if ((pr.h_idx[0].empty() && !pr.dyn[0].on) || (pr.h_idx[1].empty() && !pr.dyn[1].on)) return bail(MDGPU_ERR_INVALID_ARG, "'" + pr.name + "': empty argument");
            { size_t cnt[2]; const std::string er = take_groups(pr, d, cnt); if (!er.empty()) return bail(MDGPU_ERR_INVALID_ARG, er); }   // arrays of selections: one centre of mass per selection
            e = set_temporal(pr, num_frames, 1);
            break;
        case MDGPU_OP_DISTANCE: case MDGPU_OP_ANGLE: case MDGPU_OP_DIHEDRAL: {
            const int need = pr.op == MDGPU_OP_DISTANCE ? 2 : (pr.op == MDGPU_OP_ANGLE ? 3 : 4);
            if (pr.n_struct) {   // `expr in contexts` (evaluate_context md_script.c:3418): idx[k][c] = argument k's atom in context c, one value per context
                // an argument that is a selection: idx[k] = the atoms of (selection AND context c) for every context back to back, arg_offsets[k] their
                // n_contexts + 1 offsets (arg_parts[k] == num_structures); its position in context c is that group's centre of mass
                // (coordinate_extract_com with ctx->mol_ctx, md_script_functions.inl:1812-1823). Integer arguments: one atom per context.
                for (int k = 0; k < need; ++k) {
                    if (d.arg_parts[k]) {
                        if (d.arg_parts[k] != pr.n_struct) return bail(MDGPU_ERR_INVALID_ARG, "'" + pr.name + "': one group of atoms per context expected for a selection argument");
                        const std::string er = take_arg_parts(pr, d, k); if (!er.empty()) return bail(MDGPU_ERR_INVALID_ARG, er);
                    } else if (pr.h_idx[k].size() != pr.n_struct) return bail(MDGPU_ERR_INVALID_ARG, "'" + pr.name + "': one atom per context and argument expected");
                }
                e = set_temporal(pr, num_frames, pr.n_struct);
                break;
            }
            pr.com_mask = d.com_args & ((1u << need) - 1u);
            for (int k = 0; k < need; ++k) if (d.arg_parts[k] > 1u) { const std::string er = take_arg_parts(pr, d, k); if (!er.empty()) return bail(MDGPU_ERR_INVALID_ARG, er); }
            for (int k = 0; k < need; ++k) {
                if (pr.dyn[k].on) { pr.com_mask |= 1u << k; continue; }   // a dynamic selection is a bitfield: its centre of mass
                if (pr.h_idx[k].empty()) return bail(MDGPU_ERR_INVALID_ARG, "'" + pr.name + "': empty argument");
                if (pr.h_idx[k].size() != 1) pr.com_mask |= 1u << k;   // several indices: centre of mass (coordinate_extract_com :1759)
            }
            e = set_temporal(pr, num_frames, 1);
            break; }
        case MDGPU_OP_DISTANCE_PAIR: {
            if (pr.h_idx[0].empty() || pr.h_idx[1].empty()) return bail(MDGPU_ERR_INVALID_ARG, "'" + pr.name + "': empty argument");
            // an argument that was an ARRAY of selections contributes one position per selection: extract_com (:857, no periodic treatment; coordinate_extract :1503)
            size_t cnt[2];
            { const std::string er = take_groups(pr, d, cnt); if (!er.empty()) return bail(MDGPU_ERR_INVALID_ARG, er); }
            const size_t len = cnt[0] * cnt[1];
            if (len > 1000000) return bail(MDGPU_ERR_INVALID_ARG, "'" + pr.name + "': The size produced by the operation is " + std::to_string(len) + ", which exceeds the upper limit of 1'000'000");   // :4056
            e = set_temporal(pr, num_frames, len);
            break; }
        case MDGPU_OP_WITHIN_COUNT:   // count(within(radius, selection)); an empty selection is valid (nothing is within reach of nothing). count(<range>): dyn[0]
            if (d.com_args & 2u) {   // count(x, 'residue' | 'chain' | 'structure'): the groups in idx[1]
                const std::string er = take_count_groups(pr, d, sys->num_atoms, &e); if (!er.empty()) return bail(MDGPU_ERR_INVALID_ARG, er);
                if (e != cudaSuccess) return bail(MDGPU_ERR_CUDA, "device allocation failed (atom groups)");
            }
            if (pr.dyn[0].range) { e = set_temporal(pr, num_frames, 1); break; }
            if (!(pr.cutoff_max > 0.0f)) return bail(MDGPU_ERR_INVALID_ARG, "'" + pr.name + "': The supplied radius is negative or zero, please supply a positive value");   // :2528
            if (pr.cutoff_min < 0.0f || pr.cutoff_max < pr.cutoff_min) return bail(MDGPU_ERR_INVALID_ARG, "'" + pr.name + "': The supplied radius range is invalid");          // :2654
            e = set_temporal(pr, num_frames, 1);
            break;
        case MDGPU_OP_SHAPE_WEIGHTS: {   // shape weights of n structures: [F, n*3]; groups as for rdf's centre-of-mass references
            if (!pr.n_struct || pr.h_idx[0].empty()) return bail(MDGPU_ERR_INVALID_ARG, "'" + pr.name + "': No structures present");   // shapespace.cpp:371
            { const std::string er = take_structures(pr, d, "'" + pr.name + "'"); if (!er.empty()) return bail(MDGPU_ERR_INVALID_ARG, er); }
            if (pr.d_soff.upload(pr.h_soff.data(), pr.h_soff.size()) != cudaSuccess) return bail(MDGPU_ERR_CUDA, "device allocation failed (structure offsets)");
            pr.com_mask = d.com_args & 1u;   // bit 0: weights are the atom masses (else 1)
            e = set_temporal(pr, num_frames, 3 * pr.n_struct);
            break; }
        case MDGPU_OP_COORD_X: case MDGPU_OP_COORD_Y: case MDGPU_OP_COORD_Z:   // coord_x/_y/_z(selection): [F, n]
            if (pr.h_idx[0].empty()) return bail(MDGPU_ERR_INVALID_ARG, "'" + pr.name + "': empty argument");
            { size_t cnt[2]; const std::string er = take_groups(pr, d, cnt); if (!er.empty()) return bail(MDGPU_ERR_INVALID_ARG, er);   // an array of selections: one value per selection
              e = set_temporal(pr, num_frames, cnt[0]); }
            break;
        case MDGPU_OP_COM: {   // com(x): a [F, 3] temporal (TI_FLOAT3)
            if (pr.h_idx[0].empty() && !pr.dyn[0].on) return bail(MDGPU_ERR_INVALID_ARG, "'" + pr.name + "': empty argument");
            pr.com_mask = (d.com_args & 1u) | (pr.h_idx[0].size() != 1 ? 1u : 0u) | (pr.dyn[0].on ? 1u : 0u);
            if (d.arg_parts[0] > 1u) { const std::string er = take_arg_parts(pr, d, 0); if (!er.empty()) return bail(MDGPU_ERR_INVALID_ARG, er); }
            e = set_temporal(pr, num_frames, 3);
            break; }
        case MDGPU_OP_PLANE: {   // plane(selection): a [F, 4] temporal (TI_FLOAT4)
            size_t cnt[2];   // an array of selections: its positions are the selections' centres of mass (coordinate_extract :1503)
            { const std::string er = take_groups(pr, d, cnt); if (!er.empty()) return bail(MDGPU_ERR_INVALID_ARG, er); }
            if (cnt[0] < 3) return bail(MDGPU_ERR_INVALID_ARG, "'" + pr.name + "': Invalid number of positions, need at least 3 to compute a plane");   // :4815
            // md_util_unwrap_vec4 is called without indices (:4771): position i is unwrapped along the bonds of ATOM i, whatever was selected — as written
            std::vector<int2> pairs; build_unwrap_pairs(pairs, cnt[0], p->conn_off, p->conn_idx);
            pr.n_unwrap = (uint32_t)pairs.size();
            e = pr.d_unwrap.upload(pairs.data(), pairs.size());
            if (e == cudaSuccess) e = set_temporal(pr, num_frames, 4);
            break; }
        case MDGPU_OP_CONTACT_COUNT: {   // contact_count(A[], B, cutoff): per set the pairs (a in A_i, b in B) within the cutoff, b outside the set's exclusion list
            if (!pr.n_struct || pr.h_idx[0].empty()) return bail(MDGPU_ERR_INVALID_ARG, "'" + pr.name + "': no sets");
            if (pr.n_struct > MDGPU_DIST_BINS) return bail(MDGPU_ERR_UNSUPPORTED, "'" + pr.name + "': more than 1024 sets");
            if (!(pr.cutoff_max > 0.0f)) return bail(MDGPU_ERR_INVALID_ARG, "'" + pr.name + "': The cutoff distance must be positive.");   // :2862
            if (pr.h_idx[1].empty()) return bail(MDGPU_ERR_INVALID_ARG, "'" + pr.name + "': empty second set");
            { const std::string er = take_structures(pr, d, "'" + pr.name + "'"); if (!er.empty()) return bail(MDGPU_ERR_INVALID_ARG, er); }
            std::vector<uint32_t> set_of(pr.h_idx[0].size());
            for (size_t k = 0; k < pr.n_struct; ++k) for (uint32_t j = pr.h_soff[k]; j < pr.h_soff[k + 1]; ++j) set_of[j] = (uint32_t)k;
            // exclusion lists (A_i & B grown along the bonds, md_util_mask_grow_by_bonds): CSR in idx[2] / structure_offsets_b, empty when absent
            std::vector<uint32_t> excl_off(pr.n_struct + 1, 0u);
            if (d.structure_offsets_b) { if (d.num_structures_b != pr.n_struct || d.structure_offsets_b[0] != 0 || d.structure_offsets_b[pr.n_struct] != pr.h_idx[2].size()) return bail(MDGPU_ERR_INVALID_ARG, "'" + pr.name + "': exclusion offsets do not cover idx[2]");
                                         excl_off.assign(d.structure_offsets_b, d.structure_offsets_b + pr.n_struct + 1); }
            else if (!pr.h_idx[2].empty()) return bail(MDGPU_ERR_INVALID_ARG, "'" + pr.name + "': exclusion atoms without offsets");
            e = pr.d_set_of.upload(set_of.data(), set_of.size());
            if (e == cudaSuccess) e = pr.d_excl_off.upload(excl_off.data(), excl_off.size());
            if (e == cudaSuccess) e = set_temporal(pr, num_frames, pr.n_struct);
            break; }
        case MDGPU_OP_BACKBONE_ANGLES: {   // two `dihedral in context` values per segment: phi = (C', N, CA, C), psi = (N, CA, C, N')
            const size_t ns = pr.n_struct;
            if (!ns || pr.h_idx[0].size() != 5 * ns) return bail(MDGPU_ERR_INVALID_ARG, "'" + pr.name + "': idx[0] must hold (C', N, CA, C, N') for each of the num_structures backbone segments");
            const std::vector<int32_t> five = pr.h_idx[0];
            std::vector<int32_t> ctx[4];
            for (int k = 0; k < 4; ++k) ctx[k].resize(2 * ns);
            for (size_t i = 0; i < ns; ++i) {
                const int32_t* q = &five[5 * i];
                const bool ok = q[0] >= 0 && q[1] >= 0 && q[2] >= 0 && q[3] >= 0 && q[4] >= 0;   // both angles or none (md_util.c:2592)
                for (int k = 0; k < 4; ++k) { ctx[k][2 * i] = ok ? q[k] : -1; ctx[k][2 * i + 1] = ok ? q[k + 1] : -1; }
            }
            for (int k = 0; k < 4; ++k) {
                pr.h_idx[k] = ctx[k];
                if (pr.d_idx[SPACE_FULL][k].upload(pr.h_idx[k].data(), pr.h_idx[k].size()) != cudaSuccess) return bail(MDGPU_ERR_CUDA, "device allocation failed (indices)");
            }
            pr.op = MDGPU_OP_DIHEDRAL; pr.n_struct = 2 * ns; pr.backbone_segments = ns;
            e = set_temporal(pr, num_frames, 2 * ns);
            break; }
        case MDGPU_OP_SECONDARY_STRUCTURE: {   // (N, CA, C, O, HN) per segment, the backbone ranges in structure_offsets_b: [F, S] codes
            const size_t ns = pr.n_struct, nr = d.num_structures_b; const uint32_t* ro = d.structure_offsets_b;
            if (!ns) return bail(MDGPU_ERR_INVALID_ARG, "'" + pr.name + "': no backbone segments (num_structures = 0)");
            if (pr.h_idx[0].size() != 5 * ns) return bail(MDGPU_ERR_INVALID_ARG, "'" + pr.name + "': idx[0] must hold (N, CA, C, O, HN) for each of the num_structures backbone segments");
            for (size_t i = 0; i < 5 * ns; ++i) if (pr.h_idx[0][i] < 0 && i % 5 != 4) return bail(MDGPU_ERR_INVALID_ARG, "property '" + pr.name + "': atom index out of range");
            if (!ro || !nr) return bail(MDGPU_ERR_INVALID_ARG, "'" + pr.name + "': no backbone range offsets (structure_offsets_b / num_structures_b)");
            if (ro[0] != 0 || ro[nr] != ns) return bail(MDGPU_ERR_INVALID_ARG, "'" + pr.name + "': backbone range offsets must start at 0 and end at the segment count");
            for (size_t r = 0; r < nr; ++r) if (ro[r] > ro[r + 1]) return bail(MDGPU_ERR_INVALID_ARG, "'" + pr.name + "': backbone range offsets are not ascending");
            std::vector<uint32_t> seg(3 * ns);
            for (size_t r = 0; r < nr; ++r) for (uint32_t i = ro[r]; i < ro[r + 1]; ++i) { seg[3 * i] = (uint32_t)r; seg[3 * i + 1] = ro[r]; seg[3 * i + 2] = ro[r + 1]; }
            pr.h_idx[1].resize(ns); for (size_t i = 0; i < ns; ++i) pr.h_idx[1][i] = pr.h_idx[0][5 * i + 1];   // the CA atoms: the walk's AABB on open axes
            e = pr.d_idx[SPACE_FULL][1].upload(pr.h_idx[1].data(), ns);
            if (e == cudaSuccess) e = pr.d_ss_seg.upload(seg.data(), seg.size());
            pr.ss_segments = ns;
            if (e == cudaSuccess) e = set_temporal(pr, num_frames, ns);
            break; }
        case MDGPU_OP_POROSITY:   // porosity(selection): [F, 1]; an empty selection is valid and evaluates to 0 (:5896-5899)
            e = set_temporal(pr, num_frames, 1);
            if (e == cudaSuccess) e = pr.d_frame_total.alloc(num_frames);
            if (e == cudaSuccess) e = pr.d_frame_n.alloc(num_frames);
            break;
        case MDGPU_OP_RMSD: {   // an empty selection is valid and evaluates to 0 (_rmsd :4311, :4336-4338)
            std::vector<int2> pairs;   // without bonds md_util_unwrap_vec4 fails and its result is ignored (:4327): nothing is unwrapped
            if (!pr.n_struct) {
                build_unwrap_pairs(pairs, pr.h_idx[0].size(), p->conn_off, p->conn_idx);
                pr.n_unwrap = (uint32_t)pairs.size();
                e = pr.d_unwrap.upload(pairs.data(), pairs.size());
                if (e == cudaSuccess) e = set_temporal(pr, num_frames, 1);
                break;
            }
            // `rmsd(x) in <n contexts>`: n groups of idx[0], one value each. A group's unwrap pairs depend on its size only: built once per size.
            { const std::string er = take_structures(pr, d, "rmsd '" + pr.name + "'"); if (!er.empty()) return bail(MDGPU_ERR_INVALID_ARG, er); }
            std::map<uint32_t, uint2> by_size; std::vector<uint2> gp(pr.n_struct);
            for (size_t g = 0; g < pr.n_struct; ++g) {
                const uint32_t sz = pr.h_soff[g + 1] - pr.h_soff[g];
                auto it = by_size.find(sz);
                if (it == by_size.end()) {
                    std::vector<int2> one; build_unwrap_pairs(one, sz, p->conn_off, p->conn_idx);
                    it = by_size.emplace(sz, make_uint2((uint32_t)pairs.size(), (uint32_t)one.size())).first;
                    pairs.insert(pairs.end(), one.begin(), one.end());
                }
                gp[g] = it->second;
            }
            pr.n_unwrap = (uint32_t)pairs.size();
            e = pr.d_unwrap.upload(pairs.data(), pairs.size());
            if (e == cudaSuccess) e = pr.d_group_pairs.upload(gp.data(), gp.size());
            if (e == cudaSuccess) e = pr.d_soff.upload(pr.h_soff.data(), pr.h_soff.size());
            if (e == cudaSuccess) e = set_temporal(pr, num_frames, pr.n_struct);
            break; }
        case MDGPU_OP_EXPRESSION:   // its values per frame follow from its program's operands: take_expressions, once every property is set up
            continue;
        default:
            return bail(MDGPU_ERR_UNSUPPORTED, "property '" + pr.name + "': unsupported operation " + std::to_string(pr.op));
        }
        if (e != cudaSuccess) return bail(MDGPU_ERR_CUDA, std::string("device allocation failed: ") + cudaGetErrorString(e));
        pr.vptr = pr.values.data(); pr.amean = pr.agg_mean.data(); pr.avar = pr.agg_var.data(); pr.aext = pr.agg_ext.data();
        pr.data.num_values = pr.values.size(); pr.data.values = pr.vptr;
        pr.data.weights = pr.is_dist() ? pr.vptr + MDGPU_DIST_BINS : nullptr;
    }
    {
        cudaError_t e = cudaSuccess;
        const std::string er = take_expressions(p, props, num_props, exprs, num_exprs, e);
        if (!er.empty()) return bail(MDGPU_ERR_INVALID_ARG, er);
        if (e != cudaSuccess) return bail(MDGPU_ERR_CUDA, std::string("device allocation failed: ") + cudaGetErrorString(e));
        for (auto& pr : p->props) if (pr.op == MDGPU_OP_EXPRESSION) {
            pr.vptr = pr.values.data(); pr.amean = pr.agg_mean.data(); pr.avar = pr.agg_var.data(); pr.aext = pr.agg_ext.data();
            pr.data.num_values = pr.values.size(); pr.data.values = pr.vptr;
        }
    }
    for (size_t i = 0; i < num_props; ++i) for (size_t j = 0; j < i; ++j) {
        Prop& a = p->props[i]; Prop& b = p->props[j];
        if (a.needs_cells() && b.needs_cells() && b.share_trg < 0 && a.cutoff_max == b.cutoff_max && a.h_idx[1] == b.h_idx[1] && !a.dyn[1].on && !b.dyn[1].on && !a.trg_groups && !b.trg_groups) { a.share_trg = (int)j; break; }
    }
    {   // compact atom space: what host ingest has to copy
        const size_t N = sys->num_atoms; bool all_atoms = false;
        std::vector<uint8_t> mark(N, 0);
        for (auto& pr : p->props) {
            if (pr.op == MDGPU_OP_WITHIN_COUNT || pr.any_dyn()) all_atoms = true;   // within() searches the whole system
            for (int k = 0; k < 4; ++k) for (int32_t a : pr.h_idx[k]) if (a >= 0) mark[(size_t)a] = 1;
        }
        for (size_t a = 0; a < N; ++a) if (mark[a]) p->needed.push_back((int32_t)a);
        const char* env = getenv("MDGPU_INGEST_MODE");
        const uint32_t mode = env ? (uint32_t)atoi(env) : p->ingest_mode;
        p->compact = !all_atoms && mode == 0 && p->needed.size() * 4 <= N * 3;
        for (auto& pr : p->props) for (int k = 0; k < 4; ++k) if (!pr.h_idx[k].empty()) pr.first[SPACE_FULL][k] = pr.h_idx[k][0];
        if (p->compact) {
            AtomSpace& cs = p->space[SPACE_COMPACT];
            std::vector<int32_t> map(N, -1); for (size_t j = 0; j < p->needed.size(); ++j) map[(size_t)p->needed[j]] = (int32_t)j;
            cs.num_atoms = p->needed.size(); cs.axis_stride = (cs.num_atoms + 3) & ~(size_t)3;
            std::vector<float> mc(cs.num_atoms); for (size_t j = 0; j < mc.size(); ++j) mc[j] = p->h_mass[(size_t)p->needed[j]];
            if (cs.d_mass.upload(mc.data(), mc.size()) != cudaSuccess) return bail(MDGPU_ERR_CUDA, "device allocation failed (masses)");
            if (!p->h_radius.empty()) {
                std::vector<float> rc(cs.num_atoms); for (size_t j = 0; j < rc.size(); ++j) rc[j] = p->h_radius[(size_t)p->needed[j]];
                if (cs.d_radius.upload(rc.data(), rc.size()) != cudaSuccess) return bail(MDGPU_ERR_CUDA, "device allocation failed (radii)");
            }
            for (auto& pr : p->props) for (int k = 0; k < 4; ++k) if (!pr.h_idx[k].empty()) {
                std::vector<int32_t> ci(pr.h_idx[k].size()); for (size_t j = 0; j < ci.size(); ++j) ci[j] = pr.h_idx[k][j] < 0 ? -1 : map[(size_t)pr.h_idx[k][j]];
                pr.first[SPACE_COMPACT][k] = ci[0];
                if (pr.d_idx[SPACE_COMPACT][k].upload(ci.data(), ci.size()) != cudaSuccess) return bail(MDGPU_ERR_CUDA, "device allocation failed (indices)");
            }
            if (cs.d_init.alloc(3 * cs.axis_stride) != cudaSuccess) return bail(MDGPU_ERR_CUDA, "device allocation failed (initial frame)");
        }
    }
    p->frame_mask.assign((num_frames + 63) / 64, 0);
    if (full.d_init.alloc(3 * full.axis_stride) != cudaSuccess) return bail(MDGPU_ERR_CUDA, "device allocation failed (initial frame)");
    if (mdgpu_plan_clear(p) != 0) { destroy_plan(p); return nullptr; }
    return p;
}

void mdgpu_plan_destroy(mdgpu_plan* plan) { destroy_plan(plan); }

}  // extern "C"

static int zero_accumulators(Prop& pr) {
    return Prop::for_each_accumulator([&](auto member) -> int {
        auto& b = pr.*member;
        if (b.get()) CUDA_TRY(cudaMemset(b.get(), 0, b.bytes()));
        return 0;
    });
}

extern "C" {

int mdgpu_plan_clear(mdgpu_plan* p) {
    if (!p) return fail(MDGPU_ERR_INVALID_ARG, "null plan");
    if (p->multi) for (auto* q : p->multi->peers) { int rc = mdgpu_plan_clear(q); if (rc) return rc; }
    CUDA_TRY(cudaSetDevice(p->device));
    CUDA_TRY(cudaDeviceSynchronize());
    for (auto& s : p->slots) { s.busy = false; s.h_err[0] = 0; CUDA_TRY(cudaMemset(s.d_err.get(), 0, sizeof(int))); }
    for (auto& pr : p->props) {
        { const int rc = zero_accumulators(pr); if (rc) return rc; }
        if (!pr.agg_mean.empty()) { std::fill(pr.amean, pr.amean + p->num_frames, 0.0f); std::fill(pr.avar, pr.avar + p->num_frames, 0.0f); std::fill(pr.aext, pr.aext + 2 * p->num_frames, 0.0f); }
        std::fill(pr.vptr, pr.vptr + pr.values.size(), 0.0f);
        if (pr.is_dist()) std::fill(pr.vptr + MDGPU_DIST_BINS, pr.vptr + pr.values.size(), 1.0f);   // allocate_property_data :5613-5618
        pr.data.min_value = +FLT_MAX; pr.data.max_value = -FLT_MAX;                                 // clear_property_data :5726-5727
        pr.data.min_range[0] = pr.data.min_range[1] = pr.data.max_range[0] = pr.data.max_range[1] = 0.0f;
        pr.frames_accumulated = 0; pr.frames_overridden = false; pr.data.frames_accumulated = 0;
    }
    { std::lock_guard<std::mutex> lk(p->mask_mutex); std::fill(p->frame_mask.begin(), p->frame_mask.end(), 0ull); }
    p->interrupt = false; p->frames_retired = 0;
    for (int k = 0; k < TIMED_KINDS; ++k) { p->timed_ms[k] = 0; p->timed_n[k] = 0; }
    if (p->d_counters.get()) CUDA_TRY(cudaMemset(p->d_counters.get(), 0, p->d_counters.bytes()));
    p->dirty = true;
    return 0;
}

int mdgpu_plan_set_initial_frame(mdgpu_plan* p, const float* x, const float* y, const float* z, const mdgpu_unitcell_t* cell) {
    if (!p || !x || !y || !z || !cell) return fail(MDGPU_ERR_INVALID_ARG, "mdgpu_plan_set_initial_frame: null argument");
    if (p->multi) for (auto* q : p->multi->peers) { int rc = mdgpu_plan_set_initial_frame(q, x, y, z, cell); if (rc) return rc; }
    CUDA_TRY(cudaSetDevice(p->device));
    const AtomSpace& full = p->space[SPACE_FULL]; const float* src[3] = { x, y, z };
    for (int ax = 0; ax < 3; ++ax) CUDA_TRY(cudaMemcpy(full.d_init.get() + (size_t)ax * full.axis_stride, src[ax], sizeof(float) * full.num_atoms, cudaMemcpyHostToDevice));
    if (p->compact) {
        const AtomSpace& cs = p->space[SPACE_COMPACT];
        std::vector<float> c(3 * cs.axis_stride, 0.0f);
        for (int ax = 0; ax < 3; ++ax) gather_axis(c.data() + (size_t)ax * cs.axis_stride, src[ax], p->needed.data(), cs.num_atoms);
        CUDA_TRY(cudaMemcpy(cs.d_init.get(), c.data(), sizeof(float) * c.size(), cudaMemcpyHostToDevice));
    }
    p->init_cell = *cell; p->have_init = true;
    for (auto& pr : p->props) {
        if (pr.is_density()) {
            // reference point / extent from the initial frame's unit cell (md_script_functions.inl:4871-4903, :4930-4933)
            const int axis = (int)pr.op - MDGPU_OP_DENSITY_X;
            const float A[3][3] = { { (float)cell->x, 0.f, 0.f }, { (float)cell->xy, (float)cell->y, 0.f }, { (float)cell->xz, (float)cell->yz, (float)cell->z } };
            float rc[3], re[3];
            for (int r = 0; r < 3; ++r) { float v = A[0][r] * 0.5f; v = v + A[1][r] * 0.5f; v = v + A[2][r] * 0.5f; rc[r] = v; re[r] = A[r][r]; }
            pr.rc = rc[axis]; pr.re = re[axis];
            pr.inv_ext = re[axis] > 0.0f ? 1.0f / re[axis] : 0.0f;
            pr.min_point = rc[axis] - re[axis] * 0.5f;
            const float vol = (re[0] * re[1] * re[2]) / (float)MDGPU_DIST_BINS;
            const double slice_vol = vol;
            pr.dens_factor = 1660.5390666 / slice_vol;
        }
    }
    return 0;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------------------------
// slot set-up
// ---------------------------------------------------------------------------------------------------------------
// rdf candidate lists of the packed pair kernel, entries per frame for frames of `cell`: every target appears in at most (2n+1)^3 home cells'
// lists, n the neighbour reach of the cell (an NPT or sheared cell can cross from 27 to 125 offsets); a grid fitted to the data (AABB) gets
// the widest reach the reference allows. A dynamic target set is sized for a quarter of the system; frames that select more are finished by
// the overflow pass.
static size_t rdf_list_stride(const mdgpu_plan* p, const Prop& pr, const mdgpu_unitcell_t* cell) {
    FrameGeom g; host_frame_geom(&g, cell, pr.cutoff_max, pr.cutoff_max, nullptr, 0xffffffffu);
    size_t nn = (size_t)(2 * std::max(g.ncell[0], 1) + 1) * (2 * std::max(g.ncell[1], 1) + 1) * (2 * std::max(g.ncell[2], 1) + 1);
    if (g.valid <= 0 || (cell->flags & MDGPU_CELL_PBC_ALL) != MDGPU_CELL_PBC_ALL) nn = 125;
    return std::min<size_t>(nn, 125) * (pr.dyn[1].on ? std::max<size_t>(p->num_atoms / 4, 1024) : pr.h_idx[1].size()) + 1024;
}

// the scratch of one within() query over a selection of n_sel atoms; `list`: with the per-frame index list of a dynamic argument.
// A coordinate range (`cells` false) needs no grid and no cell lists: only the marks and the list.
static int alloc_within(mdgpu_plan* p, WithinScratch& w, size_t n_sel, uint32_t cap, bool list, bool cells = true) {
    if (cells) {
        CUDA_TRY(w.d_geom.alloc(p->B)); CUDA_TRY(w.d_aabb.alloc((size_t)6 * p->B));
        CUDA_TRY(w.trg.alloc(p->B, (uint32_t)p->num_atoms, cap));
        CUDA_TRY(w.ref.alloc(p->B, (uint32_t)std::max<size_t>(n_sel, 1), cap));
    }
    CUDA_TRY(w.d_flags.alloc((size_t)p->B * p->num_atoms));
    if (list) { CUDA_TRY(w.d_idx.alloc((size_t)p->B * p->num_atoms)); CUDA_TRY(w.d_n.alloc(p->B)); }
    return 0;
}

// One stream slot with the scratch of every property, for cell capacity `cap`.
static int build_slot(mdgpu_plan* p, Slot& s, const mdgpu_unitcell_t* first_cell, uint32_t cap) {
    CUDA_TRY(cudaStreamCreateWithFlags(s.stream.out(), cudaStreamNonBlocking));
    CUDA_TRY(cudaEventCreateWithFlags(s.done.out(), cudaEventDisableTiming));
    CUDA_TRY(cudaEventCreateWithFlags(s.copied.out(), cudaEventDisableTiming));
    CUDA_TRY(s.h_err.alloc(1)); s.h_err[0] = 0;
    CUDA_TRY(s.d_cells.alloc(p->B));
    CUDA_TRY(s.h_cells.alloc(p->B));
    CUDA_TRY(s.d_err.alloc(1)); CUDA_TRY(cudaMemset(s.d_err.get(), 0, sizeof(int)));
    s.ps.resize(p->props.size());
    for (size_t i = 0; i < p->props.size(); ++i) {
        Prop& pr = p->props[i]; PropScratch& ps = s.ps[i];
        for (int k = 0; k < 4; ++k) if (pr.dyn[k].on) {
            const int rc = alloc_within(p, ps.within[k], pr.h_idx[k].size(), cap, pr.op != MDGPU_OP_WITHIN_COUNT, !pr.dyn[k].range); if (rc) return rc;
        }
        // an argument that is an array of selections: one position per selection
        for (int k = 0; k < 2; ++k) if (!pr.h_goff[k].empty()) CUDA_TRY(ps.d_gpos[k].alloc((size_t)p->B * (pr.h_goff[k].size() - 1) * 3));
        if (pr.needs_cells() && pr.share_trg < 0) {
            CUDA_TRY(ps.d_geom.alloc(p->B)); CUDA_TRY(ps.d_aabb.alloc((size_t)6 * p->B));
            CUDA_TRY(ps.trg.alloc(p->B, (uint32_t)(pr.dyn[1].on ? p->num_atoms : (pr.trg_groups ? pr.trg_groups : pr.h_idx[1].size())), cap));
        }
        if (pr.op == MDGPU_OP_RDF) {
            CUDA_TRY(ps.ref.alloc(p->B, (uint32_t)(pr.dyn[0].on ? p->num_atoms : (pr.n_struct ? pr.n_struct : pr.h_idx[0].size())), cap));
            if (pr.n_struct) CUDA_TRY(ps.d_com.alloc((size_t)p->B * pr.n_struct * 3));
            else {
                CUDA_TRY(ps.d_pair_list.alloc((size_t)p->B * rdf_list_stride(p, pr, first_cell)));
                CUDA_TRY(ps.d_list_hdr.alloc((size_t)p->B * cap));
                CUDA_TRY(ps.d_list_cursor.alloc(p->B));
            }
            CUDA_TRY(ps.d_frame_bins.alloc((size_t)p->B * (MDGPU_DIST_BINS + 1)));   // + one work counter per frame (k_rdf_pairs_v2)
        } else if (pr.op == MDGPU_OP_CONTACT_COUNT) {
            CUDA_TRY(ps.ref.alloc(p->B, (uint32_t)pr.h_idx[0].size(), cap));
            CUDA_TRY(ps.d_frame_bins.alloc((size_t)p->B * (MDGPU_DIST_BINS + 1)));
        } else if (pr.op == MDGPU_OP_SDF) {
            CUDA_TRY(ps.d_sdf_xyzw.alloc((size_t)p->B * (pr.n_struct + 1) * pr.struct_size));
            CUDA_TRY(ps.d_sdf_ref0.alloc((size_t)p->B * 20));
            CUDA_TRY(ps.d_sdf_mats.alloc((size_t)p->B * pr.n_struct * 32));
        } else if (pr.op == MDGPU_OP_WITHIN_COUNT) {   // a range's scratch was allocated with the dynamic arguments above
            if (!pr.dyn[0].on) { const int rc = alloc_within(p, ps.within[0], pr.h_idx[0].size(), cap, false); if (rc) return rc; }
            if (pr.count_groups) CUDA_TRY(ps.within[0].d_hits.alloc((size_t)p->B * pr.n_groups));   // count over groups: one hit byte per group and frame
        } else if (pr.op == MDGPU_OP_POROSITY) {
            CUDA_TRY(ps.d_poro_xyzr.alloc((size_t)PORO_FRAMES * pr.h_idx[0].size())); CUDA_TRY(ps.d_poro_hdr.alloc(PORO_FRAMES));
            CUDA_TRY(ps.d_poro_grid.alloc((size_t)PORO_FRAMES * PORO_GRID_WORDS)); CUDA_TRY(ps.d_poro_count.alloc(PORO_FRAMES));
            CUDA_TRY(cudaMemset(ps.d_poro_grid.get(), 0, ps.d_poro_grid.bytes()));
            CUDA_TRY(cudaMemset(ps.d_poro_count.get(), 0, ps.d_poro_count.bytes()));
        } else if (pr.op == MDGPU_OP_SECONDARY_STRUCTURE) {
            CUDA_TRY(ps.d_geom.alloc(p->B)); CUDA_TRY(ps.d_aabb.alloc((size_t)6 * p->B));
            CUDA_TRY(ps.d_ss_res.alloc((size_t)p->B * pr.ss_segments * SS_RES_FLOATS));
            CUDA_TRY(ps.d_ss_hb.alloc((size_t)p->B * pr.ss_segments)); CUDA_TRY(ps.d_ss_bits.alloc((size_t)p->B * 2 * pr.ss_segments));
        } else if (pr.op == MDGPU_OP_RMSD) {
            CUDA_TRY(ps.d_sdf_xyzw.alloc((size_t)p->B * 2 * pr.h_idx[0].size()));   // [B][initial, current][atoms]
        } else if (pr.op == MDGPU_OP_PLANE || pr.op == MDGPU_OP_SHAPE_WEIGHTS) {
            CUDA_TRY(ps.d_sdf_xyzw.alloc((size_t)p->B * pr.h_idx[0].size()));   // the fit's xyzw scratch
        } else if (pr.is_density()) {
            CUDA_TRY(ps.d_frame_bins64.alloc((size_t)p->B * MDGPU_DIST_BINS));
        } else if (pr.com_mask) {
            if (!pr.n_struct) CUDA_TRY(ps.d_argpos.alloc((size_t)p->B * 12));
            for (int k = 0; k < 4; ++k) if (!pr.h_aoff[k].empty()) CUDA_TRY(ps.d_parts[k].alloc((size_t)p->B * (pr.h_aoff[k].size() - 1)));
        }
    }
    return 0;
}

// The frames of the evaluation that builds the slots, when they are in host memory: a grid fitted to them sizes the default cell capacity.
struct FitFrames { const float* xyz; size_t frame_stride, axis_stride; uint32_t count; };

// min[3], max[3] over every atom of every frame, starting from the origin as k_aabb does: it holds the box each frame's grid is fitted to
static void fit_frames_aabb(const FitFrames& fr, size_t num_atoms, float box[6]) {
    for (int k = 0; k < 6; ++k) box[k] = 0.0f;
    for (uint32_t f = 0; f < fr.count; ++f) for (int k = 0; k < 3; ++k) {
        const float* v = fr.xyz + (size_t)f * fr.frame_stride + (size_t)k * fr.axis_stride;
        for (size_t i = 0; i < num_atoms; ++i) { box[k] = fminf(box[k], v[i]); box[3 + k] = fmaxf(box[3 + k], v[i]); }
    }
}

// slot set-up (lazy: needs the first frame's cell for the default cell capacity). All or nothing: the slots and each slot's host staging
// become the plan's only once all their allocations have succeeded; after a failure the owners free what was built and the next call
// builds again.
static int ensure_slots(mdgpu_plan* p, const mdgpu_unitcell_t* first_cell, bool need_host_staging, const FitFrames* fit = nullptr) {
    std::lock_guard<std::mutex> guard(p->slot_mutex);   // concurrent callers: the first one builds the slots
    if (p->slots.empty()) {
        // default cell capacity: twice the grid the reference would build for the first frame, per property cutoff. A non-periodic axis takes
        // its extent from the data (AABB fit): with host frames that is the box of all the evaluation's frames (a superset of every
        // property's points, so no frame of it needs more cells); frames on the device or in XTC blobs are not seen here, and get the floor.
        uint32_t cap = p->cell_cap;
        if (!cap) {
            float box[6]; const float* aabb = nullptr;
            if (fit && (first_cell->flags & MDGPU_CELL_PBC_ALL) != MDGPU_CELL_PBC_ALL) { fit_frames_aabb(*fit, p->num_atoms, box); aabb = box; }
            uint64_t need = 1u << 16;   // floor: room for later frames that spread beyond the first evaluation's
            auto grid = [&](double cell_ext, float cutoff) {
                FrameGeom g; host_frame_geom(&g, first_cell, cell_ext, cutoff, aabb, 0xffffffffu);
                need = std::max<uint64_t>(need, 2ull * std::max<uint64_t>(g.num_cells, g.num_home) + 2);
            };
            for (auto& pr : p->props) {
                if (pr.needs_cells()) grid((double)pr.cutoff_max, pr.cutoff_max);
                if (pr.op == MDGPU_OP_WITHIN_COUNT && !pr.dyn[0].on) grid(within_cell_ext(pr.cutoff_max), pr.cutoff_max);
                for (auto& dy : pr.dyn) if (dy.on && !dy.range) grid(within_cell_ext(dy.rmax), dy.rmax);
            }
            cap = (uint32_t)std::min<uint64_t>(need, 1u << 26);
        }
        std::vector<Slot> slots(p->S);
        for (auto& s : slots) { const int rc = build_slot(p, s, first_cell, cap); if (rc) return rc; }
        p->slots = std::move(slots); p->cell_cap = cap;
    }
    if (need_host_staging) for (auto& s : p->slots) if (!s.d_frames.get()) {   // host ingest staging, in the ingest (compact or full) atom space
        const size_t n = (size_t)p->B * 3 * p->space[p->ingest_space()].axis_stride;
        DevBuf<float> d; PinnedBuf<float> h;
        CUDA_TRY(d.alloc(n));
        CUDA_TRY(h.alloc(n));
        s.d_frames = std::move(d); s.h_frames = std::move(h);
    }
    return 0;
}

// position of argument k of distance / angle / dihedral / com when it is a selection: its centre of mass (coordinate_extract_com
// md_script_functions.inl:1717), or for an array of selections the centre of the selections' centres (:1826-1842) -> ps.d_argpos[f][k]
static void arg_position(Prop& pr, PropScratch& ps, int k, const BatchFrames& fr, Slot& s, int32_t* const* didx, const float* dmass, DynSel dsel) {
    if (!pr.h_aoff[k].empty()) {
        const uint32_t n = (uint32_t)pr.h_aoff[k].size() - 1u;
        launch_arg_com_parts(fr, s.d_cells.get(), didx[k], pr.d_aoff[k].get(), n, dmass, ps.d_parts[k].get(), s.stream);
        launch_arg_combine(ps.d_parts[k].get(), n, s.d_cells.get(), ps.d_argpos.get(), k, (int)fr.count, s.stream);
    } else launch_arg_com(fr, s.d_cells.get(), didx[k], (uint32_t)pr.h_idx[k].size(), dmass, ps.d_argpos.get(), k, s.stream, dsel);
}

// Argument k as positions: an array of selections contributes one position per selection, its centre of mass (extract_com :857, no periodic
// treatment; coordinate_extract :1503) -> ps.d_gpos[k]; any other argument is the atoms of idx[k] (pos == null)
struct ArgPoints { uint32_t n; const float* pos; };
static ArgPoints group_positions(Prop& pr, PropScratch& ps, int k, const BatchFrames& fr, const int32_t* didx, const float* dmass, cudaStream_t st) {
    if (pr.h_goff[k].empty()) return ArgPoints{ (uint32_t)pr.h_idx[k].size(), nullptr };
    const uint32_t n = (uint32_t)pr.h_goff[k].size() - 1;
    launch_group_com(fr, didx, pr.d_goff[k].get(), n, dmass, ps.d_gpos[k].get(), st);
    return ArgPoints{ n, ps.d_gpos[k].get() };
}

// within([rmin:]rmax, sel) of every frame of the batch up to the marking kernel: the grid over every atom of the system (get_spatial_acc :734),
// the cell lists of all atoms and of the selection, and the arguments of launch_within_count / launch_within_list (`out` is the caller's)
static WithinArgs enqueue_within(mdgpu_plan* p, Slot& s, WithinScratch& w, const BatchFrames& fr, bool all_pbc, const int32_t* sel, size_t n_sel, float rmin, float rmax, const uint8_t* and_mask, uint32_t frame0) {
    const float* aabb = nullptr;
    if (!all_pbc) { launch_aabb(fr, nullptr, (uint32_t)p->num_atoms, w.d_aabb.get(), s.stream); aabb = w.d_aabb.get(); }
    launch_geom(s.d_cells.get(), aabb, w.d_geom.get(), within_cell_ext(rmax), (double)rmax, p->cell_cap, (int)fr.count, s.d_err.get(), s.stream);
    launch_cell_list(0, fr, nullptr, nullptr, (uint32_t)p->num_atoms, w.d_geom.get(), w.trg.cl, 0, s.stream);
    launch_cell_list(1, fr, sel, nullptr, (uint32_t)n_sel, w.d_geom.get(), w.ref.cl, 0, s.stream);
    WithinArgs a{};
    a.geom = w.d_geom.get(); a.trg = w.trg.cl; a.ref = w.ref.cl; a.sel = sel; a.n_sel = (uint32_t)n_sel;
    a.num_atoms = (uint32_t)p->num_atoms; a.flags = w.d_flags.get(); a.out = nullptr; a.frame0 = frame0; a.min_r2 = rmin * rmin; a.and_mask = and_mask;   // :2641
    return a;
}

// a coordinate range of every frame of the batch: the arguments of launch_range_list / launch_range_count (frames in the full atom space:
// a range consumer makes host ingest copy whole frames)
static RangeArgs range_args(const mdgpu_plan* p, const Prop::DynArg& dy, WithinScratch& w, const BatchFrames& fr) {
    RangeArgs a{};
    a.frames = fr;
    for (int c = 0; c < 3; ++c) { a.lo[c] = dy.lo[c]; a.hi[c] = dy.hi[c]; }
    a.has_and = dy.has_and ? 1u : 0u; a.and_idx = dy.d_and_idx.get(); a.n_and = (uint32_t)dy.d_and_idx.size();
    a.num_atoms = (uint32_t)p->num_atoms; a.flags = w.d_flags.get();
    return a;
}

// what `launch` enqueues on `st`, timed as one TimedLaunch of `kind` when kernel timing is enabled
template <typename F> static void timed_launch(mdgpu_plan* p, cudaStream_t st, int kind, F&& launch) {
    TimedLaunch tl{ nullptr, nullptr, kind };
    if (p->timing) { cudaEventCreate(&tl.a); cudaEventCreate(&tl.b); cudaEventRecord(tl.a, st); }
    launch();
    if (p->timing) { cudaEventRecord(tl.b, st); p->timed.push_back(tl); }
}

// md_spatial_acc_init(&acc, CA, 9.0, cell) and its pair walk at cutoff 9.0 (md_util.c:2122, 2150)
constexpr double SS_CUTOFF = 9.0;
// why the candidate walk of a frame with this cell cannot be restated (nullptr: it can). A triclinic cell must be periodic on all axes
// (md_spatial_acc.c:201-202) and not degenerate; a periodic axis needs at least 2n + 1 cells for the neighbour reach n, so that no pair of cells
// is joined by two offsets (a narrower cell could report a pair twice).
static const char* ss_cell_unsupported(const mdgpu_unitcell_t& c) {
    if ((c.flags & MDGPU_CELL_TRICLINIC) && (c.flags & MDGPU_CELL_PBC_ALL) != MDGPU_CELL_PBC_ALL) return "a triclinic cell must be periodic on all axes";
    FrameGeom g; host_frame_geom(&g, &c, SS_CUTOFF, SS_CUTOFF, nullptr, 0xffffffffu);
    if ((c.flags & MDGPU_CELL_TRICLINIC) && g.valid <= 0) return "degenerate triclinic cell";
    for (int k = 0; k < 3; ++k)
        if ((c.flags & (MDGPU_CELL_PBC_X << k)) && (g.ncell[k] > 2 || g.cdim[k] < 2 * g.ncell[k] + 1))
            return "a periodic axis of the cell is too narrow for the 9 A candidate search to visit each residue pair once (at least 27 A, or wider when skewed)";
    return nullptr;
}

// enqueue the property kernels of one batch whose frames are already in device memory, in atom space `sp`: SPACE_COMPACT when host ingest
// copied only the atoms the properties read (index lists, masses and the initial frame of that space are used), SPACE_FULL for whole frames
// with global atom indices.
static int enqueue_batch(mdgpu_plan* p, Slot& s, const BatchFrames& fr, uint32_t frame0, Space sp) {
    std::lock_guard<std::mutex> guard(p->submit_mutex);
    const int B = (int)fr.count;
    const AtomSpace& as = p->space[sp];
    const float* dmass = as.d_mass.get(); const float* dinit = as.d_init.get(); const size_t init_as = as.axis_stride;
    // all frames of a batch must agree on ortho vs triclinic (kernel template parameter)
    bool tri = (s.h_cells[0].flags & MDGPU_CELL_TRICLINIC) != 0;
    for (int i = 1; i < B; ++i) if (((s.h_cells[i].flags & MDGPU_CELL_TRICLINIC) != 0) != tri)
        return fail(MDGPU_ERR_UNSUPPORTED, "frames %u..%u mix orthorhombic and triclinic unit cells inside one batch", frame0, frame0 + B - 1);
    CUDA_TRY(cudaMemcpyAsync(s.d_cells.get(), s.h_cells.get(), sizeof(mdgpu_unitcell_t) * B, cudaMemcpyHostToDevice, s.stream));
    bool all_pbc = true; for (int i = 0; i < B; ++i) all_pbc = all_pbc && ((s.h_cells[i].flags & MDGPU_CELL_PBC_ALL) == MDGPU_CELL_PBC_ALL);
    for (size_t i = 0; i < p->props.size(); ++i) {
        Prop& pr = p->props[i]; PropScratch& ps = s.ps[i];
        int32_t* didx[4]; for (int k = 0; k < 4; ++k) didx[k] = pr.d_idx[sp][k].get();
        const PropScratch& cs = (pr.share_trg >= 0) ? s.ps[pr.share_trg] : ps;   // owner of the target cell list + geometry
        DynSel dsel[4];
        for (int k = 0; k < 4; ++k) {   // dynamic arguments first: within([min:]max, idx[k]) [and mask] of every frame of the batch -> ascending per-frame lists
            dsel[k] = DynSel{ nullptr, nullptr, 0 };
            if (!pr.dyn[k].on || pr.op == MDGPU_OP_WITHIN_COUNT) continue;   // count() of a range reads the marks itself (below)
            auto& w = ps.within[k];
            dsel[k] = DynSel{ w.d_idx.get(), w.d_n.get(), (uint32_t)p->num_atoms };
            if (pr.dyn[k].range) { launch_range_list(range_args(p, pr.dyn[k], w, fr), B, p->sm_count, w.d_idx.get(), w.d_n.get(), s.stream); continue; }
            const WithinArgs wa = enqueue_within(p, s, w, fr, all_pbc, didx[k], pr.h_idx[k].size(), pr.dyn[k].rmin, pr.dyn[k].rmax, pr.dyn[k].d_and_mask.get(), frame0);
            launch_within_list(wa, B, tri, p->sm_count, w.d_idx.get(), w.d_n.get(), s.stream);
        }
        if (pr.needs_cells() && pr.share_trg < 0) {
            // target groups: the target points are the groups' centres of mass, an AoS stream, j = position index (compute_rdf :5299-5301);
            // otherwise the atoms of idx[1], or of the frame's dynamic selection (an array of selections is never dynamic: dsel[1] is empty then)
            const ArgPoints t = group_positions(pr, ps, 1, fr, didx[1], dmass, s.stream);
            const int32_t* tidx = t.pos ? nullptr : didx[1];
            const float* aabb = nullptr;
            if (!all_pbc) { launch_aabb(fr, tidx, t.n, ps.d_aabb.get(), s.stream, dsel[1], t.pos); aabb = ps.d_aabb.get(); }
            launch_geom(s.d_cells.get(), aabb, ps.d_geom.get(), (double)pr.cutoff_max, (double)pr.cutoff_max, p->cell_cap, B, s.d_err.get(), s.stream);
            launch_cell_list(0, fr, tidx, t.pos, t.n, ps.d_geom.get(), ps.trg.cl, 0, s.stream, dsel[1]);
        }
        switch (pr.op) {
        case MDGPU_OP_RDF: {
            if (pr.dyn[0].on) {   // references = the frame's dynamic selection (coordinate_extract on a single bitfield: ascending atoms; compute_rdf :5281-5290)
                launch_cell_list(1, fr, nullptr, nullptr, 0, cs.d_geom.get(), ps.ref.cl, 0, s.stream, dsel[0]);
            } else if (pr.n_struct) {
                launch_group_com(fr, didx[0], pr.d_soff.get(), (uint32_t)pr.n_struct, dmass, ps.d_com.get(), s.stream);
                launch_cell_list(1, fr, nullptr, ps.d_com.get(), (uint32_t)pr.n_struct, cs.d_geom.get(), ps.ref.cl, 0, s.stream);   // AoS stream: i = position index (:1721)
            } else {
                launch_cell_list(1, fr, didx[0], nullptr, (uint32_t)pr.h_idx[0].size(), cs.d_geom.get(), ps.ref.cl, 0, s.stream);
            }
            if (!pr.n_struct) {   // candidate lists: the neighbour reach follows the frame's cell
                size_t need = 0;
                for (int i = 0; i < B; ++i) {
                    if (!ps.nn_valid || memcmp(&ps.nn_cell, &s.h_cells[i], sizeof(mdgpu_unitcell_t)) != 0) {   // constant-cell trajectories: one evaluation
                        ps.nn_cell = s.h_cells[i]; ps.nn_stride = rdf_list_stride(p, pr, &s.h_cells[i]); ps.nn_valid = true;
                    }
                    need = std::max(need, ps.nn_stride);
                }
                if ((size_t)p->B * need > ps.d_pair_list.size()) {   // the slot was retired before this batch: its buffers are idle
                    CUDA_TRY(cudaStreamSynchronize(s.stream));
                    CUDA_TRY(ps.d_pair_list.alloc((size_t)p->B * need));   // on failure the list is empty and the next batch tries again
                }
            }
            RdfArgs a{};
            a.geom = cs.d_geom.get(); a.trg = cs.trg.cl; a.ref = ps.ref.cl;
            a.inv_cutoff_range = 1.0f / (pr.cutoff_max - pr.cutoff_min);                 // before the clamp (compute_rdf :5264)
            a.min_cutoff = pr.cutoff_min > 1e-3f ? pr.cutoff_min : 1e-3f;                 // :5269
            a.min_r2 = a.min_cutoff * a.min_cutoff;                                       // rdf_cb :5233
            a.frame_bins = ps.d_frame_bins.get(); a.frame0 = frame0;
            a.pair_list = ps.d_pair_list.get(); a.list_hdr = ps.d_list_hdr.get(); a.list_cursor = ps.d_list_cursor.get(); a.list_stride = ps.d_pair_list.size() / p->B; a.hdr_stride = p->cell_cap; a.err = s.d_err.get();
            a.excl_off = pr.n_struct ? pr.d_soff.get() : nullptr; a.excl_idx = pr.n_struct ? didx[0] : nullptr;   // md_bitfield_test_bit(&masks[i], j) :5252
            a.symmetric = (!pr.n_struct && !pr.trg_groups && !pr.dyn[0].on && !pr.dyn[1].on && pr.h_idx[0] == pr.h_idx[1]) ? 1 : 0;   // same selection on both sides: unshifted pairs are evaluated once, counted twice
            a.acc = pr.d_acc.get(); a.frame_total = pr.d_frame_total.get(); a.frame_min = pr.d_frame_min.get(); a.frame_max = pr.d_frame_max.get(); a.keep = pr.d_keep.get();
            a.counters = p->timing ? p->d_counters.get() : nullptr;
            cudaEvent_t ev4[4] = { nullptr, nullptr, nullptr, nullptr };   // before cull, after cull, before pairs, after pairs
            if (p->timing) for (auto& e : ev4) cudaEventCreate(&e);
            launch_rdf(a, B, tri, (int)p->rdf_variant, p->sm_count, s.stream, p->timing ? ev4 : nullptr);
            if (p->timing) { p->timed.push_back(TimedLaunch{ ev4[0], ev4[1], 3 }); p->timed.push_back(TimedLaunch{ ev4[2], ev4[3], 0 }); }
            break; }
        case MDGPU_OP_CONTACT_COUNT: {   // external points = the atoms of all sets (tag: position in the list), internal = B (md_script_functions.inl:2808-2846)
            launch_cell_list(1, fr, didx[0], nullptr, (uint32_t)pr.h_idx[0].size(), cs.d_geom.get(), ps.ref.cl, 1, s.stream);
            RdfArgs a{};
            a.geom = cs.d_geom.get(); a.trg = cs.trg.cl; a.ref = ps.ref.cl;
            a.inv_cutoff_range = 1.0f; a.min_cutoff = 0.0f; a.min_r2 = 0.0f;
            a.frame_bins = ps.d_frame_bins.get(); a.frame0 = frame0; a.err = s.d_err.get();
            a.excl_off = pr.d_excl_off.get(); a.excl_idx = didx[2]; a.ref_set = pr.d_set_of.get(); a.count_mode = 1;
            launch_rdf(a, B, tri, 1, p->sm_count, s.stream, nullptr);
            launch_contact_rows(ps.d_frame_bins.get(), (uint32_t)pr.n_struct, pr.d_temporal.get(), frame0, B, s.stream);
            break; }
        case MDGPU_OP_SDF: {
            if (!p->have_init) return fail(MDGPU_ERR_INVALID_ARG, "sdf '%s' needs the initial frame (mdgpu_plan_set_initial_frame)", pr.name.c_str());
            SdfArgs a{};
            a.geom = cs.d_geom.get(); a.trg = cs.trg.cl; a.frames = fr; a.cells = s.d_cells.get();
            a.init_xyz = dinit; a.init_axis_stride = init_as; a.mass = dmass;
            a.struct_idx = didx[0]; a.n_struct = (uint32_t)pr.n_struct; a.struct_size = (uint32_t)pr.struct_size;
            a.unwrap_pairs = pr.d_unwrap.get(); a.n_unwrap = pr.n_unwrap; a.cutoff = pr.cutoff_max;
            a.scratch_xyzw = ps.d_sdf_xyzw.get(); a.ref0 = ps.d_sdf_ref0.get(); a.matrices = ps.d_sdf_mats.get();
            a.vol = pr.d_vol.get(); a.frame_total = pr.d_frame_total.get(); a.frame0 = frame0;
            timed_launch(p, s.stream, 1, [&] { launch_sdf(a, B, tri, s.stream); });
            break; }
        case MDGPU_OP_DENSITY_X: case MDGPU_OP_DENSITY_Y: case MDGPU_OP_DENSITY_Z: {
            if (!p->have_init) return fail(MDGPU_ERR_INVALID_ARG, "density '%s' needs the initial frame (mdgpu_plan_set_initial_frame)", pr.name.c_str());
            DensityArgs a{};
            a.frames = fr; a.idx = didx[0]; a.n = (uint32_t)pr.h_idx[0].size(); a.mass = dmass; a.axis = (int)pr.op - MDGPU_OP_DENSITY_X; a.dyn = dsel[0];
            a.rc = pr.rc; a.re = pr.re; a.inv_ext = pr.inv_ext; a.min_point = pr.min_point;
            a.acc = pr.d_acc.get(); a.frame_bins = ps.d_frame_bins64.get(); a.frame_min = pr.d_frame_min64.get(); a.frame_max = pr.d_frame_max64.get(); a.keep = pr.d_keep64.get(); a.frame0 = frame0;
            timed_launch(p, s.stream, 2, [&] { launch_density(a, B, s.stream); });
            break; }
        case MDGPU_OP_WITHIN_COUNT: {
            const GroupArgs grp{ pr.count_groups ? pr.d_group_of.get() : nullptr, ps.within[0].d_hits.get(), pr.n_groups };
            if (pr.dyn[0].on) { launch_range_count(range_args(p, pr.dyn[0], ps.within[0], fr), grp, B, p->sm_count, pr.d_temporal.get(), frame0, s.stream); break; }
            WithinArgs a = enqueue_within(p, s, ps.within[0], fr, all_pbc, didx[0], pr.h_idx[0].size(), pr.cutoff_min, pr.cutoff_max, pr.d_and_mask.get(), frame0);
            a.out = pr.d_temporal.get(); a.grp = grp;
            launch_within_count(a, B, tri, p->sm_count, s.stream);
            break; }
        case MDGPU_OP_COM: {
            TemporalArgs a{};
            a.frames = fr; a.cells = s.d_cells.get(); a.op = (int)pr.op; a.out = pr.d_temporal.get(); a.frame0 = frame0;
            a.atom[0] = pr.first[sp][0]; a.pos = ps.d_argpos.get(); a.com_mask = pr.com_mask;
            if (pr.com_mask & 1u) arg_position(pr, ps, 0, fr, s, didx, dmass, dsel[0]);
            launch_com_rows(a, B, s.stream);
            break; }
        case MDGPU_OP_COORD_X: case MDGPU_OP_COORD_Y: case MDGPU_OP_COORD_Z: {
            const ArgPoints g = group_positions(pr, ps, 0, fr, didx[0], dmass, s.stream);
            if (g.pos) launch_coord_rows_pos(g.pos, g.n, (int)pr.op - MDGPU_OP_COORD_X, pr.d_temporal.get(), frame0, B, s.stream);
            else launch_coord_rows(fr, didx[0], g.n, (int)pr.op - MDGPU_OP_COORD_X, pr.d_temporal.get(), frame0, s.stream);
            break; }
        case MDGPU_OP_SHAPE_WEIGHTS: {
            ShapeArgs a{};
            a.frames = fr; a.cells = s.d_cells.get(); a.mass = dmass; a.use_mass = (int)(pr.com_mask & 1u);
            a.idx = didx[0]; a.soff = pr.d_soff.get(); a.n_struct = (uint32_t)pr.n_struct; a.n_atoms_total = (uint32_t)pr.h_idx[0].size();
            a.scratch_xyzw = ps.d_sdf_xyzw.get(); a.out = pr.d_temporal.get(); a.frame0 = frame0;
            launch_shape_weights(a, B, s.stream);
            break; }
        case MDGPU_OP_PLANE: {
            RmsdArgs a{};
            const ArgPoints g = group_positions(pr, ps, 0, fr, didx[0], dmass, s.stream);
            a.frames = fr; a.cells = s.d_cells.get(); a.mass = dmass; a.idx = didx[0]; a.n = g.n; a.pos = g.pos;
            a.unwrap_pairs = pr.d_unwrap.get(); a.n_unwrap = pr.n_unwrap; a.scratch_xyzw = ps.d_sdf_xyzw.get(); a.out = pr.d_temporal.get(); a.frame0 = frame0;
            launch_plane(a, B, s.stream);
            break; }
        case MDGPU_OP_DISTANCE_PAIR: {
            const ArgPoints g0 = group_positions(pr, ps, 0, fr, didx[0], dmass, s.stream), g1 = group_positions(pr, ps, 1, fr, didx[1], dmass, s.stream);
            launch_distance_pair(fr, s.d_cells.get(), didx[0], g0.n, didx[1], g1.n, g0.pos, g1.pos, pr.d_temporal.get(), frame0, s.stream);
            break; }
        case MDGPU_OP_POROSITY:   // sub-batches of PORO_FRAMES frames through the slot's grids
            for (uint32_t f0 = 0; f0 < (uint32_t)B; f0 += PORO_FRAMES) {
                const uint32_t nf = std::min<uint32_t>(PORO_FRAMES, (uint32_t)B - f0);
                PorosityArgs a{};
                a.frames = BatchFrames{ fr.xyz + (size_t)f0 * fr.frame_stride, fr.frame_stride, fr.axis_stride, nf }; a.cells = s.d_cells.get() + f0;
                a.idx = didx[0]; a.n = (uint32_t)pr.h_idx[0].size(); a.radius = as.d_radius.get();
                a.xyzr = ps.d_poro_xyzr.get(); a.hdr = ps.d_poro_hdr.get(); a.grid = ps.d_poro_grid.get(); a.count = ps.d_poro_count.get();
                a.frame_set = pr.d_frame_total.get(); a.frame_n = pr.d_frame_n.get(); a.out = pr.d_temporal.get(); a.frame0 = frame0 + f0;
                launch_porosity(a, (int)nf, s.stream);
            }
            break;
        case MDGPU_OP_SECONDARY_STRUCTURE: {
            for (int i = 0; i < B; ++i) {   // the walk must reach each pair of cells by one offset (see dssp.cu); periodic axes decide it without the data
                const mdgpu_unitcell_t& c = s.h_cells[i];
                const char* why = ss_cell_unsupported(c);
                if (why) return fail(MDGPU_ERR_UNSUPPORTED, "secondary structure '%s': frame %u: %s", pr.name.c_str(), frame0 + i, why);
            }
            const float* aabb = nullptr;
            if (!all_pbc) { launch_aabb(fr, didx[1], (uint32_t)pr.ss_segments, ps.d_aabb.get(), s.stream); aabb = ps.d_aabb.get(); }
            launch_geom(s.d_cells.get(), aabb, ps.d_geom.get(), SS_CUTOFF, SS_CUTOFF, 0xffffffffu, B, s.d_err.get(), s.stream);
            SsArgs a{};
            a.frames = fr; a.atoms = didx[0]; a.seg = pr.d_ss_seg.get(); a.S = (uint32_t)pr.ss_segments; a.geom = ps.d_geom.get();
            a.res = ps.d_ss_res.get(); a.hb = ps.d_ss_hb.get(); a.bits = ps.d_ss_bits.get(); a.out = pr.d_temporal.get(); a.frame0 = frame0; a.err = s.d_err.get();
            launch_secondary_structure(a, B, tri, s.stream);
            break; }
        case MDGPU_OP_RMSD: {
            if (!p->have_init) return fail(MDGPU_ERR_INVALID_ARG, "rmsd '%s' needs the initial frame (mdgpu_plan_set_initial_frame)", pr.name.c_str());
            RmsdArgs a{};
            a.frames = fr; a.cells = s.d_cells.get(); a.init_xyz = dinit; a.init_axis_stride = init_as; a.mass = dmass;
            a.idx = didx[0]; a.n = (uint32_t)pr.h_idx[0].size(); a.unwrap_pairs = pr.d_unwrap.get(); a.n_unwrap = pr.n_unwrap;
            a.scratch_xyzw = ps.d_sdf_xyzw.get(); a.out = pr.d_temporal.get(); a.frame0 = frame0;
            if (pr.n_struct) {   // one value per context
                a.soff = pr.d_soff.get(); a.group_pairs = pr.d_group_pairs.get(); a.n_groups = (uint32_t)pr.n_struct;
                launch_rmsd_groups(a, B, s.stream);
            } else launch_rmsd(a, B, s.stream);
            break; }
        case MDGPU_OP_DISTANCE_MIN: case MDGPU_OP_DISTANCE_MAX: {   // both evaluate md_util_min_distance (md_script_functions.inl:3904, 3944)
            const ArgPoints g0 = group_positions(pr, ps, 0, fr, didx[0], dmass, s.stream), g1 = group_positions(pr, ps, 1, fr, didx[1], dmass, s.stream);
            if (g0.pos || g1.pos) launch_min_distance_pos(fr, s.d_cells.get(), didx[0], g0.n, didx[1], g1.n, g0.pos, g1.pos, pr.d_temporal.get(), frame0, s.stream);
            else launch_min_distance(fr, s.d_cells.get(), didx[0], g0.n, didx[1], g1.n, pr.d_temporal.get(), frame0, s.stream, dsel[0], dsel[1]);
            break; }
        case MDGPU_OP_DISTANCE: case MDGPU_OP_ANGLE: case MDGPU_OP_DIHEDRAL: {
            TemporalArgs a{};
            a.frames = fr; a.cells = s.d_cells.get(); a.op = (int)pr.op; a.out = pr.d_temporal.get(); a.frame0 = frame0;
            if (pr.n_struct) {
                for (int k = 0; k < 4; ++k) {
                    a.ctx_idx[k] = didx[k]; a.ctx_pos[k] = nullptr;
                    if (!pr.h_aoff[k].empty()) {   // a selection inside the contexts: one centre of mass per context
                        launch_arg_com_parts(fr, s.d_cells.get(), didx[k], pr.d_aoff[k].get(), (uint32_t)pr.n_struct, dmass, ps.d_parts[k].get(), s.stream);
                        a.ctx_pos[k] = ps.d_parts[k].get();
                    }
                }
                a.n_ctx = (uint32_t)pr.n_struct;
                launch_temporal_ctx(a, B, s.stream);
                break;
            }
            for (int k = 0; k < 4; ++k) a.atom[k] = pr.first[sp][k];
            a.pos = ps.d_argpos.get(); a.com_mask = pr.com_mask;
            for (int k = 0; k < 4; ++k) if (pr.com_mask & (1u << k)) arg_position(pr, ps, k, fr, s, didx, dmass, dsel[k]);
            launch_temporal(a, B, s.stream);
            break; }
        default: break;
        }
        pr.frames_accumulated += (uint64_t)B;
    }
    for (size_t l = 0; l + 1 < p->expr_level.size(); ++l)   // temporal expressions, after the rows they read: level by level, on the batch's stream
        launch_temporal_expr(p->d_expr_progs.get() + p->expr_level[l], p->expr_level[l + 1] - p->expr_level[l], p->d_expr_nodes.get(), p->expr_level_len[l], frame0, B, s.stream);
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaMemcpyAsync(s.h_err.get(), s.d_err.get(), sizeof(int), cudaMemcpyDeviceToHost, s.stream));   // read when the slot is retired
    CUDA_TRY(cudaEventRecord(s.done, s.stream));
    s.busy = true; s.pending_beg = frame0; s.pending_cnt = (uint32_t)B;
    p->dirty = true;
    return 0;
}

static void mark_frames(mdgpu_plan* p, uint32_t beg, uint32_t cnt) {
    std::lock_guard<std::mutex> lk(p->mask_mutex);
    for (uint32_t f = beg; f < beg + cnt && f < p->num_frames; ++f) p->frame_mask[f >> 6] |= (1ull << (f & 63));
}

static int publish_batch(mdgpu_plan* p, uint32_t beg, uint32_t cnt);

static int device_error(mdgpu_plan* p, int err) {
    if (err == MDGPU_ERR_CAPACITY) return fail(err, "a frame needs more cells than the plan reserved from its first frame (cell capacity %u); raise mdgpu_plan_options_t.cell_capacity", p->cell_cap);
    if (err == MDGPU_ERR_FRAME_SOURCE) return fail(err, "XTC: Failed to decode frame data (%d)", err);
    if (err == MDGPU_ERR_UNSUPPORTED) return fail(err, "a property kernel found a frame outside what it supports (device-side check; the unit cells of the batch are the usual cause)");
    return fail(err, "device-side error %d", err);
}

// wait until a slot's previous batch has finished (its staging buffers become reusable). Only the thread that owns the slot calls this.
// The batch's device-side error word is inspected BEFORE its frames are declared done: a failed batch never shows up in the frame mask.
static int retire_slot(mdgpu_plan* p, Slot& s) {
    if (!s.busy) return 0;
    CUDA_TRY(cudaEventSynchronize(s.done));
    s.busy = false;
    if (s.h_err.get() && *s.h_err.get()) {
        const int err = *s.h_err.get(); *s.h_err.get() = 0;
        cudaMemsetAsync(s.d_err.get(), 0, sizeof(int), s.stream); cudaStreamSynchronize(s.stream);
        return device_error(p, err);
    }
    mark_frames(p, s.pending_beg, s.pending_cnt);
    p->frames_retired.fetch_add(s.pending_cnt);
    if (p->progress_fn) return publish_batch(p, s.pending_beg, s.pending_cnt);
    return 0;
}

// Slot ownership: the calling thread gets exclusive use of one slot (stream + staging buffers), with that slot's previous batch retired,
// for as long as it holds the lease (move-only); the slot is handed back when the lease is destroyed or reset.
struct SlotRelease {
    mdgpu_plan* p = nullptr;
    void operator()(Slot* s) const { { std::lock_guard<std::mutex> lk(p->slot_mutex); s->owned = false; } p->slot_cv.notify_all(); }
};
using SlotLease = std::unique_ptr<Slot, SlotRelease>;
static int acquire_slot(mdgpu_plan* p, SlotLease& out, int want = -1) {   // the next free slot in ring order, or slot `want`: waits until it is free
    Slot* s = nullptr;
    {
        std::unique_lock<std::mutex> lk(p->slot_mutex);
        for (;;) {
            const size_t S = p->slots.size();
            if (want >= 0) { if (!p->slots[(size_t)want].owned) s = &p->slots[(size_t)want]; }
            else for (size_t i = 0; i < S && !s; ++i) { Slot& c = p->slots[(p->next_slot + i) % S]; if (!c.owned) { s = &c; p->next_slot = (p->next_slot + i + 1) % S; } }
            if (s) break;
            p->slot_cv.wait(lk);
        }
        s->owned = true;
    }
    out = SlotLease(s, SlotRelease{ p });
    const int rc = retire_slot(p, *s);
    if (rc) out.reset();
    return rc;
}
// retire every slot (waits for all batches in flight, whoever enqueued them)
static int drain_slots(mdgpu_plan* p) {
    int rc = 0;
    for (size_t i = 0; i < p->slots.size(); ++i) { SlotLease lease; const int r = acquire_slot(p, lease, (int)i); if (r && !rc) rc = r; }
    return rc;
}

static const mdgpu_unitcell_t* cell_at(const mdgpu_unitcell_t* cells, size_t stride_bytes, size_t i) {
    return (const mdgpu_unitcell_t*)((const char*)cells + i * stride_bytes);
}

static int eval_host_frames_1(mdgpu_plan* p, const float* h_xyz, size_t frame_stride, size_t axis_stride, const mdgpu_unitcell_t* cells, size_t cell_stride_bytes, uint32_t frame_beg, uint32_t count);
static int eval_trajectory_1(mdgpu_plan* p, const mdgpu_trajectory_i* traj, uint32_t frame_beg, uint32_t frame_end, uint32_t loader_threads);
static int multi_eval_host_frames(mdgpu_plan* p, const float* h_xyz, size_t frame_stride, size_t axis_stride, const mdgpu_unitcell_t* cells, size_t cell_stride_bytes, uint32_t frame_beg, uint32_t count);
static int multi_eval_trajectory(mdgpu_plan* p, const mdgpu_trajectory_i* traj, uint32_t frame_beg, uint32_t frame_end, uint32_t loader_threads);
static int multi_sync(mdgpu_plan* p);

// ---------------------------------------------------------------------------------------------------------------
// Several GPUs from ONE process (VIAMD is one process, src/main.cpp:982-1011): the root plan owns one peer plan per further device. A frame
// range is cut into contiguous blocks, one per device (SURVEY.md 8(e)), each block evaluated by its own host thread into that device's
// integer accumulators — no data-path collective. The single exchange step happens at mdgpu_plan_sync: NCCL reduce(sum) of the RDF bins,
// SDF voxels, density sums, per-frame rows and the (disjoint, zero elsewhere) temporal rows onto the root device over NVLink, where the
// usual fold then runs; the peers' accumulators are zeroed so every contribution is counted once.
// NCCL is bound at run time (dlopen "libnccl.so.2", or $MDGPU_NCCL_LIB): single-device users never load it, and a process that already
// carries a NCCL (torch) shares that one.
// ---------------------------------------------------------------------------------------------------------------
static int nccl_load(NcclApi& n) {
    if (n.lib) return 0;
    const char* path = getenv("MDGPU_NCCL_LIB");
    n.lib = dlopen(path && *path ? path : "libnccl.so.2", RTLD_NOW | RTLD_LOCAL);
    if (!n.lib) return fail(MDGPU_ERR_CUDA, "multi-device plan: cannot load NCCL (%s)", dlerror());
    n.CommInitAll = (decltype(n.CommInitAll))dlsym(n.lib, "ncclCommInitAll"); n.CommDestroy = (decltype(n.CommDestroy))dlsym(n.lib, "ncclCommDestroy");
    n.GroupStart = (decltype(n.GroupStart))dlsym(n.lib, "ncclGroupStart"); n.GroupEnd = (decltype(n.GroupEnd))dlsym(n.lib, "ncclGroupEnd");
    n.Reduce = (decltype(n.Reduce))dlsym(n.lib, "ncclReduce"); n.GetErrorString = (decltype(n.GetErrorString))dlsym(n.lib, "ncclGetErrorString");
    if (!n.CommInitAll || !n.CommDestroy || !n.GroupStart || !n.GroupEnd || !n.Reduce) return fail(MDGPU_ERR_CUDA, "multi-device plan: NCCL library lacks a required entry point");
    return 0;
}
#define NCCL_TRY(m, expr) do { const int r_ = (expr); if (r_ != 0) return fail(MDGPU_ERR_CUDA, "%s failed: %s", #expr, (m)->nccl.GetErrorString ? (m)->nccl.GetErrorString(r_) : "nccl error"); } while (0)

static void destroy_multi(mdgpu_plan* p) {
    MultiDevice* m = p->multi; if (!m) return;
    for (size_t g = 0; g < m->comms.size(); ++g) if (m->comms[g]) { cudaSetDevice(m->devices[g]); m->nccl.CommDestroy(m->comms[g]); }
    for (auto* q : m->peers) destroy_plan(q);
    delete m; p->multi = nullptr;
}

// contiguous block of device g out of G (the partition VIAMD's range task uses per thread, src/task_system.cpp:73-87)
static void frame_block(uint32_t count, size_t g, size_t G, uint32_t& off, uint32_t& cnt) {
    const uint64_t a = (uint64_t)count * g / G, b = (uint64_t)count * (g + 1) / G; off = (uint32_t)a; cnt = (uint32_t)(b - a);
}

template <typename F> static int multi_run(mdgpu_plan* p, F&& body) {
    MultiDevice* m = p->multi; const size_t G = m->peers.size() + 1;
    std::vector<int> rcs(G, 0); std::vector<std::string> msgs(G);
    std::vector<std::thread> th;
    for (size_t g = 0; g < G; ++g) th.emplace_back([&, g]() { mdgpu_plan* q = g ? m->peers[g - 1] : p; rcs[g] = body(q, g, G); if (rcs[g]) msgs[g] = g_last_error; });
    for (auto& t : th) t.join();
    for (size_t g = 0; g < G; ++g) if (rcs[g]) { g_last_error = msgs[g]; return rcs[g]; }
    return 0;
}

static int multi_eval_host_frames(mdgpu_plan* p, const float* h_xyz, size_t frame_stride, size_t axis_stride, const mdgpu_unitcell_t* cells, size_t cell_stride_bytes, uint32_t frame_beg, uint32_t count) {
    return multi_run(p, [&](mdgpu_plan* q, size_t g, size_t G) -> int {
        uint32_t off, cnt; frame_block(count, g, G, off, cnt); if (!cnt) return 0;
        return eval_host_frames_1(q, h_xyz + (size_t)off * frame_stride, frame_stride, axis_stride, cell_at(cells, cell_stride_bytes, off), cell_stride_bytes, frame_beg + off, cnt);
    });
}
static int multi_eval_trajectory(mdgpu_plan* p, const mdgpu_trajectory_i* traj, uint32_t frame_beg, uint32_t frame_end, uint32_t loader_threads) {
    return multi_run(p, [&](mdgpu_plan* q, size_t g, size_t G) -> int {
        uint32_t off, cnt; frame_block(frame_end - frame_beg, g, G, off, cnt); if (!cnt) return 0;
        return eval_trajectory_1(q, traj, frame_beg + off, frame_beg + off + cnt, std::max<uint32_t>(1u, (loader_threads ? loader_threads : 4u) / (uint32_t)G));
    });
}

// the exchange step: everything the peers accumulated moves onto the root device
static int multi_sync(mdgpu_plan* p) {
    MultiDevice* m = p->multi; const size_t G = m->peers.size() + 1;
    uint64_t fresh = 0;
    for (auto* q : m->peers) { CUDA_TRY(cudaSetDevice(q->device)); int rc = drain_slots(q); if (rc) return rc; CUDA_TRY(cudaDeviceSynchronize()); fresh += q->frames_retired.load(); }
    CUDA_TRY(cudaSetDevice(p->device)); { int rc = drain_slots(p); if (rc) return rc; } CUDA_TRY(cudaDeviceSynchronize());
    if (!fresh) return 0;
    { int rc = nccl_load(m->nccl); if (rc) return rc; }
    if (m->comms.empty()) { m->comms.assign(G, nullptr); NCCL_TRY(m, m->nccl.CommInitAll(m->comms.data(), (int)G, m->devices.data())); }
    cudaEvent_t t0 = nullptr, t1 = nullptr; cudaEventCreate(&t0); cudaEventCreate(&t1); cudaEventRecord(t0, 0);
    NCCL_TRY(m, m->nccl.GroupStart());
    for (size_t i = 0; i < p->props.size(); ++i) {
        // rows of frames a device did not evaluate are zero: the sum merges them (float temporal rows: x + 0 is exact)
        NCCL_TRY(m, Prop::for_each_accumulator([&](auto member) -> int {
            const auto& root = p->props[i].*member;
            if (!root.get()) return 0;
            for (size_t g = 0; g < G; ++g) {
                mdgpu_plan* q = g ? m->peers[g - 1] : p; void* buf = (q->props[i].*member).get();
                cudaSetDevice(q->device);
                const int r = m->nccl.Reduce(buf, buf, root.size(), nccl_type<typename std::remove_reference_t<decltype(root)>::value_type>(), NCCL_SUM, 0, m->comms[g], 0);
                if (r != 0) return r;
            }
            return 0;
        }));
    }
    NCCL_TRY(m, m->nccl.GroupEnd());
    for (auto* q : m->peers) { CUDA_TRY(cudaSetDevice(q->device)); CUDA_TRY(cudaDeviceSynchronize()); }
    CUDA_TRY(cudaSetDevice(p->device)); cudaEventRecord(t1, 0); CUDA_TRY(cudaDeviceSynchronize());
    { float ms = 0; if (cudaEventElapsedTime(&ms, t0, t1) == cudaSuccess) { m->last_reduce_ms = ms; m->reduces++; } cudaEventDestroy(t0); cudaEventDestroy(t1); }
    for (auto* q : m->peers) {   // moved, not copied: zero the peers so the next exchange does not count them again
        CUDA_TRY(cudaSetDevice(q->device));
        for (auto& pr : q->props) { const int rc = zero_accumulators(pr); if (rc) return rc; }
        p->frames_retired.fetch_add(q->frames_retired.exchange(0));
        std::lock_guard<std::mutex> la(p->mask_mutex); std::lock_guard<std::mutex> lb(q->mask_mutex);
        for (size_t w = 0; w < p->frame_mask.size(); ++w) { p->frame_mask[w] |= q->frame_mask[w]; q->frame_mask[w] = 0; }
    }
    CUDA_TRY(cudaSetDevice(p->device));
    p->dirty = true;
    return 0;
}


extern "C" {

int mdgpu_eval_device_frames(mdgpu_plan* p, const float* d_xyz, size_t frame_stride, size_t axis_stride,
                             const mdgpu_unitcell_t* cells, size_t cell_stride_bytes, uint32_t frame_beg, uint32_t count) {
    if (!p || !d_xyz || !cells) return fail(MDGPU_ERR_INVALID_ARG, "mdgpu_eval_device_frames: null argument");
    if ((size_t)frame_beg + count > p->num_frames) return fail(MDGPU_ERR_INVALID_ARG, "Script eval: Invalid frame range");   // md_script.c:6594-6597
    if (p->multi) return fail(MDGPU_ERR_UNSUPPORTED, "mdgpu_eval_device_frames: frames resident on one device cannot feed a multi-device plan; use the host or trajectory entry points");
    CUDA_TRY(cudaSetDevice(p->device));
    if (!count) return 0;
    int rc = ensure_slots(p, cell_at(cells, cell_stride_bytes, 0), false); if (rc) return rc;
    for (uint32_t b0 = 0; b0 < count; b0 += p->B) {
        if (p->interrupt.load()) return fail(MDGPU_ERR_INTERRUPTED, "evaluation interrupted");
        const uint32_t nb = std::min(p->B, count - b0);
        SlotLease s; rc = acquire_slot(p, s); if (rc) return rc;
        for (uint32_t i = 0; i < nb; ++i) s->h_cells[i] = *cell_at(cells, cell_stride_bytes, b0 + i);
        BatchFrames fr{ d_xyz + (size_t)b0 * frame_stride, frame_stride, axis_stride, nb };
        rc = enqueue_batch(p, *s, fr, frame_beg + b0, SPACE_FULL); if (rc) return rc;
    }
    return 0;
}

// Host frames -> the slot's staging. Compact plans gather the atoms the properties read (ingest threads, pinned staging, one DMA of
// |needed| / num_atoms of the bytes); otherwise whole frames: straight from the caller's buffer when it is pinned, through staging when not.
int mdgpu_eval_host_frames(mdgpu_plan* p, const float* h_xyz, size_t frame_stride, size_t axis_stride,
                           const mdgpu_unitcell_t* cells, size_t cell_stride_bytes, uint32_t frame_beg, uint32_t count) {
    if (!p || !h_xyz || !cells) return fail(MDGPU_ERR_INVALID_ARG, "mdgpu_eval_host_frames: null argument");
    if ((size_t)frame_beg + count > p->num_frames) return fail(MDGPU_ERR_INVALID_ARG, "Script eval: Invalid frame range");
    if (p->multi) return multi_eval_host_frames(p, h_xyz, frame_stride, axis_stride, cells, cell_stride_bytes, frame_beg, count);
    return eval_host_frames_1(p, h_xyz, frame_stride, axis_stride, cells, cell_stride_bytes, frame_beg, count);
}
}  // extern "C"

static int eval_host_frames_1(mdgpu_plan* p, const float* h_xyz, size_t frame_stride, size_t axis_stride,
                              const mdgpu_unitcell_t* cells, size_t cell_stride_bytes, uint32_t frame_beg, uint32_t count) {
    CUDA_TRY(cudaSetDevice(p->device));
    if (!count) return 0;
    const FitFrames fit{ h_xyz, frame_stride, axis_stride, count };
    int rc = ensure_slots(p, cell_at(cells, cell_stride_bytes, 0), true, &fit); if (rc) return rc;
    cudaPointerAttributes attr{}; bool pinned = false;
    if (cudaPointerGetAttributes(&attr, h_xyz) == cudaSuccess) pinned = (attr.type == cudaMemoryTypeHost); else cudaGetLastError();
    const Space sp = p->ingest_space(); const bool c = sp == SPACE_COMPACT;
    const size_t N = p->num_atoms, AS = p->space[sp].axis_stride, M = p->space[SPACE_COMPACT].num_atoms;
    std::vector<cudaEvent_t> direct;   // copies that read the caller's buffer: it may be refilled once they are done
    for (uint32_t b0 = 0; b0 < count; b0 += p->B) {
        if (p->interrupt.load()) return fail(MDGPU_ERR_INTERRUPTED, "evaluation interrupted");
        const uint32_t nb = std::min(p->B, count - b0);
        SlotLease s; rc = acquire_slot(p, s); if (rc) return rc;
        for (uint32_t i = 0; i < nb; ++i) s->h_cells[i] = *cell_at(cells, cell_stride_bytes, b0 + i);
        const float* src = h_xyz + (size_t)b0 * frame_stride;
        cudaError_t e = cudaSuccess;
        if (c) {
            float* dst = s->h_frames.get(); const int32_t* idx = p->needed.data();
            ingest_pool(p)->parallel_for(nb * 3, [&](uint32_t w) {
                const uint32_t i = w / 3, ax = w % 3;
                gather_axis(dst + ((size_t)i * 3 + ax) * AS, src + (size_t)i * frame_stride + (size_t)ax * axis_stride, idx, M);
            });
            e = cudaMemcpyAsync(s->d_frames.get(), s->h_frames.get(), sizeof(float) * (size_t)nb * 3 * AS, cudaMemcpyHostToDevice, s->stream);
        } else if (pinned) {
            if (frame_stride == 3 * axis_stride && axis_stride == AS && AS == N) {   // fully contiguous: one linear DMA
                e = cudaMemcpyAsync(s->d_frames.get(), src, sizeof(float) * (size_t)nb * 3 * AS, cudaMemcpyHostToDevice, s->stream);
            } else if (frame_stride == 3 * axis_stride) {
                e = cudaMemcpy2DAsync(s->d_frames.get(), sizeof(float) * AS, src, sizeof(float) * axis_stride, sizeof(float) * N, (size_t)nb * 3, cudaMemcpyHostToDevice, s->stream);
            } else {
                for (uint32_t i = 0; i < nb && e == cudaSuccess; ++i)
                    e = cudaMemcpy2DAsync(s->d_frames.get() + (size_t)i * 3 * AS, sizeof(float) * AS, src + (size_t)i * frame_stride, sizeof(float) * axis_stride,
                                          sizeof(float) * N, 3, cudaMemcpyHostToDevice, s->stream);
            }
            if (e == cudaSuccess) e = cudaEventRecord(s->copied, s->stream);
            if (std::find(direct.begin(), direct.end(), s->copied) == direct.end()) direct.push_back(s->copied);
        } else {
            for (uint32_t i = 0; i < nb; ++i) for (int ax = 0; ax < 3; ++ax)
                memcpy(s->h_frames.get() + ((size_t)i * 3 + ax) * AS, src + (size_t)i * frame_stride + (size_t)ax * axis_stride, sizeof(float) * N);
            e = cudaMemcpyAsync(s->d_frames.get(), s->h_frames.get(), sizeof(float) * (size_t)nb * 3 * AS, cudaMemcpyHostToDevice, s->stream);
        }
        if (e != cudaSuccess) return fail(MDGPU_ERR_CUDA, "H2D copy failed: %s", cudaGetErrorString(e));
        BatchFrames fr{ s->d_frames.get(), 3 * AS, AS, nb };
        rc = enqueue_batch(p, *s, fr, frame_beg + b0, sp); if (rc) return rc;
    }
    // "copied host->device batch by batch inside the call": when the call returns, the caller's buffer has been read
    for (cudaEvent_t ev : direct) CUDA_TRY(cudaEventSynchronize(ev));
    return 0;
}

extern "C" {
// ---- XTC input ---------------------------------------------------------------------------------------------------------------
static uint32_t xtc_be32(const uint8_t* p) { return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3]; }
static float xtc_bef32(const uint8_t* p) { const uint32_t u = xtc_be32(p); float f; memcpy(&f, &u, 4); return f; }

// frame header -> unit cell as xtc_reader_load_frame builds it: box * 10 in float (md_xtc.c:765-768), md_unitcell_from_matrix_float
// (md_unitcell.inl:109) -> md_unitcell_from_basis_parameters (:12-31)
static bool xtc_header_cell(const uint8_t* fr, size_t nbytes, mdgpu_unitcell_t* cell, int32_t* step, float* time) {
    if (nbytes < 56 || xtc_be32(fr) != 1995u) return false;
    float box[9]; for (int i = 0; i < 9; ++i) box[i] = xtc_bef32(fr + 16 + 4 * i) * 10.0f;
    const double cx = box[0], cy = box[4], cz = box[8], xy = box[3], xz = box[6], yz = box[7];
    uint32_t flags = 0;
    if (xy == 0.0 && xz == 0.0 && yz == 0.0) { if (!(cx == 0.0 && cy == 0.0 && cz == 0.0) && !(cx == 1.0 && cy == 1.0 && cz == 1.0)) flags |= MDGPU_CELL_ORTHO; }
    else flags |= MDGPU_CELL_TRICLINIC;
    if (flags) { if (cx != 0.0) flags |= MDGPU_CELL_PBC_X; if (cy != 0.0) flags |= MDGPU_CELL_PBC_Y; if (cz != 0.0) flags |= MDGPU_CELL_PBC_Z; }
    cell->x = cx; cell->xy = xy; cell->xz = xz; cell->y = cy; cell->yz = yz; cell->z = cz; cell->flags = flags;
    if (step) *step = (int32_t)xtc_be32(fr + 8);
    if (time) *time = xtc_bef32(fr + 12);
    return true;
}

// the stage is built whole (a stage with a stream is complete) or not at all, so a failed set-up is repeated by the next call
static int ensure_xtc_stage(mdgpu_plan* p, XtcStage& st, size_t need_bytes) {
    const size_t nf = (size_t)p->B * XTC_SUPER;
    if (!st.stream) {
        XtcStage b;
        CUDA_TRY(cudaStreamCreateWithFlags(b.stream.out(), cudaStreamNonBlocking));
        CUDA_TRY(cudaEventCreateWithFlags(b.ready.out(), cudaEventDisableTiming));
        for (auto& e : b.consumed) CUDA_TRY(cudaEventCreateWithFlags(e.out(), cudaEventDisableTiming));
        CUDA_TRY(b.d_off.alloc(nf + 1));
        CUDA_TRY(b.h_off.alloc(nf + 1));
        CUDA_TRY(b.d_info.alloc(nf));
        CUDA_TRY(b.d_rec.alloc(nf * p->num_atoms));
        CUDA_TRY(b.d_state.alloc(nf * p->num_atoms));
        st = std::move(b);
    }
    if (need_bytes + 32 > st.d_blob.size()) CUDA_TRY(st.d_blob.alloc(std::max(need_bytes + 32, nf * (p->num_atoms * 6 + 128)) + 4096));
    return 0;
}

int mdgpu_eval_xtc_frames(mdgpu_plan* p, const uint8_t* h_blob, const uint64_t* frame_offsets, uint32_t frame_beg, uint32_t count) {
    if (!p || !h_blob || !frame_offsets) return fail(MDGPU_ERR_INVALID_ARG, "mdgpu_eval_xtc_frames: null argument");
    if ((size_t)frame_beg + count > p->num_frames) return fail(MDGPU_ERR_INVALID_ARG, "Script eval: Invalid frame range");
    CUDA_TRY(cudaSetDevice(p->device));
    if (!count) return 0;
    for (uint32_t i = 0; i < count; ++i) if (frame_offsets[i + 1] <= frame_offsets[i] || (frame_offsets[i] & 3u)) return fail(MDGPU_ERR_FRAME_SOURCE, "XTC: Invalid frame offset range");
    mdgpu_unitcell_t first{};
    if (!xtc_header_cell(h_blob + frame_offsets[0], frame_offsets[1] - frame_offsets[0], &first, nullptr, nullptr)) return fail(MDGPU_ERR_FRAME_SOURCE, "XTC: Magic number did not match");
    if (p->multi) return fail(MDGPU_ERR_UNSUPPORTED, "XTC input is evaluated on one device; create a single-device plan");
    std::lock_guard<std::mutex> xtc_guard(p->xtc_mutex);   // the scan stages are one pipeline: one XTC evaluation at a time per plan
    int rc = ensure_slots(p, &first, false); if (rc) return rc;
    const size_t AS = p->space[SPACE_FULL].axis_stride, NA = p->num_atoms;
    const uint32_t SB = p->B * XTC_SUPER;
    const uint32_t nsuper = (count + SB - 1) / SB;
    // stage k+1 (copy + scan, on its own stream) is issued BEFORE the batches of stage k are enqueued, so it overlaps their kernels
    auto issue = [&](uint32_t k) -> int {
        const uint32_t s0 = k * SB, ns = std::min(SB, count - s0);
        XtcStage& st = p->xtc[(p->next_xtc + k) % XTC_STAGES];
        const uint64_t beg = frame_offsets[s0], end = frame_offsets[s0 + ns];
        int r = ensure_xtc_stage(p, st, (size_t)(end - beg)); if (r) return r;
        CUDA_TRY(cudaEventSynchronize(st.ready));                                   // the pinned offset table of its previous use has been read
        for (uint32_t q = 0; q < st.n_consumed; ++q) CUDA_TRY(cudaStreamWaitEvent(st.stream, st.consumed[q], 0));   // ... and its bytes expanded
        st.n_consumed = 0;
        for (uint32_t i = 0; i <= ns; ++i) st.h_off[i] = frame_offsets[s0 + i] - beg;
        CUDA_TRY(cudaMemcpyAsync(st.d_blob.get(), h_blob + beg, (size_t)(end - beg), cudaMemcpyHostToDevice, st.stream));
        CUDA_TRY(cudaMemsetAsync(st.d_blob.get() + (end - beg), 0, 32, st.stream));   // guard bytes for the word-wise bit reader
        CUDA_TRY(cudaMemcpyAsync(st.d_off.get(), st.h_off.get(), sizeof(unsigned long long) * (ns + 1), cudaMemcpyHostToDevice, st.stream));
        launch_xtc_scan(st.d_blob.get(), st.d_off.get(), (uint32_t)NA, (int)ns, st.d_info.get(), st.d_rec.get(), st.d_state.get(), NA, st.stream);
        CUDA_TRY(cudaEventRecord(st.ready, st.stream));
        return 0;
    };
    for (uint32_t k = 0; k + 1 < XTC_STAGES && k < nsuper; ++k) { rc = issue(k); if (rc) return rc; }
    for (uint32_t k = 0; k < nsuper; ++k) {
        if (k + XTC_STAGES - 1 < nsuper) { rc = issue(k + XTC_STAGES - 1); if (rc) return rc; }
        const uint32_t s0 = k * SB, ns = std::min(SB, count - s0);
        XtcStage& st = p->xtc[(p->next_xtc + k) % XTC_STAGES];
        for (uint32_t b0 = 0; b0 < ns; b0 += p->B) {
            if (p->interrupt.load()) return fail(MDGPU_ERR_INTERRUPTED, "evaluation interrupted");
            const uint32_t nb = std::min(p->B, ns - b0);
            SlotLease lease; rc = acquire_slot(p, lease); if (rc) return rc;
            Slot& s = *lease;
            bool ok = true;
            for (uint32_t i = 0; i < nb && ok; ++i) {
                const uint64_t o = frame_offsets[s0 + b0 + i];
                ok = xtc_header_cell(h_blob + o, (size_t)(frame_offsets[s0 + b0 + i + 1] - o), &s.h_cells[i], nullptr, nullptr);
            }
            if (!ok) return fail(MDGPU_ERR_FRAME_SOURCE, "XTC: Magic number did not match");
            cudaError_t e = cudaSuccess;
            if (!s.d_xtc_frames.get()) e = s.d_xtc_frames.alloc((size_t)p->B * 3 * AS);   // whole decoded frames (global atom indices)
            if (e == cudaSuccess) e = cudaStreamWaitEvent(s.stream, st.ready, 0);
            if (e != cudaSuccess) return fail(MDGPU_ERR_CUDA, "XTC stage set-up failed: %s", cudaGetErrorString(e));
            launch_xtc_expand(st.d_blob.get(), st.d_off.get() + b0, (uint32_t)NA, (int)nb, st.d_info.get() + b0, st.d_rec.get() + (size_t)b0 * NA, st.d_state.get() + (size_t)b0 * NA, NA,
                              s.d_xtc_frames.get(), 3 * AS, AS, s.d_err.get(), s.stream);
            cudaEventRecord(st.consumed[st.n_consumed++], s.stream);
            BatchFrames fr{ s.d_xtc_frames.get(), 3 * AS, AS, nb };
            rc = enqueue_batch(p, s, fr, frame_beg + s0 + b0, SPACE_FULL); if (rc) return rc;
        }
    }
    p->next_xtc += nsuper;
    // the compressed bytes are read from the caller's buffer by the stage copies: wait for them, as mdgpu_eval_host_frames does for its source
    for (auto& st : p->xtc) if (st.ready) CUDA_TRY(cudaEventSynchronize(st.ready));
    return 0;
}

// whole-file convenience: read (a range of) an .xtc file into pinned memory, find the frame starts, evaluate frames [frame_beg, frame_end)
int mdgpu_eval_xtc_file(mdgpu_plan* p, const char* path, uint32_t frame_beg, uint32_t frame_end) {
    if (!p || !path) return fail(MDGPU_ERR_INVALID_ARG, "mdgpu_eval_xtc_file: null argument");
    FILE* fp = fopen(path, "rb");
    if (!fp) return fail(MDGPU_ERR_FRAME_SOURCE, "XTC: Failed to open file '%s'", path);
    fseek(fp, 0, SEEK_END); const long fsz = ftell(fp); fseek(fp, 0, SEEK_SET);
    if (fsz <= 0) { fclose(fp); return fail(MDGPU_ERR_FRAME_SOURCE, "XTC: Failed extract filesize"); }
    CUDA_TRY(cudaSetDevice(p->device));
    PinnedBuf<uint8_t> buf;
    if (buf.alloc((size_t)fsz) != cudaSuccess) { fclose(fp); return fail(MDGPU_ERR_CUDA, "pinned allocation of %ld bytes failed", fsz); }
    const size_t got = fread(buf.get(), 1, (size_t)fsz, fp); fclose(fp);
    std::vector<uint64_t> offs((size_t)fsz / 56 + 2);
    size_t nf = 0, na = 0;
    if (got != (size_t)fsz) return fail(MDGPU_ERR_FRAME_SOURCE, "XTC: Failed to read frame data from file, expected %ld bytes, got %zu bytes", fsz, got);
    int rc = mdgpu_xtc_frame_offsets(buf.get(), (size_t)fsz, offs.data(), offs.size(), &nf, &na); if (rc) return rc;
    if (na != p->num_atoms) return fail(MDGPU_ERR_INVALID_ARG, "XTC: Number of atoms in frame header does not match expected number of atoms");
    if (frame_beg > frame_end || frame_end > nf) return fail(MDGPU_ERR_INVALID_ARG, "Script eval: Invalid frame range");
    if (!p->have_init && nf) {   // initial configuration = frame 0 of the trajectory (md_script.c:5808)
        std::vector<float> f0(3 * na); mdgpu_unitcell_t c0{};
        rc = mdgpu_xtc_decode_frames(p->device, buf.get(), offs.data(), 1, na, f0.data(), &c0, nullptr, nullptr); if (rc) return rc;
        rc = mdgpu_plan_set_initial_frame(p, f0.data(), f0.data() + na, f0.data() + 2 * na, &c0); if (rc) return rc;
    }
    rc = mdgpu_eval_xtc_frames(p, buf.get(), offs.data() + frame_beg, frame_beg, frame_end - frame_beg); if (rc) return rc;
    return mdgpu_plan_sync(p);   // the pinned file image must outlive the copies
}

// frame starts of an XTC file image (md_xtc_read_frame_offsets_and_times md_xtc.c:436-570): offsets[0..n], offsets[n] = end of the last frame
int mdgpu_xtc_frame_offsets(const uint8_t* file, size_t nbytes, uint64_t* offsets, size_t capacity, size_t* num_frames, size_t* num_atoms) {
    if (!file || !offsets || capacity < 2) return fail(MDGPU_ERR_INVALID_ARG, "mdgpu_xtc_frame_offsets: invalid argument");
    if (nbytes < 56 || xtc_be32(file) != 1995u) return fail(MDGPU_ERR_FRAME_SOURCE, "XTC: File does not appear to be a valid xtc trajectory");
    const int32_t natoms = (int32_t)xtc_be32(file + 4);
    if (natoms <= 0) return fail(MDGPU_ERR_FRAME_SOURCE, "XTC: Invalid number of atoms in header");
    size_t n = 0, pos = 0;
    if (natoms <= 9) {
        const size_t fb = 56 + 12u * (size_t)natoms;
        while (pos + fb <= nbytes && n + 1 < capacity && xtc_be32(file + pos) == 1995u) { offsets[n++] = pos; pos += fb; }
    } else {
        while (pos != nbytes && n + 1 < capacity) {
            if (pos + 92 > nbytes || xtc_be32(file + pos) != 1995u) break;                 // "encountered corrupted frame header": keep what was found
            const size_t fb = ((size_t)xtc_be32(file + pos + 88) + 3u) & ~(size_t)3;        // rounding to the next 32-bit boundary
            if (pos + 92 + fb > nbytes) break;
            offsets[n++] = pos; pos += 92 + fb;
        }
    }
    offsets[n] = pos;
    if (num_frames) *num_frames = n; if (num_atoms) *num_atoms = (size_t)natoms;
    return 0;
}

// stand-alone decode (tests, tools): frames -> host arrays [count][3][num_atoms], cells, steps, times
int mdgpu_xtc_decode_frames(int device, const uint8_t* h_blob, const uint64_t* frame_offsets, uint32_t count, size_t num_atoms,
                            float* h_xyz, mdgpu_unitcell_t* h_cells, int32_t* h_steps, float* h_times) {
    if (!h_blob || !frame_offsets || !h_xyz) return fail(MDGPU_ERR_INVALID_ARG, "mdgpu_xtc_decode_frames: null argument");
    CUDA_TRY(cudaSetDevice(device));
    if (!count) return 0;
    const uint64_t beg = frame_offsets[0], end = frame_offsets[count];
    std::vector<unsigned long long> off(count + 1);
    for (uint32_t i = 0; i <= count; ++i) { if ((frame_offsets[i] & 3u) || (i && frame_offsets[i] <= frame_offsets[i - 1])) return fail(MDGPU_ERR_FRAME_SOURCE, "XTC: Invalid frame offset range"); off[i] = frame_offsets[i] - beg; }
    for (uint32_t i = 0; i < count; ++i) {
        mdgpu_unitcell_t c{}; int32_t st = 0; float tm = 0;
        if (!xtc_header_cell(h_blob + frame_offsets[i], (size_t)(frame_offsets[i + 1] - frame_offsets[i]), &c, &st, &tm)) return fail(MDGPU_ERR_FRAME_SOURCE, "XTC: Magic number did not match");
        if (h_cells) h_cells[i] = c; if (h_steps) h_steps[i] = st; if (h_times) h_times[i] = tm;
    }
    DevBuf<uint8_t> d_blob; DevBuf<unsigned long long> d_off; DevBuf<XtcFrameInfo> d_info; DevBuf<uint2> d_rec; DevBuf<uint16_t> d_state; DevBuf<float> d_out; DevBuf<int> d_err;
    if (d_blob.alloc((size_t)(end - beg) + 32) != cudaSuccess || d_off.alloc((size_t)count + 1) != cudaSuccess || d_info.alloc(count) != cudaSuccess ||
        d_rec.alloc((size_t)count * num_atoms) != cudaSuccess || d_state.alloc((size_t)count * num_atoms) != cudaSuccess ||
        d_out.alloc((size_t)count * 3 * num_atoms) != cudaSuccess || d_err.alloc(1) != cudaSuccess) return fail(MDGPU_ERR_CUDA, "device allocation failed (xtc decode)");
    cudaMemset(d_err.get(), 0, sizeof(int)); cudaMemset(d_blob.get() + (end - beg), 0, 32);
    cudaMemcpy(d_blob.get(), h_blob + beg, (size_t)(end - beg), cudaMemcpyHostToDevice);
    cudaMemcpy(d_off.get(), off.data(), sizeof(unsigned long long) * (count + 1), cudaMemcpyHostToDevice);
    launch_xtc_decode(d_blob.get(), d_off.get(), (uint32_t)num_atoms, (int)count, d_info.get(), d_rec.get(), d_state.get(), num_atoms, d_out.get(), 3 * num_atoms, num_atoms, d_err.get(), 0);
    int err = 0;
    if (cudaMemcpy(&err, d_err.get(), sizeof(int), cudaMemcpyDeviceToHost) != cudaSuccess) return fail(MDGPU_ERR_CUDA, "xtc decode failed: %s", cudaGetErrorString(cudaGetLastError()));
    if (err) return fail(MDGPU_ERR_FRAME_SOURCE, "XTC: Failed to decode frame data");
    if (cudaMemcpy(h_xyz, d_out.get(), sizeof(float) * (size_t)count * 3 * num_atoms, cudaMemcpyDeviceToHost) != cudaSuccess) return fail(MDGPU_ERR_CUDA, "xtc decode copy failed");
    return 0;
}

// md_script_eval_frame_range's frame loop (md_script.c:6573-6612 -> eval_properties :5730): re-entrant on one plan from many threads with
// disjoint ranges (VIAMD's enkiTS range task, task_system.cpp:73-87). Every call creates its own readers (:5754) — `loader_threads` of them —
// which decode frames into a slot's pinned staging (compact plans: into a per-reader scratch frame, then the needed atoms are gathered).
int mdgpu_eval_trajectory(mdgpu_plan* p, const mdgpu_trajectory_i* traj, uint32_t frame_beg, uint32_t frame_end, uint32_t loader_threads) {
    if (!p) return fail(MDGPU_ERR_INVALID_ARG, "null plan");
    if (!traj || !traj->inst || !traj->get_header || !traj->init_reader) return fail(MDGPU_ERR_INVALID_ARG, "Script eval: Trajectory was null");
    mdgpu_trajectory_header_t hdr{};
    if (!traj->get_header(traj->inst, &hdr) || hdr.num_frames == 0) return fail(MDGPU_ERR_INVALID_ARG, "Script eval: Trajectory was empty");
    if (frame_beg > frame_end || frame_end > hdr.num_frames || frame_end > p->num_frames) return fail(MDGPU_ERR_INVALID_ARG, "Script eval: Invalid frame range");
    if (hdr.num_atoms != p->num_atoms) return fail(MDGPU_ERR_INVALID_ARG, "trajectory has %zu atoms, plan has %zu", hdr.num_atoms, p->num_atoms);
    if (p->multi) return multi_eval_trajectory(p, traj, frame_beg, frame_end, loader_threads);
    return eval_trajectory_1(p, traj, frame_beg, frame_end, loader_threads);
}
}  // extern "C"

static int eval_trajectory_1(mdgpu_plan* p, const mdgpu_trajectory_i* traj, uint32_t frame_beg, uint32_t frame_end, uint32_t loader_threads) {
    CUDA_TRY(cudaSetDevice(p->device));
    const uint32_t T = std::max(1u, std::min(loader_threads ? loader_threads : 4u, 64u));
    struct Readers { std::vector<mdgpu_trajectory_reader_i> v; ~Readers() { for (auto& r : v) if (r.free) r.free(&r); } } owner;   // this call's readers, freed when it returns
    std::vector<mdgpu_trajectory_reader_i>& readers = owner.v; readers.resize(T);
    memset(readers.data(), 0, sizeof(readers[0]) * T);
    for (uint32_t t = 0; t < T; ++t) if (!traj->init_reader(&readers[t], traj->inst)) return fail(MDGPU_ERR_FRAME_SOURCE, "Failed to initialize trajectory reader for evaluation");
    const Space sp = p->ingest_space(); const bool c = sp == SPACE_COMPACT;
    const size_t ASF = p->space[SPACE_FULL].axis_stride, AS = p->space[sp].axis_stride, M = p->space[SPACE_COMPACT].num_atoms;
    {   // initial configuration = frame 0 (md_script.c:5808); the first caller loads it
        std::lock_guard<std::mutex> guard(p->init_mutex);
        if (!p->have_init) {
            std::vector<float> tmp(3 * ASF); mdgpu_frame_header_t fh{};
            if (!readers[0].load_frame(readers[0].inst, 0, &fh, tmp.data(), tmp.data() + ASF, tmp.data() + 2 * ASF)) return fail(MDGPU_ERR_FRAME_SOURCE, "Failed to load frame during evaluation");
            int rc = mdgpu_plan_set_initial_frame(p, tmp.data(), tmp.data() + ASF, tmp.data() + 2 * ASF, &fh.unitcell); if (rc) return rc;
        }
    }
    std::vector<std::vector<float>> scratch(c ? T : 0);
    for (auto& v : scratch) v.resize(3 * ASF);
    bool slots_ready = false;
    for (uint32_t b0 = frame_beg; b0 < frame_end; b0 += p->B) {
        if (p->interrupt.load()) return fail(MDGPU_ERR_INTERRUPTED, "evaluation interrupted");
        const uint32_t nb = std::min(p->B, frame_end - b0);
        if (!slots_ready) {   // need one header for the cell capacity
            mdgpu_frame_header_t fh{}; if (!readers[0].load_frame(readers[0].inst, b0, &fh, nullptr, nullptr, nullptr)) fh.unitcell = p->init_cell;
            const int rc = ensure_slots(p, &fh.unitcell, true); if (rc) return rc;
            slots_ready = true;
        }
        SlotLease lease; int rc = acquire_slot(p, lease); if (rc) return rc;
        Slot& s = *lease;
        std::atomic<int> failed{0};
        auto work = [&](uint32_t t) {
            for (uint32_t i = t; i < nb; i += T) {
                mdgpu_frame_header_t fh{};
                float* dst = s.h_frames.get() + (size_t)i * 3 * AS;
                if (c) {
                    float* tmp = scratch[t].data();
                    if (!readers[t].load_frame(readers[t].inst, (int64_t)(b0 + i), &fh, tmp, tmp + ASF, tmp + 2 * ASF)) { failed = 1; return; }
                    for (int ax = 0; ax < 3; ++ax) gather_axis(dst + (size_t)ax * AS, tmp + (size_t)ax * ASF, p->needed.data(), M);
                } else if (!readers[t].load_frame(readers[t].inst, (int64_t)(b0 + i), &fh, dst, dst + AS, dst + 2 * AS)) { failed = 1; return; }
                s.h_cells[i] = fh.unitcell;
            }
        };
        if (T == 1) work(0);
        else { std::vector<std::thread> th; for (uint32_t t = 0; t < T; ++t) th.emplace_back(work, t); for (auto& x : th) x.join(); }
        if (failed) return fail(MDGPU_ERR_FRAME_SOURCE, "Failed to load frame during evaluation");
        cudaError_t e = cudaMemcpyAsync(s.d_frames.get(), s.h_frames.get(), sizeof(float) * (size_t)nb * 3 * AS, cudaMemcpyHostToDevice, s.stream);
        if (e != cudaSuccess) return fail(MDGPU_ERR_CUDA, "H2D copy failed: %s", cudaGetErrorString(e));
        BatchFrames fr{ s.d_frames.get(), 3 * AS, AS, nb };
        rc = enqueue_batch(p, s, fr, b0, sp); if (rc) return rc;
    }
    return 0;
}

extern "C" {
void mdgpu_plan_interrupt(mdgpu_plan* p) { if (!p) return; p->interrupt = true; if (p->multi) for (auto* q : p->multi->peers) q->interrupt = true; }
}

static double sphere_volume(double r) { return (4.0 / 3.0) * 3.1415926535897932 * (r * r * r); }

// temporal rows [beg, beg+cnt) that are already in the host values: per-frame aggregates + running min / max + ranges
// (compute_min_max_mean_variance md_script.c:5646-5677: two passes over the frame's values, in float)
static void fold_temporal_rows(Prop& pr, uint32_t f, bool reset) {
    if (reset) { pr.data.min_value = +FLT_MAX; pr.data.max_value = -FLT_MAX; }
    float mn, mx, s1, s2; fold_frame_values(pr.vptr + (size_t)f * pr.len, pr.len, mn, mx, s1, s2);
    pr.data.min_value = ref_min(pr.data.min_value, mn); pr.data.max_value = ref_max(pr.data.max_value, mx);   // md_script.c:5885-5886
    if (pr.len > 1) { pr.amean[f] = s1; pr.avar[f] = s2; pr.aext[2 * f] = mn; pr.aext[2 * f + 1] = mx; }
}
static void temporal_ranges(Prop& pr) {
    if (pr.op == MDGPU_OP_DISTANCE || pr.op == MDGPU_OP_DISTANCE_MIN || pr.op == MDGPU_OP_DISTANCE_MAX || pr.op == MDGPU_OP_DISTANCE_PAIR) { pr.data.min_range[0] = 0.0f; pr.data.max_range[0] = pr.data.max_value; }   // value_range {0, FLT_MAX} (:3884)
    else if (pr.op == MDGPU_OP_POROSITY) { pr.data.min_range[0] = 0.0f; pr.data.max_range[0] = 1.0f; }   // value_range {0, 1} (:5866)
    else { pr.data.min_range[0] = pr.data.min_value; pr.data.max_range[0] = pr.data.max_value; }
}

// Fold the device accumulators of the distribution / volume properties into the host-visible property data, over the frames in `done`.
// `st`: stream the copies run on (the fold of a running evaluation uses the plan's publication stream and never drains the device).
// A distribution's accumulator -> acc[1024], and its per-frame minimum / maximum rows reduced over the frames in `done` into the property's
// min_value / max_value; `value` turns a row entry into the reported float. Waits for `st` (and so for copies the caller enqueued before).
template <typename T, typename V> static int fold_distribution(Prop& pr, const DevBuf<T>& d_min, const DevBuf<T>& d_max, const std::vector<uint32_t>& done, std::vector<unsigned long long>& acc, V&& value, cudaStream_t st) {
    std::vector<T> mn(d_min.size()), mx(d_max.size()); acc.resize(MDGPU_DIST_BINS);
    CUDA_TRY(cudaMemcpyAsync(acc.data(), pr.d_acc.get(), sizeof(unsigned long long) * MDGPU_DIST_BINS, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(mn.data(), d_min.get(), d_min.bytes(), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(mx.data(), d_max.get(), d_max.bytes(), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    float vmin = +FLT_MAX, vmax = -FLT_MAX;
    for (uint32_t f : done) { vmin = std::min(vmin, value(mn[f])); vmax = std::max(vmax, value(mx[f])); }
    pr.data.min_value = vmin; pr.data.max_value = vmax;
    return 0;
}

static int fold_accumulators(mdgpu_plan* p, const std::vector<uint32_t>& done, uint64_t evaluated, cudaStream_t st) {
    for (auto& pr : p->props) {
        // mean divisor = number of frame evaluations that went into the accumulators (the reference's count++ moving average, md_script.c:5912:
        // a frame evaluated twice counts twice); after a cross-GPU exchange the caller states the global count
        const uint64_t n = pr.frames_overridden ? pr.frames_accumulated : evaluated;
        pr.data.frames_accumulated = n;
        if (pr.op == MDGPU_OP_RDF) {
            std::vector<unsigned long long> acc, tot(p->num_frames);
            CUDA_TRY(cudaMemcpyAsync(tot.data(), pr.d_frame_total.get(), pr.d_frame_total.bytes(), cudaMemcpyDeviceToHost, st));
            { const int rc = fold_distribution(pr, pr.d_frame_min, pr.d_frame_max, done, acc, [](uint32_t v) { return (float)v; }, st); if (rc) return rc; }
            // mean of the per-frame integer bins: exact sum, one division (the reference keeps a float cumulative moving
            // average, md_script.c:5912-5921, which drifts by ~1e-5 from this value after 4096 frames: tests/test_oracle_golden.py)
            for (int b = 0; b < MDGPU_DIST_BINS; ++b) pr.vptr[b] = n ? (float)((double)acc[b] / (double)n) : 0.0f;
            // weights of the last evaluated frame (the reference copies "whichever frame finished last", :5924); compute_rdf :5323-5337
            if (!done.empty()) {
                const float min_cutoff = pr.cutoff_min > 1e-3f ? pr.cutoff_min : 1e-3f, max_cutoff = pr.cutoff_max;
                const double total_vol = sphere_volume(max_cutoff) - sphere_volume(min_cutoff);
                const double ref_rho = (double)tot[done.back()] / total_vol;
                const float drf = (max_cutoff - min_cutoff) / (float)MDGPU_DIST_BINS; const double dr = drf;
                double prev = 0;
                for (int64_t i = 0; i < MDGPU_DIST_BINS; ++i) { const double sv = sphere_volume(min_cutoff + (i + 0.5) * dr); const double bv = sv - prev; prev = sv; pr.vptr[MDGPU_DIST_BINS + i] = (float)(ref_rho * bv); }
            }
            pr.data.min_range[0] = pr.cutoff_min; pr.data.max_range[0] = pr.cutoff_max;   // value_range set by internal_rdf :5415
        } else if (pr.op == MDGPU_OP_SDF) {
            launch_mean_u32(pr.d_vol.get(), pr.d_vol_mean.get(), pr.values.size(), n, st);   // exact mean, one division per voxel, on the device
            CUDA_TRY(cudaMemcpyAsync(pr.vptr, pr.d_vol_mean.get(), sizeof(float) * pr.values.size(), cudaMemcpyDeviceToHost, st));
            CUDA_TRY(cudaStreamSynchronize(st));
            // min_value / max_value are never updated for volumes in the reference (md_script.c:5936-5956)
        } else if (pr.is_density()) {
            std::vector<unsigned long long> acc;
            const double unit = 1.0 / 16777216.0;
            { const int rc = fold_distribution(pr, pr.d_frame_min64, pr.d_frame_max64, done, acc, [&](unsigned long long v) { return (float)((double)(float)((double)v * unit) * pr.dens_factor); }, st); if (rc) return rc; }
            for (int b = 0; b < MDGPU_DIST_BINS; ++b) pr.vptr[b] = n ? (float)(((double)acc[b] * unit / (double)n) * pr.dens_factor) : 0.0f;
            for (int b = 0; b < MDGPU_DIST_BINS; ++b) pr.vptr[MDGPU_DIST_BINS + b] = 1.0f;
            const float rad = pr.re * 0.5f;   // value_range {-rad, rad} (:4983-4995)
            pr.data.min_range[0] = -rad; pr.data.max_range[0] = rad;
        }
    }
    return 0;
}

// the frame mask as it stands now -> d_mask
static cudaError_t upload_frame_mask(mdgpu_plan* p, DevBuf<unsigned long long>& d_mask) {
    std::vector<uint64_t> mask; { std::lock_guard<std::mutex> lk(p->mask_mutex); mask = p->frame_mask; }
    return d_mask.upload((const unsigned long long*)mask.data(), mask.size());
}

static void done_frames(mdgpu_plan* p, std::vector<uint32_t>& done) {
    std::lock_guard<std::mutex> lk(p->mask_mutex);
    for (size_t f = 0; f < p->num_frames; ++f) if (p->frame_mask[f >> 6] >> (f & 63) & 1ull) done.push_back((uint32_t)f);
}

// Called by the thread that retires a batch when a progress callback is installed (the md_script shim): the rows of the batch's temporal
// properties go to the host values at once, the running means of distributions / volumes at most every 100 ms; then the callback — the
// shim sets the frame-mask bits there, so VIAMD's UI (src/main.cpp:1513-1524) sees partial results while the evaluation runs.
static int publish_batch(mdgpu_plan* p, uint32_t beg, uint32_t cnt) {
    {
        std::lock_guard<std::mutex> guard(p->sync_mutex);
        if (!p->pub_stream) CUDA_TRY(cudaStreamCreateWithFlags(p->pub_stream.out(), cudaStreamNonBlocking));
        const uint32_t end = (uint32_t)std::min<size_t>((size_t)beg + cnt, p->num_frames);
        for (auto& pr : p->props) if (pr.d_temporal.get() && end > beg) {
            CUDA_TRY(cudaMemcpyAsync(pr.vptr + (size_t)beg * pr.len, pr.d_temporal.get() + (size_t)beg * pr.len, sizeof(float) * (size_t)(end - beg) * pr.len, cudaMemcpyDeviceToHost, p->pub_stream));
        }
        CUDA_TRY(cudaStreamSynchronize(p->pub_stream));
        for (auto& pr : p->props) if (pr.d_temporal.get()) { for (uint32_t f = beg; f < end; ++f) fold_temporal_rows(pr, f, false); temporal_ranges(pr); pr.data.frames_accumulated = p->frames_retired.load(); }
        const auto now = std::chrono::steady_clock::now();
        if (now - p->last_pub >= std::chrono::milliseconds(100)) {
            p->last_pub = now;
            std::vector<uint32_t> done; done_frames(p, done);
            int rc = fold_accumulators(p, done, p->frames_retired.load(), p->pub_stream); if (rc) return rc;
        }
    }
    p->progress_fn(p->progress_user, beg, cnt);
    return 0;
}

extern "C" {

int mdgpu_plan_sync(mdgpu_plan* p) {
    if (!p) return fail(MDGPU_ERR_INVALID_ARG, "null plan");
    if (p->multi) { int rc = multi_sync(p); if (rc) return rc; }
    CUDA_TRY(cudaSetDevice(p->device));
    { int rc = drain_slots(p); if (rc) return rc; }
    std::lock_guard<std::mutex> guard(p->sync_mutex);
    if (!p->dirty.load()) return 0;
    CUDA_TRY(cudaDeviceSynchronize());
    p->dirty = false;   // batches enqueued from here on set it again
    for (auto& s : p->slots) {
        int err = 0; CUDA_TRY(cudaMemcpy(&err, s.d_err.get(), sizeof(int), cudaMemcpyDeviceToHost));
        if (err) { cudaMemset(s.d_err.get(), 0, sizeof(int)); if (s.h_err.get()) *s.h_err.get() = 0; p->dirty = true; return device_error(p, err); }
    }
    {
        std::lock_guard<std::mutex> tl(p->submit_mutex);
        for (auto& t : p->timed) { float ms = 0; if (cudaEventElapsedTime(&ms, t.a, t.b) == cudaSuccess) { p->timed_ms[t.kind] += ms; p->timed_n[t.kind] += 1; } cudaEventDestroy(t.a); cudaEventDestroy(t.b); }
        p->timed.clear();
    }
    std::vector<uint32_t> done; done_frames(p, done);
    { int rc = fold_accumulators(p, done, p->frames_retired.load(), 0); if (rc) { p->dirty = true; return rc; } }
    const size_t F = p->num_frames;
    for (auto& pr : p->props) if (pr.d_temporal.get()) {
        CUDA_TRY(cudaMemcpy(pr.vptr, pr.d_temporal.get(), sizeof(float) * F * pr.len, cudaMemcpyDeviceToHost));
        pr.data.min_value = +FLT_MAX; pr.data.max_value = -FLT_MAX;
        for (uint32_t f : done) fold_temporal_rows(pr, f, false);
        temporal_ranges(pr);
        pr.data.frames_accumulated = pr.frames_overridden ? pr.frames_accumulated : p->frames_retired.load();
    }
    return 0;
}

size_t mdgpu_plan_property_count(const mdgpu_plan* p) { return p ? p->props.size() : 0; }

int mdgpu_plan_property_index(const mdgpu_plan* p, const char* name) {
    if (!p || !name) return -1;
    for (size_t i = 0; i < p->props.size(); ++i) if (p->props[i].name == name) return (int)i;
    return -1;
}

int mdgpu_plan_property_data(mdgpu_plan* p, size_t prop, mdgpu_property_data_t* out) {
    if (!p || !out || prop >= p->props.size()) return fail(MDGPU_ERR_INVALID_ARG, "mdgpu_plan_property_data: invalid argument");
    int rc = mdgpu_plan_sync(p); if (rc) return rc;
    *out = p->props[prop].data;
    return 0;
}

// the property data as last folded, without waiting for anything (progress callbacks read the scalars this way)
int mdgpu_plan_property_peek(mdgpu_plan* p, size_t prop, mdgpu_property_data_t* out) {
    if (!p || !out || prop >= p->props.size()) return fail(MDGPU_ERR_INVALID_ARG, "mdgpu_plan_property_peek: invalid argument");
    *out = p->props[prop].data;
    return 0;
}

int mdgpu_plan_property_histogram(mdgpu_plan* p, size_t prop, uint32_t num_bins, float range_min, float range_max, int aggregate, float* out_bins, float* out_min_max) {
    if (!p || prop >= p->props.size() || !out_bins || !num_bins) return fail(MDGPU_ERR_INVALID_ARG, "mdgpu_plan_property_histogram: invalid argument");
    int rc = mdgpu_plan_sync(p); if (rc) return rc;
    Prop& pr = p->props[prop];
    if (!pr.d_temporal.get()) return fail(MDGPU_ERR_INVALID_ARG, "property '%s' is not a temporal", pr.name.c_str());
    const uint32_t dim = (uint32_t)pr.len, rows = aggregate ? 1u : dim;
    DevBuf<unsigned long long> d_mask; DevBuf<uint32_t> d_counts, d_tot;
    if (upload_frame_mask(p, d_mask) != cudaSuccess || d_counts.alloc((size_t)rows * num_bins) != cudaSuccess || d_tot.alloc(rows) != cudaSuccess) return fail(MDGPU_ERR_CUDA, "device allocation failed (histogram)");
    cudaMemset(d_counts.get(), 0, d_counts.bytes()); cudaMemset(d_tot.get(), 0, d_tot.bytes());
    const float range_ext = range_max - range_min, inv_range = range_ext > 0.0f ? 1.0f / range_ext : 0.0f;   // src/main.cpp:188-189
    launch_temporal_histogram(pr.d_temporal.get(), d_mask.get(), (uint32_t)p->num_frames, dim, range_min, range_max, inv_range, num_bins, aggregate, d_counts.get(), d_tot.get(), 0);
    std::vector<uint32_t> counts((size_t)rows * num_bins), tot(rows);
    if (cudaMemcpy(counts.data(), d_counts.get(), sizeof(uint32_t) * counts.size(), cudaMemcpyDeviceToHost) != cudaSuccess || cudaMemcpy(tot.data(), d_tot.get(), sizeof(uint32_t) * rows, cudaMemcpyDeviceToHost) != cudaSuccess)
        return fail(MDGPU_ERR_CUDA, "histogram copy failed: %s", cudaGetErrorString(cudaGetLastError()));
    float min_bin = FLT_MAX, max_bin = -FLT_MAX;
    const float width = range_ext / (float)num_bins;                                  // :213-222
    for (uint32_t i = 0; i < rows; ++i) {
        const float scl = 1.0f / (width * (float)(int)tot[i]);
        for (uint32_t j = 0; j < num_bins; ++j) { float v = (float)counts[(size_t)i * num_bins + j]; v *= scl; out_bins[(size_t)i * num_bins + j] = v; min_bin = std::min(min_bin, v); max_bin = std::max(max_bin, v); }
    }
    if (out_min_max) { out_min_max[0] = min_bin; out_min_max[1] = max_bin; }
    return 0;
}

// Radii of the three box passes per axis that approximate a Gaussian of `sigma` texels: boxes_for_gauss(., 3, sigma) of VIAMD's Ramachandran
// component (src/components/ramachandran/ramachandran.cpp:333-344), with the same float expressions so that the radii agree for every sigma.
static void rama_box_radii(int r[3], float sigma) {
    const float ideal = sqrtf(12 * sigma * sigma / 3 + 1);                                  // ideal width of one of three boxes
    int lo = (int)ideal; if (lo % 2 == 0) --lo;                                              // the odd width at or below it
    const float passes_lo = (12 * sigma * sigma - 3 * lo * lo - 12 * lo - 9) / (-4 * lo - 4);   // how many passes use lo, the rest lo + 2
    const int n_lo = (int)(passes_lo + 0.5f);
    for (int i = 0; i < 3; ++i) r[i] = i < n_lo ? lo : lo + 2;
}

int mdgpu_plan_rama_density(mdgpu_plan* p, size_t prop, const uint32_t* segments, const uint32_t class_offsets[5], uint32_t frame_beg, uint32_t frame_end,
                            float sigma, float* out_tex, float out_sum[4]) {
    if (!p || prop >= p->props.size() || !class_offsets || !out_tex || !out_sum) return fail(MDGPU_ERR_INVALID_ARG, "mdgpu_plan_rama_density: invalid argument");
    Prop& pr = p->props[prop];
    if (!pr.backbone_segments) return fail(MDGPU_ERR_INVALID_ARG, "property '%s' is not a backbone-angles property", pr.name.c_str());
    for (int c = 0; c < 4; ++c) if (class_offsets[c] > class_offsets[c + 1]) return fail(MDGPU_ERR_INVALID_ARG, "mdgpu_plan_rama_density: class offsets decrease");
    const uint32_t n_entries = class_offsets[4] - class_offsets[0];
    if (n_entries && !segments) return fail(MDGPU_ERR_INVALID_ARG, "mdgpu_plan_rama_density: no segment list");
    for (uint32_t e = class_offsets[0]; e < class_offsets[4]; ++e)
        if (segments[e] >= pr.backbone_segments) return fail(MDGPU_ERR_INVALID_ARG, "mdgpu_plan_rama_density: segment %u out of range (%zu segments)", segments[e], pr.backbone_segments);
    if (frame_beg > frame_end || frame_end > p->num_frames) return fail(MDGPU_ERR_INVALID_ARG, "mdgpu_plan_rama_density: frame range [%u, %u) outside [0, %zu)", frame_beg, frame_end, p->num_frames);
    // VIAMD's blur slider range; it keeps every box radius far below 256, which the wrap of the box passes assumes
    if (!(sigma >= 0.1f && sigma <= 10.0f)) return fail(MDGPU_ERR_INVALID_ARG, "mdgpu_plan_rama_density: sigma %g outside [0.1, 10]", (double)sigma);
    int rc = mdgpu_plan_sync(p); if (rc) return rc;   // multi-device plans hold every frame's rows on devices[0] = p->device from here on
    CUDA_TRY(cudaSetDevice(p->device));
    const size_t texels = 512 * 512 * 4;
    RamaArgs a{};
    DevBuf<unsigned long long> d_mask, d_counts, d_samples; DevBuf<uint32_t> d_seg; DevBuf<float> d_buf;
    if (upload_frame_mask(p, d_mask) != cudaSuccess) return fail(MDGPU_ERR_CUDA, d_mask.get() ? "frame mask upload failed (rama density)" : "device allocation failed (rama density)");
    if (d_seg.upload(segments ? segments + class_offsets[0] : nullptr, n_entries) != cudaSuccess ||
        d_counts.alloc(texels) != cudaSuccess || d_samples.alloc(4) != cudaSuccess || d_buf.alloc(3 * texels) != cudaSuccess)
        return fail(MDGPU_ERR_CUDA, "device allocation failed (rama density)");
    a.angles = pr.d_temporal.get(); a.n_seg = (uint32_t)pr.backbone_segments; a.seg = d_seg.get(); a.n_entries = n_entries;
    for (int c = 0; c < 3; ++c) a.class_end[c] = class_offsets[c + 1] - class_offsets[0];
    a.frame_beg = frame_beg; a.frame_count = frame_end - frame_beg; a.mask = d_mask.get();
    a.scale = (float)(1.0 / (2.0 * 3.1415926535897932));   // 1.0f / (2.0f * PI) with the double PI of md_common.h:157
    a.counts = d_counts.get(); a.samples = d_samples.get(); a.buf[0] = d_buf.get(); a.buf[1] = d_buf.get() + texels; a.buf[2] = d_buf.get() + 2 * texels;
    rama_box_radii(a.box, sigma); a.sm_count = p->sm_count;
    launch_rama_density(a, 0);
    uint64_t samples[4] = { 0, 0, 0, 0 };
    if (cudaMemcpy(out_tex, a.buf[1], sizeof(float) * texels, cudaMemcpyDeviceToHost) != cudaSuccess || cudaMemcpy(samples, d_samples.get(), sizeof(samples), cudaMemcpyDeviceToHost) != cudaSuccess)
        return fail(MDGPU_ERR_CUDA, "rama density failed: %s", cudaGetErrorString(cudaGetLastError()));
    for (int c = 0; c < 4; ++c) out_sum[c] = (float)(double)samples[c];   // den_sum: (float) of the task's double sum
    return 0;
}

int mdgpu_plan_secondary_structure(mdgpu_plan* p, size_t prop, uint32_t frame_beg, uint32_t frame_end, int32_t* out) {
    if (!p || prop >= p->props.size()) return fail(MDGPU_ERR_INVALID_ARG, "mdgpu_plan_secondary_structure: invalid argument");
    Prop& pr = p->props[prop];
    if (!pr.ss_segments) return fail(MDGPU_ERR_INVALID_ARG, "property '%s' is not a secondary-structure property", pr.name.c_str());
    if (!out && frame_end > frame_beg) return fail(MDGPU_ERR_INVALID_ARG, "mdgpu_plan_secondary_structure: no output array");
    if (frame_beg > frame_end || frame_end > p->num_frames) return fail(MDGPU_ERR_INVALID_ARG, "mdgpu_plan_secondary_structure: frame range [%u, %u) outside [0, %zu)", frame_beg, frame_end, p->num_frames);
    int rc = mdgpu_plan_sync(p); if (rc) return rc;   // multi-device plans hold every frame's rows on devices[0] = p->device from here on
    if (frame_end == frame_beg) return 0;
    CUDA_TRY(cudaSetDevice(p->device));
    const size_t n = (size_t)(frame_end - frame_beg) * pr.ss_segments;
    std::vector<float> rows(n);
    CUDA_TRY(cudaMemcpy(rows.data(), pr.d_temporal.get() + (size_t)frame_beg * pr.ss_segments, sizeof(float) * n, cudaMemcpyDeviceToHost));
    for (size_t k = 0; k < n; ++k) out[k] = (int32_t)rows[k];   // rows of frames not evaluated are 0 (MD_SECONDARY_STRUCTURE_UNKNOWN)
    return 0;
}

int mdgpu_plan_property_counts(mdgpu_plan* p, size_t prop, uint64_t* out, size_t out_len) {
    if (!p || !out || prop >= p->props.size()) return fail(MDGPU_ERR_INVALID_ARG, "mdgpu_plan_property_counts: invalid argument");
    int rc = mdgpu_plan_sync(p); if (rc) return rc;
    Prop& pr = p->props[prop];
    if (pr.d_acc.get()) {
        if (out_len < MDGPU_DIST_BINS) return fail(MDGPU_ERR_INVALID_ARG, "output too small");
        CUDA_TRY(cudaMemcpy(out, pr.d_acc.get(), sizeof(uint64_t) * MDGPU_DIST_BINS, cudaMemcpyDeviceToHost));
    } else if (pr.d_vol.get()) {
        const size_t nv = (size_t)MDGPU_VOL_DIM * MDGPU_VOL_DIM * MDGPU_VOL_DIM;
        if (out_len < nv) return fail(MDGPU_ERR_INVALID_ARG, "output too small");
        std::vector<uint32_t> v(nv); CUDA_TRY(cudaMemcpy(v.data(), pr.d_vol.get(), sizeof(uint32_t) * nv, cudaMemcpyDeviceToHost));
        for (size_t i = 0; i < nv; ++i) out[i] = v[i];
    } else return fail(MDGPU_ERR_UNSUPPORTED, "property '%s' has no integer accumulator", pr.name.c_str());
    return 0;
}

int mdgpu_plan_property_frame_counts(mdgpu_plan* p, size_t prop, uint32_t frame, uint32_t* out_bins, uint64_t* out_total) {
    if (!p || prop >= p->props.size() || frame >= p->num_frames) return fail(MDGPU_ERR_INVALID_ARG, "mdgpu_plan_property_frame_counts: invalid argument");
    int rc = mdgpu_plan_sync(p); if (rc) return rc;
    Prop& pr = p->props[prop];
    if (pr.op == MDGPU_OP_SDF && out_bins) return fail(MDGPU_ERR_UNSUPPORTED, "sdf '%s' keeps the per-frame hit total only, no bins", pr.name.c_str());
    if (pr.op != MDGPU_OP_RDF && pr.op != MDGPU_OP_SDF) return fail(MDGPU_ERR_UNSUPPORTED, "per-frame counts are kept for rdf and sdf properties only");
    if (out_bins) {
        if (!pr.d_keep.get()) return fail(MDGPU_ERR_INVALID_ARG, "plan was created without keep_frame_results");
        CUDA_TRY(cudaMemcpy(out_bins, pr.d_keep.get() + (size_t)frame * MDGPU_DIST_BINS, sizeof(uint32_t) * MDGPU_DIST_BINS, cudaMemcpyDeviceToHost));
    }
    if (out_total) { unsigned long long t = 0; CUDA_TRY(cudaMemcpy(&t, pr.d_frame_total.get() + frame, sizeof(t), cudaMemcpyDeviceToHost)); *out_total = t; }
    return 0;
}

int mdgpu_plan_property_aggregate(mdgpu_plan* p, size_t prop, float* out_mean, float* out_var, float* out_ext, size_t num_frames) {
    if (!p || prop >= p->props.size() || num_frames > p->num_frames) return fail(MDGPU_ERR_INVALID_ARG, "mdgpu_plan_property_aggregate: invalid argument");
    int rc = mdgpu_plan_sync(p); if (rc) return rc;
    const Prop& pr = p->props[prop];
    if (pr.agg_mean.empty()) return fail(MDGPU_ERR_INVALID_ARG, "property '%s' has one value per frame: no aggregate (md_script.c:5618)", pr.name.c_str());
    if (out_mean && out_mean != pr.amean) memcpy(out_mean, pr.amean, sizeof(float) * num_frames);
    if (out_var && out_var != pr.avar) memcpy(out_var, pr.avar, sizeof(float) * num_frames);
    if (out_ext && out_ext != pr.aext) memcpy(out_ext, pr.aext, sizeof(float) * 2 * num_frames);
    return 0;
}

// The md_script shim hands over md_script_property_data_t::values (and the aggregate arrays): results are written where VIAMD reads them.
int mdgpu_plan_bind_property_storage(mdgpu_plan* p, size_t prop, float* values, size_t num_values, float* agg_mean, float* agg_var, float* agg_ext) {
    if (!p || prop >= p->props.size() || !values) return fail(MDGPU_ERR_INVALID_ARG, "mdgpu_plan_bind_property_storage: invalid argument");
    Prop& pr = p->props[prop];
    if (num_values != pr.values.size()) return fail(MDGPU_ERR_INVALID_ARG, "property '%s' has %zu values, the bound array %zu", pr.name.c_str(), pr.values.size(), num_values);
    { int rc = mdgpu_plan_sync(p); if (rc) return rc; }
    std::lock_guard<std::mutex> guard(p->sync_mutex);
    memcpy(values, pr.vptr, sizeof(float) * num_values);
    pr.vptr = values; pr.data.values = values; pr.data.weights = pr.is_dist() ? values + MDGPU_DIST_BINS : nullptr;
    if (!pr.agg_mean.empty() && agg_mean && agg_var && agg_ext) {
        memcpy(agg_mean, pr.amean, sizeof(float) * p->num_frames); memcpy(agg_var, pr.avar, sizeof(float) * p->num_frames); memcpy(agg_ext, pr.aext, sizeof(float) * 2 * p->num_frames);
        pr.amean = agg_mean; pr.avar = agg_var; pr.aext = agg_ext;
    }
    return 0;
}

int mdgpu_plan_set_progress_callback(mdgpu_plan* p, mdgpu_progress_fn fn, void* user) {
    if (!p) return fail(MDGPU_ERR_INVALID_ARG, "null plan");
    std::lock_guard<std::mutex> guard(p->sync_mutex);
    p->progress_fn = fn; p->progress_user = user;
    if (p->multi) for (auto* q : p->multi->peers) { q->progress_fn = nullptr; }   // peers publish through the root at sync
    return 0;
}

// Run the calling thread (and the threads it creates later: ingest pool, loaders) on the CPUs next to the GPU: reads the device's
// local_cpulist from sysfs. Pinned buffers the thread allocates and first touches afterwards land on that NUMA node.
int mdgpu_bind_host_to_device(int device) {
    char bus[32] = {0};
    if (cudaDeviceGetPCIBusId(bus, sizeof(bus), device) != cudaSuccess) { cudaGetLastError(); return fail(MDGPU_ERR_CUDA, "cudaDeviceGetPCIBusId(%d) failed", device); }
    for (char* c = bus; *c; ++c) *c = (char)tolower(*c);
    char path[128]; snprintf(path, sizeof(path), "/sys/bus/pci/devices/%s/local_cpulist", bus);
    FILE* f = fopen(path, "r"); if (!f) return fail(MDGPU_ERR_UNSUPPORTED, "no %s", path);
    char line[4096] = {0}; if (!fgets(line, sizeof(line), f)) { fclose(f); return fail(MDGPU_ERR_UNSUPPORTED, "empty %s", path); } fclose(f);
    cpu_set_t set; CPU_ZERO(&set); int n = 0;
    for (char* tok = strtok(line, ",\n"); tok; tok = strtok(nullptr, ",\n")) {
        int a = 0, b = 0; const int k = sscanf(tok, "%d-%d", &a, &b); if (k < 1) continue; if (k == 1) b = a;
        for (int c = a; c <= b && c < CPU_SETSIZE; ++c) { CPU_SET(c, &set); ++n; }
    }
    if (!n) return fail(MDGPU_ERR_UNSUPPORTED, "no CPUs listed in %s", path);
    if (sched_setaffinity(0, sizeof(set), &set) != 0) return fail(MDGPU_ERR_UNSUPPORTED, "sched_setaffinity failed");
    return n;
}

int mdgpu_plan_exchange_stats(mdgpu_plan* p, double* last_ms, uint64_t* count) {
    if (!p) return fail(MDGPU_ERR_INVALID_ARG, "null plan");
    if (last_ms) *last_ms = p->multi ? p->multi->last_reduce_ms : 0.0; if (count) *count = p->multi ? p->multi->reduces : 0;
    return 0;
}
int mdgpu_plan_ingest_info(mdgpu_plan* p, size_t* atoms_per_frame, uint32_t* threads) {
    if (!p) return fail(MDGPU_ERR_INVALID_ARG, "null plan");
    if (atoms_per_frame) *atoms_per_frame = p->space[p->ingest_space()].num_atoms;
    if (threads) *threads = p->compact ? (uint32_t)(ingest_pool(p)->th.size() + 1) : 0u;
    return 0;
}

int mdgpu_debug_aggregate(const float* values, size_t count, float* out4) {
    if (!values || !out4 || !count) return fail(MDGPU_ERR_INVALID_ARG, "mdgpu_debug_aggregate: invalid argument");
    fold_frame_values(values, count, out4[0], out4[1], out4[2], out4[3]);
    return 0;
}

int mdgpu_plan_frame_mask(mdgpu_plan* p, uint64_t* out_words, size_t num_words) {
    if (!p || !out_words) return fail(MDGPU_ERR_INVALID_ARG, "null argument");
    std::lock_guard<std::mutex> lk(p->mask_mutex);
    for (size_t i = 0; i < num_words; ++i) out_words[i] = i < p->frame_mask.size() ? p->frame_mask[i] : 0ull;
    return 0;
}

int mdgpu_plan_property_accum_ptr(mdgpu_plan* p, size_t prop, void** d_ptr, size_t* bytes, uint32_t* elem_bytes) {
    if (!p || prop >= p->props.size() || !d_ptr || !bytes) return fail(MDGPU_ERR_INVALID_ARG, "invalid argument");
    Prop& pr = p->props[prop];
    auto give = [&](const auto& b) { *d_ptr = b.get(); *bytes = b.bytes(); if (elem_bytes) *elem_bytes = (uint32_t)(b.bytes() / b.size()); return 0; };
    if (pr.d_acc.get()) return give(pr.d_acc);
    if (pr.d_vol.get()) return give(pr.d_vol);
    if (pr.d_temporal.get()) return give(pr.d_temporal);   // float rows, zero where not evaluated
    return fail(MDGPU_ERR_UNSUPPORTED, "property '%s' has no accumulator", pr.name.c_str());
}

int mdgpu_plan_property_frame_rows(mdgpu_plan* p, size_t prop, uint32_t which, void** d_ptr, size_t* bytes, uint32_t* elem_bytes) {
    if (!p || prop >= p->props.size() || !d_ptr || !bytes || !elem_bytes) return fail(MDGPU_ERR_INVALID_ARG, "invalid argument");
    Prop& pr = p->props[prop];
    *d_ptr = nullptr; *bytes = 0; *elem_bytes = 0;
    auto give = [&](const auto& b) { *d_ptr = b.get(); *bytes = b.bytes(); *elem_bytes = (uint32_t)(b.bytes() / b.size()); };
    if (which == 0 && pr.d_frame_total.get()) give(pr.d_frame_total);
    else if (which == 1 && pr.d_frame_n.get()) give(pr.d_frame_n);
    else if (which == 1 && pr.d_frame_min.get()) give(pr.d_frame_min);
    else if (which == 1 && pr.d_frame_min64.get()) give(pr.d_frame_min64);
    else if (which == 2 && pr.d_frame_max.get()) give(pr.d_frame_max);
    else if (which == 2 && pr.d_frame_max64.get()) give(pr.d_frame_max64);
    return 0;   // a property without that row returns a null pointer
}

int mdgpu_plan_mark_frames_done(mdgpu_plan* p, uint32_t frame_beg, uint32_t count) {
    if (!p || (size_t)frame_beg + count > p->num_frames) return fail(MDGPU_ERR_INVALID_ARG, "mdgpu_plan_mark_frames_done: frame range out of bounds");
    mark_frames(p, frame_beg, count);
    p->dirty = true;
    return 0;
}

int mdgpu_plan_set_frames_accumulated(mdgpu_plan* p, size_t prop, uint64_t frames) {
    if (!p || prop >= p->props.size()) return fail(MDGPU_ERR_INVALID_ARG, "invalid argument");
    p->props[prop].frames_accumulated = frames; p->props[prop].frames_overridden = true; p->dirty = true;
    return 0;
}

int mdgpu_plan_enable_kernel_timing(mdgpu_plan* p, int enable) {
    if (!p) return MDGPU_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> guard(p->submit_mutex);
    if (enable && !p->d_counters.get()) { CUDA_TRY(cudaSetDevice(p->device)); CUDA_TRY(p->d_counters.alloc(8)); CUDA_TRY(cudaMemset(p->d_counters.get(), 0, p->d_counters.bytes())); }
    p->timing = enable != 0; return 0;
}

// measurement counters of the pair kernel (filled while kernel timing is enabled): which = 0 executed pair tests (padding lanes included), 1 useful ones
int mdgpu_plan_kernel_counter(mdgpu_plan* p, uint32_t which, uint64_t* value) {
    if (!p || !value || which >= 8) return fail(MDGPU_ERR_INVALID_ARG, "mdgpu_plan_kernel_counter: invalid argument");
    int rc = mdgpu_plan_sync(p); if (rc) return rc;
    *value = 0;
    if (p->d_counters.get()) { unsigned long long v = 0; CUDA_TRY(cudaMemcpy(&v, p->d_counters.get() + which, sizeof(v), cudaMemcpyDeviceToHost)); *value = v; }
    return 0;
}

int mdgpu_plan_kernel_time_ms(mdgpu_plan* p, const char* kernel, double* total_ms, uint64_t* launches) {
    if (!p) return fail(MDGPU_ERR_INVALID_ARG, "null plan");
    const int kind = (kernel && strncmp(kernel, "k_sdf", 5) == 0) ? 1 : (kernel && strncmp(kernel, "k_density", 9) == 0) ? 2 : (kernel && strncmp(kernel, "k_rdf_cull", 10) == 0) ? 3 : 0;
    int rc = mdgpu_plan_sync(p); if (rc) return rc;
    if (total_ms) *total_ms = p->timed_ms[kind]; if (launches) *launches = p->timed_n[kind];
    return 0;
}

int mdgpu_plan_timer_begin(mdgpu_plan* p) {
    if (!p) return fail(MDGPU_ERR_INVALID_ARG, "null plan");
    CUDA_TRY(cudaSetDevice(p->device));
    for (auto& s : p->slots) { int rc = retire_slot(p, s); if (rc) return rc; }
    CUDA_TRY(cudaDeviceSynchronize());
    if (!p->t_begin) CUDA_TRY(cudaEventCreate(p->t_begin.out()));
    // the device is idle: an event on the legacy default stream is reached immediately and precedes everything enqueued later
    CUDA_TRY(cudaEventRecord(p->t_begin, p->slots.empty() ? (cudaStream_t)0 : p->slots[0].stream));
    return 0;
}

int mdgpu_plan_timer_end(mdgpu_plan* p, double* elapsed_ms) {
    if (!p || !elapsed_ms || !p->t_begin) return fail(MDGPU_ERR_INVALID_ARG, "mdgpu_plan_timer_end without _begin");
    CUDA_TRY(cudaSetDevice(p->device));
    while (p->t_end.size() < p->slots.size()) { Event e; CUDA_TRY(cudaEventCreate(e.out())); p->t_end.push_back(std::move(e)); }
    for (size_t i = 0; i < p->slots.size(); ++i) CUDA_TRY(cudaEventRecord(p->t_end[i], p->slots[i].stream));
    double best = 0.0;
    for (size_t i = 0; i < p->slots.size(); ++i) {
        CUDA_TRY(cudaEventSynchronize(p->t_end[i]));
        float ms = 0.f; CUDA_TRY(cudaEventElapsedTime(&ms, p->t_begin, p->t_end[i]));
        if (ms > best) best = ms;
    }
    *elapsed_ms = best;
    return 0;
}

int mdgpu_debug_frame_geom(const mdgpu_unitcell_t* cell, double cell_ext, double cutoff, const float* aabb, int32_t* out_i, float* out_f) {
    if (!cell || !out_i || !out_f) return fail(MDGPU_ERR_INVALID_ARG, "null argument");
    FrameGeom g; host_frame_geom(&g, cell, cell_ext, cutoff, aabb, 0xffffffffu);
    for (int k = 0; k < 3; ++k) { out_i[k] = g.cdim[k]; out_i[3 + k] = g.ncell[k]; out_i[6 + k] = g.hlo[k]; out_i[9 + k] = g.hdim[k]; }
    out_i[12] = g.valid;
    out_f[0] = g.G00; out_f[1] = g.G11; out_f[2] = g.G22; out_f[3] = g.H01; out_f[4] = g.H02; out_f[5] = g.H12; out_f[6] = g.r2;
    return 0;
}

int mdgpu_debug_sqrt_sweep(int device, uint32_t lo_bits, uint32_t hi_bits, uint64_t* mismatches) {
    if (!mismatches) return fail(MDGPU_ERR_INVALID_ARG, "null argument");
    CUDA_TRY(cudaSetDevice(device));
    *mismatches = run_sqrt_sweep(lo_bits, hi_bits);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

int mdgpu_debug_rdf_config(char* out, size_t n) {
    if (!out) return fail(MDGPU_ERR_INVALID_ARG, "null argument");
    const RdfCullConfig c = rdf_cull_config();
    char name[16];
    if (c.kind == RDF_CULL_HALF) snprintf(name, sizeof(name), "half");
    else snprintf(name, sizeof(name), "%s%d", c.kind == RDF_CULL_FLAT ? "flat" : "full", c.occ);
    if (strlen(name) >= n) return fail(MDGPU_ERR_INVALID_ARG, "mdgpu_debug_rdf_config: buffer of %zu bytes too small", n);
    memcpy(out, name, strlen(name) + 1);
    return 0;
}

// ------------------------------------------------------------------------------------------------- synthetic workloads
int mdgpu_synth_water_desc(uint32_t n, uint32_t seed, uint32_t* num_atoms, float* L) {
    const mdsynth_water_t w = mdsynth_water_desc(n, seed);
    if (num_atoms) *num_atoms = w.num_atoms; if (L) *L = w.L;
    return 0;
}

int mdgpu_synth_water_base(uint32_t n, uint32_t seed, float* base_xyz, float* whole_xyz) {
    const mdsynth_water_t w = mdsynth_water_desc(n, seed);
    const size_t N = w.num_atoms;
    mdsynth_water_base(&w, base_xyz, base_xyz ? base_xyz + N : nullptr, base_xyz ? base_xyz + 2 * N : nullptr,
                       whole_xyz, whole_xyz ? whole_xyz + N : nullptr, whole_xyz ? whole_xyz + 2 * N : nullptr);
    return 0;
}

int mdgpu_synth_water_frames_host(uint32_t n, uint32_t seed, const float* base_xyz, uint32_t frame_beg, uint32_t count,
                                  float* out_xyz, size_t frame_stride, size_t axis_stride) {
    if (!base_xyz || !out_xyz) return fail(MDGPU_ERR_INVALID_ARG, "null argument");
    const mdsynth_water_t w = mdsynth_water_desc(n, seed); const size_t N = w.num_atoms;
    for (uint32_t i = 0; i < count; ++i) {
        float* o = out_xyz + (size_t)i * frame_stride;
        mdsynth_water_frame(&w, frame_beg + i, base_xyz, base_xyz + N, base_xyz + 2 * N, o, o + axis_stride, o + 2 * axis_stride);
    }
    return 0;
}

// frames [frame_beg, frame_beg + count) of a synthetic trajectory, 32768 frames per launch (mol_id null: water)
static int synth_frames_device(int device, uint32_t seed, float Lx, float Ly, float Lz, uint32_t num_atoms, const float* d_base_xyz, const uint32_t* d_mol_id,
                               uint32_t frame_beg, uint32_t count, float* d_out_xyz, size_t frame_stride, size_t axis_stride) {
    CUDA_TRY(cudaSetDevice(device));
    for (uint32_t c0 = 0; c0 < count; c0 += 32768) {
        const uint32_t c = std::min(32768u, count - c0);
        launch_synth_frames(seed, Lx, Ly, Lz, num_atoms, d_base_xyz, num_atoms, d_mol_id, frame_beg + c0, c, d_out_xyz + (size_t)c0 * frame_stride, frame_stride, axis_stride, 0);
    }
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaDeviceSynchronize());
    return 0;
}

int mdgpu_synth_water_frames_device(int device, uint32_t n, uint32_t seed, const float* d_base_xyz, uint32_t frame_beg, uint32_t count,
                                    float* d_out_xyz, size_t frame_stride, size_t axis_stride) {
    if (!d_base_xyz || !d_out_xyz) return fail(MDGPU_ERR_INVALID_ARG, "null argument");
    const mdsynth_water_t w = mdsynth_water_desc(n, seed);
    return synth_frames_device(device, seed, w.L, w.L, w.L, w.num_atoms, d_base_xyz, nullptr, frame_beg, count, d_out_xyz, frame_stride, axis_stride);
}

int mdgpu_synth_membrane_desc(uint32_t nl, uint32_t nw_xy, uint32_t nwz, uint32_t seed, uint32_t* num_atoms, uint32_t* num_lipids, float* L3) {
    const mdsynth_membrane_t m = mdsynth_membrane_desc(nl, nw_xy, nwz, seed);
    if (num_atoms) *num_atoms = m.num_atoms; if (num_lipids) *num_lipids = m.num_lipids;
    if (L3) { L3[0] = m.Lx; L3[1] = m.Ly; L3[2] = m.Lz; }
    return 0;
}

int mdgpu_synth_membrane_base(uint32_t nl, uint32_t nw_xy, uint32_t nwz, uint32_t seed, float* base_xyz, float* whole_xyz, uint32_t* mol_id) {
    const mdsynth_membrane_t m = mdsynth_membrane_desc(nl, nw_xy, nwz, seed);
    mdsynth_membrane_base(&m, base_xyz, whole_xyz, mol_id);
    return 0;
}

int mdgpu_synth_membrane_frames_host(uint32_t nl, uint32_t nw_xy, uint32_t nwz, uint32_t seed, const float* base_xyz, const uint32_t* mol_id,
                                     uint32_t frame_beg, uint32_t count, float* out_xyz, size_t frame_stride, size_t axis_stride) {
    if (!base_xyz || !mol_id || !out_xyz) return fail(MDGPU_ERR_INVALID_ARG, "null argument");
    const mdsynth_membrane_t m = mdsynth_membrane_desc(nl, nw_xy, nwz, seed);
    for (uint32_t i = 0; i < count; ++i) {
        float* o = out_xyz + (size_t)i * frame_stride;
        mdsynth_membrane_frame(&m, frame_beg + i, base_xyz, mol_id, o, o + axis_stride, o + 2 * axis_stride);
    }
    return 0;
}

int mdgpu_synth_membrane_frames_device(int device, uint32_t nl, uint32_t nw_xy, uint32_t nwz, uint32_t seed, const float* d_base_xyz, const uint32_t* d_mol_id,
                                       uint32_t frame_beg, uint32_t count, float* d_out_xyz, size_t frame_stride, size_t axis_stride) {
    if (!d_base_xyz || !d_mol_id || !d_out_xyz) return fail(MDGPU_ERR_INVALID_ARG, "null argument");
    const mdsynth_membrane_t m = mdsynth_membrane_desc(nl, nw_xy, nwz, seed);
    return synth_frames_device(device, seed, m.Lx, m.Ly, m.Lz, m.num_atoms, d_base_xyz, d_mol_id, frame_beg, count, d_out_xyz, frame_stride, axis_stride);
}

// ------------------------------------------------------------------------------------------------- memory helpers
int mdgpu_device_alloc(int device, size_t bytes, void** out) { if (!out) return MDGPU_ERR_INVALID_ARG; CUDA_TRY(cudaSetDevice(device)); CUDA_TRY(cudaMalloc(out, bytes)); return 0; }
int mdgpu_device_free(int device, void* ptr) { CUDA_TRY(cudaSetDevice(device)); CUDA_TRY(cudaFree(ptr)); return 0; }
int mdgpu_host_alloc_pinned(size_t bytes, void** out) { if (!out) return MDGPU_ERR_INVALID_ARG; CUDA_TRY(cudaMallocHost(out, bytes)); return 0; }
int mdgpu_host_free_pinned(void* ptr) { CUDA_TRY(cudaFreeHost(ptr)); return 0; }
int mdgpu_memcpy_h2d(int device, void* dst, const void* src, size_t bytes) { CUDA_TRY(cudaSetDevice(device)); CUDA_TRY(cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice)); return 0; }
int mdgpu_memcpy_d2h(int device, void* dst, const void* src, size_t bytes) { CUDA_TRY(cudaSetDevice(device)); CUDA_TRY(cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost)); return 0; }
int mdgpu_device_synchronize(int device) { CUDA_TRY(cudaSetDevice(device)); CUDA_TRY(cudaDeviceSynchronize()); return 0; }

}  // extern "C"
