// binding.cpp -- pybind11 module `_pcu_internal`, the layer between the Python package and the C ABI of
// libpcu_b200.so (include/pcu_b200.h).  All computation goes through that ABI; there is no CPU implementation
// behind these functions.  The drop-in boundary is the Python package: it checks every argument, with the reference's
// rules and messages, before it calls in here.  The module has three kinds of functions:
//   - numpy entry points, which run the library's host entry points.  The nearest-neighbour family's (`_*_host` and
//     `_chamfer_stats`) take arrays the package has checked and keep only a guard against arrays their C entry point
//     would read out of bounds; they return the library's int64 indices, squeezed k-NN outputs and statistics records
//     as numpy records of pcu_b200_nn_stats.  The
//     Morton-code functions are still named after the reference's bindings and keep its checks;
//   - device entry points (`_*_device`), which the Python package uses for CUDA torch tensors: the caller passes
//     data_ptr()s, a device and a stream handle; nothing is copied and nothing synchronises unless the C entry point
//     says so.  Those that only forward to the C ABI are generated from the C signatures (Forward below); the rest
//     build host arrays or option structs, or return handles, counts or vectors;
//   - handle destroyers and diagnostics.
#include <pybind11/pybind11.h>
#include <pybind11/numpy.h>
#include <pybind11/stl.h>

#include <algorithm>
#include <array>
#include <cstdint>
#include <map>
#include <memory>
#include <mutex>
#include <stdexcept>
#include <string>
#include <tuple>
#include <type_traits>
#include <utility>
#include <vector>

#include "../../include/pcu_b200.h"

namespace py = pybind11;

namespace {

[[noreturn]] void raise_status(int status) {
    const std::string msg = pcu_b200_last_error();
    switch (status) {
        case PCU_B200_INVALID_ARGUMENT: throw py::value_error(msg);
        case PCU_B200_OUT_OF_MEMORY: throw std::bad_alloc();
        default: throw std::runtime_error("pcu_b200: " + msg);
    }
}
inline void check(int status) { if (status != PCU_B200_OK) raise_status(status); }

// One workspace per (device, stream): a workspace serves one stream at a time.  Calls that share a
// workspace (several Python threads on the same stream) are serialised by that workspace's own mutex:
// enqueueing is what must not interleave, the work itself is ordered by the stream.  Calls on different
// devices or streams never wait for each other.
// The numpy (host-pointer) entry points run on the workspace's private stream; they get workspaces of
// their own under the key kHostKey, so they never share scratch with a device-pointer call that may still
// be queued on one of the caller's streams (stream handle 0 is torch's default stream, not "host").
constexpr uintptr_t kHostKey = ~(uintptr_t)0;
struct Slot {
    pcu_b200_workspace* ws = nullptr;
    std::mutex busy;
};
struct Pool {
    std::mutex mu;
    std::map<std::pair<int, uintptr_t>, std::unique_ptr<Slot>> items;
    Slot& get(int device, uintptr_t stream) {
        std::lock_guard<std::mutex> lock(mu);
        auto key = std::make_pair(device, stream);
        auto it = items.find(key);
        if (it != items.end()) return *it->second;
        std::unique_ptr<Slot> slot(new Slot());
        check(pcu_b200_workspace_create(device, &slot->ws));
        Slot& ref = *slot;
        items[key] = std::move(slot);
        return ref;
    }
    void clear() {
        std::lock_guard<std::mutex> lock(mu);
        for (auto& kv : items) pcu_b200_workspace_destroy(kv.second->ws);
        items.clear();
    }
};
Pool& pool() { static Pool p; return p; }
// Released GIL + exclusive use of one workspace for the duration of one call.
struct CallScope {
    py::gil_scoped_release nogil;
    std::lock_guard<std::mutex> lock;
    explicit CallScope(Slot& slot) : nogil(), lock(slot.busy) {}
};

// Result arrays of 1 MiB and more are backed by page-locked host memory: the device-to-host copy of a large
// k-NN result into a fresh pageable numpy array is bound by page faults, into pinned memory by PCIe.  Page-locking is slow itself, so blocks are
// recycled: when the numpy array that owns one is garbage-collected the block returns to this pool (at most
// kKeepBytes stay cached; anything beyond is unpinned and released).  Allocation failure or a pool over its
// budget of outstanding blocks falls back to an ordinary numpy array.
class PinnedPool {
public:
    static constexpr size_t kMinBytes = size_t(1) << 20;
    static constexpr size_t kKeepBytes = size_t(6) << 30;
    static constexpr size_t kMaxOutstanding = size_t(24) << 30;
    void* take(size_t bytes, size_t& capacity) {
        capacity = (bytes + (size_t(2) << 20) - 1) & ~((size_t(2) << 20) - 1);
        {
            std::lock_guard<std::mutex> lock(mu_);
            auto it = free_.lower_bound(capacity);
            if (it != free_.end() && it->first <= capacity + capacity / 4) {
                void* p = it->second;
                capacity = it->first;
                cached_ -= it->first;
                free_.erase(it);
                outstanding_ += capacity;
                return p;
            }
            if (outstanding_ + capacity > kMaxOutstanding) return nullptr;
            outstanding_ += capacity;
        }
        void* p = nullptr;
        if (pcu_b200_host_alloc(&p, (int64_t)capacity) != PCU_B200_OK) {
            std::lock_guard<std::mutex> lock(mu_);
            outstanding_ -= capacity;
            return nullptr;
        }
        return p;
    }
    void give(void* p, size_t capacity) {
        bool release = false;
        {
            std::lock_guard<std::mutex> lock(mu_);
            outstanding_ -= capacity;
            if (closed_ || cached_ + capacity > kKeepBytes) release = true;
            else { free_.emplace(capacity, p); cached_ += capacity; }
        }
        if (release) pcu_b200_host_free(p);
    }
    void clear(bool close) {
        std::multimap<size_t, void*> drop;
        {
            std::lock_guard<std::mutex> lock(mu_);
            drop.swap(free_);
            cached_ = 0;
            if (close) closed_ = true;
        }
        for (auto& kv : drop) pcu_b200_host_free(kv.second);
    }
private:
    std::mutex mu_;
    std::multimap<size_t, void*> free_;
    size_t cached_ = 0, outstanding_ = 0;
    bool closed_ = false;
};
PinnedPool& pinned_pool() { static PinnedPool* p = new PinnedPool(); return *p; }   // outlives late array destructors

struct PinnedBlock { void* ptr; size_t capacity; };

// A C-contiguous (rows, cols) array of T: page-locked and pool-backed when it is large, ordinary otherwise.
template <typename T>
py::array_t<T> result_array(py::ssize_t rows, py::ssize_t cols) {
    const size_t bytes = (size_t)rows * (size_t)cols * sizeof(T);
    if (bytes >= PinnedPool::kMinBytes) {
        size_t capacity = 0;
        void* p = pinned_pool().take(bytes, capacity);
        if (p != nullptr) {
            auto* block = new PinnedBlock{p, capacity};
            py::capsule owner(block, [](void* b) {
                auto* blk = static_cast<PinnedBlock*>(b);
                pinned_pool().give(blk->ptr, blk->capacity);
                delete blk;
            });
            return py::array_t<T>({rows, cols}, {(py::ssize_t)(cols * sizeof(T)), (py::ssize_t)sizeof(T)}, static_cast<T*>(p), owner);
        }
    }
    return py::array_t<T>({rows, cols});
}

// pcu.pinned_empty: an (n, 3) array of T in page-locked memory next to the current GPU, for callers who fill their
// clouds in place (what torch's pin_memory() gives, with the placement taken care of: pcu_b200_host_alloc)
template <typename T>
py::array pinned_cloud(py::ssize_t rows, py::ssize_t cols) {
    if (rows <= 0 || cols <= 0) throw py::value_error("shape must be positive");
    const size_t bytes = (size_t)rows * (size_t)cols * sizeof(T);
    void* p = nullptr;
    check(pcu_b200_host_alloc(&p, (int64_t)bytes));
    py::capsule owner(p, [](void* q) { pcu_b200_host_free(q); });
    return py::array_t<T>({rows, cols}, {(py::ssize_t)(cols * sizeof(T)), (py::ssize_t)sizeof(T)}, static_cast<T*>(p), owner);
}

struct Options { float occupancy = 0.f; int disable_replay = 0; int binning = 0; int host_staging = 0; };
Options& defaults() { static Options o; return o; }
constexpr int kDefaultLeaf = 10;   // the leaf size of calls that take none

// Validates the per-call options (with the GIL held); they are applied to the workspace inside the
// call's exclusive section so that concurrent callers cannot mix them up.
pcu_b200_options make_options(int max_points_per_leaf) {
    if (max_points_per_leaf <= 0) throw py::value_error("max_points_per_leaf must be greater than 0.");
    pcu_b200_options o{};
    o.max_points_per_leaf = max_points_per_leaf;
    o.cell_occupancy = defaults().occupancy;
    o.disable_tie_replay = defaults().disable_replay;
    o.binning = defaults().binning;
    o.host_staging = defaults().host_staging;
    return o;
}

// Every binding enters a workspace here: the workspace of (device, key), the process defaults plus this call's leaf
// size, then `call(ws)` with the GIL released and the workspace held exclusively, under exactly those options (never
// what an earlier call left behind).  A failed status becomes a Python exception.
template <class F>
void on_workspace(int device, uintptr_t key, int leaf, F&& call) {
    Slot& slot = pool().get(device, key);
    const pcu_b200_options opts = make_options(leaf);
    int status;
    {
        CallScope scope(slot);
        status = pcu_b200_workspace_set_options(slot.ws, &opts);
        if (status == PCU_B200_OK) status = call(slot.ws);
    }
    check(status);
}

// The _f32 or the _f64 entry point of a pair, for inputs of type T.
template <typename T, class F32, class F64>
auto pick(F32 f32, F64 f64) {
    static_assert(std::is_same_v<T, float> || std::is_same_v<T, double>, "inputs are float or double");
    if constexpr (std::is_same_v<T, float>) return f32;
    else return f64;
}

// Device bindings that only forward to one C entry point int f(pcu_b200_workspace*, A..., void* stream), or to one of a
// pair f_f32 / f_f64, are built from that signature.  The Python function takes ([is_f64,] A'..., [max_points_per_leaf,]
// device, stream), A' being A with every pointer passed as an integer address; it runs f on the workspace of (device,
// stream), with each address converted to f's own parameter type and stream passed on as f's stream.
template <class F> struct CParams;
template <class... A> struct CParams<int (*)(pcu_b200_workspace*, A...)> { using type = std::tuple<A...>; };
template <class F, size_t I> using c_param_t = std::tuple_element_t<I, typename CParams<F>::type>;
template <class F> constexpr size_t c_arity = std::tuple_size_v<typename CParams<F>::type>;
template <class T> using py_param_t = std::conditional_t<std::is_pointer_v<T>, uintptr_t, T>;
template <class T> T from_py(py_param_t<T> a) {
    if constexpr (std::is_pointer_v<T>) return reinterpret_cast<T>(a);
    else return a;
}
template <class A, class B> constexpr bool same_up_to_pointee = std::is_pointer_v<A> ? std::is_pointer_v<B> : std::is_same_v<A, B>;

template <class F32, class F64, class = std::make_index_sequence<c_arity<F32> - 1>> struct Forward;
template <class F32, class F64, size_t... I> struct Forward<F32, F64, std::index_sequence<I...>> {
    static_assert(std::is_same_v<c_param_t<F32, sizeof...(I)>, void*>, "an entry point's last parameter is its stream");
    static_assert(c_arity<F64> == c_arity<F32> && (same_up_to_pointee<c_param_t<F32, I>, c_param_t<F64, I>> && ...),
                  "the _f32 and _f64 entry points differ only in pointer types");
    F32 f32;
    F64 f64;

    void run(bool is_f64, int leaf, int device, uintptr_t stream, py_param_t<c_param_t<F32, I>>... a) const {
        on_workspace(device, stream, leaf, [&](pcu_b200_workspace* ws) {
            return is_f64 ? f64(ws, from_py<c_param_t<F64, I>>(a)..., (void*)stream)
                          : f32(ws, from_py<c_param_t<F32, I>>(a)..., (void*)stream);
        });
    }
    auto single() const {
        return [e = *this](py_param_t<c_param_t<F32, I>>... a, int device, uintptr_t stream) {
            e.run(false, kDefaultLeaf, device, stream, a...);
        };
    }
    auto single_with_leaf() const {
        return [e = *this](py_param_t<c_param_t<F32, I>>... a, int max_points_per_leaf, int device, uintptr_t stream) {
            e.run(false, max_points_per_leaf, device, stream, a...);
        };
    }
    auto pair() const {
        return [e = *this](bool is_f64, py_param_t<c_param_t<F32, I>>... a, int device, uintptr_t stream) {
            e.run(is_f64, kDefaultLeaf, device, stream, a...);
        };
    }
    auto pair_with_leaf() const {
        return [e = *this](bool is_f64, py_param_t<c_param_t<F32, I>>... a, int max_points_per_leaf, int device, uintptr_t stream) {
            e.run(is_f64, max_points_per_leaf, device, stream, a...);
        };
    }
};
template <class F> Forward<F, F> forward_to(F f) { return {f, f}; }
template <class F32, class F64> Forward<F32, F64> forward_to(F32 f32, F64 f64) { return {f32, f64}; }

// Frees a handle with the library's destroy function f, without the GIL.
template <class H> auto destroy(int (*f)(H*)) {
    return [f](uintptr_t handle) {
        py::gil_scoped_release nogil;
        f(reinterpret_cast<H*>(handle));
    };
}

template <typename T>
py::array_t<T, py::array::c_style> dense(const py::array& a) {
    return py::array_t<T, py::array::c_style | py::array::forcecast>::ensure(a);
}

// The host entry points take arrays the Python package has checked against the reference's rules.  This guard only
// keeps an array of another dtype or shape from reaching a C entry point, which would read out of bounds: a C-contiguous
// (rows, 3) array of T (rows < 0: any number of rows), copied into one when it is laid out otherwise.
template <typename T>
py::array_t<T, py::array::c_style> points_of(const py::array& a, int64_t rows = -1) {
    if (!a.dtype().is(py::dtype::of<T>()) || a.ndim() != 2 || a.shape(1) != 3 || (rows >= 0 && a.shape(0) != rows))
        throw py::value_error("pcu_b200: expected an (n, 3) array of the points' dtype");
    return dense<T>(a);
}
bool is_f64(const py::array& a) { return a.dtype().is(py::dtype::of<double>()); }

// device < 0: the caller named none (the reference's interface has no such argument) -> the library's rule
// (PCU_B200_DEVICE, the CUDA runtime's current device, LOCAL_RANK, 0; see pcu_b200_current_device)
int current_device_or_default(int device) { return device < 0 ? pcu_b200_current_device() : device; }

// k nearest neighbours of numpy queries: (dists, corrs), squeezed as npe::move squeezes them (pinned for (n, 1) -> (n,)
// by tests/test_examples.py:363-368).  knn(ws, queries, n, dists, corrs) runs the host entry point against the dataset.
template <typename T, class F>
py::tuple knn_host(const py::array& q_in, int k, int leaf, int device, F&& knn) {
    auto q = points_of<T>(q_in);
    const int64_t n = q.shape(0);
    py::array_t<T> dists = result_array<T>((py::ssize_t)n, (py::ssize_t)k);
    py::array_t<int64_t> corrs = result_array<int64_t>((py::ssize_t)n, (py::ssize_t)k);
    on_workspace(device, kHostKey, leaf, [&](pcu_b200_workspace* ws) { return knn(ws, q.data(), n, dists.mutable_data(), corrs.mutable_data()); });
    return py::make_tuple(dists.attr("squeeze")(), corrs.attr("squeeze")());
}

template <typename T>
py::tuple knn_numpy_t(const py::array& q, const py::array& d_in, int k, bool squared, int leaf, int device) {
    auto d = points_of<T>(d_in);
    return knn_host<T>(q, k, leaf, device, [&](pcu_b200_workspace* ws, const T* qp, int64_t n, T* dists, int64_t* corrs) {
        int64_t tied = 0;
        return pick<T>(pcu_b200_knn_host_f32, pcu_b200_knn_host_f64)(ws, qp, n, d.data(), d.shape(0), k, squared, dists, corrs, &tied);
    });
}
py::tuple knn_numpy(const py::array& q, const py::array& d, int k, bool squared, int leaf, int device) {
    const int dev = current_device_or_default(device);
    return is_f64(q) ? knn_numpy_t<double>(q, d, k, squared, leaf, dev) : knn_numpy_t<float>(q, d, k, squared, leaf, dev);
}

// The fused statistics sweep(s) of numpy points x, one way or both: (the Chamfer value in the input precision, or None
// one way; the record x -> y; the record y -> x, zero one way).  The records are numpy records of the struct itself
// (PYBIND11_NUMPY_DTYPE below), the type the Python package reads device records as.
// sweep(ws, x, n, records, value or nullptr) runs the host entry point against the second cloud.
template <typename T, class F>
py::tuple stats_host(const py::array& x_in, bool both, int leaf, int device, F&& sweep) {
    auto x = points_of<T>(x_in);
    py::array_t<pcu_b200_nn_stats> recs(2);
    std::fill_n(recs.mutable_data(), 2, pcu_b200_nn_stats{});
    T v = 0;
    on_workspace(device, kHostKey, leaf, [&](pcu_b200_workspace* ws) { return sweep(ws, x.data(), x.shape(0), recs.mutable_data(), both ? &v : nullptr); });
    return py::make_tuple(both ? py::object(py::dtype::of<T>().attr("type")(v)) : py::object(py::none()), recs[py::int_(0)], recs[py::int_(1)]);
}

template <typename T>
py::tuple stats_numpy_t(const py::array& x, const py::array& y_in, bool both, int leaf, int device) {
    auto y = points_of<T>(y_in);
    return stats_host<T>(x, both, leaf, device, [&](pcu_b200_workspace* ws, const T* xp, int64_t n, pcu_b200_nn_stats* st, T* v) {
        return v ? pick<T>(pcu_b200_chamfer_host_f32, pcu_b200_chamfer_host_f64)(ws, xp, n, y.data(), y.shape(0), st, v)
                 : pick<T>(pcu_b200_nn_stats_host_f32, pcu_b200_nn_stats_host_f64)(ws, xp, n, y.data(), y.shape(0), st);
    });
}
py::tuple stats_numpy(const py::array& x, const py::array& y, int leaf, int device, bool both) {
    const int dev = current_device_or_default(device);
    return is_f64(x) ? stats_numpy_t<double>(x, y, both, leaf, dev) : stats_numpy_t<float>(x, y, both, leaf, dev);
}

// The normal estimators on numpy points (src/point_cloud_normals.cpp:303-411): (indices of the kept points, their unit
// normals).  view_dirs is a (0, 3) array when no view directions are given, as in the reference's wrapper.
// estimate(ws, points, n, view_dirs or nullptr, idx, normals, &kept) runs the host entry point.
template <typename T, class F>
py::tuple normals_host(const py::array& p_in, const py::array& v_in, int leaf, int device, F&& estimate) {
    auto pts = points_of<T>(p_in);
    const int64_t n = pts.shape(0);
    auto dirs = points_of<T>(v_in, v_in.ndim() == 2 && v_in.shape(0) == 0 ? 0 : n);
    const bool has_dirs = dirs.shape(0) != 0;
    py::array_t<int64_t> idx({(py::ssize_t)n});
    py::array_t<T> normals({(py::ssize_t)n, (py::ssize_t)3});
    int64_t kept = 0;
    on_workspace(device, kHostKey, leaf, [&](pcu_b200_workspace* ws) {
        return estimate(ws, pts.data(), n, has_dirs ? dirs.data() : nullptr, idx.mutable_data(), normals.mutable_data(), &kept);
    });
    idx.resize({(py::ssize_t)kept});
    normals.resize({(py::ssize_t)kept, (py::ssize_t)3});
    return py::make_tuple(idx, normals);
}

template <typename T>
py::tuple normals_knn_t(const py::array& p, const py::array& v, int k, double drop_angle, int leaf, int device) {
    return normals_host<T>(p, v, leaf, device, [&](pcu_b200_workspace* ws, const T* pts, int64_t n, const T* dirs, int64_t* idx,
                                                   T* normals, int64_t* kept) {
        return pick<T>(pcu_b200_normals_knn_host_f32, pcu_b200_normals_knn_host_f64)(ws, pts, n, dirs, k, drop_angle, idx, normals, kept);
    });
}
py::tuple normals_knn_numpy(const py::array& p, const py::array& v, int k, double drop_angle, int leaf, int device) {
    const int dev = current_device_or_default(device);
    return is_f64(p) ? normals_knn_t<double>(p, v, k, drop_angle, leaf, dev) : normals_knn_t<float>(p, v, k, drop_angle, leaf, dev);
}

// estimate_point_cloud_normals_ball_internal (src/point_cloud_normals.cpp:303-370), argument order of the reference
pcu_b200_ball_options ball_options(double radius, int min_pts, int max_pts, double drop_angle, const std::string& weight_function, int seed) {
    if (radius <= 0.0) throw py::value_error("Invalid radius (" + std::to_string(radius) + ") must be greater than 0.");
    if (min_pts < 3) throw py::value_error("Invalid min_pts_per_ball (" + std::to_string(min_pts) + ") must be greater than 3.");
    if (max_pts > 0 && max_pts < 3)
        throw py::value_error("Invalid max_pts_per_ball (" + std::to_string(max_pts) +
                              ") must either be negative (no max) or a number greater than 3.");
    pcu_b200_ball_options o;
    o.radius = radius; o.drop_angle_threshold = drop_angle; o.min_pts_per_ball = min_pts; o.max_pts_per_ball = max_pts;
    if (weight_function == "constant") o.weight_function = 0;
    else if (weight_function == "rbf") o.weight_function = 1;
    else throw py::value_error("Invalid weight_function, must be one of 'constant' or 'rbf'.");
    o.seed = (uint32_t)seed;
    return o;
}

template <typename T>
py::tuple normals_ball_t(const py::array& p, const py::array& v, const pcu_b200_ball_options& o, int device) {
    return normals_host<T>(p, v, kDefaultLeaf, device, [&](pcu_b200_workspace* ws, const T* pts, int64_t n, const T* dirs,
                                                            int64_t* idx, T* normals, int64_t* kept) {
        return pick<T>(pcu_b200_normals_ball_host_f32, pcu_b200_normals_ball_host_f64)(ws, pts, n, dirs, &o, idx, normals, kept);
    });
}
py::tuple normals_ball_numpy(const py::array& p, const py::array& v, double radius, int min_pts_per_ball, int max_pts_per_ball,
                             double drop_angle_threshold, const std::string& weight_function, int random_seed, int device) {
    const pcu_b200_ball_options o = ball_options(radius, min_pts_per_ball, max_pts_per_ball, drop_angle_threshold, weight_function, random_seed);
    const int dev = current_device_or_default(device);
    return is_f64(p) ? normals_ball_t<double>(p, v, o, dev) : normals_ball_t<float>(p, v, o, dev);
}

void normals_ball_device(bool is_f64, uintptr_t points, int64_t n, uintptr_t view_dirs, double radius, int min_pts, int max_pts,
                         double drop_angle, const std::string& weight_function, int seed, uintptr_t out_idx, uintptr_t out_normals,
                         uintptr_t out_count, int device, uintptr_t stream) {
    const pcu_b200_ball_options o = ball_options(radius, min_pts, max_pts, drop_angle, weight_function, seed);
    on_workspace(device, stream, kDefaultLeaf, [&](pcu_b200_workspace* ws) {
        return is_f64 ? pcu_b200_normals_ball_f64(ws, (const double*)points, n, (const double*)view_dirs, &o, (int64_t*)out_idx,
                                                  (double*)out_normals, (int64_t*)out_count, (void*)stream)
                      : pcu_b200_normals_ball_f32(ws, (const float*)points, n, (const float*)view_dirs, &o, (int64_t*)out_idx,
                                                  (float*)out_normals, (int64_t*)out_count, (void*)stream);
    });
}

// Voronoi centroids of device seeds (n, dim) fp64 -> device out (and the cells' moments, (n, 5), when out_moments is
// not 0); returns the cells each pass handled.
py::tuple voronoi_centroids_device(uintptr_t centers, int64_t n, int dim, uintptr_t out, uintptr_t out_moments, int device,
                                   uintptr_t stream) {
    int64_t passes[3] = {0, 0, 0};
    on_workspace(device, stream, kDefaultLeaf, [&](pcu_b200_workspace* ws) {
        return pcu_b200_voronoi_centroids(ws, (const double*)centers, n, dim, (double*)out, (double*)out_moments, passes,
                                          (void*)stream);
    });
    return py::make_tuple(passes[0], passes[1], passes[2]);
}

// Lloyd relaxation into device out (n, dim) fp64; returns (energies of the Newton phase, cells each pass handled).
py::tuple lloyd_device(int64_t n, int dim, uint32_t seed, int num_lloyd, int num_newton, uintptr_t out, int device, uintptr_t stream) {
    int64_t passes[3] = {0, 0, 0};
    int32_t steps = 0;
    std::vector<double> energy((size_t)std::max(num_newton, 0) + 1, 0.0);
    on_workspace(device, stream, kDefaultLeaf, [&](pcu_b200_workspace* ws) {
        return pcu_b200_lloyd(ws, n, dim, seed, num_lloyd, num_newton, (double*)out, energy.data(), &steps, passes, (void*)stream);
    });
    energy.resize(num_newton > 0 ? (size_t)steps + 1 : 0);
    return py::make_tuple(energy, py::make_tuple(passes[0], passes[1], passes[2]));
}

// Moments (n, 5) of the cells of device seeds (n, 3) restricted to a device mesh (fp64 v) into device out_moments;
// returns the pairs each pass handled.
py::tuple restricted_voronoi_moments_device(uintptr_t seeds, int64_t n, uintptr_t v, int64_t nv, uintptr_t f, int64_t nf, int f_kind,
                                            uintptr_t out_moments, int device, uintptr_t stream) {
    int64_t passes[3] = {0, 0, 0};
    on_workspace(device, stream, kDefaultLeaf, [&](pcu_b200_workspace* ws) {
        return pcu_b200_restricted_voronoi_moments(ws, (const double*)seeds, n, (const double*)v, nv, (const void*)f, nf, f_kind,
                                                   (double*)out_moments, passes, (void*)stream);
    });
    return py::make_tuple(passes[0], passes[1], passes[2]);
}

// Lloyd sampling of a device mesh (fp64 v) into device out (num_samples, 3) fp64; returns (energies of the Newton
// phase, pairs each pass handled).
py::tuple sample_mesh_lloyd_device(uintptr_t v, int64_t nv, uintptr_t f, int64_t nf, int f_kind, int64_t num_samples, uint32_t seed,
                                   int num_lloyd, int num_newton, uintptr_t out, int device, uintptr_t stream) {
    int64_t passes[3] = {0, 0, 0};
    int32_t steps = 0;
    std::vector<double> energy((size_t)std::max(num_newton, 0) + 1, 0.0);
    on_workspace(device, stream, kDefaultLeaf, [&](pcu_b200_workspace* ws) {
        return pcu_b200_sample_mesh_lloyd(ws, (const double*)v, nv, (const void*)f, nf, f_kind, num_samples, seed, num_lloyd, num_newton,
                                          (double*)out, energy.data(), &steps, passes, (void*)stream);
    });
    energy.resize(num_newton > 0 ? (size_t)steps + 1 : 0);
    return py::make_tuple(energy, py::make_tuple(passes[0], passes[1], passes[2]));
}

// A prepared mesh (RayMeshIntersector); out_bad: one device uint64, the faces with a corner out of range.
uintptr_t mesh_prepare_device(bool is_f64, uintptr_t v, int64_t nv, uintptr_t f, int64_t nf, int f_kind, uintptr_t out_bad, int device,
                              uintptr_t stream) {
    pcu_b200_mesh* mesh = nullptr;
    on_workspace(device, stream, kDefaultLeaf, [&](pcu_b200_workspace* ws) {
        return is_f64 ? pcu_b200_mesh_prepare_f64(ws, (const double*)v, nv, (const void*)f, nf, f_kind, &mesh, (uint64_t*)out_bad,
                                                  (void*)stream)
                      : pcu_b200_mesh_prepare_f32(ws, (const float*)v, nv, (const void*)f, nf, f_kind, &mesh, (uint64_t*)out_bad,
                                                  (void*)stream);
    });
    return (uintptr_t)mesh;
}

// Prepared surfels (RaySurfelIntersector); freed by _mesh_destroy.
uintptr_t surfel_prepare_device(bool is_f64, uintptr_t p, uintptr_t n, uintptr_t r, int64_t np, int subdivs, int device, uintptr_t stream) {
    pcu_b200_mesh* h = nullptr;
    on_workspace(device, stream, kDefaultLeaf, [&](pcu_b200_workspace* ws) {
        return is_f64 ? pcu_b200_surfel_prepare_f64(ws, (const double*)p, (const double*)n, (const double*)r, np, subdivs, &h, (void*)stream)
                      : pcu_b200_surfel_prepare_f32(ws, (const float*)p, (const float*)n, (const float*)r, np, subdivs, &h, (void*)stream);
    });
    return (uintptr_t)h;
}

// Marching cubes (marching_cubes_sparse_voxel_grid, _sparse_voxels.py): classifies and numbers the vertices (two
// synchronisations of `stream`), returns (handle, #v, #f); _marching_cubes_emit writes v and f; _marching_cubes_destroy.
py::tuple marching_cubes_prepare_device(bool t_f64, uintptr_t scalars, bool s_f64, uintptr_t coords, int64_t n, uintptr_t idx, int64_t m,
                                        int idx_kind, double isovalue, int device, uintptr_t stream) {
    pcu_b200_marching_cubes* mc = nullptr;
    int64_t counts[2] = {0, 0};
    on_workspace(device, stream, kDefaultLeaf, [&](pcu_b200_workspace* ws) {
        return t_f64 ? pcu_b200_marching_cubes_prepare_f64(ws, (const void*)scalars, s_f64, (const double*)coords, n, (const void*)idx, m,
                                                           idx_kind, isovalue, &mc, counts, (void*)stream)
                     : pcu_b200_marching_cubes_prepare_f32(ws, (const void*)scalars, s_f64, (const float*)coords, n, (const void*)idx, m,
                                                           idx_kind, isovalue, &mc, counts, (void*)stream);
    });
    return py::make_tuple((uintptr_t)mc, counts[0], counts[1]);
}

// Sparse voxel grids (_sparse_voxels.py): one code-set handle, prepared from points, by a dilation round or from a grid's
// cube corners (one synchronisation of `stream` each), returns (handle, rows, records); _sparse_grid_emit writes the
// outputs; _sparse_grid_destroy.
py::tuple sparse_grid_from_points_device(bool is_f64, uintptr_t points, int64_t n, std::vector<double> size, std::vector<double> origin,
                                         int device, uintptr_t stream) {
    if (size.size() != 3 || origin.size() != 3) throw py::value_error("Invalid shape");
    pcu_b200_sparse_grid* sg = nullptr;
    int64_t counts[2] = {0, 0};
    on_workspace(device, stream, kDefaultLeaf, [&](pcu_b200_workspace* ws) {
        return is_f64 ? pcu_b200_sparse_grid_from_points_f64(ws, (const double*)points, n, size.data(), origin.data(), &sg, counts, (void*)stream)
                      : pcu_b200_sparse_grid_from_points_f32(ws, (const float*)points, n, size.data(), origin.data(), &sg, counts, (void*)stream);
    });
    return py::make_tuple((uintptr_t)sg, counts[0], counts[1]);
}
py::tuple sparse_grid_dilate_prepare_device(uintptr_t grid, int64_t n, int idx_kind, int device, uintptr_t stream) {
    pcu_b200_sparse_grid* sg = nullptr;
    int64_t counts[2] = {0, 0};
    on_workspace(device, stream, kDefaultLeaf, [&](pcu_b200_workspace* ws) {
        return pcu_b200_sparse_grid_dilate_prepare(ws, (const void*)grid, n, idx_kind, &sg, counts, (void*)stream);
    });
    return py::make_tuple((uintptr_t)sg, counts[0], counts[1]);
}
py::tuple sparse_grid_hex_prepare_device(uintptr_t grid, int64_t n, int idx_kind, std::vector<double> size, std::vector<double> origin,
                                         bool vertices_f64, int device, uintptr_t stream) {
    if (size.size() != 3 || origin.size() != 3) throw py::value_error("Invalid shape");
    pcu_b200_sparse_grid* sg = nullptr;
    int64_t counts[2] = {0, 0};
    on_workspace(device, stream, kDefaultLeaf, [&](pcu_b200_workspace* ws) {
        return pcu_b200_sparse_grid_hex_prepare(ws, (const void*)grid, n, idx_kind, size.data(), origin.data(), vertices_f64 ? 1 : 0, &sg,
                                                counts, (void*)stream);
    });
    return py::make_tuple((uintptr_t)sg, counts[0], counts[1]);
}
// voxel_grid_geometry (_voxels.py): out_v (8 n, 3) float32, out_f (12 n, 3) int32; no synchronisation.
void voxel_grid_geometry_device(uintptr_t ijk, int64_t n, int idx_kind, std::vector<double> size, std::vector<double> origin, double gap,
                                uintptr_t out_v, uintptr_t out_f, int device, uintptr_t stream) {
    if (size.size() != 3 || origin.size() != 3) throw py::value_error("Invalid shape");
    on_workspace(device, stream, kDefaultLeaf, [&](pcu_b200_workspace* ws) {
        return pcu_b200_voxel_grid_geometry(ws, (const void*)ijk, n, idx_kind, size.data(), origin.data(), gap, (float*)out_v,
                                            (int32_t*)out_f, (void*)stream);
    });
}

// Voxelization (voxelize_triangle_mesh, _voxels.py): tests and sorts (two synchronisations of `stream`), returns
// (handle, n, accepted (face, voxel) pairs); _voxelize_emit writes the (n, 3) int32 voxels; _voxelize_destroy.
py::tuple voxelize_prepare_device(bool is_f64, uintptr_t v, int64_t nv, uintptr_t f, int64_t nf, int f_kind, std::vector<double> size,
                                  std::vector<double> origin, int device, uintptr_t stream) {
    if (size.size() != 3 || origin.size() != 3) throw py::value_error("Invalid shape");
    pcu_b200_voxelize* vx = nullptr;
    int64_t counts[2] = {0, 0};
    on_workspace(device, stream, kDefaultLeaf, [&](pcu_b200_workspace* ws) {
        return is_f64 ? pcu_b200_voxelize_prepare_f64(ws, (const double*)v, nv, (const void*)f, nf, f_kind, size.data(), origin.data(), &vx,
                                                      counts, (void*)stream)
                      : pcu_b200_voxelize_prepare_f32(ws, (const float*)v, nv, (const void*)f, nf, f_kind, size.data(), origin.data(), &vx,
                                                      counts, (void*)stream);
    });
    return py::make_tuple((uintptr_t)vx, counts[0], counts[1]);
}

// Watertight remeshing (make_mesh_watertight, _watertight.py): the whole remeshing (synchronises `stream` per phase and
// per flip pass), returns (handle, #v, #f, depth); _make_mesh_watertight_emit writes v and f; _make_mesh_watertight_destroy.
py::tuple make_mesh_watertight_prepare_device(bool is_f64, uintptr_t v, int64_t nv, uintptr_t f, int64_t nf, int f_kind, double resolution,
                                              int device, uintptr_t stream) {
    pcu_b200_watertight* wt = nullptr;
    int64_t counts[3] = {0, 0, 0};
    on_workspace(device, stream, kDefaultLeaf, [&](pcu_b200_workspace* ws) {
        return is_f64 ? pcu_b200_make_mesh_watertight_prepare_f64(ws, (const double*)v, nv, (const void*)f, nf, f_kind, resolution, &wt,
                                                                  counts, (void*)stream)
                      : pcu_b200_make_mesh_watertight_prepare_f32(ws, (const float*)v, nv, (const void*)f, nf, f_kind, resolution, &wt,
                                                                  counts, (void*)stream);
    });
    return py::make_tuple((uintptr_t)wt, counts[0], counts[1], counts[2]);
}

// Decimation (decimate_triangle_mesh, _decimate.py): the whole decimation (synchronises `stream` before the rounds, per
// round and for the counts), returns (handle, #v_out, #f_out, rounds); _decimate_triangle_mesh_emit writes v_out, f_out
// and the correspondences; _decimate_triangle_mesh_destroy.
py::tuple decimate_triangle_mesh_prepare_device(bool is_f64, uintptr_t v, int64_t nv, uintptr_t f, int64_t nf, int f_kind, int64_t max_faces,
                                                int device, uintptr_t stream) {
    pcu_b200_decimate* dc = nullptr;
    int64_t counts[3] = {0, 0, 0};
    on_workspace(device, stream, kDefaultLeaf, [&](pcu_b200_workspace* ws) {
        return is_f64 ? pcu_b200_decimate_triangle_mesh_prepare_f64(ws, (const double*)v, nv, (const void*)f, nf, f_kind, max_faces, &dc,
                                                                    counts, (void*)stream)
                      : pcu_b200_decimate_triangle_mesh_prepare_f32(ws, (const float*)v, nv, (const void*)f, nf, f_kind, max_faces, &dc,
                                                                    counts, (void*)stream);
    });
    return py::make_tuple((uintptr_t)dc, counts[0], counts[1], counts[2]);
}

// Connected components (connected_components, _mesh_topology.py): validates f and labels (two synchronisations of
// `stream`), returns (handle, n = max(f) + 1, components); _connected_components_emit writes cv, nv, cf and nf in f's
// width; _connected_components_destroy.
py::tuple connected_components_prepare_device(uintptr_t f, int64_t nf, int f_cols, int f_kind, int device, uintptr_t stream) {
    pcu_b200_components* cc = nullptr;
    int64_t counts[2] = {0, 0};
    on_workspace(device, stream, kDefaultLeaf, [&](pcu_b200_workspace* ws) {
        return pcu_b200_connected_components_prepare(ws, (const void*)f, nf, f_cols, f_kind, &cc, counts, (void*)stream);
    });
    return py::make_tuple((uintptr_t)cc, counts[0], counts[1]);
}
// Adjacency lists (adjacency_list, _mesh_topology.py): validates f and builds the CSR (two synchronisations of `stream`),
// returns (handle, n = max(f) + 1, nnz); _adjacency_list_emit writes the offsets and neighbours in f's width;
// _adjacency_list_destroy.
py::tuple adjacency_list_prepare_device(uintptr_t f, int64_t nf, int f_kind, int device, uintptr_t stream) {
    pcu_b200_adjacency* adj = nullptr;
    int64_t counts[2] = {0, 0};
    on_workspace(device, stream, kDefaultLeaf, [&](pcu_b200_workspace* ws) {
        return pcu_b200_adjacency_list_prepare(ws, (const void*)f, nf, f_kind, &adj, counts, (void*)stream);
    });
    return py::make_tuple((uintptr_t)adj, counts[0], counts[1]);
}
// remove_mesh_vertices: out_v (capacity nv rows), out_f (capacity nf rows, f's width); one synchronisation; returns
// (kept vertices, kept faces).
py::tuple remove_mesh_vertices_device(bool is_f64, uintptr_t v, int64_t nv, uintptr_t f, int64_t nf, int f_kind, uintptr_t mask,
                                      uintptr_t out_v, uintptr_t out_f, int device, uintptr_t stream) {
    int64_t counts[2] = {0, 0};
    on_workspace(device, stream, kDefaultLeaf, [&](pcu_b200_workspace* ws) {
        return is_f64 ? pcu_b200_remove_mesh_vertices_f64(ws, (const double*)v, nv, (const void*)f, nf, f_kind, (const uint8_t*)mask,
                                                          (double*)out_v, (void*)out_f, counts, (void*)stream)
                      : pcu_b200_remove_mesh_vertices_f32(ws, (const float*)v, nv, (const void*)f, nf, f_kind, (const uint8_t*)mask,
                                                          (float*)out_v, (void*)out_f, counts, (void*)stream);
    });
    return py::make_tuple(counts[0], counts[1]);
}
// remove_unreferenced_mesh_vertices: out_v and out_corr_v (capacity nv rows), out_f (nf, 3) and out_corr_f (nv), the
// index arrays in f's width; one synchronisation; returns the kept vertex count.
int64_t remove_unreferenced_device(bool is_f64, uintptr_t v, int64_t nv, uintptr_t f, int64_t nf, int f_kind, uintptr_t out_v,
                                   uintptr_t out_f, uintptr_t out_corr_v, uintptr_t out_corr_f, int device, uintptr_t stream) {
    int64_t kept = 0;
    on_workspace(device, stream, kDefaultLeaf, [&](pcu_b200_workspace* ws) {
        return is_f64 ? pcu_b200_remove_unreferenced_mesh_vertices_f64(ws, (const double*)v, nv, (const void*)f, nf, f_kind, (double*)out_v,
                                                                       (void*)out_f, (void*)out_corr_v, (void*)out_corr_f, &kept,
                                                                       (void*)stream)
                      : pcu_b200_remove_unreferenced_mesh_vertices_f32(ws, (const float*)v, nv, (const void*)f, nf, f_kind, (float*)out_v,
                                                                       (void*)out_f, (void*)out_corr_v, (void*)out_corr_f, &kept,
                                                                       (void*)stream);
    });
    return kept;
}

// mesh_face_areas (normal false) / estimate_mesh_face_normals (normal true): out (nf) or (nf, 3) in v's type; one
// synchronisation.
void mesh_face_device(bool is_f64, bool normal, uintptr_t v, int64_t nv, uintptr_t f, int64_t nf, int f_kind, uintptr_t out, int device,
                      uintptr_t stream) {
    on_workspace(device, stream, kDefaultLeaf, [&](pcu_b200_workspace* ws) {
        if (normal)
            return is_f64 ? pcu_b200_mesh_face_normals_f64(ws, (const double*)v, nv, (const void*)f, nf, f_kind, (double*)out, (void*)stream)
                          : pcu_b200_mesh_face_normals_f32(ws, (const float*)v, nv, (const void*)f, nf, f_kind, (float*)out, (void*)stream);
        return is_f64 ? pcu_b200_mesh_face_areas_f64(ws, (const double*)v, nv, (const void*)f, nf, f_kind, (double*)out, (void*)stream)
                      : pcu_b200_mesh_face_areas_f32(ws, (const float*)v, nv, (const void*)f, nf, f_kind, (float*)out, (void*)stream);
    });
}
// laplacian_smooth_mesh: out (nv, 3) in v's type; returns (CG iterations of every step, largest relative residual of
// every step).
py::tuple laplacian_smooth_device(bool is_f64, uintptr_t v, int64_t nv, uintptr_t f, int64_t nf, int f_kind, int num_iters, double step_size,
                                  bool use_cotan_weights, int max_cg_iters, uintptr_t out, int device, uintptr_t stream) {
    std::vector<int32_t> iters((size_t)std::max(num_iters, 0));
    std::vector<double> residual(iters.size());
    on_workspace(device, stream, kDefaultLeaf, [&](pcu_b200_workspace* ws) {
        return is_f64 ? pcu_b200_laplacian_smooth_mesh_f64(ws, (const double*)v, nv, (const void*)f, nf, f_kind, num_iters, step_size,
                                                           use_cotan_weights, max_cg_iters, (double*)out, iters.data(), residual.data(),
                                                           (void*)stream)
                      : pcu_b200_laplacian_smooth_mesh_f32(ws, (const float*)v, nv, (const void*)f, nf, f_kind, num_iters, step_size,
                                                           use_cotan_weights, max_cg_iters, (float*)out, iters.data(), residual.data(),
                                                           (void*)stream);
    });
    py::list it, res;
    for (size_t i = 0; i < iters.size(); ++i) {
        it.append(iters[i]);
        res.append(residual[i]);
    }
    return py::make_tuple(it, res);
}

// out is float64 when bc or attribute is (numpy's promotion), else float32; out_bad: one device uint64.
void interpolate_barycentric_device(uintptr_t f, int64_t nf, int f_kind, uintptr_t fi, int64_t n, int fi_kind, uintptr_t bc,
                                    bool bc_f64, uintptr_t attr, bool attr_f64, int64_t nv, int64_t dim, uintptr_t out,
                                    uintptr_t out_bad, int device, uintptr_t stream) {
    on_workspace(device, stream, kDefaultLeaf, [&](pcu_b200_workspace* ws) {
        return (bc_f64 || attr_f64)
                   ? pcu_b200_interpolate_barycentric_f64(ws, (const void*)f, nf, f_kind, (const void*)fi, n, fi_kind, (const void*)bc,
                                                          bc_f64, (const void*)attr, attr_f64, nv, dim, (double*)out,
                                                          (uint64_t*)out_bad, (void*)stream)
                   : pcu_b200_interpolate_barycentric_f32(ws, (const void*)f, nf, f_kind, (const void*)fi, n, fi_kind, (const float*)bc,
                                                          (const float*)attr, nv, dim, (float*)out, (uint64_t*)out_bad, (void*)stream);
    });
}

// ---- Morton codes (src/morton.cpp) ----------------------------------------------------------------
// dtype rules of the bindings: pts int32 / int64; codes uint32 / uint64 (uint32 codes are widened, as the
// reference's MortonCode64(uint64_t) constructor does implicitly); results are uint64 / int32 / int64 like the reference's.
py::array_t<uint64_t, py::array::c_style> as_codes(const py::array& a, const char* name) {
    if (!a.dtype().is(py::dtype::of<uint64_t>()) && !a.dtype().is(py::dtype::of<uint32_t>()))
        throw py::value_error(std::string("Invalid scalar type (") + std::string(py::str(a.dtype())) + ") for argument '" + name +
                              "'. Expected one of ['uint32', 'uint64'].");
    if (a.ndim() == 0 || a.size() == 0) throw py::value_error(std::string(name) + " must be an array of shape [n] but got an empty array");
    if (!(a.ndim() == 1 || (a.ndim() == 2 && a.shape(1) == 1)))
        throw py::value_error(std::string(name) + " must be an array of shape [n] but got an invalid number of columns");
    return py::array_t<uint64_t, py::array::c_style | py::array::forcecast>::ensure(a);
}

py::array morton_encode(const py::array& pts, int num_threads, int device) {
    (void)num_threads;
    const bool i32 = pts.dtype().is(py::dtype::of<int32_t>()), i64 = pts.dtype().is(py::dtype::of<int64_t>());
    if (!i32 && !i64)
        throw py::value_error("Invalid scalar type (" + std::string(py::str(pts.dtype())) + ") for argument 'pts'. Expected one of ['int32', 'int64'].");
    if (pts.ndim() != 2 || pts.shape(0) <= 0) throw py::value_error("pts must be an array of shape [n, 3] but got an empty array");
    if (pts.shape(1) != 3) throw py::value_error("pts must be an array of shape [n, 3] but got an invalid number of columns");
    const int64_t n = pts.shape(0);
    py::array_t<uint64_t> codes({(py::ssize_t)n});
    const int dev = current_device_or_default(device);
    if (i32) {
        auto p = py::array_t<int32_t, py::array::c_style | py::array::forcecast>::ensure(pts);
        on_workspace(dev, kHostKey, kDefaultLeaf, [&](pcu_b200_workspace* ws) {
            return pcu_b200_morton_encode_host_i32(ws, p.data(), n, codes.mutable_data());
        });
    } else {
        auto p = py::array_t<int64_t, py::array::c_style | py::array::forcecast>::ensure(pts);
        on_workspace(dev, kHostKey, kDefaultLeaf, [&](pcu_b200_workspace* ws) {
            return pcu_b200_morton_encode_host_i64(ws, p.data(), n, codes.mutable_data());
        });
    }
    return codes;
}

py::array morton_decode(const py::array& codes_in, int num_threads, int device) {
    (void)num_threads;
    auto codes = as_codes(codes_in, "codes");
    const int64_t n = codes.size();
    py::array_t<int32_t> pts({(py::ssize_t)n, (py::ssize_t)3});
    on_workspace(current_device_or_default(device), kHostKey, kDefaultLeaf, [&](pcu_b200_workspace* ws) {
        return pcu_b200_morton_decode_host(ws, codes.data(), n, pts.mutable_data());
    });
    return pts;
}

py::array morton_addsub(const py::array& a_in, const py::array& b_in, int num_threads, int device, bool subtract) {
    (void)num_threads;
    auto a = as_codes(a_in, "codes_1");
    auto b = as_codes(b_in, "codes_2");
    if (a.size() != b.size()) throw py::value_error("codes_1 and codes_2 must have the same number of entries.");
    const int64_t n = a.size();
    py::array_t<uint64_t> out({(py::ssize_t)n});
    on_workspace(current_device_or_default(device), kHostKey, kDefaultLeaf, [&](pcu_b200_workspace* ws) {
        return subtract ? pcu_b200_morton_subtract_host(ws, a.data(), b.data(), n, out.mutable_data())
                        : pcu_b200_morton_add_host(ws, a.data(), b.data(), n, out.mutable_data());
    });
    return out;
}

py::array morton_knn(const py::array& codes_in, const py::array& qcodes_in, int k, bool sort_dist, int device) {
    if (k <= 0) throw py::value_error("k must be greater than 0");
    auto codes = as_codes(codes_in, "codes");
    auto qcodes = as_codes(qcodes_in, "qcodes");
    if (!qcodes_in.dtype().is(codes_in.dtype()))
        throw py::value_error("Invalid scalar type for argument 'qcodes'. Expected it to match argument 'codes'.");
    const int64_t n = codes.size(), m = qcodes.size();
    k = (int)std::min<int64_t>(k, n);                       // morton.cpp:351
    py::array_t<int64_t> idx({(py::ssize_t)m, (py::ssize_t)k});
    on_workspace(current_device_or_default(device), kHostKey, kDefaultLeaf, [&](pcu_b200_workspace* ws) {
        return pcu_b200_morton_knn_host(ws, codes.data(), n, qcodes.data(), m, k, sort_dist ? 1 : 0, idx.mutable_data());
    });
    return idx;
}

// ---- prepared clouds (handles travel as integers; point-cloud-utils_b200/__init__.py wraps them in PreparedCloud) ----
template <typename T>
pcu_b200_cloud* cloud_prepare_numpy_t(const py::array& pts_in, int knn_k, int leaf, int device) {
    auto p = points_of<T>(pts_in);
    pcu_b200_cloud* cloud = nullptr;
    on_workspace(device, kHostKey, leaf > 0 ? leaf : kDefaultLeaf, [&](pcu_b200_workspace* ws) {   // leaf 0: the library's default
        if (knn_k > 0)
            return pick<T>(pcu_b200_cloud_prepare_knn_host_f32, pcu_b200_cloud_prepare_knn_host_f64)(ws, p.data(), p.shape(0), knn_k, leaf,
                                                                                                     &cloud);
        return pick<T>(pcu_b200_cloud_prepare_host_f32, pcu_b200_cloud_prepare_host_f64)(ws, p.data(), p.shape(0), &cloud);
    });
    return cloud;
}
uintptr_t cloud_prepare_numpy(const py::array& pts, int device, int knn_k, int leaf) {
    const int dev = current_device_or_default(device);
    return (uintptr_t)(is_f64(pts) ? cloud_prepare_numpy_t<double>(pts, knn_k, leaf, dev) : cloud_prepare_numpy_t<float>(pts, knn_k, leaf, dev));
}
uintptr_t cloud_prepare_device(bool is_f64, uintptr_t pts, int64_t n, int device, uintptr_t stream, int knn_k, int leaf) {
    pcu_b200_cloud* cloud = nullptr;
    on_workspace(device, stream, leaf > 0 ? leaf : kDefaultLeaf, [&](pcu_b200_workspace* ws) {
        if (knn_k > 0)
            return is_f64 ? pcu_b200_cloud_prepare_knn_f64(ws, (const double*)pts, n, knn_k, leaf, &cloud, (void*)stream)
                          : pcu_b200_cloud_prepare_knn_f32(ws, (const float*)pts, n, knn_k, leaf, &cloud, (void*)stream);
        return is_f64 ? pcu_b200_cloud_prepare_f64(ws, (const double*)pts, n, &cloud, (void*)stream)
                      : pcu_b200_cloud_prepare_f32(ws, (const float*)pts, n, &cloud, (void*)stream);
    });
    return (uintptr_t)cloud;
}
// k_nearest_neighbors and the statistics sweeps of numpy points against a prepared cloud of the precision cloud_is_f64
template <typename T>
py::tuple knn_prepared_numpy_t(const py::array& q, pcu_b200_cloud* cloud, int k, bool squared, int leaf, int device) {
    return knn_host<T>(q, k, leaf, device, [&](pcu_b200_workspace* ws, const T* qp, int64_t n, T* dists, int64_t* corrs) {
        int64_t tied = 0;
        return pick<T>(pcu_b200_knn_prepared_host_f32, pcu_b200_knn_prepared_host_f64)(ws, qp, n, cloud, k, squared, dists, corrs, &tied);
    });
}
py::tuple knn_prepared_numpy(const py::array& q, uintptr_t cloud, bool cloud_is_f64, int k, bool squared, int leaf, int device) {
    auto* y = (pcu_b200_cloud*)cloud;
    return cloud_is_f64 ? knn_prepared_numpy_t<double>(q, y, k, squared, leaf, device) : knn_prepared_numpy_t<float>(q, y, k, squared, leaf, device);
}

template <typename T>
py::tuple stats_prepared_numpy_t(const py::array& x, const pcu_b200_cloud* y, bool both, int leaf, int device) {
    return stats_host<T>(x, both, leaf, device, [&](pcu_b200_workspace* ws, const T* xp, int64_t n, pcu_b200_nn_stats* st, T* v) {
        return v ? pick<T>(pcu_b200_chamfer_prepared_host_f32, pcu_b200_chamfer_prepared_host_f64)(ws, xp, n, y, st, v)
                 : pick<T>(pcu_b200_nn_stats_prepared_host_f32, pcu_b200_nn_stats_prepared_host_f64)(ws, xp, n, y, st);
    });
}
py::tuple stats_prepared_numpy(const py::array& x, uintptr_t cloud, bool cloud_is_f64, bool both, int leaf, int device) {
    auto* y = (const pcu_b200_cloud*)cloud;
    return cloud_is_f64 ? stats_prepared_numpy_t<double>(x, y, both, leaf, device) : stats_prepared_numpy_t<float>(x, y, both, leaf, device);
}

// ---- voxel-grid down-sampling on device pointers (the Python layer owns the arrays) ----
void voxel_downsample_device(bool is_f64, uintptr_t pts, int64_t n, uintptr_t attr, int attr_cols, bool attr_is_f64,
                             std::array<double, 3> size, std::array<double, 3> lo, std::array<double, 3> hi, int min_points,
                             uintptr_t out_pts, uintptr_t out_attr, uintptr_t out_counts, uintptr_t out_rows, int device, uintptr_t stream) {
    on_workspace(device, stream, kDefaultLeaf, [&](pcu_b200_workspace* ws) {
        return is_f64 ? pcu_b200_voxel_downsample_f64(ws, (const double*)pts, n, (const void*)attr, attr_cols, attr_is_f64 ? 1 : 0,
                                                      size.data(), lo.data(), hi.data(), min_points, (double*)out_pts, (void*)out_attr,
                                                      (int32_t*)out_counts, (int64_t*)out_rows, (void*)stream)
                      : pcu_b200_voxel_downsample_f32(ws, (const float*)pts, n, (const void*)attr, attr_cols, attr_is_f64 ? 1 : 0,
                                                      size.data(), lo.data(), hi.data(), min_points, (float*)out_pts, (void*)out_attr,
                                                      (int32_t*)out_counts, (int64_t*)out_rows, (void*)stream);
    });
}

// Batched Chamfer on numpy inputs: x (B, n, 3), y (B, m, 3) float32 -> ((B,) float32, fp64 sum)
py::tuple batched_chamfer_numpy(const py::array& x_in, const py::array& y_in, int max_points_per_leaf, int device) {
    // the guard of points_of for batches: float32, (B, n, 3) and (B, m, 3)
    for (const py::array* a : {&x_in, &y_in})
        if (!a->dtype().is(py::dtype::of<float>()) || a->ndim() != 3 || a->shape(2) != 3 || a->shape(0) != x_in.shape(0))
            throw py::value_error("pcu_b200: expected (B, n, 3) float32 arrays");
    auto x = dense<float>(x_in);
    auto y = dense<float>(y_in);
    const int64_t B = x.shape(0), n = x.shape(1), m = y.shape(1);
    py::array_t<float> out({(py::ssize_t)B});
    double sum = 0.0;
    on_workspace(current_device_or_default(device), kHostKey, max_points_per_leaf, [&](pcu_b200_workspace* ws) {
        return pcu_b200_batched_chamfer_host_f32(ws, x.data(), y.data(), B, n, m, out.mutable_data(), &sum);
    });
    return py::make_tuple(out, sum);
}

template <typename T>
py::dict debug_kd_tree_t(const py::array& pts_in, int leaf, int device) {
    auto pts = dense<T>(pts_in);
    const int64_t m = pts.shape(0);
    const int64_t cap = 2 * m + 2;
    py::array_t<int32_t> order(m), feat(cap), first(cap), last(cap), kid0(cap), kid1(cap);
    py::array_t<T> lo(cap), hi(cap);
    int64_t nn = 0;
    on_workspace(device, kHostKey, leaf, [&](pcu_b200_workspace* ws) {
        return pick<T>(pcu_b200_debug_kd_tree_f32, pcu_b200_debug_kd_tree_f64)(ws, pts.data(), m, leaf, order.mutable_data(), cap,
                                                                                feat.mutable_data(), lo.mutable_data(), hi.mutable_data(),
                                                                                first.mutable_data(), last.mutable_data(),
                                                                                kid0.mutable_data(), kid1.mutable_data(), &nn);
    });
    py::dict d;
    d["order"] = order; d["feat"] = feat; d["div_lo"] = lo; d["div_hi"] = hi; d["first"] = first; d["last"] = last;
    d["kid0"] = kid0; d["kid1"] = kid1; d["n_nodes"] = nn;
    return d;
}

py::dict debug_kd_tree(const py::array& pts, int leaf, int device) {
    if (pts.ndim() != 2 || pts.shape(1) != 3 || pts.shape(0) == 0) throw py::value_error("points must be (m, 3)");
    const int dev = current_device_or_default(device);
    if (pts.dtype().is(py::dtype::of<float>())) return debug_kd_tree_t<float>(pts, leaf, dev);
    if (pts.dtype().is(py::dtype::of<double>())) return debug_kd_tree_t<double>(pts, leaf, dev);
    throw py::value_error("points must be float32 or float64");
}

}  // namespace

PYBIND11_MODULE(_pcu_internal, mod) {
    mod.doc() = "pcu_b200's native layer: host and device entry points of libpcu_b200.so for the Python package, which "
                "checks every argument (the drop-in boundary is the package, not this module)";
    mod.def("_knn_host", &knn_numpy);
    mod.def("_knn_device", forward_to(pcu_b200_knn_f32, pcu_b200_knn_f64).pair_with_leaf());
    PYBIND11_NUMPY_DTYPE(pcu_b200_nn_stats, sum_dist, sum_sq_dist, max_sq_dist, argmax_query, argmax_data, n_queries, n_tied, n_far,
                         witness_tied, pair_value);
    mod.def("_stats_dtype", []() { return py::dtype::of<pcu_b200_nn_stats>(); });
    mod.def("_chamfer_stats", &stats_numpy, py::arg("x"), py::arg("y"), py::arg("max_points_per_leaf") = 10, py::arg("device") = -1,
            py::arg("both") = true);
    mod.def("_nn_stats_device", forward_to(pcu_b200_nn_stats_f32, pcu_b200_nn_stats_f64).pair_with_leaf());
    mod.def("_chamfer_device", forward_to(pcu_b200_chamfer_f32, pcu_b200_chamfer_f64).pair_with_leaf());
    mod.def("_resolve_witness_device", forward_to(pcu_b200_resolve_witness_f32, pcu_b200_resolve_witness_f64).pair_with_leaf());
    mod.def("_normals_knn_host", &normals_knn_numpy);
    mod.def("_normals_knn_device", forward_to(pcu_b200_normals_knn_f32, pcu_b200_normals_knn_f64).pair_with_leaf());
    mod.def("_normals_ball_host", &normals_ball_numpy);
    mod.def("_normals_ball_device", &normals_ball_device);
    mod.def("_poisson_disk_device", forward_to(pcu_b200_poisson_disk_f32, pcu_b200_poisson_disk_f64).pair());
    mod.def("_voronoi_centroids_device", &voronoi_centroids_device);
    mod.def("_lloyd_device", &lloyd_device);
    mod.def("_restricted_voronoi_moments_device", &restricted_voronoi_moments_device);
    mod.def("_sample_mesh_lloyd_device", &sample_mesh_lloyd_device);
    mod.def("_mesh_area_device", forward_to(pcu_b200_mesh_area_f32, pcu_b200_mesh_area_f64).pair());
    mod.def("_sample_mesh_random_device", forward_to(pcu_b200_sample_mesh_random_f32, pcu_b200_sample_mesh_random_f64).pair());
    mod.def("_closest_points_on_mesh_device", forward_to(pcu_b200_closest_points_on_mesh_f32, pcu_b200_closest_points_on_mesh_f64).pair());
    mod.def("_fast_winding_number_device", forward_to(pcu_b200_fast_winding_number_f32, pcu_b200_fast_winding_number_f64).pair());
    mod.def("_point_cloud_fast_winding_number_device",
            forward_to(pcu_b200_point_cloud_fast_winding_number_f32, pcu_b200_point_cloud_fast_winding_number_f64).pair());
    mod.def("_estimate_point_cloud_areas_device",
            forward_to(pcu_b200_estimate_point_cloud_areas_f32, pcu_b200_estimate_point_cloud_areas_f64).pair());
    mod.def("_apss_device", forward_to(pcu_b200_apss_project_f32, pcu_b200_apss_project_f64).pair());
    mod.def("_signed_distance_to_mesh_device",
            forward_to(pcu_b200_signed_distance_to_mesh_f32, pcu_b200_signed_distance_to_mesh_f64).pair());
    mod.def("_sample_mesh_poisson_disk_device",
            forward_to(pcu_b200_sample_mesh_poisson_disk_f32, pcu_b200_sample_mesh_poisson_disk_f64).pair());
    mod.def("_ray_mesh_intersection_device", forward_to(pcu_b200_ray_mesh_intersection_f32, pcu_b200_ray_mesh_intersection_f64).pair());
    mod.def("_mesh_prepare_device", &mesh_prepare_device);
    mod.def("_mesh_destroy", destroy(pcu_b200_mesh_destroy));
    mod.def("_ray_mesh_prepared_device",
            forward_to(pcu_b200_ray_mesh_intersection_prepared_f32, pcu_b200_ray_mesh_intersection_prepared_f64).pair());
    mod.def("_ray_surfel_intersection_device",
            forward_to(pcu_b200_ray_surfel_intersection_f32, pcu_b200_ray_surfel_intersection_f64).pair());
    mod.def("_surfel_prepare_device", &surfel_prepare_device);
    mod.def("_ray_surfel_prepared_device",
            forward_to(pcu_b200_ray_surfel_intersection_prepared_f32, pcu_b200_ray_surfel_intersection_prepared_f64).pair());
    mod.def("_surfel_geometry_device", forward_to(pcu_b200_pointcloud_surfel_geometry_f32, pcu_b200_pointcloud_surfel_geometry_f64).pair());
    mod.def("_sphere_geometry_device", forward_to(pcu_b200_pointcloud_sphere_geometry_f32, pcu_b200_pointcloud_sphere_geometry_f64).pair());
    mod.def("_interpolate_barycentric_device", &interpolate_barycentric_device);
    mod.def("_marching_cubes_prepare_device", &marching_cubes_prepare_device);
    mod.def("_marching_cubes_emit_device", forward_to(pcu_b200_marching_cubes_emit).single());
    mod.def("_marching_cubes_destroy", destroy(pcu_b200_marching_cubes_destroy));
    mod.def("_sparse_voxel_grid_boundary_device", forward_to(pcu_b200_sparse_voxel_grid_boundary).single());
    mod.def("_sparse_grid_from_points_device", &sparse_grid_from_points_device);
    mod.def("_sparse_grid_dilate_prepare_device", &sparse_grid_dilate_prepare_device);
    mod.def("_sparse_grid_hex_prepare_device", &sparse_grid_hex_prepare_device);
    mod.def("_sparse_grid_emit_device", forward_to(pcu_b200_sparse_grid_emit).single());
    mod.def("_sparse_grid_destroy", destroy(pcu_b200_sparse_grid_destroy));
    mod.def("_sparse_grid_erode_device", forward_to(pcu_b200_sparse_grid_erode).single());
    mod.def("_voxel_grid_geometry_device", &voxel_grid_geometry_device);
    mod.def("_voxelize_prepare_device", &voxelize_prepare_device);
    mod.def("_voxelize_emit_device", forward_to(pcu_b200_voxelize_emit).single());
    mod.def("_voxelize_destroy", destroy(pcu_b200_voxelize_destroy));
    mod.def("_make_mesh_watertight_prepare_device", &make_mesh_watertight_prepare_device);
    mod.def("_make_mesh_watertight_emit_device", forward_to(pcu_b200_make_mesh_watertight_emit).single());
    mod.def("_make_mesh_watertight_destroy", destroy(pcu_b200_make_mesh_watertight_destroy));
    mod.def("_decimate_triangle_mesh_prepare_device", &decimate_triangle_mesh_prepare_device);
    mod.def("_decimate_triangle_mesh_emit_device", forward_to(pcu_b200_decimate_triangle_mesh_emit).single());
    mod.def("_decimate_triangle_mesh_destroy", destroy(pcu_b200_decimate_triangle_mesh_destroy));
    mod.def("_flood_fill_3d_device", forward_to(pcu_b200_flood_fill_3d).single());
    mod.def("_connected_components_prepare_device", &connected_components_prepare_device);
    mod.def("_connected_components_emit_device", forward_to(pcu_b200_connected_components_emit).single());
    mod.def("_connected_components_destroy", destroy(pcu_b200_connected_components_destroy));
    mod.def("_remove_mesh_vertices_device", &remove_mesh_vertices_device);
    mod.def("_remove_unreferenced_device", &remove_unreferenced_device);
    mod.def("_orient_mesh_faces_device", forward_to(pcu_b200_orient_mesh_faces).single());
    mod.def("_adjacency_list_prepare_device", &adjacency_list_prepare_device);
    mod.def("_adjacency_list_emit_device", forward_to(pcu_b200_adjacency_list_emit).single());
    mod.def("_adjacency_list_destroy", destroy(pcu_b200_adjacency_list_destroy));
    mod.def("_mesh_face_device", &mesh_face_device);
    mod.def("_mesh_vertex_normals_device", forward_to(pcu_b200_mesh_vertex_normals_f32, pcu_b200_mesh_vertex_normals_f64).pair());
    mod.def("_mesh_curvatures_device",
            forward_to(pcu_b200_mesh_principal_curvatures_f32, pcu_b200_mesh_principal_curvatures_f64).pair());
    mod.def("_laplacian_smooth_device", &laplacian_smooth_device);
    mod.def("_cloud_prepare_host", &cloud_prepare_numpy);
    mod.def("_cloud_prepare_device", &cloud_prepare_device, py::arg("is_f64"), py::arg("points"), py::arg("n"), py::arg("device"),
            py::arg("stream"), py::arg("knn_k") = 0, py::arg("max_points_per_leaf") = 10);
    mod.def("_knn_prepared_host", &knn_prepared_numpy);
    mod.def("_knn_prepared_device", forward_to(pcu_b200_knn_prepared_f32, pcu_b200_knn_prepared_f64).pair_with_leaf());
    mod.def("_cloud_destroy", destroy(pcu_b200_cloud_destroy));
    mod.def("_cloud_points", [](uintptr_t cloud) { return (uintptr_t)pcu_b200_cloud_points((const pcu_b200_cloud*)cloud); });
    mod.def("_stats_prepared_host", &stats_prepared_numpy);
    mod.def("_nn_stats_prepared_device", forward_to(pcu_b200_nn_stats_prepared_f32, pcu_b200_nn_stats_prepared_f64).pair_with_leaf());
    mod.def("_chamfer_prepared_device", forward_to(pcu_b200_chamfer_prepared_f32, pcu_b200_chamfer_prepared_f64).pair_with_leaf());
    mod.def("_voxel_downsample_device", &voxel_downsample_device);
    mod.def("_deduplicate_device", forward_to(pcu_b200_deduplicate_f32, pcu_b200_deduplicate_f64).pair());
    mod.def("_pairwise_device", forward_to(pcu_b200_pairwise_distances_f32, pcu_b200_pairwise_distances_f64).pair());
    mod.def("_sinkhorn_device", forward_to(pcu_b200_sinkhorn_f32, pcu_b200_sinkhorn_f64).pair());
    mod.def("morton_encode", &morton_encode, py::arg("pts"), py::arg("num_threads") = -1, py::arg("device") = -1,
            "Encode n 3D integer points into Morton codes: (n, 3) int32 / int64 -> (n,) uint64.");
    mod.def("morton_decode", &morton_decode, py::arg("codes"), py::arg("num_threads") = -1, py::arg("device") = -1,
            "Decode n Morton codes into 3D integer points: (n,) -> (n, 3) int32.");
    mod.def("morton_add", [](const py::array& a, const py::array& b, int t, int d) { return morton_addsub(a, b, t, d, false); },
            py::arg("codes_1"), py::arg("codes_2"), py::arg("num_threads") = -1, py::arg("device") = -1,
            "Add morton codes together (corresponding to adding the vectors they encode).");
    mod.def("morton_subtract", [](const py::array& a, const py::array& b, int t, int d) { return morton_addsub(a, b, t, d, true); },
            py::arg("codes_1"), py::arg("codes_2"), py::arg("num_threads") = -1, py::arg("device") = -1,
            "Subtract morton codes from each other (codes_1 - codes_2).");
    mod.def("morton_knn", &morton_knn, py::arg("codes"), py::arg("qcodes"), py::arg("k"), py::arg("sort_dist") = true,
            py::arg("device") = -1,
            "Queries a sorted array of morton encoded points to find the (approximate) k nearest neighbors: (m, min(k, n)) int64.");
    mod.def("_batched_chamfer_host", &batched_chamfer_numpy);
    mod.def("_batched_chamfer_device", forward_to(pcu_b200_batched_chamfer_f32).single_with_leaf());
    mod.def("_batched_chamfer_stats_device", forward_to(pcu_b200_debug_batched_chamfer_stats_f32).single_with_leaf());
    // diagnostics address a workspace by (device, stream); stream None = the numpy path's own workspace,
    // device < 0 = the device a call that names none would use
    auto key_of = [](const py::object& stream) { return stream.is_none() ? kHostKey : stream.cast<uintptr_t>(); };
    mod.def("_debug_kd_times", [key_of](int device, py::object stream) {
        std::array<uint64_t, 40> t{};
        on_workspace(current_device_or_default(device), key_of(stream), kDefaultLeaf,
                     [&](pcu_b200_workspace* ws) { return pcu_b200_debug_kd_times(ws, t.data()); });
        return t;
    }, py::arg("device") = -1, py::arg("stream") = py::none());
    mod.def("_debug_kd_tree", &debug_kd_tree, py::arg("points"), py::arg("max_points_per_leaf") = 10,
            py::arg("device") = -1);
    mod.def("_stats_nbytes", []() { return (int)sizeof(pcu_b200_nn_stats); });
    mod.def("_device_count", []() { return pcu_b200_device_count(); });
    mod.def("_launch_count", []() { return (int64_t)pcu_b200_launch_count(); });
    mod.def("_abi_version", []() { return pcu_b200_abi_version(); });
    mod.def("_current_device", []() { return pcu_b200_current_device(); });
    mod.def("_grid_refinement", [key_of](int device, py::object stream) {
        float m[2] = {1.f, 1.f};
        on_workspace(current_device_or_default(device), key_of(stream), kDefaultLeaf, [&](pcu_b200_workspace* ws) {
            pcu_b200_workspace_grid_refinement(ws, m);
            return PCU_B200_OK;
        });
        return py::make_tuple(m[0], m[1]);
    }, py::arg("device") = -1, py::arg("stream") = py::none());
    mod.def("_workspace_bytes", [key_of](int device, py::object stream) {
        int64_t bytes = 0;
        on_workspace(current_device_or_default(device), key_of(stream), kDefaultLeaf, [&](pcu_b200_workspace* ws) {
            bytes = pcu_b200_workspace_bytes(ws);
            return PCU_B200_OK;
        });
        return bytes;
    }, py::arg("device") = -1, py::arg("stream") = py::none());
    mod.def("_workspace_exists", [key_of](int device, py::object stream) {
        std::lock_guard<std::mutex> lock(pool().mu);
        return pool().items.count(std::make_pair(current_device_or_default(device), key_of(stream))) != 0;
    }, py::arg("device") = -1, py::arg("stream") = py::none());
    mod.def("_set_profiling", [key_of](int device, py::object stream, bool on) {
        on_workspace(current_device_or_default(device), key_of(stream), kDefaultLeaf,
                     [&](pcu_b200_workspace* ws) { return pcu_b200_workspace_set_profiling(ws, on ? 1 : 0); });
    });
    mod.def("_last_profile", [key_of](int device, py::object stream) {
        float ms[10];
        int n = 0;
        on_workspace(current_device_or_default(device), key_of(stream), kDefaultLeaf, [&](pcu_b200_workspace* ws) {
            n = pcu_b200_workspace_last_profile(ws, ms, 10);   // the number of stages, or -1
            return PCU_B200_OK;
        });
        py::dict d;
        for (int i = 0; i < n; ++i) d[py::str(pcu_b200_profile_stage_name(i))] = ms[i];
        return d;
    });
    mod.def("_set_defaults", [](float cell_occupancy, int disable_tie_replay, int binning, int host_staging) {
        if (host_staging < 0 || host_staging > 2) throw py::value_error("host_staging must be 0 (auto), 1 (always) or 2 (never)");
        defaults().host_staging = host_staging;
        if (disable_tie_replay < 0 || disable_tie_replay > 3) throw py::value_error("disable_tie_replay must be 0 .. 3");
        if (binning < 0 || binning > 3) throw py::value_error("binning must be 0 (auto), 1 (cell-wise passes), 2 (one CTA per cloud) or 3 (slab build)");
        defaults().occupancy = cell_occupancy;
        defaults().disable_replay = disable_tie_replay;
        defaults().binning = binning;
    }, py::arg("cell_occupancy") = 0.f, py::arg("disable_tie_replay") = 0, py::arg("binning") = 0, py::arg("host_staging") = 0);
    mod.def("_pinned_empty", [](py::ssize_t rows, py::ssize_t cols, bool is_f64) {
        return is_f64 ? pinned_cloud<double>(rows, cols) : pinned_cloud<float>(rows, cols);
    });
    mod.def("_release_workspaces", []() { pool().clear(); });
    mod.def("_release_pinned_results", []() { pinned_pool().clear(false); });
    // destroy workspaces and cached pinned blocks before the CUDA context goes away at interpreter exit
    py::module_::import("atexit").attr("register")(py::cpp_function([]() { pool().clear(); pinned_pool().clear(true); }));
}
