// api.cu — the C ABI of libbyzagg (include/byzagg.h): argument checks, the launch geometry
// (vector width and alignment shift shared by all rows), and the kernel chains of every rule.  No device memory is allocated here and nothing synchronises the host.
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <type_traits>
#include <utility>

#include "launch.cuh"
#include "dist.cuh"
#include "api_shared.cuh"

namespace bz {

static thread_local char g_error[512] = "";

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_error, sizeof(g_error), fmt, ap);
  va_end(ap);
  return code;
}

int sm_count() {
  static int cached[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  int& c = cached[dev & 63];
  if (c == 0) cudaDeviceGetAttribute(&c, cudaDevAttrMultiProcessorCount, dev);
  return c > 0 ? c : 132;
}

int check_launch(const char* what) {
  const cudaError_t err = cudaGetLastError();
  if (err != cudaSuccess) return fail(BZ_ECUDA, "%s: %s", what, cudaGetErrorString(err));
  return BZ_OK;
}

Geom make_geom(const float* const* rows, int n, const void* out, const void* extra, int64_t d, int want_vec) {
  Geom g{d, d, 0, 1, 1, -1, 0};
  if (want_vec <= 1 || d < 1) return g;
  const uintptr_t bytes = (uintptr_t)want_vec * sizeof(float);
  const uintptr_t mis = (uintptr_t)rows[0] % bytes;
  bool same = ((uintptr_t)out % bytes) == mis;
  if (extra != nullptr) same = same && ((uintptr_t)extra % bytes) == mis;
  for (int r = 1; r < n && same; ++r) same = ((uintptr_t)rows[r] % bytes) == mis;
  if (!same) return g;
  g.vec = want_vec;
  g.shift = (int)(mis / sizeof(float));        // element e sits at (e + shift) modulo VEC
  g.nv = (d + g.shift + want_vec - 1) / want_vec;
  return g;
}

// max_n: kMaxN, or kMaxNCoordinate for bz_coordinate (the limit's name goes into the message)
static int check_rows(const float* const* rows, int n, int64_t d, const void* out, const char* who, int max_n = kMaxN) {
  if (rows == nullptr) return fail(BZ_EINVAL, "%s: rows is NULL", who);
  if (n < 1) return fail(BZ_EINVAL, "%s: n = %d, expected n >= 1", who, n);
  if (n > max_n) return fail(BZ_EUNSUPPORTED, "%s: n = %d exceeds %s = %d", who, n, max_n == kMaxN ? "BZ_MAX_N" : "BZ_MAX_N_COORDINATE", max_n);
  if (d < 0) return fail(BZ_EINVAL, "%s: d = %lld < 0", who, (long long)d);
  if (d > 0) {
    if (out == nullptr) return fail(BZ_EINVAL, "%s: output pointer is NULL", who);
    for (int r = 0; r < n; ++r) {
      if (rows[r] == nullptr) return fail(BZ_EINVAL, "%s: rows[%d] is NULL", who, r);
      if (((uintptr_t)rows[r] % sizeof(float)) != 0) return fail(BZ_EINVAL, "%s: rows[%d] is not 4-byte aligned", who, r);
    }
    if (((uintptr_t)out % sizeof(float)) != 0) return fail(BZ_EINVAL, "%s: output is not 4-byte aligned", who);
  }
  return BZ_OK;
}

template <class Rows>
static void fill_table(Rows& t, const float* const* rows, int n) {
  constexpr int slots = sizeof(t.p) / sizeof(t.p[0]);
  for (int r = 0; r < n; ++r) t.p[r] = rows[r];
  for (int r = n; r < slots; ++r) t.p[r] = rows[0];
}

// Unique rows by pointer equality: uniq[k] = first row with that address, to_unique[i] = its k.
// by_address = false: every row counts as distinct (rows of an empty shard: every empty tensor has
// address 0, so equal addresses say nothing there).
static int dedupe_rows(const float* const* rows, int n, const float** uniq, int* to_unique, bool by_address = true) {
  int u = 0;
  for (int i = 0; i < n; ++i) {
    int k = by_address ? 0 : u;
    while (k < u && uniq[k] != rows[i]) ++k;
    if (k == u) uniq[u++] = rows[i];
    to_unique[i] = k;
  }
  return u;
}

// The pointer table the kernels of n rows take, RowTable up to kMaxN rows and WideRowTable above, handed to `fn`.
template <class Fn>
static void with_table(const float* const* rows, int n, Fn fn) {
  if (n > kMaxN) {
    WideRowTable t;
    fill_table(t, rows, n);
    fn(t);
  } else {
    RowTable t;
    fill_table(t, rows, n);
    fn(t);
  }
}

// First n of every range of K1's kernels: each has a median and a sorted object in the Makefile (K1FIRST).
using K1Ranges = std::integer_sequence<int, 1, 17, 33, 49, 65, 73, 81, 89, 97, 105, 113, 121>;

// The launcher of the range that holds n.  A range whose kernels take the other table never does.
template <int FIRST, class Rows>
static bool median_range(int n, const Rows& t, const Geom& g, float* out, cudaStream_t st) {
  if constexpr (std::is_same<Rows, RowsOf<FIRST>>::value) return launch_median_range<FIRST>(n, t, g, out, st);
  else return false;
}
template <int FIRST, class Rows>
static bool sorted_range(int n, const Rows& t, const Geom& g, int mode, int f, float* out, cudaStream_t st) {
  if constexpr (std::is_same<Rows, RowsOf<FIRST>>::value) return launch_sorted_range<FIRST>(n, t, g, mode, f, out, st);
  else return false;
}
template <class Rows, int... FIRST>
static bool launch_median(std::integer_sequence<int, FIRST...>, int n, const Rows& t, const Geom& g, float* out, cudaStream_t st) {
  return (median_range<FIRST>(n, t, g, out, st) || ...);
}
template <class Rows, int... FIRST>
static bool launch_sorted(std::integer_sequence<int, FIRST...>, int n, const Rows& t, const Geom& g, int mode, int f, float* out, cudaStream_t st) {
  return (sorted_range<FIRST>(n, t, g, mode, f, out, st) || ...);
}
// The (n, f) specialisations exist up to kMaxN rows only.
static bool launch_special(int n, const RowTable& t, const Geom& g, int mode, int f, float* out, cudaStream_t st) {
  return (mode == kModeTrmean) ? launch_trmean_special(n, f, t, g, out, st)
       : (mode == kModePhocas) ? launch_phocas_special(n, f, t, g, out, st)
                               : launch_meamed_special(n, f, t, g, out, st);
}
static bool launch_special(int, const WideRowTable&, const Geom&, int, int, float*, cudaStream_t) { return false; }

int run_median(const float* const* rows, int n, int64_t d, float* out, cudaStream_t st) {
  const Geom g = make_geom(rows, n, out, nullptr, d, body_vec(n));
  with_table(rows, n, [&](const auto& t) { launch_median(K1Ranges{}, n, t, g, out, st); });
  return check_launch("k1_median");
}

int run_sorted(const float* const* rows, int n, int mode, int f, int64_t d, float* out, cudaStream_t st) {
  const Geom g = make_geom(rows, n, out, nullptr, d, body_vec(n));
  with_table(rows, n, [&](const auto& t) {
    if (!launch_special(n, t, g, mode, f, out, st)) launch_sorted(K1Ranges{}, n, t, g, mode, f, out, st);
  });
  return check_launch("k1_sorted");
}

int run_average_selected(const float* const* rows, int n, const int32_t* sel, int count, int zero_init,
                         float divisor, const int32_t* status, int64_t d, float* out, cudaStream_t st, int reverse = 0) {
  Geom g = make_geom(rows, n, out, nullptr, d, 4);
  g.reverse = reverse;
  with_table(rows, n, [&](const auto& t) { launch_average(t, g, sel, count, zero_init, divisor, status, out, st); });
  return check_launch("k3_average");
}

static int check_f_trim(int n, int f, const char* who) {
  // executable range (the reference's check(), trmean.py:52-64, is the caller's job)
  if (f < 0 || n - 2 * f < 1) return fail(BZ_EINVAL, "%s: f = %d not executable with n = %d (need n - 2f >= 1)", who, f, n);
  return BZ_OK;
}

// The launches of coordinate-wise rule `rule` over checked rows, d >= 1.
static int run_coordinate(int rule, const float* const* rows, int n, int f, int64_t d, float* out, cudaStream_t st) {
  switch (rule) {
    case BZ_RULE_AVERAGE: return run_average_selected(rows, n, nullptr, n, 1, (float)n, nullptr, d, out, st);
    case BZ_RULE_MEDIAN:  return run_median(rows, n, d, out, st);
    case BZ_RULE_TRMEAN:  return run_sorted(rows, n, kModeTrmean, f, d, out, st);
    case BZ_RULE_PHOCAS:  return run_sorted(rows, n, kModePhocas, f, d, out, st);
    default:              return run_sorted(rows, n, kModeMeamed, f, d, out, st);
  }
}

// Entry point `who` of a coordinate-wise rule, for up to max_n rows.
static int coordinate_entry(const char* who, int max_n, int rule, const float* const* rows, int n, int f, int64_t d, float* out, void* stream) {
  if (int rc = check_rows(rows, n, d, out, who, max_n)) return rc;
  if (rule >= BZ_RULE_TRMEAN) if (int rc = check_f_trim(n, f, who)) return rc;
  if (d == 0) return BZ_OK;
  return run_coordinate(rule, rows, n, f, d, out, (cudaStream_t)stream);
}

}  // namespace bz

using namespace bz;

extern "C" {

int bz_version(void) { return 100; }
int bz_max_n(void) { return kMaxN; }
const char* bz_last_error(void) { return g_error; }

int bz_average(const float* const* rows, int n, int64_t d, float* out, void* stream) {
  return coordinate_entry("bz_average", kMaxN, BZ_RULE_AVERAGE, rows, n, 0, d, out, stream);
}
int bz_median(const float* const* rows, int n, int64_t d, float* out, void* stream) {
  return coordinate_entry("bz_median", kMaxN, BZ_RULE_MEDIAN, rows, n, 0, d, out, stream);
}
int bz_trmean(const float* const* rows, int n, int f, int64_t d, float* out, void* stream) {
  return coordinate_entry("bz_trmean", kMaxN, BZ_RULE_TRMEAN, rows, n, f, d, out, stream);
}
int bz_phocas(const float* const* rows, int n, int f, int64_t d, float* out, void* stream) {
  return coordinate_entry("bz_phocas", kMaxN, BZ_RULE_PHOCAS, rows, n, f, d, out, stream);
}
int bz_meamed(const float* const* rows, int n, int f, int64_t d, float* out, void* stream) {
  return coordinate_entry("bz_meamed", kMaxN, BZ_RULE_MEAMED, rows, n, f, d, out, stream);
}

int bz_average_selected(const float* const* rows, int n, const int32_t* sel, int count, int zero_init,
                        double divisor, const int32_t* status, int64_t d, float* out, void* stream) {
  if (int rc = check_rows(rows, n, d, out, "bz_average_selected")) return rc;
  if (count < 1 || count > n) return fail(BZ_EINVAL, "bz_average_selected: count = %d, expected 1..%d", count, n);
  if (d == 0) return BZ_OK;
  return run_average_selected(rows, n, sel, count, zero_init, (float)divisor, status, d, out, (cudaStream_t)stream);
}

// n host->device copies of `bytes` each as ONE batch (cudaMemcpyBatchAsync, CUDA >= 12.8; not on the
// legacy default stream): separate cudaMemcpyAsync calls cost ~5.7 us each on the copy engine (measured:
// n pinned rows vs one contiguous copy of the same bytes, bench.py h2d_probe).  Falls back to the loop.
static void h2d_rows(void** dsts, void** srcs, int count, size_t bytes, cudaStream_t s) {
  static const bool batch_allowed = [] { const char* e = getenv("BYZAGG_H2D_BATCH"); return e == nullptr || e[0] != '0'; }();
  static bool batch_works = true;
  if (batch_allowed && batch_works && s != nullptr && count > 1) {
    size_t sizes[kMaxN];
    for (int k = 0; k < count; ++k) sizes[k] = bytes;
    cudaMemcpyAttributes attr;
    memset(&attr, 0, sizeof(attr));
    attr.srcAccessOrder = cudaMemcpySrcAccessOrderStream;
    size_t attr_index = 0, fail_index = 0;
    if (cudaMemcpyBatchAsync(dsts, srcs, sizes, (size_t)count, &attr, &attr_index, 1, &fail_index, s) == cudaSuccess) return;
    cudaGetLastError();
    batch_works = false;          // older driver: the plain loop from now on
  }
  for (int k = 0; k < count; ++k) cudaMemcpyAsync(dsts[k], srcs[k], bytes, cudaMemcpyHostToDevice, s);
}

int bz_stage_rows(const float* const* host_rows, int n, int64_t d, float* staging, int64_t pitch, void* stream) {
  if (int rc = check_rows(host_rows, n, d, staging, "bz_stage_rows")) return rc;
  if (d == 0) return BZ_OK;
  if (pitch < d) return fail(BZ_EINVAL, "bz_stage_rows: pitch = %lld < d = %lld", (long long)pitch, (long long)d);
  void* dsts[kMaxN];
  void* srcs[kMaxN];
  for (int k = 0; k < n; ++k) {
    dsts[k] = staging + (size_t)k * pitch;
    srcs[k] = const_cast<float*>(host_rows[k]);
  }
  h2d_rows(dsts, srcs, n, (size_t)d * sizeof(float), (cudaStream_t)stream);
  return check_launch("bz_stage_rows");
}

// Host buffers in, host buffer out, for the coordinate-wise rules: every coordinate is independent, so
// the vector is cut into `chunks` column ranges and the three engines of the GPU work at once — while
// chunk c+1 crosses PCIe host->device (in_stream), chunk c is reduced (stream) and the result of chunk
// c-1 crosses device->host (out_stream; PCIe is full duplex).  The step then costs the H2D time of the
// n rows plus the kernel and the D2H of ONE chunk, instead of H2D + kernel + D2H of the whole vector.
int bz_coordinate_host(int rule, const float* const* host_rows, int n, int f, int64_t d, float* host_out,
                       float* staging, int64_t pitch, float* dev_out, int chunks,
                       void* stream, void* in_stream, void* out_stream) {
  if (rule < BZ_RULE_AVERAGE || rule > BZ_RULE_MEAMED) return fail(BZ_EINVAL, "bz_coordinate_host: unknown rule %d", rule);
  if (int rc = check_rows(host_rows, n, d, host_out, "bz_coordinate_host")) return rc;
  if (rule >= BZ_RULE_TRMEAN) if (int rc = check_f_trim(n, f, "bz_coordinate_host")) return rc;
  if (d == 0) return BZ_OK;
  if (staging == nullptr || dev_out == nullptr) return fail(BZ_EINVAL, "bz_coordinate_host: staging / dev_out is NULL");
  if ((((uintptr_t)staging | (uintptr_t)dev_out) % sizeof(float)) != 0) return fail(BZ_EINVAL, "bz_coordinate_host: staging / dev_out is not 4-byte aligned");
  if (pitch < d || pitch % 4 != 0) return fail(BZ_EINVAL, "bz_coordinate_host: pitch = %lld must be >= d and a multiple of 4 floats", (long long)pitch);
  if (chunks < 1 || chunks > BZ_MAX_HOST_CHUNKS) return fail(BZ_EINVAL, "bz_coordinate_host: chunks = %d outside 1..%d", chunks, BZ_MAX_HOST_CHUNKS);
  cudaStream_t st = (cudaStream_t)stream, sin = (cudaStream_t)in_stream, sout = (cudaStream_t)out_stream;
  // every distinct host row is staged once (the attack rows of the reference are one tensor f times)
  const float* uniq[kMaxN];
  int slot[kMaxN];
  const int u = dedupe_rows(host_rows, n, uniq, slot);
  int64_t cs = (d + chunks - 1) / chunks;
  cs = (cs + 63) / 64 * 64;                       // chunk starts keep the 256-byte alignment of the staged rows
  cudaEvent_t ev[2 * BZ_MAX_HOST_CHUNKS + 2];
  int nev = 0;
  auto event_on = [&](cudaStream_t s) -> cudaEvent_t {
    cudaEvent_t e = nullptr;
    cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
    cudaEventRecord(e, s);
    ev[nev++] = e;
    return e;
  };
  int rc = BZ_OK;
  // the previous user of the staging rows and of dev_out (work queued on `stream`) must be done
  if (sin != st) cudaStreamWaitEvent(sin, event_on(st), 0);
  const float* dev_rows[kMaxN];
  for (int64_t c0 = 0; c0 < d && rc == BZ_OK; c0 += cs) {
    const int64_t cnt = (d - c0 < cs) ? d - c0 : cs;
    void* dsts[kMaxN];
    void* srcs[kMaxN];
    for (int k = 0; k < u; ++k) {
      dsts[k] = staging + (size_t)k * pitch + c0;
      srcs[k] = const_cast<float*>(uniq[k] + c0);
    }
    h2d_rows(dsts, srcs, u, (size_t)cnt * sizeof(float), sin);
    if (sin != st) cudaStreamWaitEvent(st, event_on(sin), 0);
    for (int i = 0; i < n; ++i) dev_rows[i] = staging + (size_t)slot[i] * pitch + c0;
    rc = run_coordinate(rule, dev_rows, n, f, cnt, dev_out + c0, st);
    if (rc != BZ_OK) break;
    if (sout != st) cudaStreamWaitEvent(sout, event_on(st), 0);
    cudaMemcpyAsync(host_out + c0, dev_out + c0, (size_t)cnt * sizeof(float), cudaMemcpyDeviceToHost, sout);
  }
  // whoever synchronises `stream` afterwards has the whole result
  if (sout != st) cudaStreamWaitEvent(st, event_on(sout), 0);
  for (int k = 0; k < nev; ++k) cudaEventDestroy(ev[k]);      // released by the runtime once they have completed
  if (rc != BZ_OK) return rc;
  return check_launch("bz_coordinate_host");
}

int bz_coordinate(int rule, const float* const* rows, int n, int f, int64_t d, float* out, void* stream) {
  if (rule < BZ_RULE_AVERAGE || rule > BZ_RULE_MEAMED) return fail(BZ_EINVAL, "bz_coordinate: unknown rule %d", rule);
  return coordinate_entry("bz_coordinate", kMaxNCoordinate, rule, rows, n, f, d, out, stream);
}

}  // extern "C"

#include "api_dist.inc"
#include "api_search.inc"
#include "api_search_shards.inc"
#include "api_search_peers.inc"
#include "api_peers_next.inc"
#include "api_distance.inc"
#include "api_distance_shards.inc"
#include "api_anticge.inc"
#include "api_anticge_peers.inc"
#include "api_distance_search.inc"
#include "api_distance_search_shards.inc"
