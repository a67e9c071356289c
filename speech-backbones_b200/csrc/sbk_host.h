// Host-side core of the four engines' C ABIs (sbk_api.cu: the U-Net, sbk_vocoder.cu, sbk_postnet.cu, sbk_textenc.cu): the
// error text, strict weight loading, keyed uploads of packed weight images, grow-only workspaces and per-name debug snapshots.
#pragma once
#include "../../include/sbk.h"
#include "sbk_internal.h"

#include <math.h>
#include <string.h>

#include <map>
#include <string>
#include <vector>

namespace sbk {

// Sets the calling thread's error text (sbk_last_error, sbk_api.cu) and returns `code`.
int fail(int code, const char* fmt, ...);

#define CU(x)                                                                                          \
    do {                                                                                               \
        cudaError_t e_ = (x);                                                                          \
        if (e_ != cudaSuccess)                                                                         \
            return sbk::fail(SBK_ERR_CUDA, "%s failed: %s (%s:%d)", #x, cudaGetErrorString(e_), __FILE__, __LINE__); \
    } while (0)

#define TRY(x) do { int rc_ = (x); if (rc_ != SBK_OK) return rc_; } while (0)

// Device buffers by name; the map owns them (freed by free_all).
struct DeviceBuf { void* ptr = nullptr; size_t bytes = 0; };
using BufMap = std::map<std::string, DeviceBuf>;

// Copy `bytes` from `src` (host or device) into the buffer `key`, (re)allocating it when absent or of another size (a
// packed image of another precision mode).
inline int upload(BufMap& m, const std::string& key, size_t bytes, const void* src) {
    DeviceBuf& d = m[key];
    if (d.ptr && d.bytes != bytes) { CU(cudaFree(d.ptr)); d = DeviceBuf(); }
    if (!d.ptr) { CU(cudaMalloc(&d.ptr, bytes)); d.bytes = bytes; }
    CU(cudaMemcpy(d.ptr, src, bytes, cudaMemcpyDefault));
    return SBK_OK;
}
inline void free_all(BufMap& m) {
    for (auto& kv : m) cudaFree(kv.second.ptr);
    m.clear();
}

// The strict weight inventory of one handle: the reference's names and shapes, their device copies (`raw`) and the kernel
// layouts packed from them (`packed`).  `api` names the C entry point in error messages.
struct WeightSet {
    struct Spec { std::string name; std::vector<int64_t> shape; };
    std::vector<Spec> spec;
    BufMap raw, packed;

    WeightSet() = default;
    WeightSet(const WeightSet&) = delete;
    WeightSet& operator=(const WeightSet&) = delete;
    ~WeightSet() { free_all(raw); free_all(packed); }

    void add(const std::string& name, std::vector<int64_t> shape) { spec.push_back({name, std::move(shape)}); }
    int count() const { return (int)spec.size(); }
    const char* name(int i) const { return i >= 0 && i < count() ? spec[i].name.c_str() : nullptr; }
    const Spec* find(const std::string& name) const {
        for (auto& s : spec) if (s.name == name) return &s;
        return nullptr;
    }
    static size_t numel(const Spec& s) { size_t n = 1; for (auto v : s.shape) n *= (size_t)v; return n; }

    // name, rank and shape are checked before any CUDA call
    int set(const char* name, const void* data, const int64_t* shape, int ndim, int device, const char* api) {
        const Spec* ws = find(name);
        if (!ws) return fail(SBK_ERR_ARG, "%s: unexpected key '%s' (strict)", api, name);
        if ((int)ws->shape.size() != ndim) return fail(SBK_ERR_ARG, "%s: '%s' rank %d, expected %d", api, name, ndim, (int)ws->shape.size());
        for (int i = 0; i < ndim; ++i)
            if (ws->shape[i] != shape[i]) return fail(SBK_ERR_ARG, "%s: '%s' dim %d is %lld, expected %lld", api, name, i, (long long)shape[i], (long long)ws->shape[i]);
        CU(cudaSetDevice(device));
        return upload(raw, name, numel(*ws) * sizeof(float), data);
    }
    int require_all(const char* api) const {
        for (auto& s : spec) if (!raw.count(s.name)) return fail(SBK_ERR_STATE, "%s: missing key '%s' (strict)", api, s.name.c_str());
        return SBK_OK;
    }
    // host copy of the raw tensor `name` (for the packers)
    int fetch(const std::string& name, std::vector<float>& out) const {
        const Spec* s = find(name);
        auto it = raw.find(name);
        if (!s || it == raw.end()) return fail(SBK_ERR_STATE, "no loaded weight %s", name.c_str());
        out.resize(numel(*s));
        CU(cudaMemcpy(out.data(), it->second.ptr, out.size() * sizeof(float), cudaMemcpyDeviceToHost));
        return SBK_OK;
    }
    // the packed image `key`, else the raw tensor `key`, else null
    const float* get(const std::string& key) const {
        auto it = packed.find(key);
        if (it != packed.end()) return (const float*)it->second.ptr;
        it = raw.find(key);
        return it != raw.end() ? (const float*)it->second.ptr : nullptr;
    }
};

// Bump allocator over a workspace, 256-byte aligned; with a null base it only measures (bytes()).
struct Arena {
    char* base = nullptr; size_t off = 0;
    void* take(size_t bytes) {
        off = (off + 255) & ~size_t(255);
        void* r = base ? base + off : nullptr;
        off += bytes;
        return r;
    }
    size_t bytes() const { return off + 256; }
};

// Grow-only device workspace: shapes change from call to call, and a cudaFree/cudaMalloc pair is a device-wide sync.
// An engine describes its buffers in one carve function over an Arena, run with a null base to size the workspace
// (reserve) and again over arena() to lay it out.
struct Workspace {
    void* mem = nullptr; size_t cap = 0;

    Workspace() = default;
    Workspace(const Workspace&) = delete;
    Workspace& operator=(const Workspace&) = delete;
    ~Workspace() { if (mem) cudaFree(mem); }

    // On failure the CUDA error is cleared and returned; the caller words the out-of-memory message.
    cudaError_t reserve(size_t bytes) {
        if (bytes <= cap) return cudaSuccess;
        if (mem) cudaFree(mem);
        mem = nullptr; cap = 0;
        const cudaError_t e = cudaMalloc(&mem, bytes);
        if (e != cudaSuccess) { mem = nullptr; cudaGetLastError(); return e; }
        cap = bytes;
        return cudaSuccess;
    }
    Arena arena() const { Arena a; a.base = (char*)mem; return a; }
};

// Element size of a debug-snapshot layout: 2 = bf16, 4 = fp16 (both [B][H][C/8][W][8]), 3 = float64, every other layout fp32.
inline size_t snap_elem_bytes(int fmt) { return fmt == 2 || fmt == 4 ? 2 : (fmt == 3 ? 8 : 4); }

// IEEE binary16 bits -> fp32 (exact)
inline float f16_bits_to_f32(uint16_t h) {
    const uint32_t s = (uint32_t)(h & 0x8000u) << 16, e = (h >> 10) & 0x1Fu, m = h & 0x3FFu;
    if (e == 0) { const float f = ldexpf((float)m, -24); return s ? -f : f; }       // zero / subnormal
    const uint32_t u = s | (e == 31 ? 0x7F800000u : (e + 112) << 23) | (m << 13);
    float f; memcpy(&f, &u, 4);
    return f;
}

// Copy `numel` elements of layout `fmt` from device memory to `dst` (host or device); bf16 and fp16 are widened to fp32
// (exact), element order unchanged.
inline int read_widened(void* dst, const void* src, size_t numel, int fmt) {
    if (fmt != 2 && fmt != 4) { CU(cudaMemcpy(dst, src, numel * snap_elem_bytes(fmt), cudaMemcpyDefault)); return SBK_OK; }
    std::vector<uint16_t> h16(numel);
    CU(cudaMemcpy(h16.data(), src, numel * 2, cudaMemcpyDeviceToHost));
    std::vector<float> h32(numel);
    for (size_t i = 0; i < numel; ++i) {
        if (fmt == 4) { h32[i] = f16_bits_to_f32(h16[i]); continue; }
        const uint32_t u = (uint32_t)h16[i] << 16; memcpy(&h32[i], &u, 4);
    }
    CU(cudaMemcpy(dst, h32.data(), numel * sizeof(float), cudaMemcpyDefault));
    return SBK_OK;
}

// Per-name copies of the intermediates of a handle's last call (the debug_capture test hooks).  The workspace is
// overwritten within a call, so each tensor is copied (stream-ordered) right after the launch that wrote it, into a buffer
// kept per name across calls.  The copies are not launches.
struct Snapshots {
    struct Snap { std::string name; void* buf = nullptr; size_t cap = 0, numel = 0; int fmt = 0; };
    bool on = false;              // capture the next calls
    std::vector<Snap> list;       // in launch order

    Snapshots() = default;
    Snapshots(const Snapshots&) = delete;
    Snapshots& operator=(const Snapshots&) = delete;
    ~Snapshots() { for (auto& sn : list) cudaFree(sn.buf); }

    void begin() { n_ = 0; err_ = cudaSuccess; }
    // after the first failed allocation or copy nothing more is recorded; finish() reports it
    void record(const std::string& name, const void* src, size_t numel, int fmt, cudaStream_t s) {
        if (!on || err_ != cudaSuccess) return;
        if (n_ == list.size()) list.emplace_back();
        Snap& sn = list[n_++];
        const size_t bytes = numel * snap_elem_bytes(fmt);
        sn.name = name; sn.numel = numel; sn.fmt = fmt;
        if (bytes > sn.cap) {
            cudaFree(sn.buf); sn.buf = nullptr; sn.cap = 0;
            if ((err_ = cudaMalloc(&sn.buf, bytes)) != cudaSuccess) { sn.buf = nullptr; sn.numel = 0; return; }
            sn.cap = bytes;
        }
        err_ = cudaMemcpyAsync(sn.buf, src, bytes, cudaMemcpyDeviceToDevice, s);
    }
    // drops the entries the call did not record (when capturing); returns the first capture error
    cudaError_t finish() {
        if (on) {
            for (size_t i = n_; i < list.size(); ++i) cudaFree(list[i].buf);
            list.resize(n_);
        }
        return err_;
    }
    const Snap* find(const char* name) const {
        for (auto& sn : list) if (sn.name == name) return &sn;
        return nullptr;
    }
    int read(const char* name, void* dst, int64_t* numel, int device, const char* api) const {
        const Snap* sn = find(name);
        if (!sn) return fail(SBK_ERR_ARG, "%s: no intermediate named '%s'", api, name);
        if (numel) *numel = (int64_t)sn->numel;
        if (dst && sn->numel > 0) {
            CU(cudaSetDevice(device));
            CU(cudaDeviceSynchronize());
            return read_widened(dst, sn->buf, sn->numel, sn->fmt);
        }
        return SBK_OK;
    }

private:
    size_t n_ = 0;
    cudaError_t err_ = cudaSuccess;
};

// The tensor-core form of a precision mode: the fp32-class modes (fp32x3, and fp32 wherever it runs on tensor cores) use
// the fp32x3 split.
inline bool prec_runs_x3(int precision) { return precision == SBK_PREC_FP32X3 || precision == SBK_PREC_FP32; }

// Grid of a grid-stride element-wise kernel: 256-thread blocks, at most 16 blocks per SM.
inline int ew_grid(long long n) {
    const long long g = (n + 255) / 256, cap = 16LL * device_sm_count();
    return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace sbk
