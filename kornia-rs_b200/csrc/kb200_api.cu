// kb200_api.cu — error model, device info and the host-side helpers of the C ABI
// (matrix inversion, Gaussian taps, preprocess geometry, std_mean finalisation).
// Host arithmetic mirrors the reference's f32/f64 expression trees; this file is compiled by
// nvcc with -fmad=false and the host compiler flags -ffp-contract=off (see build()).
#include <atomic>
#include <cmath>
#include <cstring>
#include <mutex>

#include "kb200_common.cuh"

namespace kb200 {

std::string& last_error_ref() {
    static thread_local std::string s;
    return s;
}

int fail(int status, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    last_error_ref() = buf;
    return status;
}

static const char*& last_kernel_ref() {
    static thread_local const char* s = "";
    return s;
}

static std::atomic<int> g_knobs[KNOB_COUNT];
static const char* const g_knob_names[KNOB_COUNT] = {
    "fr.npx", "fr.stages", "fr.ctas", "fr.rows", "ss.stages", "ss.ctas", "ss.rc", "warp.pf", "warp.path",
    "ws.stages", "ws.ctas", "ws.rc", "ws.npx", "rs.stages", "rs.ctas", "rs.npx", "a", "b", "c", "d"};
int knob(Knob k) { return g_knobs[k].load(std::memory_order_relaxed); }

int check_launch(const char* what) {
    last_kernel_ref() = what;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail(KB200_ERR_CUDA, "CUDA launch of %s failed: %s", what, cudaGetErrorString(e));
    return KB200_OK;
}

const DeviceInfo& device_info() {
    static DeviceInfo infos[64];
    static std::mutex mu;
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) dev = 0;
    DeviceInfo& d = infos[dev];
    if (d.device == dev) return d;
    std::lock_guard<std::mutex> lk(mu);
    if (d.device != dev) {
        cudaDeviceGetAttribute(&d.sm_count, cudaDevAttrMultiProcessorCount, dev);
        cudaDeviceGetAttribute(&d.cc_major, cudaDevAttrComputeCapabilityMajor, dev);
        cudaDeviceGetAttribute(&d.cc_minor, cudaDevAttrComputeCapabilityMinor, dev);
        cudaDeviceGetAttribute(&d.max_smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
        d.device = dev;
    }
    return d;
}

}  // namespace kb200

using namespace kb200;

extern "C" {

KB200_API int kb200_version(void) { return 100; }

KB200_API const char* kb200_last_error(void) { return last_error_ref().c_str(); }

KB200_API const char* kb200_status_name(int st) {
    switch (st) {
        case KB200_OK: return "KB200_OK";
        case KB200_ERR_INVALID_ARGUMENT: return "KB200_ERR_INVALID_ARGUMENT";
        case KB200_ERR_SLICE_TOO_SMALL: return "KB200_ERR_SLICE_TOO_SMALL";
        case KB200_ERR_SINGULAR_MATRIX: return "KB200_ERR_SINGULAR_MATRIX";
        case KB200_ERR_UNSUPPORTED: return "KB200_ERR_UNSUPPORTED";
        case KB200_ERR_CUDA: return "KB200_ERR_CUDA";
        case KB200_ERR_INVALID_KERNEL: return "KB200_ERR_INVALID_KERNEL";
        case KB200_ERR_DIMS_TOO_LARGE: return "KB200_ERR_DIMS_TOO_LARGE";
        case KB200_ERR_INVALID_SOURCE: return "KB200_ERR_INVALID_SOURCE";
        default: return "KB200_ERR_UNKNOWN";
    }
}

KB200_API const char* kb200_last_kernel(void) { return last_kernel_ref(); }

KB200_API int kb200_debug_set_knob(const char* name, int value) {
    if (!name) return fail(KB200_ERR_INVALID_ARGUMENT, "null knob name");
    for (int k = 0; k < KNOB_COUNT; ++k)
        if (strcmp(name, g_knob_names[k]) == 0) { g_knobs[k].store(value, std::memory_order_relaxed); return KB200_OK; }
    return fail(KB200_ERR_INVALID_ARGUMENT, "unknown knob '%s'", name);
}

KB200_API int kb200_set_device(int ordinal) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) {
        cudaGetLastError();
        return fail(KB200_ERR_CUDA, "no CUDA device visible");
    }
    if (ordinal < 0 || ordinal >= n) return fail(KB200_ERR_INVALID_ARGUMENT, "device ordinal %d out of range (0..%d)", ordinal, n - 1);
    cudaError_t e = cudaSetDevice(ordinal);
    if (e != cudaSuccess) return fail(KB200_ERR_CUDA, "cudaSetDevice(%d) failed: %s", ordinal, cudaGetErrorString(e));
    return KB200_OK;
}

KB200_API int kb200_device_info(int* sm_count, int* cc_major, int* cc_minor) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) {
        cudaGetLastError();
        return fail(KB200_ERR_CUDA, "no CUDA device visible");
    }
    const DeviceInfo& d = device_info();
    if (sm_count) *sm_count = d.sm_count;
    if (cc_major) *cc_major = d.cc_major;
    if (cc_minor) *cc_minor = d.cc_minor;
    return KB200_OK;
}

// warp/affine.rs:18-38
KB200_API void kb200_invert_affine_transform(const float m[6], float out[6]) {
    const float a = m[0], b = m[1], c = m[2], d = m[3], e = m[4], f = m[5];
    const float determinant = a * e - b * d;
    const float inv_determinant = (determinant != 0.0f) ? 1.0f / determinant : 0.0f;
    const float new_a = e * inv_determinant;
    const float new_b = -b * inv_determinant;
    const float new_d = -d * inv_determinant;
    const float new_e = a * inv_determinant;
    const float new_c = -(new_a * c + new_b * f);
    const float new_f = -(new_d * c + new_e * f);
    out[0] = new_a; out[1] = new_b; out[2] = new_c;
    out[3] = new_d; out[4] = new_e; out[5] = new_f;
}

// warp/affine.rs:70-79
KB200_API void kb200_get_rotation_matrix2d(float cx, float cy, float angle_deg, float scale, float out[6]) {
    const float PI_F = 3.14159265358979323846f;
    const float angle = angle_deg * PI_F / 180.0f;
    const float alpha = scale * cosf(angle);
    const float beta = scale * sinf(angle);
    const float tx = (1.0f - alpha) * cx - beta * cy;
    const float ty = beta * cx + (1.0f - alpha) * cy;
    out[0] = alpha; out[1] = beta; out[2] = tx; out[3] = -beta; out[4] = alpha; out[5] = ty;
}

// warp/perspective.rs:11-60
KB200_API int kb200_invert_homography(const float m[9], float inv[9]) {
    const float det = m[0] * (m[4] * m[8] - m[5] * m[7]) - m[1] * (m[3] * m[8] - m[5] * m[6]) +
                      m[2] * (m[3] * m[7] - m[4] * m[6]);
    const float h8_sq = m[8] * m[8];
    const float det_norm = (h8_sq > 1.1920929e-07f) ? det / (h8_sq * fabsf(m[8])) : det;
    if (fabsf(det_norm) < 1e-10f) return fail(KB200_ERR_SINGULAR_MATRIX, "homography matrix is singular (|det| < 1e-10)");
    const float adj[9] = {
        m[4] * m[8] - m[5] * m[7], m[2] * m[7] - m[1] * m[8], m[1] * m[5] - m[2] * m[4],
        m[5] * m[6] - m[3] * m[8], m[0] * m[8] - m[2] * m[6], m[2] * m[3] - m[0] * m[5],
        m[3] * m[7] - m[4] * m[6], m[1] * m[6] - m[0] * m[7], m[0] * m[4] - m[1] * m[3]};
    const float inv_det = 1.0f / det;
    for (int i = 0; i < 9; ++i) inv[i] = adj[i] * inv_det;
    return KB200_OK;
}

// filter/kernels.rs:25-41
KB200_API void kb200_gaussian_kernel_1d(uint32_t ksize, float sigma, float* out) {
    const float mean = (float)(ksize - 1) / 2.0f;
    const float sigma_sq = sigma * sigma;
    for (uint32_t i = 0; i < ksize; ++i) {
        const float x = (float)i - mean;
        out[i] = expf(-(x * x) / (2.0f * sigma_sq));
    }
    float norm = 0.0f;
    for (uint32_t i = 0; i < ksize; ++i) norm += out[i];
    for (uint32_t i = 0; i < ksize; ++i) out[i] /= norm;
}

// filter/ops.rs:122-153
KB200_API int kb200_gaussian_resolve(uint32_t kx_in, uint32_t ky_in, float sx_in, float sy_in, uint32_t* kx,
                                     uint32_t* ky, float* sx, float* sy) {
    size_t kernel_x = kx_in, kernel_y = ky_in;
    float sigma_x = sx_in, sigma_y = sy_in;
    if (sigma_y <= 0.0f) sigma_y = sigma_x;
    auto auto_k = [](float s) -> size_t {
        const float v = 2.0f * roundf(4.0f * s) + 1.0f;
        const size_t k = v <= 0.0f ? 0 : (size_t)v;
        return k | 1;
    };
    if (kernel_x == 0 && sigma_x > 0.0f) kernel_x = auto_k(sigma_x);
    if (kernel_y == 0 && sigma_y > 0.0f) kernel_y = auto_k(sigma_y);
    if (!(kernel_x > 0 && kernel_x % 2 == 1 && kernel_y > 0 && kernel_y % 2 == 1))
        return fail(KB200_ERR_INVALID_KERNEL, "invalid gaussian kernel size / sigma (%g, %g)", sigma_x, sigma_y);
    sigma_x = fmaxf(sigma_x, 0.0f);
    sigma_y = fmaxf(sigma_y, 0.0f);
    if (sigma_x == 0.0f) sigma_x = ((float)kernel_x - 1.0f) / 8.0f;
    if (sigma_y == 0.0f) sigma_y = ((float)kernel_y - 1.0f) / 8.0f;
    *kx = (uint32_t)kernel_x; *ky = (uint32_t)kernel_y; *sx = sigma_x; *sy = sigma_y;
    return KB200_OK;
}

// preprocess.rs:349-370
KB200_API void kb200_preprocess_affine(int mode, uint32_t sw, uint32_t sh, uint32_t dw, uint32_t dh, float out[4]) {
    if (mode == 0) {
        const float s = fminf((float)dw / (float)sw, (float)dh / (float)sh);
        out[0] = s; out[1] = s;
        out[2] = ((float)dw - (float)sw * s) * 0.5f;
        out[3] = ((float)dh - (float)sh * s) * 0.5f;
    } else {
        out[0] = (float)dw / (float)sw; out[1] = (float)dh / (float)sh;
        out[2] = 0.0f; out[3] = 0.0f;
    }
}

// core.rs:58-66
KB200_API void kb200_std_mean_finalize(const uint64_t sums[6], size_t npixels, double std_out[3], double mean_out[3]) {
    const double n = (double)npixels;
    for (int c = 0; c < 3; ++c) {
        const double sum = (double)sums[c], sq = (double)sums[3 + c];
        const double mean = sum / n;
        mean_out[c] = mean;
        std_out[c] = std::sqrt(sq / n - mean * mean);
    }
}

}  // extern "C"
