// ref_shim.h — minimal stand-ins for the TensorFlow / Eigen declarations that the
// reference's *_gpu.cu.cc files mention, so that those files compile UNMODIFIED with nvcc
// for sm_90a (oracle/Makefile `ref` target).  TEST INFRASTRUCTURE ONLY; written from
// scratch (the kernels need nothing from TF beyond a stream handle and temp allocations).
#pragma once
#include <cuda_runtime.h>

#include <cassert>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <vector>

namespace Eigen {

struct GpuDevice {
    cudaStream_t s = 0;
    cudaStream_t stream() const { return s; }
    bool ok() const { return true; }
};

enum { DontAlign = 0x2 };

template <typename T, int R, int C, int Opt = 0>
struct Matrix {
    T v[R * C];
    __host__ __device__ T& operator()(int r, int c) { return v[r * C + c]; }
    __host__ __device__ const T& operator()(int r, int c) const { return v[r * C + c]; }
    __host__ __device__ Matrix<T, C, R, Opt> transpose() const
    {
        Matrix<T, C, R, Opt> t;
        for (int r = 0; r < R; r++)
            for (int c = 0; c < C; c++) t(c, r) = (*this)(r, c);
        return t;
    }
};

// coefficient-wise (lazy) product, the evaluation Eigen uses for small fixed sizes
template <typename T, int R, int K, int C, int O1, int O2>
__host__ __device__ Matrix<T, R, C, O2> operator*(const Matrix<T, R, K, O1>& a, const Matrix<T, K, C, O2>& b)
{
    Matrix<T, R, C, O2> o;
    for (int i = 0; i < R; i++)
        for (int j = 0; j < C; j++) {
            T acc = a(i, 0) * b(0, j);
            for (int k = 1; k < K; k++) acc += a(i, k) * b(k, j);
            o(i, j) = acc;
        }
    return o;
}

typedef Matrix<float, 3, 3> Matrix3f;

template <typename T>
struct Quaternion {
    T w_, x_, y_, z_;
    __host__ __device__ Quaternion(T w, T x, T y, T z) : w_(w), x_(x), y_(y), z_(z) {}
    // rotation matrix of a unit quaternion (standard formula, as in Eigen::QuaternionBase)
    __host__ __device__ Matrix<T, 3, 3> toRotationMatrix() const
    {
        Matrix<T, 3, 3> res;
        const T tx = T(2) * x_, ty = T(2) * y_, tz = T(2) * z_;
        const T twx = tx * w_, twy = ty * w_, twz = tz * w_;
        const T txx = tx * x_, txy = ty * x_, txz = tz * x_;
        const T tyy = ty * y_, tyz = tz * y_, tzz = tz * z_;
        res(0, 0) = T(1) - (tyy + tzz); res(0, 1) = txy - twz; res(0, 2) = txz + twy;
        res(1, 0) = txy + twz; res(1, 1) = T(1) - (txx + tzz); res(1, 2) = tyz - twx;
        res(2, 0) = txz - twy; res(2, 1) = tyz + twx; res(2, 2) = T(1) - (txx + tyy);
        return res;
    }
};
typedef Quaternion<float> Quaternionf;

}  // namespace Eigen

namespace tensorflow {

struct Status {
    bool ok() const { return true; }
};
enum DataType { DT_INT32, DT_FLOAT };

struct TensorShape {
    std::vector<long long> dims;
    long long num_elements() const
    {
        long long n = 1;
        for (long long d : dims) n *= d;
        return n;
    }
};

struct TensorShapeUtils {
    static Status MakeShape(const int* d, int n, TensorShape* out)
    {
        out->dims.assign(d, d + n);
        return Status();
    }
};

template <typename T>
struct FlatView {
    T* p;
    T* data() { return p; }
};

struct Tensor {
    void* p = nullptr;
    template <typename T>
    FlatView<T> flat() { return FlatView<T>{static_cast<T*>(p)}; }
};

// temp allocations with reuse across calls (cudaMalloc per call would dominate timings)
struct OpKernelContext {
    std::multimap<size_t, void*> free_list;
    std::vector<std::pair<size_t, void*>> in_use;
    Status allocate_temp(DataType, const TensorShape& shape, Tensor* t)
    {
        size_t bytes = (size_t)shape.num_elements() * 4;
        if (bytes == 0) bytes = 4;
        auto it = free_list.find(bytes);
        void* p = nullptr;
        if (it != free_list.end()) {
            p = it->second;
            free_list.erase(it);
        } else if (cudaMalloc(&p, bytes) != cudaSuccess) {
            fprintf(stderr, "ref_shim: cudaMalloc(%zu) failed\n", bytes);
            abort();
        }
        in_use.emplace_back(bytes, p);
        t->p = p;
        return Status();
    }
    void release_all()
    {
        for (auto& a : in_use) free_list.insert(a);
        in_use.clear();
    }
    ~OpKernelContext()
    {
        release_all();
        for (auto& a : free_list) cudaFree(a.second);
    }
};

#define OP_REQUIRES_OK(ctx, expr) \
    do {                          \
        (void)(ctx);              \
        (expr);                   \
    } while (0)

}  // namespace tensorflow
