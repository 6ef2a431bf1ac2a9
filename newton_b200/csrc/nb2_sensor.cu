// nb2_sensor.cu - contact sensor: Contacts.force summed per sensing object and per counterpart (reference
// newton.sensors.SensorContact, sensors/sensor_contact.py).
//
// The reference accumulates with float atomics (accumulate_contact_forces_kernel, :67-156), so on a GPU the last bit of every
// reading depends on thread timing.  Here every output entry is the sum of its contributions in ascending contact index, the
// shape0 side of a contact before its shape1 side - the reference's serial order - for any order of the contact buffer:
//   1. sensor_records_kernel: one thread per contact slot evaluates force, friction and the force-weighted midpoint once and
//      emits two sort records (key = row of side 0 / side 1 or the sentinel row_count, value = 2 i + side);
//   2. cub::DeviceRadixSort::SortPairs over the 2 rigid_contact_max records, end_bit = bits of row_count; the sort is stable, so
//      inside one row the records stay in (i, side) order;
//   3. sensor_rows_kernel: one thread per row finds its run by binary search and walks it in order.  It is the only writer of
//      its row (totals, matrix entries, position weights), so no atomics are needed.  The matrices and weights are cleared by
//      memsets before it (coalesced; a row-per-thread clear of 13 columns strides 156 bytes between lanes), the totals are
//      written whole.  A second walk over the run divides each touched position entry by its weight, once, and the thread
//      finally writes the sensing transform.
// The caller owns all memory (outputs and one scratch buffer); nothing here allocates or synchronises.
#include <cub/device/device_radix_sort.cuh>

#include "nb2_internal.cuh"
#include "nb2_math.cuh"

namespace nb2 {
namespace {

struct SensorScratch {
    int *keys, *vals, *keys_sorted, *vals_sorted;
    float4* rec;    // 3 per contact: (force, |force|), (friction, col of shape1), (|force| * midpoint, col of shape0)
    float* weight;  // [row_count, col_count] position weights
    void* temp;     // CUB temp storage
    size_t temp_bytes, total;
};

size_t align256(size_t x) { return (x + 255) & ~size_t(255); }

int sensor_end_bit(int rows) {  // keys are 0 .. rows (rows = sentinel)
    int b = 1;
    while ((1ll << b) <= rows) ++b;
    return b;
}

// Carves `base` (nullptr: sizes only) into the scratch regions.
cudaError_t sensor_scratch_layout(int C, int R, int K, char* base, SensorScratch& s) {
    const int N = 2 * C;
    size_t temp = 0;
    if (N > 0) {
        cudaError_t e = cub::DeviceRadixSort::SortPairs(nullptr, temp, (const int*)nullptr, (int*)nullptr, (const int*)nullptr, (int*)nullptr,
                                                        N, 0, sensor_end_bit(R));
        if (e != cudaSuccess) return e;
    }
    size_t off = 0;
    auto take = [&](size_t bytes) -> char* {
        char* p = base ? base + off : nullptr;
        off += align256(bytes);
        return p;
    };
    s.keys = reinterpret_cast<int*>(take(size_t(N) * sizeof(int)));
    s.vals = reinterpret_cast<int*>(take(size_t(N) * sizeof(int)));
    s.keys_sorted = reinterpret_cast<int*>(take(size_t(N) * sizeof(int)));
    s.vals_sorted = reinterpret_cast<int*>(take(size_t(N) * sizeof(int)));
    s.rec = reinterpret_cast<float4*>(take(size_t(C) * 3 * sizeof(float4)));
    s.weight = reinterpret_cast<float*>(take(size_t(R) * size_t(K) * sizeof(float)));
    s.temp = take(temp);
    s.temp_bytes = temp;
    s.total = off;
    return cudaSuccess;
}

// accumulate_contact_forces_kernel (:67-156) up to the atomics: the per-contact terms and the two sort records.
__global__ void __launch_bounds__(256) sensor_records_kernel(nb2_sensor_contact_view S, nb2_contacts_view c, const float* __restrict__ body_q,
                                                             int* __restrict__ keys, int* __restrict__ vals, float4* __restrict__ rec) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= c.rigid_contact_max) return;
    const int R = S.row_count;
    int key0 = R, key1 = R;
    if (i < *c.rigid_contact_count) {
        const int s0 = c.shape0[i], s1 = c.shape1[i];
        // malformed ids: the reference only asserts shape0 >= 0 and shape1 >= 0 (and reads out of bounds past the end)
        if (s0 >= 0 && s0 < S.shape_count && s1 >= 0 && s1 < S.shape_count) {
            const int row0 = S.shape_to_row[s0], row1 = S.shape_to_row[s1];
            if (row0 >= 0 || row1 >= 0) {
                const V3 f = ld3(c.force + 6 * size_t(i));  // spatial_top
                V3 n = ld3(c.normal + 3 * size_t(i));
                if (fabsf(dot(n, n) - 1.0f) > 1.0e-4f) n = unit(n);
                const V3 fr = f - dot(f, n) * n;
                int col0 = -1, col1 = -1;
                float weight = 0.0f;
                V3 wm;
                if (S.col_count > 0) {
                    col0 = S.shape_to_col[s0];
                    col1 = S.shape_to_col[s1];
                    if (body_q) {
                        weight = len(f);
                        if (weight > 0.0f && ((row0 >= 0 && col1 >= 0) || (row1 >= 0 && col0 >= 0))) {
                            const int b0 = S.shape_body[s0], b1 = S.shape_body[s1];
                            const Xf X0 = b0 >= 0 ? ldx(body_q + 7 * size_t(b0)) : Xf();
                            const Xf X1 = b1 >= 0 ? ldx(body_q + 7 * size_t(b1)) : Xf();
                            // contact_surface_point (sim/contacts.py:96-115)
                            const V3 p0 = xpoint(X0, ld3(c.point0 + 3 * size_t(i)) + ld3(c.offset0 + 3 * size_t(i)));
                            const V3 p1 = xpoint(X1, ld3(c.point1 + 3 * size_t(i)) + ld3(c.offset1 + 3 * size_t(i)));
                            wm = weight * (0.5f * (p0 + p1));
                        }
                    }
                }
                rec[3 * size_t(i) + 0] = make_float4(f.x, f.y, f.z, weight);
                rec[3 * size_t(i) + 1] = make_float4(fr.x, fr.y, fr.z, __int_as_float(col1));
                rec[3 * size_t(i) + 2] = make_float4(wm.x, wm.y, wm.z, __int_as_float(col0));
                if (row0 >= 0) key0 = row0;
                if (row1 >= 0) key1 = row1;
            }
        }
    }
    keys[2 * i] = key0;
    keys[2 * i + 1] = key1;
    vals[2 * i] = 2 * i;
    vals[2 * i + 1] = 2 * i + 1;
}

NB2_DEV void add3(float* p, V3 v) { st3(p, ld3(p) + v); }

// The atomics of accumulate_contact_forces_kernel in serial order, normalize_contact_positions_kernel (:159-168) and
// compute_sensing_transforms_kernel (:44-64) for one row.
__global__ void __launch_bounds__(128) sensor_rows_kernel(nb2_sensor_contact_view S, const float* __restrict__ body_q, int N,
                                                          const int* __restrict__ keys, const int* __restrict__ vals,
                                                          const float4* __restrict__ rec, float* __restrict__ weight) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= S.row_count) return;
    const int K = S.col_count;  // the matrices and weights of this row are zero (memsets before the launch)
    float* fm = K ? S.force_matrix + size_t(r) * K * 3 : nullptr;
    float* fmf = K ? S.force_matrix_friction + size_t(r) * K * 3 : nullptr;
    float* pm = K ? S.position_matrix + size_t(r) * K * 3 : nullptr;
    float* w = K ? weight + size_t(r) * K : nullptr;
    int lo = 0, hi = N;  // first record of this row
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (keys[mid] < r) lo = mid + 1;
        else hi = mid;
    }
    V3 tot, totf;
    int end = lo;
    for (int k = lo; k < N && keys[k] == r; ++k, ++end) {
        const int v = vals[k], i = v >> 1, side = v & 1;
        const float4 a = rec[3 * size_t(i)], b = rec[3 * size_t(i) + 1];
        V3 f(a.x, a.y, a.z), fr(b.x, b.y, b.z);
        if (side) {  // the shape1 side receives -force
            f = -f;
            fr = -fr;
        }
        tot += f;
        totf += fr;
        if (K > 0) {
            const float4 m = rec[3 * size_t(i) + 2];
            const int col = __float_as_int(side ? m.w : b.w);  // the counterpart is the other side
            if (col >= 0) {
                add3(fm + 3 * col, f);
                add3(fmf + 3 * col, fr);
                if (body_q && a.w > 0.0f) {
                    add3(pm + 3 * col, V3(m.x, m.y, m.z));
                    w[col] += a.w;
                }
            }
        }
    }
    if (S.total_force) {
        st3(S.total_force + 3 * size_t(r), tot);
        st3(S.total_force_friction + 3 * size_t(r), totf);
    }
    if (!body_q) return;
    if (K > 0) {  // normalize_contact_positions_kernel for the entries this row touched; the weight is cleared once used
        for (int k = lo; k < end; ++k) {
            const int v = vals[k], i = v >> 1;
            const int col = __float_as_int((v & 1) ? rec[3 * size_t(i) + 2].w : rec[3 * size_t(i) + 1].w);
            if (col >= 0 && w[col] > 0.0f) {
                st3(pm + 3 * col, ld3(pm + 3 * col) / w[col]);
                w[col] = 0.0f;
            }
        }
    }
    const int idx = S.sensing_indices[r];
    Xf X;
    if (S.sensing_kind == NB2_SENSING_BODY) {
        X = ldx(body_q + 7 * size_t(idx));
    } else {
        const int b = S.shape_body[idx];
        const Xf Xs = ldx(S.shape_transform + 7 * size_t(idx));
        X = b >= 0 ? xmul(ldx(body_q + 7 * size_t(b)), Xs) : Xs;
    }
    stx(S.sensing_transforms + 7 * size_t(r), X);
}

}  // namespace

nb2_status sensor_contact_scratch_bytes(int C, int R, int K, size_t* bytes) {
    SensorScratch s{};
    NB2_CUDA_CHECK(sensor_scratch_layout(C, R, K, nullptr, s));
    *bytes = s.total;
    return NB2_OK;
}

nb2_status launch_sensor_contact_update(const nb2_sensor_contact_view& S, const nb2_contacts_view& c, const float* body_q, void* scratch,
                                        size_t scratch_bytes, cudaStream_t stream) {
    const int C = c.rigid_contact_max, N = 2 * C;
    SensorScratch s{};
    NB2_CUDA_CHECK(sensor_scratch_layout(C, S.row_count, S.col_count, static_cast<char*>(scratch), s));
    if (s.total > scratch_bytes) {
        set_error("nb2_sensor_contact_update: scratch buffer of " + std::to_string(scratch_bytes) + " bytes, the call needs " +
                  std::to_string(s.total) + " (nb2_sensor_contact_scratch_bytes)");
        return NB2_ERR_INVALID_ARGUMENT;
    }
    if (S.row_count == 0) return NB2_OK;
    if (S.col_count > 0) {
        const size_t entries = size_t(S.row_count) * size_t(S.col_count);
        NB2_CUDA_CHECK(cudaMemsetAsync(S.force_matrix, 0, entries * 3 * sizeof(float), stream));
        NB2_CUDA_CHECK(cudaMemsetAsync(S.force_matrix_friction, 0, entries * 3 * sizeof(float), stream));
        NB2_CUDA_CHECK(cudaMemsetAsync(S.position_matrix, 0, entries * 3 * sizeof(float), stream));
        NB2_CUDA_CHECK(cudaMemsetAsync(s.weight, 0, entries * sizeof(float), stream));
    }
    int launches = 1;
    if (C > 0) {
        sensor_records_kernel<<<(C + 255) / 256, 256, 0, stream>>>(S, c, body_q, s.keys, s.vals, s.rec);
        size_t temp = s.temp_bytes;
        NB2_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(s.temp, temp, s.keys, s.keys_sorted, s.vals, s.vals_sorted, N, 0,
                                                       sensor_end_bit(S.row_count), stream));
        launches = 2;
    }
    sensor_rows_kernel<<<(S.row_count + 127) / 128, 128, 0, stream>>>(S, body_q, N, s.keys_sorted, s.vals_sorted, s.rec, s.weight);
    count_launch(launches);  // plus the radix sort's own kernels
    NB2_CUDA_CHECK(cudaGetLastError());
    return NB2_OK;
}

}  // namespace nb2
