// nb2_selection.cu - ArticulationView attribute gather / masked scatter / articulation-mask kernels (SURVEY.md §8(f) rank 2).
//
// Reference: newton/_src/utils/selection.py
//   _gather_indexed_{3,4}d_kernel                          :185-203   -> view_gather_kernel
//   set_articulation_attribute_{3,4}d[_per_world]_kernel   :85-152    -> view_scatter_kernel
//   set_model_articulation_mask[_per_world]_kernel         :35-61     -> view_articulation_mask_kernel
// The reference launches one thread per (world, articulation, value[, component]) of a strided Warp array; here one thread
// copies one 32-bit word of the contiguous values array, so the staging side is always fully coalesced and the attribute
// side is coalesced over each articulation's run of selected values (K * row_words words).  These are pure bandwidth
// kernels: 8 bytes of traffic per word and no arithmetic besides the index split (DESIGN.md §3).
#include "nb2_internal.cuh"
#include "nb2_selection.cuh"

namespace nb2 {

template <typename I>
__global__ void __launch_bounds__(256) view_gather_kernel(const uint32_t* __restrict__ attrib, nb2_view_layout L, uint32_t* __restrict__ values,
                                                          long long n) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const ViewElem e = view_elem<I>(L, L.indices, (I)i);
        values[i] = attrib[e.word];
    }
}

template <typename I>
__global__ void __launch_bounds__(256) view_scatter_kernel(uint32_t* __restrict__ attrib, nb2_view_layout L, const uint32_t* __restrict__ values,
                                                           const uint8_t* __restrict__ mask, int mask_ndim, long long n) {
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        const ViewElem e = view_elem<I>(L, L.indices, (I)i);
        if (view_selected(L, mask, mask_ndim, e)) attrib[e.word] = values[i];
    }
}

__global__ void __launch_bounds__(256) view_articulation_mask_kernel(const uint8_t* __restrict__ mask, int mask_ndim,
                                                                     const int32_t* __restrict__ articulation_ids, int world_count,
                                                                     int count_per_world, uint8_t* __restrict__ model_mask,
                                                                     int articulation_count) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= world_count * count_per_world) return;
    const int w = i / count_per_world;
    const bool on = mask_ndim == 0 ? true : (mask_ndim == 1 ? mask[w] != 0 : mask[i] != 0);
    const int id = articulation_ids[i];
    if (on && id >= 0 && id < articulation_count) model_mask[id] = 1;
}

static bool layout_ok(const nb2_view_layout* L) {
    return L && L->world_count >= 0 && L->count_per_world >= 0 && L->value_count >= 0 && L->row_words > 0;
}

static int copy_grid(long long n) {
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const long long blocks = (n + 255) / 256;
    const long long cap = (long long)sms * 8;  // 8 resident 256-thread blocks per SM: one wave, grid-stride beyond it
    return (int)(blocks < cap ? blocks : cap);
}

}  // namespace nb2

using namespace nb2;

extern "C" {

nb2_status nb2_view_gather(const void* attrib, const nb2_view_layout* layout, void* values, void* cuda_stream) {
    if (!layout_ok(layout)) {
        set_error("nb2_view_gather: invalid layout");
        return NB2_ERR_INVALID_ARGUMENT;
    }
    const long long n = (long long)layout->world_count * layout->count_per_world * layout->value_count * layout->row_words;
    if (n == 0) return NB2_OK;
    if (!attrib || !values) {
        set_error("nb2_view_gather: NULL argument");
        return NB2_ERR_INVALID_ARGUMENT;
    }
    cudaStream_t s = static_cast<cudaStream_t>(cuda_stream);
    if (n < (1ll << 32))
        view_gather_kernel<unsigned><<<copy_grid(n), 256, 0, s>>>(static_cast<const uint32_t*>(attrib), *layout, static_cast<uint32_t*>(values), n);
    else
        view_gather_kernel<long long><<<copy_grid(n), 256, 0, s>>>(static_cast<const uint32_t*>(attrib), *layout, static_cast<uint32_t*>(values), n);
    count_launch();
    NB2_CUDA_CHECK(cudaGetLastError());
    return NB2_OK;
}

nb2_status nb2_view_scatter(void* attrib, const nb2_view_layout* layout, const void* values, const uint8_t* mask, int32_t mask_ndim,
                            void* cuda_stream) {
    if (!layout_ok(layout) || mask_ndim < 0 || mask_ndim > 2 || (mask_ndim != 0 && !mask)) {
        set_error("nb2_view_scatter: invalid layout or mask");
        return NB2_ERR_INVALID_ARGUMENT;
    }
    const long long n = (long long)layout->world_count * layout->count_per_world * layout->value_count * layout->row_words;
    if (n == 0) return NB2_OK;
    if (!attrib || !values) {
        set_error("nb2_view_scatter: NULL argument");
        return NB2_ERR_INVALID_ARGUMENT;
    }
    cudaStream_t s = static_cast<cudaStream_t>(cuda_stream);
    if (n < (1ll << 32))
        view_scatter_kernel<unsigned><<<copy_grid(n), 256, 0, s>>>(static_cast<uint32_t*>(attrib), *layout, static_cast<const uint32_t*>(values), mask,
                                                                   mask_ndim, n);
    else
        view_scatter_kernel<long long><<<copy_grid(n), 256, 0, s>>>(static_cast<uint32_t*>(attrib), *layout, static_cast<const uint32_t*>(values), mask,
                                                                    mask_ndim, n);
    count_launch();
    NB2_CUDA_CHECK(cudaGetLastError());
    return NB2_OK;
}

nb2_status nb2_view_articulation_mask(const uint8_t* mask, int32_t mask_ndim, const int32_t* articulation_ids, int32_t world_count,
                                      int32_t count_per_world, uint8_t* model_mask, int32_t articulation_count, void* cuda_stream) {
    if (world_count < 0 || count_per_world < 0 || articulation_count < 0 || mask_ndim < 0 || mask_ndim > 2 || (mask_ndim != 0 && !mask)) {
        set_error("nb2_view_articulation_mask: invalid argument");
        return NB2_ERR_INVALID_ARGUMENT;
    }
    if (articulation_count == 0) return NB2_OK;
    if (!model_mask || (!articulation_ids && world_count * count_per_world > 0)) {
        set_error("nb2_view_articulation_mask: NULL argument");
        return NB2_ERR_INVALID_ARGUMENT;
    }
    cudaStream_t s = static_cast<cudaStream_t>(cuda_stream);
    NB2_CUDA_CHECK(cudaMemsetAsync(model_mask, 0, (size_t)articulation_count, s));
    const int n = world_count * count_per_world;
    if (n == 0) return NB2_OK;
    view_articulation_mask_kernel<<<(n + 255) / 256, 256, 0, s>>>(mask, mask_ndim, articulation_ids, world_count, count_per_world, model_mask,
                                                                  articulation_count);
    count_launch();
    NB2_CUDA_CHECK(cudaGetLastError());
    return NB2_OK;
}

}  // extern "C"
