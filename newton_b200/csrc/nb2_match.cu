// nb2_match.cu - frame-to-frame contact matching, CollisionPipeline(contact_matching="latest" | "sticky", contact_report=...)
// (reference geometry/contact_match.py: _match_contacts_kernel :266-354, _resolve_claims_kernel :357-390,
// _save_sorted_state_kernel :442-477, _replay_matched_kernel :529-561, _collect_contact_report_kernel :568-595; call sites
// sim/collide.py:2033-2137).
//
// Runs on the exported, key-sorted `Contacts` arrays (matching implies deterministic=True upstream, collide.py:1269-1271): for
// each new contact the previous frame's contacts of the same shape pair are found by binary search on the sorted keys, the closest
// one (world-space midpoint) whose normal passes the dot threshold is claimed with one 64-bit atomicMin (distance, then key),
// and losers of a claim become MATCH_BROKEN.  The history (keys, midpoints, normals) lives with the nb2_model.
#include <cstdint>

#include "nb2_internal.cuh"
#include "nb2_math.cuh"

namespace nb2 {

enum { MATCH_NOT_FOUND = -1, MATCH_BROKEN = -2 };
static const long long CLAIM_SENTINEL = 0x7FFFFFFFFFFFFFFFll;

__device__ __forceinline__ long long pair_prefix(int s0, int s1) {  // make_contact_sort_key without the sub key (contact_data.py:59-87)
    return ((long long)(s0 & 0xFFFFF) << 43) | ((long long)(s1 & 0xFFFFF) << 23);
}
__device__ __forceinline__ int lower_bound64(const long long* keys, int lo, int hi, long long v) {
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (keys[mid] < v) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}
__device__ __forceinline__ unsigned float_flip(float f) {
    const unsigned i = __float_as_uint(f);
    const unsigned mask = (unsigned)(-(int)(i >> 31)) | 0x80000000u;
    return i ^ mask;
}
__device__ __forceinline__ V3 contact_midpoint(const nb2_model_desc& d, const nb2_contacts_view& c, const float* body_q, int i) {
    V3 p0 = ld3(c.point0 + 3 * i), p1 = ld3(c.point1 + 3 * i);
    const int b0 = d.shape_body[c.shape0[i]], b1 = d.shape_body[c.shape1[i]];
    if (b0 != -1) p0 = xpoint(ldx(body_q + 7 * b0), p0);
    if (b1 != -1) p1 = xpoint(ldx(body_q + 7 * b1), p1);
    return 0.5f * (p0 + p1);
}

// sort keys of the new (sorted) contacts: the sub key is the contact's position inside its pair's run
__global__ void __launch_bounds__(256) match_keys_kernel(nb2_contacts_view c, long long* __restrict__ keys) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int n = min(c.rigid_contact_count[0], c.rigid_contact_max);
    if (i >= n) return;
    const long long prefix = pair_prefix(c.shape0[i], c.shape1[i]);
    int lo = 0, hi = i;  // first contact of the run: shapes are sorted, so search on (shape0, shape1) directly
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (pair_prefix(c.shape0[mid], c.shape1[mid]) < prefix) lo = mid + 1;
        else hi = mid;
    }
    keys[i] = prefix | (long long)((i - lo) & 0x7FFFFF);
}

__global__ void __launch_bounds__(256) match_contacts_kernel(nb2_model_desc d, nb2_contacts_view c, const float* __restrict__ body_q,
                                                             const long long* __restrict__ new_keys, const long long* __restrict__ prev_keys,
                                                             const float* __restrict__ prev_pos, const float* __restrict__ prev_normal,
                                                             const int* __restrict__ prev_count, long long* prev_claim,
                                                             const uint8_t* __restrict__ reset_mask, float pos_threshold_sq, float normal_dot_threshold,
                                                             int* __restrict__ match_index) {
    const int tid = blockIdx.x * blockDim.x + threadIdx.x;
    if (tid >= c.rigid_contact_max) return;
    const int n_new = min(c.rigid_contact_count[0], c.rigid_contact_max);
    if (tid >= n_new) {
        match_index[tid] = MATCH_NOT_FOUND;
        return;
    }
    const int n_old = prev_count[0];
    if (n_old == 0) {
        match_index[tid] = MATCH_NOT_FOUND;
        return;
    }
    if (reset_mask) {  // reset_world_selected (core/reset.py:14-18) on both shapes
        const int w0 = d.shape_world[c.shape0[tid]], w1 = d.shape_world[c.shape1[tid]];
        const bool r0 = (w0 >= 0 && w0 < d.world_count) ? reset_mask[w0] != 0 : (w0 == -1 && reset_mask[d.world_count] != 0);
        const bool r1 = (w1 >= 0 && w1 < d.world_count) ? reset_mask[w1] != 0 : (w1 == -1 && reset_mask[d.world_count] != 0);
        if (r0 || r1) {
            match_index[tid] = MATCH_NOT_FOUND;
            return;
        }
    }
    const long long target = new_keys[tid];
    const V3 pos = contact_midpoint(d, c, body_q, tid);
    const V3 nrm = ld3(c.normal + 3 * tid);
    const long long prefix = target & ~0x7FFFFFll, pair_end = prefix + 0x800000ll;
    const int lo = lower_bound64(prev_keys, 0, n_old, prefix), hi = lower_bound64(prev_keys, lo, n_old, pair_end);
    if (lo >= hi) {
        match_index[tid] = MATCH_NOT_FOUND;
        return;
    }
    int best = -1;
    float best_d = pos_threshold_sq;
    for (int k = lo; k < hi; ++k) {
        const V3 diff = pos - ld3(prev_pos + 3 * k);
        const float dsq = dot(diff, diff);
        if (dsq <= best_d && dot(nrm, ld3(prev_normal + 3 * k)) >= normal_dot_threshold) {
            best_d = dsq;
            best = k;
        }
    }
    if (best >= 0) {
        match_index[tid] = best;
        const long long claim = ((long long)float_flip(best_d) << 32) | (target & 0xFFFFFFFFll);
        atomicMin(prev_claim + best, claim);
    } else {
        match_index[tid] = MATCH_BROKEN;
    }
}

__global__ void __launch_bounds__(256) match_resolve_kernel(nb2_contacts_view c, const long long* __restrict__ new_keys,
                                                            const long long* __restrict__ prev_claim, int* __restrict__ match_index,
                                                            int* __restrict__ prev_was_matched) {
    const int tid = blockIdx.x * blockDim.x + threadIdx.x;
    if (tid >= min(c.rigid_contact_count[0], c.rigid_contact_max)) return;
    const int cand = match_index[tid];
    if (cand < 0) return;
    if ((prev_claim[cand] & 0xFFFFFFFFll) != (new_keys[tid] & 0xFFFFFFFFll)) match_index[tid] = MATCH_BROKEN;
    else if (prev_was_matched) prev_was_matched[cand] = 1;
}

// "sticky": a matched contact that is still touching keeps last frame's record - body-frame points and offsets, world normal
// (_replay_matched_kernel :529-561).  Runs on the sorted rows, before the history is saved.
__global__ void __launch_bounds__(256) match_replay_kernel(nb2_model_desc d, nb2_contacts_view c, const float* __restrict__ body_q,
                                                           const int* __restrict__ match_index, const float* __restrict__ prev_record,
                                                           const float* __restrict__ prev_normal, int cap) {
    const int tid = blockIdx.x * blockDim.x + threadIdx.x;
    if (tid >= min(c.rigid_contact_count[0], c.rigid_contact_max)) return;
    const int idx = match_index[tid];
    if (idx < 0) return;
    V3 p0 = ld3(c.point0 + 3 * tid), p1 = ld3(c.point1 + 3 * tid);
    const int b0 = d.shape_body[c.shape0[tid]], b1 = d.shape_body[c.shape1[tid]];
    if (b0 >= 0) p0 = xpoint(ldx(body_q + 7 * b0), p0);
    if (b1 >= 0) p1 = xpoint(ldx(body_q + 7 * b1), p1);
    const float fresh_gap = dot(p1 - p0, ld3(c.normal + 3 * tid)) - (c.margin0[tid] + c.margin1[tid]);
    if (fresh_gap > 0.0f) return;
    st3(c.point0 + 3 * tid, ld3(prev_record + 3 * idx));
    st3(c.point1 + 3 * tid, ld3(prev_record + 3 * (cap + idx)));
    st3(c.offset0 + 3 * tid, ld3(prev_record + 3 * (2 * cap + idx)));
    st3(c.offset1 + 3 * tid, ld3(prev_record + 3 * (3 * cap + idx)));
    st3(c.normal + 3 * tid, ld3(prev_normal + 3 * idx));
}

// contact_report: rows of this frame without a match ("new") and rows of the previous frame nothing matched ("broken", unless the
// row's worlds were reset), both in ascending order - the reference appends with atomics (:583-595), i.e. in no particular order.
// One CTA walks the rows in tiles with a ballot/prefix per tile: the lists are short and the order is reproducible.
__global__ void __launch_bounds__(1024) match_report_kernel(nb2_model_desc d, nb2_contacts_view c, const int* __restrict__ match_index,
                                                            const long long* __restrict__ prev_keys, const int* __restrict__ prev_count,
                                                            const int* __restrict__ prev_was_matched, const uint8_t* __restrict__ reset_mask,
                                                            int* __restrict__ new_indices, int* __restrict__ new_count,
                                                            int* __restrict__ broken_indices, int* __restrict__ broken_count) {
    __shared__ int warp_sum[2][32];
    __shared__ int base[2];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, warps = blockDim.x >> 5;
    const int n_new = min(c.rigid_contact_count[0], c.rigid_contact_max), n_old = prev_count[0];
    if (threadIdx.x == 0) base[0] = base[1] = 0;
    __syncthreads();
    for (int start = 0; start < max(n_new, n_old); start += blockDim.x) {
        const int i = start + threadIdx.x;
        const bool is_new = i < n_new && match_index[i] < 0;
        bool is_broken = false;
        if (i < n_old && prev_was_matched[i] == 0) {
            const long long key = prev_keys[i];
            const int s0 = int((key >> 43) & 0xFFFFF), s1 = int((key >> 23) & 0xFFFFF);
            bool reset = false;
            if (reset_mask) {
                const int w0 = d.shape_world[s0], w1 = d.shape_world[s1];
                reset = ((w0 >= 0 && w0 < d.world_count) ? reset_mask[w0] != 0 : (w0 == -1 && reset_mask[d.world_count] != 0)) ||
                        ((w1 >= 0 && w1 < d.world_count) ? reset_mask[w1] != 0 : (w1 == -1 && reset_mask[d.world_count] != 0));
            }
            is_broken = !reset;
        }
        const unsigned bn = __ballot_sync(0xFFFFFFFFu, is_new), bb = __ballot_sync(0xFFFFFFFFu, is_broken);
        if (lane == 0) {
            warp_sum[0][warp] = __popc(bn);
            warp_sum[1][warp] = __popc(bb);
        }
        __syncthreads();
        int off_n = base[0], off_b = base[1];
        for (int w = 0; w < warp; ++w) {
            off_n += warp_sum[0][w];
            off_b += warp_sum[1][w];
        }
        const unsigned below = (1u << lane) - 1u;
        if (is_new) new_indices[off_n + __popc(bn & below)] = i;
        if (is_broken) broken_indices[off_b + __popc(bb & below)] = i;
        __syncthreads();
        if (threadIdx.x == 0) {
            int tn = 0, tb = 0;
            for (int w = 0; w < warps; ++w) {
                tn += warp_sum[0][w];
                tb += warp_sum[1][w];
            }
            base[0] += tn;
            base[1] += tb;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        new_count[0] = base[0];
        broken_count[0] = base[1];
    }
}

__global__ void __launch_bounds__(256) match_save_kernel(nb2_model_desc d, nb2_contacts_view c, const float* __restrict__ body_q,
                                                         const long long* __restrict__ new_keys, long long* __restrict__ prev_keys,
                                                         float* __restrict__ prev_pos, float* __restrict__ prev_normal, long long* __restrict__ prev_claim,
                                                         int* __restrict__ prev_count, int* __restrict__ prev_was_matched,
                                                         float* __restrict__ prev_record, int cap) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int n = min(c.rigid_contact_count[0], c.rigid_contact_max);
    if (i == 0) prev_count[0] = n;
    if (i >= n) return;
    prev_keys[i] = new_keys[i];
    prev_claim[i] = CLAIM_SENTINEL;
    if (prev_was_matched) prev_was_matched[i] = 0;
    st3(prev_pos + 3 * i, contact_midpoint(d, c, body_q, i));
    st3(prev_normal + 3 * i, ld3(c.normal + 3 * i));
    if (prev_record) {  // sticky: the record this frame actually used, carried forward
        st3(prev_record + 3 * i, ld3(c.point0 + 3 * i));
        st3(prev_record + 3 * (cap + i), ld3(c.point1 + 3 * i));
        st3(prev_record + 3 * (2 * cap + i), ld3(c.offset0 + 3 * i));
        st3(prev_record + 3 * (3 * cap + i), ld3(c.offset1 + 3 * i));
    }
}

}  // namespace nb2

using namespace nb2;

extern "C" nb2_status nb2_contacts_match(nb2_model* m, const float* body_q, const nb2_contacts_view* c, int32_t* match_index,
                                         const nb2_match_options* opt, void* cuda_stream) {
    if (!m || !c || !opt || !match_index || !c->rigid_contact_count || !c->shape0 || !c->shape1 || !c->point0 || !c->point1 || !c->normal ||
        (!body_q && m->dev.d.body_count > 0)) {
        set_error("nb2_contacts_match: NULL argument");
        return NB2_ERR_INVALID_ARGUMENT;
    }
    const bool sticky = opt->sticky != 0;
    const bool report = opt->new_indices || opt->new_count || opt->broken_indices || opt->broken_count;
    if (report && !(opt->new_indices && opt->new_count && opt->broken_indices && opt->broken_count)) {
        set_error("nb2_contacts_match: the contact report needs all four of new_indices, new_count, broken_indices, broken_count");
        return NB2_ERR_INVALID_ARGUMENT;
    }
    if (sticky && !(c->offset0 && c->offset1 && c->margin0 && c->margin1)) {
        set_error("nb2_contacts_match: sticky matching replays offset0/offset1 and reads margin0/margin1 - all four must be given");
        return NB2_ERR_INVALID_ARGUMENT;
    }
    cudaStream_t s = static_cast<cudaStream_t>(cuda_stream);
    DeviceGuard guard(m->device);
    const int cap = c->rigid_contact_max;
    // history buffers (not capturable: the first call - or the first sticky / report call - sizes them, like the sort scratch)
    if (cap > m->match_capacity || (sticky && !m->match_prev_record.get()) || (report && !m->match_prev_was_matched.get())) {
        const size_t rows = size_t(cap > 0 ? cap : 1);
        DeviceBuffer new_keys, prev_keys, prev_claim, prev_pos, prev_normal, prev_record, prev_was_matched, prev_count;
        if (new_keys.alloc(rows * 8) || prev_keys.alloc(rows * 8) || prev_claim.alloc(rows * 8) || prev_pos.alloc(rows * 12) ||
            prev_normal.alloc(rows * 12) || (sticky && prev_record.alloc(rows * 48)) || (report && prev_was_matched.alloc(rows * 4)) ||
            (!m->match_prev_count.get() && prev_count.alloc(sizeof(int)))) {
            set_error("nb2_contacts_match: out of device memory");
            return NB2_ERR_CUDA;
        }
        m->replace_scratch(m->match_new_keys, std::move(new_keys));
        m->replace_scratch(m->match_prev_keys, std::move(prev_keys));
        m->replace_scratch(m->match_prev_claim, std::move(prev_claim));
        m->replace_scratch(m->match_prev_pos, std::move(prev_pos));
        m->replace_scratch(m->match_prev_normal, std::move(prev_normal));
        m->replace_scratch(m->match_prev_record, std::move(prev_record));
        m->replace_scratch(m->match_prev_was_matched, std::move(prev_was_matched));
        if (prev_count.get()) m->match_prev_count = std::move(prev_count);
        if (report) cudaMemsetAsync(m->match_prev_was_matched.get(), 0, rows * 4, s);
        cudaMemsetAsync(m->match_prev_count.get(), 0, sizeof(int), s);
        m->match_prev_has_record = false;
        m->match_capacity = cap;
    }
    long long* new_keys = m->match_new_keys.get<long long>();
    long long* prev_keys = m->match_prev_keys.get<long long>();
    long long* prev_claim = m->match_prev_claim.get<long long>();
    float* prev_pos = m->match_prev_pos.get<float>();
    float* prev_normal = m->match_prev_normal.get<float>();
    float* prev_record = m->match_prev_record.get<float>();
    int* prev_count = m->match_prev_count.get<int>();
    int* prev_was_matched = m->match_prev_was_matched.get<int>();
    if (opt->reset_all) cudaMemsetAsync(prev_count, 0, sizeof(int), s);
    if (cap > 0) {
        const int blocks = (cap + 255) / 256;
        // a history that was saved without sticky records / report flags keeps working: those buffers are only used when present
        match_keys_kernel<<<blocks, 256, 0, s>>>(*c, new_keys);
        match_contacts_kernel<<<blocks, 256, 0, s>>>(m->dev.d, *c, body_q, new_keys, prev_keys, prev_pos, prev_normal, prev_count, prev_claim,
                                                     opt->reset_world_mask, opt->pos_threshold * opt->pos_threshold,
                                                     opt->normal_dot_threshold, match_index);
        match_resolve_kernel<<<blocks, 256, 0, s>>>(*c, new_keys, prev_claim, match_index, prev_was_matched);
        int launched = 4;
        if (sticky && m->match_prev_has_record) {
            match_replay_kernel<<<blocks, 256, 0, s>>>(m->dev.d, *c, body_q, match_index, prev_record, prev_normal, m->match_capacity);
            ++launched;
        }
        if (report) {
            match_report_kernel<<<1, 1024, 0, s>>>(m->dev.d, *c, match_index, prev_keys, prev_count, prev_was_matched, opt->reset_world_mask,
                                                   opt->new_indices, opt->new_count, opt->broken_indices, opt->broken_count);
            ++launched;
        }
        match_save_kernel<<<blocks, 256, 0, s>>>(m->dev.d, *c, body_q, new_keys, prev_keys, prev_pos, prev_normal, prev_claim, prev_count,
                                                 prev_was_matched, sticky ? prev_record : nullptr, m->match_capacity);
        m->match_prev_has_record = sticky;
        count_launch(launched);
        if (cudaGetLastError() != cudaSuccess) {
            set_error("nb2_contacts_match: kernel launch failed");
            return NB2_ERR_CUDA;
        }
    } else if (report) {
        cudaMemsetAsync(opt->new_count, 0, sizeof(int), s);
        cudaMemsetAsync(opt->broken_count, 0, sizeof(int), s);
    }
    return NB2_OK;
}
