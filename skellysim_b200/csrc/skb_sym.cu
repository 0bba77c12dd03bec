// skb_sym.cu -- host side of the symmetric Stokeslet kernel (sym_kernels.cuh) and the fiber <-> periphery cross kernel
// (cross_kernels.cuh), the one unit that compiles them: launch attributes, the planner and ItemPlan they share, the
// symmetric path of an Evaluator (SymState), the cross pass of a flow (CrossState), and the C ABI calls about them.
#include "sym_kernels.cuh"
#include "cross_kernels.cuh"
#include "skb_internal.hpp"

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <vector>

namespace skb {

// (prepare_device) both kernels' dynamic shared memory, and the max-shared carve-out they share with the row streamer
int prepare_sym_kernels() {
    auto set_shared = [](auto kern, int bytes) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
        return e == cudaSuccess ? cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout,
                                                       cudaSharedmemCarveoutMaxShared)
                                : e;
    };
    CUDA_TRY(set_shared(pair_sym_kernel<kSymT, kSymMinB, false>, SymSmem<kSymT>::total_bytes));
    CUDA_TRY(set_shared(pair_sym_kernel<kSymT, kSymMinB, true>, SymSmem<kSymT>::total_bytes));
    CUDA_TRY(set_shared(pair_cross_kernel<kCrossT, kCrossMinB>, CrossSmem<kCrossT>::total_bytes));
    return SKB_OK;
}

__global__ void self_check_kernel(const double *__restrict__ a, const double *__restrict__ b, long long n,
                                  int *__restrict__ differs) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && __double_as_longlong(a[i]) != __double_as_longlong(b[i]))
        *differs = 1;
}

// bytes the reverse partials of the symmetric kernel may occupy: SKB_SYM_MAX_BYTES, else 30 % of the device memory
// (at least 8 GiB): 24 GB on one 80 GB H100, so a 1e6-node self-interaction (47 GB) takes the plain kernel on one GPU
// and the symmetric one from 2 GPUs on (1/P of that per rank with the row partition)
long long sym_mem_budget() {
    static long long cached = -1; // all devices of a box are alike; the environment is read once
    if (cached >= 0)
        return cached;
    if (const char *e = getenv("SKB_SYM_MAX_BYTES"))
        return cached = atoll(e);
    size_t free_b = 0, total_b = 0;
    if (cudaMemGetInfo(&free_b, &total_b) != cudaSuccess)
        return cached = 8LL << 30;
    return cached = std::max<long long>(8LL << 30, (long long)(0.30 * (double)total_b));
}
long long sym_block_nodes() { return (long long)kSymThreads * kSymT; }

// Block row I of the symmetric path's upper triangle belongs to part owner(I): serpentine assignment, so that every
// part gets the same number of long and short rows (one rank per GPU: each rank evaluates its rows, partial sums are
// all-reduced).
static int sym_row_owner(int I, int n_parts) {
    const int k = I / n_parts, m = I % n_parts;
    return (k & 1) ? n_parts - 1 - m : m;
}
static int sym_owned_rows(int nb, int part, int parts) {
    int n = 0;
    for (int I = 0; I < nb; ++I)
        n += sym_row_owner(I, parts) == part;
    return n;
}

// One row of work items: block I of the I side meets the J groups [g0, g0 + n_groups); its items write row prow of P.
struct ItemRow {
    int I, g0, n_groups, prow;
};

// The work items of one launch of the symmetric or the cross kernel: `rows` (in increasing I) cut into items (I, groups
// [g0, g1)), in units of 32-node groups.  Guided sizes: most of the work goes out in large items (about a quarter of a
// CTA slot's share each), the last ~30 % in items a quarter of that size and the last ~8 % in single stages (4 groups =
// 17 us of one CTA slot), so that all `slots` CTA slots drain together: the hardware hands the next item to whichever
// slot frees up first, in `order` (large items first).  item.slot is the item's row-major position,
// row_begin[b]..row_begin[b+1] the slots of block row b < n_blocks (their forward partials are summed in that order by
// the reduction kernel).
static void cut_items(const std::vector<ItemRow> &rows, int n_blocks, long long slots, std::vector<SymItem> &order,
                      std::vector<int> &row_begin) {
    const int sg = kSymStageGroups;
    long long work = 0;
    for (const ItemRow &r : rows)
        work += r.n_groups;
    long long big = work / std::max<long long>(1, slots * 4); // 4 large items per CTA slot (if all work were large items)
    big = std::max<long long>(sg, std::min<long long>(big / sg * sg, 1024LL * sg));
    const long long mid = std::max<long long>(sg, big / 4 / sg * sg);
    struct Piece {
        int I, g0, g1, prow;
    };
    std::vector<Piece> pieces;
    for (const ItemRow &r : rows) {
        const int len = r.n_groups;
        const int n_chunks = (int)((len + big - 1) / big);
        for (int c = 0; c < n_chunks; ++c) { // near-equal chunks, cut at stage boundaries
            const int a = (int)((long long)(len / sg) * c / n_chunks) * sg;
            const int b = c + 1 == n_chunks ? len : (int)((long long)(len / sg) * (c + 1) / n_chunks) * sg;
            if (b > a)
                pieces.push_back(Piece{r.I, r.g0 + a, r.g0 + b, r.prow});
        }
    }
    // the tail of the launch order is cut finer
    std::stable_sort(pieces.begin(), pieces.end(),
                     [](const Piece &x, const Piece &y) { return (x.g1 - x.g0) > (y.g1 - y.g0); });
    std::vector<Piece> fine;
    long long done = 0;
    // (at most ~6 items of a tier per CTA slot: more would only add forward-partial slabs)
    const long long fine_work = std::min<long long>(work * 8 / 100, slots * 6 * sg);
    const long long mid_work = std::min<long long>(work * 30 / 100, fine_work + slots * 6 * mid);
    for (const Piece &pc : pieces) {
        const long long len = pc.g1 - pc.g0;
        const long long left = work - done;
        const long long unit = left <= fine_work ? sg : left <= mid_work ? mid : len;
        for (long long g = pc.g0; g < pc.g1; g += unit)
            fine.push_back(Piece{pc.I, (int)g, (int)std::min<long long>(pc.g1, g + unit), pc.prow});
        done += len;
    }
    // slots: row-major
    std::sort(fine.begin(), fine.end(),
              [](const Piece &x, const Piece &y) { return x.I != y.I ? x.I < y.I : x.g0 < y.g0; });
    std::vector<SymItem> items(fine.size());
    row_begin.assign(n_blocks + 1, 0);
    for (size_t i = 0; i < fine.size(); ++i) {
        items[i] = SymItem{fine[i].I, fine[i].g0, fine[i].g1, (int)i, fine[i].prow, 0};
        row_begin[fine[i].I + 1] = (int)i + 1;
    }
    for (int b = 0; b < n_blocks; ++b) // rows without items inherit the running count
        row_begin[b + 1] = std::max(row_begin[b + 1], row_begin[b]);
    order = items;
    std::stable_sort(order.begin(), order.end(),
                     [](const SymItem &x, const SymItem &y) { return (x.g1 - x.g0) > (y.g1 - y.g0); });
}

// The rows of the symmetric kernel's items: the upper triangle of nb blocks INCLUDING the block diagonal (row I starts
// at its own first group), restricted to the block rows owned by `part`.  Every owned row has a P row, in increasing I
// (sym_reduce_kernel counts the same way).
static std::vector<ItemRow> sym_item_rows(int nb, int part, int parts) {
    const int gpb = kSymGroupsPerBlock;
    std::vector<ItemRow> rows;
    for (int I = 0; I < nb; ++I)
        if (sym_row_owner(I, parts) == part)
            rows.push_back(ItemRow{I, gpb * I, gpb * (nb - I), (int)rows.size()});
    return rows;
}

// Makes pl the plan of `rows` over n_blocks blocks of `block` nodes and `slots` CTA slots: the items in launch order,
// row_begin and one forward-partial slab (block x 3 doubles) per item, uploaded on st.  The caller has sized pl.P
// first: what a P that cannot be allocated means is its own decision.  Waits for every copy on st, so that host
// tables the caller uploaded before may go out of scope on return.
static int build_plan(ItemPlan &pl, const std::vector<ItemRow> &rows, int n_blocks, long long block, long long slots,
                      cudaStream_t st) {
    std::vector<SymItem> order;
    std::vector<int> row_begin;
    cut_items(rows, n_blocks, slots, order, row_begin);
    SKB_TRY(pl.items.ensure(order.size() * sizeof(SymItem) + 16));
    SKB_TRY(pl.row_begin.ensure(row_begin.size() * sizeof(int)));
    SKB_TRY(pl.F.ensure(order.size() * (size_t)block * 24 + 16));
    CUDA_TRY(cudaMemcpyAsync(pl.items.ptr, order.data(), order.size() * sizeof(SymItem), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(pl.row_begin.ptr, row_begin.data(), row_begin.size() * sizeof(int),
                             cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    pl.n_items = (int)order.size();
    pl.n_blocks = n_blocks;
    return SKB_OK;
}

int ensure_self_state(Evaluator &e, SourceSet &s, cudaStream_t st) {
    SymState &y = s.sym;
    if (y.self_state >= 0)
        return SKB_OK;
    if (e.n_trg < s.n || s.n <= 0) {
        y.self_state = 0;
        return SKB_OK;
    }
    SKB_TRY(y.flag.ensure(sizeof(int)));
    CUDA_TRY(cudaMemsetAsync(y.flag.ptr, 0, sizeof(int), st));
    const long long n3 = 3 * s.n;
    self_check_kernel<<<(unsigned)((n3 + 255) / 256), 256, 0, st>>>((const double *)e.r_trg.ptr, (const double *)s.r.ptr,
                                                                    n3, (int *)y.flag.ptr);
    CUDA_TRY(cudaGetLastError());
    count_launch(1);
    int differs = 1;
    CUDA_TRY(cudaMemcpyAsync(&differs, y.flag.ptr, sizeof(int), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    y.self_state = differs ? 0 : 1;
    return SKB_OK;
}

int sym_prepare(Evaluator &e, cudaStream_t st, int *use) {
    *use = 0;
    SourceSet &s = e.src[SKB_STOKESLET];
    SymState &y = s.sym;
    const long long block = sym_block_nodes();
    if (s.n < 4096 && e.sym_mode != 1)
        return SKB_OK; // too small to matter
    if (s.n < 2 * block || e.n_trg < s.n)
        return SKB_OK;
    const long long nb = s.n_pad / block; // n_pad is a multiple of 1024
    if ((long long)sym_owned_rows((int)nb, e.sym_part, e.sym_parts) * s.n_pad * 24 > sym_mem_budget())
        return SKB_OK;
    SKB_TRY(ensure_self_state(e, s, st));
    if (y.self_state != 1)
        return SKB_OK;
    const std::array<int, 3> key = {(int)nb, e.sym_part, e.sym_parts};
    if (y.key != key) {
        const std::vector<ItemRow> rows = sym_item_rows((int)nb, e.sym_part, e.sym_parts);
        const size_t p_bytes = rows.size() * (size_t)s.n_pad * 24;
        if (y.plan.P.ensure(p_bytes) != SKB_OK) { // not enough free memory for the reverse partials: the plain kernel
                                                  // serves this geometry
            (void)cudaGetLastError();
            if (e.layout == Evaluator::kShared) // every device holds ALL leading targets there and the caller reduce-scatters the
                                 // partial sums: a silent switch to the plain kernel would count them P times
                return set_error(SKB_ERR_ALLOC, "symmetric multi-device layout: no memory for the reverse partials "
                                                "(%zu bytes); free memory or skb_ctx_set_symmetric(ctx, 0)",
                                 p_bytes);
            y.self_state = 0;
            return SKB_OK;
        }
        std::vector<int> owned; // block rows of P's rows, for sym_reduce_kernel
        // pairs of one launch: every ordered pair of real nodes in (owned row I, any block J > I), both directions
        long long pairs = 0;
        for (const ItemRow &r : rows) {
            owned.push_back(r.I);
            const long long nI = std::max<long long>(0, std::min<long long>(s.n, (r.I + 1) * block) - r.I * block);
            const long long after = std::max<long long>(0, s.n - (r.I + 1) * block);
            pairs += 2 * nI * after + nI * nI; // both directions beyond the block + the block diagonal
        }
        SKB_TRY(y.row_ids.ensure(owned.size() * sizeof(int) + 16));
        CUDA_TRY(cudaMemcpyAsync(y.row_ids.ptr, owned.data(), owned.size() * sizeof(int), cudaMemcpyHostToDevice, st));
        SKB_TRY(build_plan(y.plan, rows, (int)nb, block, (long long)e.info.num_sms * kSymMinB, st)); // waits for owned
        y.n_owned = (int)owned.size();
        y.pairs = pairs;
        y.key = key;
    }
    *use = 1;
    return SKB_OK;
}

int sym_eval(Evaluator &ev, double *d_u_out, int accumulate, cudaStream_t st, double scale_mul, int *launches) {
    SourceSet &s = ev.src[SKB_STOKESLET];
    const SymState &y = s.sym;
    const SymArgs a{(const double *)s.r.ptr, s.f_cur, s.excl ? (const int *)s.excl_ids.ptr : nullptr,
                    (const SymItem *)y.plan.items.ptr, (double *)y.plan.P.ptr, (double *)y.plan.F.ptr, s.n_pad,
                    y.plan.n_blocks};
    cudaError_t e = cudaSuccess;
    if (y.plan.n_items > 0) {
        CUDA_TRY(cudaEventRecord(ev.ev_s0, st));
        constexpr int smem = SymSmem<kSymT>::total_bytes;
        if (s.excl)
            pair_sym_kernel<kSymT, kSymMinB, true><<<y.plan.n_items, kSymThreads, smem, st>>>(a);
        else
            pair_sym_kernel<kSymT, kSymMinB, false><<<y.plan.n_items, kSymThreads, smem, st>>>(a);
        e = cudaGetLastError();
        if (e == cudaSuccess)
            CUDA_TRY(cudaEventRecord(ev.ev_s1, st));
        ev.sym_timed = true;
        if (e != cudaSuccess)
            return set_error(SKB_ERR_CUDA, "pair_sym_kernel launch failed: %s", cudaGetErrorString(e));
        count_launch(1);
    }
    const long long n3 = 3 * s.n;
    const double scale = scale_mul / (8.0 * M_PI);
    sym_reduce_kernel<<<(unsigned)((n3 + 255) / 256), 256, 0, st>>>(
        (const double *)y.plan.P.ptr, (const double *)y.plan.F.ptr, (const int *)y.plan.row_begin.ptr,
        (const int *)y.row_ids.ptr, y.n_owned, (int)sym_block_nodes(), s.n_pad, n3, scale, accumulate, d_u_out);
    e = cudaGetLastError();
    if (e != cudaSuccess)
        return set_error(SKB_ERR_CUDA, "sym_reduce_kernel launch failed: %s", cudaGetErrorString(e));
    count_launch(1);
    if (launches)
        *launches += 2;
    return SKB_OK;
}

LaunchPlan sym_launch_plan(const SourceSet &s) { return LaunchPlan{kSymT, 1, 0, (unsigned)s.sym.plan.n_items}; }

int Evaluator::last_sym_kernel(double *ms, int64_t *pairs) const {
    if (!ms || !pairs)
        return set_error(SKB_ERR_INVALID, "skb_ctx_last_sym_kernel: NULL");
    *ms = 0;
    *pairs = 0;
    if (!sym_timed)
        return SKB_OK;
    float t = 0;
    cudaSetDevice(info.dev);
    if (cudaEventElapsedTime(&t, ev_s0, ev_s1) == cudaSuccess) {
        *ms = t;
        *pairs = src[SKB_STOKESLET].sym.pairs;
    } else {
        (void)cudaGetLastError(); // not finished yet
    }
    return SKB_OK;
}

int cross_eval(CrossState &cs, const DeviceInfo &di, const double *d_r_fib, const double *d_h, long long node0,
               long long n_rows, const double *d_r_sh, const double *d_s6, long long n_sh, long long n_sh_pad,
               double scale_dl, double scale_sl, double *d_u_fib, int acc_fib, double *d_u_shell, int acc_shell,
               cudaStream_t st, int *launches) {
    if (n_rows <= 0 || n_sh <= 0)
        return SKB_OK;
    const long long block = kCrossBlock;
    const std::array<long long, 5> key = {node0, n_rows, n_sh, n_sh_pad, di.num_sms};
    if (cs.key != key) {
        // items: rectangles (fiber block I, periphery groups [g0, g1)), every block meets every group
        const int n_blocks = (int)((n_rows + block - 1) / block);
        const int n_groups = (int)((n_sh + kSymGroup - 1) / kSymGroup);
        std::vector<ItemRow> rows;
        for (int I = 0; I < n_blocks; ++I)
            rows.push_back(ItemRow{I, 0, n_groups, I});
        SKB_TRY(cs.plan.P.ensure((size_t)n_blocks * (size_t)n_sh_pad * 24));
        SKB_TRY(build_plan(cs.plan, rows, n_blocks, block, (long long)di.num_sms * kCrossMinB, st));
        cs.key = key;
    }
    const ItemPlan &pl = cs.plan;
    const CrossArgs a{d_r_fib, d_h, d_r_sh, d_s6, (const SymItem *)pl.items.ptr, (double *)pl.P.ptr, (double *)pl.F.ptr,
                      n_sh_pad, node0, n_rows};
    pair_cross_kernel<kCrossT, kCrossMinB><<<pl.n_items, kSymThreads, CrossSmem<kCrossT>::total_bytes, st>>>(a);
    CUDA_TRY(cudaGetLastError());
    const long long nr3 = 3 * n_rows, ns3 = 3 * n_sh;
    cross_reduce_fib_kernel<<<(unsigned)((nr3 + 255) / 256), 256, 0, st>>>(
        (const double *)pl.F.ptr, (const int *)pl.row_begin.ptr, (int)block, nr3, scale_dl, acc_fib, d_u_fib);
    cross_reduce_shell_kernel<<<(unsigned)((ns3 + 255) / 256), 256, 0, st>>>((const double *)pl.P.ptr, pl.n_blocks,
                                                                              n_sh_pad, ns3, scale_sl, acc_shell,
                                                                              d_u_shell);
    CUDA_TRY(cudaGetLastError());
    count_launch(3);
    if (launches)
        *launches += 3;
    return SKB_OK;
}

} // namespace skb

using namespace skb;

extern "C" {

int skb_sym_plan_query(int n_blocks, int part, int n_parts, int num_sms, int max_items, int *items4, int *n_items,
                       int *row_begin) {
    if (n_blocks < 1 || n_parts < 1 || part < 0 || part >= n_parts || num_sms < 1 || !n_items)
        return set_error(SKB_ERR_INVALID, "skb_sym_plan_query: bad arguments");
    std::vector<SymItem> order;
    std::vector<int> rb;
    cut_items(sym_item_rows(n_blocks, part, n_parts), n_blocks, (long long)num_sms * kSymMinB, order, rb);
    *n_items = (int)order.size();
    if (items4)
        for (int i = 0; i < (int)order.size() && i < max_items; ++i) {
            items4[4 * i + 0] = order[i].I;
            items4[4 * i + 1] = order[i].g0;
            items4[4 * i + 2] = order[i].g1;
            items4[4 * i + 3] = order[i].slot;
        }
    if (row_begin)
        for (int b = 0; b <= n_blocks; ++b)
            row_begin[b] = rb[b];
    return SKB_OK;
}

int skb_sym_groups_per_block(void) { return kSymGroupsPerBlock; }

} // extern "C"
