// skb_periphery.cu -- the periphery's shape of a flow (include/skelly_b200_flow.h, skb_flow_set_periphery_shape):
// the fiber-periphery repulsion, the plus-end binding and the collision test on the device (periphery_kernels.cuh),
// which the step (skb_step.cu) runs before its fiber build and after its install.
#include "periphery_kernels.cuh"
#include "skb_flow.hpp"

#include <cmath>
#include <cstring>

using namespace skb;

static int load_periphery_kernels() {
    cudaFuncAttributes fa; // loaded now: a group step must not load a kernel lazily while its peers wait on a flag
    CUDA_TRY(cudaFuncGetAttributes(&fa, periphery_kernel));
    CUDA_TRY(cudaFuncGetAttributes(&fa, periphery_add_kernel));
    return SKB_OK;
}

static int shape_args(const char *who, const skb_periphery_shape *s, const int *minus_clamped,
                      const double *body_radius, int n_fibers, int n_bodies, long long n_shell) {
    if (!s)
        return set_error(SKB_ERR_INVALID, "%s: NULL shape", who);
    if (s->kind < SKB_PERIPHERY_NONE || s->kind > SKB_PERIPHERY_ELLIPSOID)
        return set_error(SKB_ERR_INVALID, "%s: kind = %d (must be SKB_PERIPHERY_NONE, _SPHERE or _ELLIPSOID)", who,
                         s->kind);
    if (s->kind == SKB_PERIPHERY_NONE)
        return SKB_OK;
    const double v[8] = {s->a, s->b, s->c, s->f_0, s->l_0, s->polar_angle_start, s->polar_angle_end,
                         s->binding_threshold};
    for (double x : v)
        if (!std::isfinite(x))
            return set_error(SKB_ERR_INVALID, "%s: a non-finite shape parameter", who);
    if (!(s->a > 0) || (s->kind == SKB_PERIPHERY_ELLIPSOID && (!(s->b > 0) || !(s->c > 0))))
        return set_error(SKB_ERR_INVALID, "%s: semi-axes (%g, %g, %g) must be > 0 for the shape in use", who, s->a,
                         s->b, s->c);
    if (!(s->l_0 > 0))
        return set_error(SKB_ERR_INVALID, "%s: l_0 = %g (must be > 0)", who, s->l_0);
    if (s->binding_active != 0 && s->binding_active != 1)
        return set_error(SKB_ERR_INVALID, "%s: binding_active = %d (must be 0 or 1)", who, s->binding_active);
    for (int f = 0; minus_clamped && f < n_fibers; ++f)
        if (minus_clamped[f] != 0 && minus_clamped[f] != 1)
            return set_error(SKB_ERR_INVALID, "%s: fiber_minus_clamped[%d] = %d (must be 0 or 1)", who, f,
                             minus_clamped[f]);
    for (int b = 0; body_radius && b < n_bodies; ++b)
        if (!(body_radius[b] >= 0) || !std::isfinite(body_radius[b]))
            return set_error(SKB_ERR_INVALID, "%s: body_radius[%d] = %g (must be finite and >= 0)", who, b,
                             body_radius[b]);
    if (n_shell == 0)
        return set_error(SKB_ERR_INVALID, "%s: the flow has no periphery nodes (skb_flow_set_periphery)", who);
    return SKB_OK;
}

int PeripheryShape::set(const skb_periphery_shape *shape, const int *minus_clamped, const double *body_radius,
                        int n_fibers, long long n_fib, int n_bodies, long long n_shell, cudaStream_t st) {
    const char *who = "skb_flow_set_periphery_shape";
    SKB_TRY(shape_args(who, shape, minus_clamped, body_radius, n_fibers, n_bodies, n_shell));
    active_ = false;
    if (shape->kind == SKB_PERIPHERY_NONE)
        return SKB_OK;
    SKB_TRY(load_periphery_kernels());
    std::vector<int> skip((size_t)n_fibers, 0);
    if (minus_clamped)
        std::memcpy(skip.data(), minus_clamped, (size_t)n_fibers * sizeof(int));
    std::vector<double> radius((size_t)n_bodies, 0.0);
    if (body_radius)
        std::memcpy(radius.data(), body_radius, (size_t)n_bodies * 8);
    SKB_TRY(force_skip_.ensure((size_t)n_fibers * sizeof(int) + 8));
    SKB_TRY(collide_skip_.ensure((size_t)n_fibers * sizeof(int) + 8));
    SKB_TRY(radius_.ensure((size_t)n_bodies * 8 + 8));
    if (n_fibers > 0)
        CUDA_TRY(cudaMemcpyAsync(force_skip_.ptr, skip.data(), skip.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    if (n_bodies > 0)
        CUDA_TRY(cudaMemcpyAsync(radius_.ptr, radius.data(), radius.size() * 8, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaStreamSynchronize(st)); // (the host copies above go out of scope)
    h_clamped_ = skip;
    h_force_skip_ = skip;
    n_fibers_ = n_fibers;
    n_bodies_ = n_bodies;
    s_ = *shape;
    active_ = true;
    cap_nodes_ = -1;
    return size(n_fib);
}

int PeripheryShape::size(long long n_fib) {
    if (!active_)
        return SKB_OK;
    const long long cap = cap_nodes_;
    cap_nodes_ = -1; // a failed allocation leaves the buffers unsized
    const long long nodes = n_fib > cap ? n_fib : cap;
    SKB_TRY(force_.ensure((size_t)nodes * 24 + 8));
    SKB_TRY(flags_.ensure(((size_t)n_fibers_ + 1) * sizeof(int)));
    const size_t n_flags = (size_t)n_fibers_ + 1;
    if (n_flags > flag_cap_) {
        h_flags_.reset();
        flag_cap_ = 0;
        CUDA_TRY(cudaMallocHost((void **)h_flags_.out(), n_flags * sizeof(int)));
        flag_cap_ = n_flags;
    }
    cap_nodes_ = nodes;
    return SKB_OK;
}

void PeripheryShape::note_clamped(int f0, int nf, const skb_fiber_params *params) {
    for (int f = 0; active_ && params && f < nf && f0 + f < n_fibers_; ++f)
        h_clamped_[(size_t)(f0 + f)] = params[f].minus_clamped;
}

void PeripheryShape::note_clamped_all(const std::vector<double> &flags) {
    for (size_t f = 0; active_ && f < flags.size() && f < h_clamped_.size(); ++f)
        h_clamped_[f] = flags[f] != 0.0 ? 1 : 0;
}

int PeripheryShape::carry(const int *origin, int n_old, int n_fibers, long long n_fib, cudaStream_t st) {
    if (!active_ || n_old != n_fibers_)
        return SKB_OK;
    std::vector<int> skip((size_t)n_fibers, 0), clamped((size_t)n_fibers, 0);
    for (int f = 0; f < n_fibers; ++f)
        if (origin[f] >= 0) {
            skip[(size_t)f] = h_force_skip_[(size_t)origin[f]];
            clamped[(size_t)f] = h_clamped_[(size_t)origin[f]];
        }
    SKB_TRY(force_skip_.ensure((size_t)n_fibers * sizeof(int) + 8));
    SKB_TRY(collide_skip_.ensure((size_t)n_fibers * sizeof(int) + 8));
    if (n_fibers > 0)
        CUDA_TRY(cudaMemcpyAsync(force_skip_.ptr, skip.data(), skip.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaStreamSynchronize(st)); // (the host copy above goes out of scope)
    h_force_skip_ = std::move(skip);
    h_clamped_ = std::move(clamped);
    n_fibers_ = n_fibers;
    return size(n_fib);
}

int PeripheryShape::upload_clamped(int f0, int nf, const skb_fiber_params *params, cudaStream_t st) {
    if (nf <= 0)
        return SKB_OK;
    std::vector<int> flags((size_t)nf);
    for (int f = 0; f < nf; ++f)
        flags[(size_t)f] = params[f].minus_clamped;
    // (from pageable memory: staged before the call returns, so the vector may go)
    CUDA_TRY(cudaMemcpyAsync((int *)collide_skip_.ptr + f0, flags.data(), (size_t)nf * sizeof(int),
                             cudaMemcpyHostToDevice, st));
    return SKB_OK;
}

// an error naming `who` unless the shape's tables and buffers fit the flow as it is
static int shape_fits(const skb_flow *fl, const char *who) {
    const PeripheryShape &P = fl->shape;
    if (!P.counts_fit(fl->n_fibers, fl->n_bodies))
        return set_error(SKB_ERR_INVALID, "%s: the number of fibers or bodies changed since "
                                          "skb_flow_set_periphery_shape (call it again with the new arrays)", who);
    if (!P.nodes_fit(fl->n_fib))
        return set_error(SKB_ERR_INVALID, "%s: the fibers' nodes outgrew the periphery's buffers (call skb_flow_set_gmres "
                                          "or skb_flow_set_periphery_shape)", who);
    return SKB_OK;
}

int PeripheryShape::run(const double *d_r_fib, const long long *d_off, int f0, int f1, bool with_force,
                        const double *d_centers, int n_bodies, cudaStream_t st, int *launches) {
    const int nf = f1 - f0;
    if (n_fibers_ > 0)
        CUDA_TRY(cudaMemcpyAsync(collide_skip_.ptr, h_clamped_.data(), (size_t)n_fibers_ * sizeof(int),
                                 cudaMemcpyHostToDevice, st));
    const PeriShape s{s_.kind, s_.binding_active, s_.a, s_.b, s_.c, s_.f_0, s_.l_0, s_.polar_angle_start,
                      s_.polar_angle_end, s_.binding_threshold};
    periphery_kernel<<<nf + 1, kPeriThreads, 0, st>>>(
        s, d_r_fib, d_off, f0, (const int *)force_skip_.ptr, (const int *)collide_skip_.ptr,
        with_force ? (double *)force_.ptr : nullptr, d_centers, (const double *)radius_.ptr,
        d_centers ? n_bodies : 0, (int *)flags_.ptr);
    CUDA_TRY(cudaGetLastError());
    count_launch(1);
    *launches += 1;
    CUDA_TRY(cudaMemcpyAsync(h_flags_.get(), flags_.ptr, ((size_t)nf + 1) * sizeof(int), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return SKB_OK;
}

int PeripheryShape::add_force(const double *d_in, double *d_out, long long n, cudaStream_t st, int *launches) const {
    if (n == 0)
        return SKB_OK;
    const long long blocks = (n + 255) / 256;
    periphery_add_kernel<<<(unsigned)(blocks < 1024 ? blocks : 1024), 256, 0, st>>>(d_in, (const double *)force_.ptr,
                                                                                   d_out, n);
    CUDA_TRY(cudaGetLastError());
    count_launch(1);
    *launches += 1;
    return SKB_OK;
}

// ---- what the step runs (skb_step.cu) --------------------------------------------------------------------------------
int skb::periphery_before_step(skb_flow *fl, const char *who, const StepArgs &a, StepCall &c) {
    PeripheryShape &P = fl->shape;
    c.hinged.clear();
    if (!P.active())
        return SKB_OK;
    SKB_TRY(shape_fits(fl, who));
    const int nf = c.own.count();
    if (nf == 0)
        return SKB_OK;
    int launches = 0;
    SKB_TRY(P.run((const double *)fl->r_fib.ptr, (const long long *)fl->fiber_offset.ptr, c.own.f0, c.own.f1, true,
                  nullptr, 0, fl->stream, &launches));
    c.hinged.assign(a.params, a.params + nf);
    for (int f = 0; f < nf; ++f) {
        if (P.flags()[f] & kPeriNonFinite)
            return set_error(SKB_ERR_INVALID, "%s: a non-finite fiber-periphery force on fiber %d (a node at the "
                                              "centre of the sphere)", who, c.own.f0 + f);
        c.hinged[(size_t)f].plus_hinged = (P.flags()[f] & kPeriHinged) ? 1 : 0;
    }
    return SKB_OK;
}

int skb::periphery_ready(const skb_flow *fl, const char *who) {
    if (!fl->shape.active())
        return set_error(SKB_ERR_INVALID, "%s: periphery_interaction needs skb_flow_set_periphery_shape", who);
    return shape_fits(fl, who);
}

int skb::periphery_add_repulsion(skb_flow *fl, const char *who, double *d_ff, cudaStream_t st, int *launches) {
    PeripheryShape &P = fl->shape;
    SKB_TRY(P.run((const double *)fl->r_fib.ptr, (const long long *)fl->fiber_offset.ptr, 0, fl->n_fibers, true,
                  nullptr, 0, st, launches));
    for (int f = 0; f < fl->n_fibers; ++f)
        if (P.flags()[f] & kPeriNonFinite)
            return set_error(SKB_ERR_INVALID, "%s: a non-finite fiber-periphery force on fiber %d (a node at the "
                                              "centre of the sphere)", who, f);
    return P.add_force(d_ff, d_ff, 3 * fl->n_fib, st, launches);
}

int skb::periphery_add_force(skb_flow *fl, const double *d_f_external, long long m, double *d_out, cudaStream_t st,
                             int *launches) {
    return fl->shape.add_force(d_f_external, d_out, 3 * m, st, launches);
}

int skb::periphery_collided(skb_flow *fl, int *collided, cudaStream_t st, int *launches) {
    PeripheryShape &P = fl->shape;
    *collided = 0;
    if (!P.active())
        return SKB_OK;
    SKB_TRY(P.run((const double *)fl->r_fib.ptr, (const long long *)fl->fiber_offset.ptr, 0, fl->n_fibers, false,
                  fl->n_bodies > 0 ? (const double *)fl->centers.ptr : nullptr, fl->n_bodies, st, launches));
    for (int f = 0; f <= fl->n_fibers; ++f)
        *collided |= (P.flags()[f] & kPeriCollided) ? 1 : 0;
    return SKB_OK;
}

extern "C" {

int skb_flow_set_periphery_shape(skb_flow *fl, const skb_periphery_shape *shape, const int32_t *fiber_minus_clamped,
                                 const double *body_radius) {
    if (!fl)
        return set_error(SKB_ERR_INVALID, "skb_flow_set_periphery_shape: NULL flow");
    CUDA_TRY(cudaSetDevice(fl->dev));
    return fl->shape.set(shape, fiber_minus_clamped, body_radius, fl->n_fibers, fl->n_fib, fl->n_bodies, fl->n_shell,
                         fl->stream);
}

int skb_flow_periphery_interaction(skb_flow *fl, double *f_periphery, int32_t *plus_hinged, int32_t *collided) {
    const char *who = "skb_flow_periphery_interaction";
    if (!fl)
        return set_error(SKB_ERR_INVALID, "%s: NULL flow", who);
    PeripheryShape &P = fl->shape;
    if (!P.active())
        return set_error(SKB_ERR_INVALID, "%s: no periphery shape (skb_flow_set_periphery_shape)", who);
    SKB_TRY(shape_fits(fl, who));
    CUDA_TRY(cudaSetDevice(fl->dev));
    OwnFibers own;
    SKB_TRY(own_fibers(fl, who, own));
    const cudaStream_t st = fl->stream;
    int launches = 0;
    if (f_periphery || plus_hinged) { // the own fibers
        SKB_TRY(P.run((const double *)fl->r_fib.ptr, (const long long *)fl->fiber_offset.ptr, own.f0, own.f1, true,
                      nullptr, 0, st, &launches));
        for (int f = 0; plus_hinged && f < own.count(); ++f)
            plus_hinged[f] = (P.flags()[f] & kPeriHinged) ? 1 : 0;
        if (f_periphery && own.nodes() > 0) {
            CUDA_TRY(cudaMemcpyAsync(f_periphery, P.force(), (size_t)own.nodes() * 24, cudaMemcpyDefault, st));
            CUDA_TRY(cudaStreamSynchronize(st));
        }
    }
    if (collided) {
        int hit = 0;
        SKB_TRY(periphery_collided(fl, &hit, st, &launches));
        *collided = hit;
    }
    fl->launches = launches;
    return SKB_OK;
}

} // extern "C"
