# NeuralPDEB200Ext.jl -- attaches libpinn_b200.so (include/pinn_b200.h) to NeuralPDE.jl at the object `discretize`
# returns (src/discretize.jl:776-780): `B200PINN(PhysicsInformedNN(chain, strategy; ...); mode)` keeps the reference's
# parsing, theta layout and point-set construction (`symbolic_discretize` runs unchanged), lowers every generated loss
# function to the engine's residual IR once, and returns an `OptimizationProblem` whose objective and gradient are ONE
# fused kernel launch each.
#
# No Julia toolchain exists in the build image, so this file has not been executed there.  Its `lower_loss_function`
# pass is mirrored function by function by tests/julia_expr.py and tested against the Python lowering
# (tests/test_julia_lowering.py) on the generated functions of the BASELINE configurations.
module NeuralPDEB200Ext

using NeuralPDE, CUDA, ComponentArrays, SciMLBase, Optimization
import NeuralPDE: PhysicsInformedNN, AbstractPINN, PINNRepresentation, GridTraining, StochasticTraining,
    QuasiRandomTraining, QuadratureTraining, get_bounds, generate_training_sets

const lib = "libpinn_b200"

# ---- C mirrors of include/pinn_b200.h ----------------------------------------------------------------------------------
const PINN_ABI_VERSION = Cint(2)
const PINN_MAX_IN = 8
const PINN_F32, PINN_F64 = Cint(0), Cint(1)
const PINN_MODE_FFMA, PINN_MODE_TC_BF16, PINN_MODE_TC_SPLIT, PINN_MODE_TC_F64 = Cint(0), Cint(1), Cint(2), Cint(3)
const PINN_REDUCE_MEAN, PINN_REDUCE_WSUM = Cint(0), Cint(1)
const ACT = Dict(:identity => 0, :tanh => 1, :tanh_fast => 1, :sigmoid => 2, :sigmoid_fast => 2, :σ => 2, :sin => 3,
                 :softplus => 4, :swish => 5, :logcosh => 7, :cos => 8)
const OPC = Dict(:const => 0, :coord => 1, :tap => 2, :param => 3, :add => 4, :sub => 5, :mul => 6, :div => 7, :neg => 8,
                 :pow => 9, :powi => 10, :sin => 11, :cos => 12, :exp => 13, :log => 14, :tanh => 15, :sqrt => 16, :abs => 17)

struct PinnInstr
    op::Cint; a::Cint; b::Cint; _pad::Cint; imm::Cdouble
end
struct PinnNet
    n_layers::Cint; dims::Ptr{Cint}; acts::Ptr{Cint}; theta_offset::Int64
end
struct PinnTap
    net::Cint; out::Cint; order::Cint; dir::NTuple{4, Cint}
end
struct PinnTerm
    dim::Cint; n_taps::Cint; taps::Ptr{PinnTap}; net_rows::Ptr{Cint}; n_instr::Cint; prog::Ptr{PinnInstr}
    reduction::Cint; scale::Cdouble
end
struct PinnProblem
    abi_version::Cint; dtype::Cint; mode::Cint; device::Cint; n_nets::Cint; nets::Ptr{PinnNet}; n_terms::Cint
    terms::Ptr{PinnTerm}; n_params::Cint; param_offset::Int64; n_theta::Int64
end

check(rc) = rc == 0 || throw(ArgumentError(unsafe_string(@ccall lib.pinn_last_error()::Cstring)))

"""
    B200PINN(inner::PhysicsInformedNN; mode = :tc_split)

Sibling discretizer (extension rule: src/NeuralPDE.jl:64-71).  `mode`: `:ffma` (fp32 / fp64 parity path),
`:tc_bf16`, `:tc_split` (tensor-core paths, Float32 theta), `:tc_f64` (the parity path with its layer products on the
FP64 tensor cores, Float64 theta).
"""
struct B200PINN{P <: PhysicsInformedNN} <: AbstractPINN
    inner::P
    mode::Cint
end
B200PINN(inner::PhysicsInformedNN; mode::Symbol = :tc_split) =
    B200PINN(inner, Dict(:ffma => PINN_MODE_FFMA, :tc_bf16 => PINN_MODE_TC_BF16, :tc_split => PINN_MODE_TC_SPLIT,
                         :tc_f64 => PINN_MODE_TC_F64)[mode])

# ---- lowering: generated loss function (Expr) -> residual IR ---------------------------------------------------------------
# Grammar after _transform_expression (src/symbolic_utilities.jl:132-331) and _dot_ (:29-62):
#   u(cord_k, θ_k, phi_k)                                   -> tap of order 0                         (:150-159)
#   derivative(phi_k, u, cord_k, εs, order, θ_k)            -> tap; each ε vector is one-hot: its index is the direction (:185-201)
#   x  bound by  (x, y) = (cord[[1], :], cord[[2], :])      -> PINN_OP_COORD row                       (src/discretize.jl:126)
#   x  bound by  fill(v, size(cord[[1], :]))                -> constant (Quadrature boundary terms, get_indvars_ex)
#   a  bound by  (a,) = (θ.p[1:1],)                         -> PINN_OP_PARAM (param_estim)             (src/discretize.jl:83-95)
#   a  bound by  ArrayInterface.allowed_getindex(p, i)      -> constant default_p[i]                   (:97-109)
#   (+).(a, b, ...), sin.(x), a .- b, literals, π           -> arithmetic opcodes / constants
#   cord_k = vcat(x, y, ...)                                -> net_rows of network k                   (:111-116)
mutable struct Lowered
    taps::Vector{Tuple{Int, Int, Vector{Int}}}          # (net, order, dirs), 0-based
    prog::Vector{Tuple{Symbol, Int, Int, Float64}}
    net_rows::Dict{Int, Vector{Int}}
    dim::Int
    const_rows::Dict{Int, Float64}                      # rows upload_points! appends (constant boundary coordinates)
    memo::Dict{Any, Int}
end
Lowered() = Lowered([], [], Dict(), 0, Dict(), Dict())

function emit!(L::Lowered, op::Symbol, a = 0, b = 0, imm = 0.0)
    key = (op, a, b, Float64(imm))
    get!(L.memo, key) do
        push!(L.prog, key)
        length(L.prog) - 1
    end
end

function tap!(L::Lowered, net, order, dirs)
    key = (net, order, sort(collect(Int, dirs)))
    i = findfirst(==(key), L.taps)
    if i === nothing
        push!(L.taps, key)
        i = length(L.taps)
    end
    emit!(L, :tap, i - 1)
end

flatten_block(ex) = (ex isa Expr && ex.head === :block) ? reduce(vcat, map(flatten_block, filter(a -> !(a isa LineNumberNode), ex.args)); init = Any[]) : Any[ex]

const BINOP = Dict(:+ => :add, :- => :sub, :* => :mul, :/ => :div, :^ => :pow)
const UNOP = Dict(:sin => :sin, :cos => :cos, :exp => :exp, :log => :log, :tanh => :tanh, :sqrt => :sqrt, :abs => :abs)
undot(s::Symbol) = Symbol(lstrip(String(s), '.'))
fname(f) = f isa Symbol ? undot(f) : (f isa Function ? nameof(f) : nothing)

function net_of(arg, env)
    arg isa Symbol || return 0
    v = get(env, arg, nothing)
    v !== nothing && v[1] === :net && return v[2]
    m = match(r"(\d+)$", String(arg))
    m === nothing ? 0 : parse(Int, m.captures[1]) - 1
end

function bind_tuple!(env, lhs, rhs, depvars, default_p)
    for (l, r) in zip(lhs, rhs)
        if r isa Expr && r.head === :ref && r.args[1] === :cord                              # cord[[i], :]
            env[l] = (:coord, Int(r.args[2].args[1]) - 1)
        elseif r isa Expr && r.head === :call && fname(r.args[1]) === :fill                   # fill(v, size(...))
            env[l] = (:const, Float64(r.args[2]))
        elseif r isa Expr && r.head === :. && r.args[1] isa Expr && r.args[1].head === :. &&
               r.args[1].args[2] == QuoteNode(:depvar)                                        # θ.depvar.<name>
            env[l] = (:net, findfirst(==(r.args[2].value), depvars) - 1)
        elseif r isa Expr && r.head === :ref && r.args[1] === :phi                            # phi[i]
            env[l] = (:net, Int(r.args[2]) - 1)
        elseif r isa Expr && r.head === :ref && r.args[1] isa Expr && r.args[1].head === :. &&
               r.args[1].args[2] == QuoteNode(:p)                                             # θ.p[i:i]
            rng = r.args[2]
            env[l] = (:param, Int(rng isa UnitRange ? first(rng) : (rng isa Expr ? rng.args[2] : rng)) - 1)
        elseif r isa Expr && r.head === :call && r.args[1] isa Expr && r.args[1].head === :. &&
               r.args[1].args[2] == QuoteNode(:allowed_getindex)                              # default_p[i]
            env[l] = (:const, Float64(default_p[Int(r.args[3])]))
        else
            throw(ArgumentError("NeuralPDEB200Ext: unrecognised binding $l = $r"))
        end
    end
end

function lower_expr!(L::Lowered, ex, env)
    if ex isa Number
        return emit!(L, :const, 0, 0, Float64(ex))                                            # includes π (Irrational)
    elseif ex isa Symbol
        ex === :π && return emit!(L, :const, 0, 0, Float64(π))
        kind, val = env[ex]
        kind === :coord && return emit!(L, :coord, val)
        kind === :const && return emit!(L, :const, 0, 0, val)
        kind === :param && return emit!(L, :param, val)
        throw(ArgumentError("NeuralPDEB200Ext: symbol $ex cannot appear in an expression"))
    end
    ex isa Expr || throw(ArgumentError("NeuralPDEB200Ext: cannot lower $ex"))
    # integral(u, cord, phi, ids, integrand, lb, ub, θ): the integrand is a separate RuntimeGeneratedFunction this
    # lowering does not read; the engine's integral terms (pinn_create_ex) are reachable from the Python layer only
    ex.head === :call && ex.args[1] === :integral &&
        throw(ArgumentError("NeuralPDEB200Ext: equations with Integral terms are not lowered by this extension"))
    if ex.head === :call && ex.args[1] === :u                                                  # u(cord_k, θ_k, phi_k)
        return tap!(L, net_of(ex.args[2], env), 0, Int[])
    elseif ex.head === :call && ex.args[1] === :derivative                                     # derivative(phi_k, u, cord_k, εs, order, θ_k)
        cord, εs, order = ex.args[4], ex.args[5], Int(ex.args[6])
        dirs = [findfirst(!iszero, ε) - 1 for ε in εs]
        length(dirs) == order || throw(ArgumentError("NeuralPDEB200Ext: derivative order $order with $(length(dirs)) directions"))
        (order <= 2 || (order == 3 && allequal(dirs))) ||
            throw(ArgumentError("NeuralPDEB200Ext: the engine takes derivatives up to order 2 and pure third derivatives"))
        return tap!(L, net_of(cord, env), order, dirs)
    end
    f, args = if ex.head === :. && ex.args[2] isa Expr && ex.args[2].head === :tuple
        fname(ex.args[1]), ex.args[2].args                                                     # f.(args...)
    elseif ex.head === :call
        fname(ex.args[1]), ex.args[2:end]                                                      # a .- b  parses as call(:.-, a, b)
    else
        throw(ArgumentError("NeuralPDEB200Ext: expression outside the grammar of _transform_expression: $ex"))
    end
    if haskey(BINOP, f)
        length(args) == 1 && f === :- && return emit!(L, :neg, lower_expr!(L, args[1], env))
        f === :^ && args[2] isa Integer && return emit!(L, :powi, lower_expr!(L, args[1], env), 0, Float64(args[2]))
        acc = lower_expr!(L, args[1], env)
        for a in args[2:end]                                                                   # n-ary + and * fold to the left
            acc = emit!(L, BINOP[f], acc, lower_expr!(L, a, env))
        end
        return acc
    elseif haskey(UNOP, f)
        return emit!(L, UNOP[f], lower_expr!(L, args[1], env))
    end
    # a function registered with @register_symbolic (such as phi_bound(x, y) reading a trained network) is an opaque
    # Julia call here; the engine's fixed networks (pinn_create_ex2) are reachable from the Python layer only
    throw(ArgumentError("NeuralPDEB200Ext: function $f has no residual-IR opcode (functions registered with " *
                        "@register_symbolic, such as a trained network read by a neural adapter, are not lowered by " *
                        "this extension)"))
end

"""
    lower_loss_function(fn::Expr, depvars; default_p = nothing) -> Lowered

`fn` is what `build_symbolic_loss_function` returns: `:((cord, θ, phi, derivative, integral, u, p) -> begin ... end)`.
"""
function lower_loss_function(fn::Expr, depvars::Vector{Symbol}; default_p = nothing)
    fn.head === :-> || throw(ArgumentError("NeuralPDEB200Ext: expected the generated loss function"))
    L = Lowered()
    env = Dict{Symbol, Tuple{Symbol, Any}}()
    loss = nothing
    for st in flatten_block(fn.args[2])
        if st isa Expr && st.head === :(=) && st.args[1] isa Expr && st.args[1].head === :tuple
            bind_tuple!(env, st.args[1].args, st.args[2].args, depvars, default_p)
        elseif st isa Expr && st.head === :let
            b = st.args[1]
            lhs = b.args[1] isa Expr ? b.args[1].args : Any[b.args[1]]
            rhs = b.args[1] isa Expr ? b.args[2].args : Any[b.args[2]]
            bind_tuple!(env, lhs, rhs, depvars, default_p)
            n_coord = 1 + maximum([v[2] for v in values(env) if v[1] === :coord]; init = -1)
            for s2 in flatten_block(st.args[2])
                if s2 isa Expr && s2.head === :(=) && s2.args[1] isa Symbol && startswith(String(s2.args[1]), "cord")
                    k = parse(Int, String(s2.args[1])[5:end]) - 1                              # cord<k> = vcat(vars...)
                    rows = Int[]
                    for v in s2.args[2].args[2:end]
                        kind, val = env[v]
                        if kind === :const                                                     # constant bc coordinate: appended row
                            r = findfirst(==(val), L.const_rows)
                            if r === nothing
                                r = n_coord + length(L.const_rows)
                                L.const_rows[r] = val
                            end
                            push!(rows, r)
                        else
                            push!(rows, val)
                        end
                    end
                    L.net_rows[k] = rows
                    env[s2.args[1]] = (:net, k)
                else
                    loss = s2
                end
            end
        end
    end
    loss === nothing && throw(ArgumentError("NeuralPDEB200Ext: no loss expression in the generated function"))
    L.dim = 1 + maximum([v[2] for v in values(env) if v[1] === :coord]; init = -1) + length(L.const_rows)
    lower_expr!(L, loss, env)
    return L
end

# ---- descriptor assembly ----------------------------------------------------------------------------------------------------
struct Keep            # keeps the buffers the C descriptor points into alive
    bufs::Vector{Any}
end

chain_dims(chain) = vcat(Int[first(chain.layers).in_dims], Int[l.out_dims for l in chain.layers])
chain_acts(chain) = Int[ACT[nameof(l.activation)] for l in chain.layers]
n_chain_params(chain) = sum(l.in_dims * l.out_dims + l.out_dims for l in chain.layers)

function lower(pinnrep::PINNRepresentation, chains, mode::Cint)
    keep = Keep(Any[])
    T = eltype(pinnrep.flat_init_params)
    depvars = collect(Symbol, pinnrep.depvars)
    nets = PinnNet[]
    off = 0
    for c in chains
        dims = Cint.(chain_dims(c)); acts = Cint.(chain_acts(c))
        push!(keep.bufs, dims, acts)
        push!(nets, PinnNet(length(acts), pointer(dims), pointer(acts), off))
        off += n_chain_params(c)
    end
    n_p = pinnrep.param_estim ? length(pinnrep.eq_params) : 0
    quad = pinnrep.strategy isa QuadratureTraining
    lowered = Lowered[]
    terms = PinnTerm[]
    for fn in vcat(pinnrep.symbolic_pde_loss_functions, pinnrep.symbolic_bc_loss_functions)
        L = lower_loss_function(fn, depvars; default_p = pinnrep.default_p)
        taps = [PinnTap(t[1], 0, t[2], (Cint(get(t[3], 1, 0)), Cint(get(t[3], 2, 0)), Cint(get(t[3], 3, 0)), Cint(0))) for t in L.taps]
        rows = fill(Cint(-1), length(chains) * PINN_MAX_IN)
        for (k, r) in L.net_rows, (j, v) in enumerate(r)
            rows[k * PINN_MAX_IN + j] = v
        end
        prog = [PinnInstr(OPC[i[1]], i[2], i[3], 0, i[4]) for i in L.prog]
        push!(keep.bufs, taps, rows, prog)
        push!(terms, PinnTerm(L.dim, length(taps), pointer(taps), pointer(rows), length(prog), pointer(prog),
                              quad ? PINN_REDUCE_WSUM : PINN_REDUCE_MEAN, 1.0))        # quadrature scale 1/area set by upload_points!
        push!(lowered, L)
    end
    push!(keep.bufs, nets, terms)
    desc = PinnProblem(PINN_ABI_VERSION, T === Float64 ? PINN_F64 : PINN_F32, mode, Cint(CUDA.deviceid(CUDA.device())),
                       length(nets), pointer(nets), length(terms), pointer(terms), n_p, off, off + n_p)
    return desc, keep, lowered
end

# ---- point sets ----------------------------------------------------------------------------------------------------------------
# rows appended for constant boundary coordinates (Lowered.const_rows) so that every tapped network finds its inputs
function with_const_rows(pts::AbstractMatrix, L::Lowered)
    isempty(L.const_rows) && return pts
    extra = vcat([fill(eltype(pts)(L.const_rows[r]), 1, size(pts, 2)) for r in sort(collect(keys(L.const_rows)))]...)
    return vcat(pts, extra)
end

mutable struct Sets
    dev::Vector{Any}         # CuArrays aliased by the engine (kept alive here)
    bounds::Any              # Stochastic / QuasiRandom: per-term (lb, ub)
    npoints::Vector{Int}
end

function upload_points!(h, pinnrep::PINNRepresentation, lowered)
    strategy = pinnrep.strategy
    T = eltype(pinnrep.flat_init_params)
    n_pde = length(pinnrep.eqs)
    sets = Sets(Any[], nothing, Int[])
    if strategy isa GridTraining                                                       # src/training_strategies.jl:215-221
        pde_sets, bc_sets = generate_training_sets(pinnrep.domains, strategy.dx, pinnrep.eqs, pinnrep.bcs, T,
                                                   pinnrep.dict_indvars, pinnrep.dict_depvars)
        for (i, s) in enumerate(vcat(pde_sets, bc_sets))
            d = cu(with_const_rows(T.(s), lowered[i]))
            push!(sets.dev, d)
            check(@ccall lib.pinn_set_points(h::Ptr{Cvoid}, (i - 1)::Cint, pointer(d)::CuPtr{Cvoid}, size(d, 2)::Int64,
                                             CU_NULL::CuPtr{Cvoid})::Cint)
        end
    elseif strategy isa StochasticTraining                                             # :271-282: drawn on the device instead
        pb, bb = get_bounds(pinnrep.domains, pinnrep.eqs, pinnrep.bcs, T, pinnrep.dict_indvars, pinnrep.dict_depvars, strategy)
        sets.bounds = vcat(pb, bb)
        for (i, b) in enumerate(sets.bounds)
            n = i <= n_pde ? strategy.points : strategy.bcs_points
            lb, ub = Float64.(b[1]), Float64.(b[2])
            for r in sort(collect(keys(lowered[i].const_rows)))
                push!(lb, lowered[i].const_rows[r]); push!(ub, lowered[i].const_rows[r])
            end
            check(@ccall lib.pinn_set_sampler(h::Ptr{Cvoid}, (i - 1)::Cint, n::Int64, lb::Ptr{Cdouble}, ub::Ptr{Cdouble},
                                              UInt64(i)::UInt64, CUDA.stream().handle::Ptr{Cvoid})::Cint)
            push!(sets.npoints, n)
        end
    elseif strategy isa QuasiRandomTraining                                            # :365-389: host sequence, uploaded per call
        pb, bb = get_bounds(pinnrep.domains, pinnrep.eqs, pinnrep.bcs, T, pinnrep.dict_indvars, pinnrep.dict_depvars, strategy)
        sets.bounds = vcat(pb, bb)
        resample_host!(h, pinnrep, lowered, sets)
    else
        throw(ArgumentError("NeuralPDEB200Ext: $(typeof(strategy)) is served by the reference path (adaptive cubature is " *
                            "host control flow); use GridTraining, StochasticTraining or QuasiRandomTraining"))
    end
    return sets
end

function resample_host!(h, pinnrep, lowered, sets::Sets)
    strategy = pinnrep.strategy
    T = eltype(pinnrep.flat_init_params)
    n_pde = length(pinnrep.eqs)
    for (i, b) in enumerate(sets.bounds)
        n = i <= n_pde ? strategy.points : strategy.bcs_points
        pts = with_const_rows(T.(NeuralPDE.generate_quasi_random_points(n, b, T, strategy.sampling_alg)), lowered[i])
        check(@ccall lib.pinn_set_points_host(h::Ptr{Cvoid}, (i - 1)::Cint, pts::Ptr{Cvoid}, size(pts, 2)::Int64,
                                              C_NULL::Ptr{Cvoid}, CUDA.stream().handle::Ptr{Cvoid})::Cint)
    end
end

# fresh points before an evaluation, as the reference's get_loss_function closures do on every call
function resample!(h, pinnrep, lowered, sets::Sets, first_call::Ref{Bool})
    strategy = pinnrep.strategy
    if strategy isa StochasticTraining
        first_call[] || check(@ccall lib.pinn_resample(h::Ptr{Cvoid}, CUDA.stream().handle::Ptr{Cvoid})::Cint)
    elseif strategy isa QuasiRandomTraining && strategy.resampling
        first_call[] || resample_host!(h, pinnrep, lowered, sets)
    end
    first_call[] = false
end

# ---- side effects the reference keeps outside the gradient (src/discretize.jl:574-645) --------------------------------------
function side_effects!(pinnrep::PINNRepresentation, reweight!, pde_losses, bc_losses, θ)
    pinnrep.iteration isa Ref || return                       # user-maintained counters stay the user's
    pinnrep.iteration[] += 1                                  # :574-576 (self_increment)
    reweight!(θ, pde_losses, bc_losses)                       # :578-580, generate_adaptive_loss_function(...)
    return
end

function log_terms(pinnrep, pde_losses, bc_losses, total)
    it = pinnrep.iteration[]
    it % pinnrep.log_options.log_frequency == 0 || return
    lg = pinnrep.logger
    NeuralPDE.logvector(lg, pde_losses, "unweighted_loss/pde_losses", it)
    NeuralPDE.logvector(lg, bc_losses, "unweighted_loss/bc_losses", it)
    NeuralPDE.logvector(lg, pinnrep.adaloss.pde_loss_weights .* pde_losses, "weighted_loss/weighted_pde_losses", it)
    NeuralPDE.logvector(lg, pinnrep.adaloss.bc_loss_weights .* bc_losses, "weighted_loss/weighted_bc_losses", it)
    NeuralPDE.logscalar(lg, total, "weighted_loss/full_weighted_loss", it)
    NeuralPDE.logvector(lg, pinnrep.adaloss.pde_loss_weights, "adaptive_loss/pde_loss_weights", it)
    NeuralPDE.logvector(lg, pinnrep.adaloss.bc_loss_weights, "adaptive_loss/bc_loss_weights", it)
end

# ---- discretize ---------------------------------------------------------------------------------------------------------------------
function SciMLBase.discretize(sys::NeuralPDE.PDESystem, d::B200PINN)
    pinnrep = SciMLBase.symbolic_discretize(sys, d.inner)            # reference code, unchanged
    chains = d.inner.chain isa AbstractVector ? d.inner.chain : [d.inner.chain]
    desc, keep, lowered = lower(pinnrep, chains, d.mode)
    h = Ref{Ptr{Cvoid}}(C_NULL)
    GC.@preserve keep check(@ccall lib.pinn_create(Ref(desc)::Ptr{PinnProblem}, h::Ptr{Ptr{Cvoid}})::Cint)
    sets = upload_points!(h[], pinnrep, lowered)
    T = eltype(pinnrep.flat_init_params)
    n_pde, n_bc = length(pinnrep.eqs), length(pinnrep.bcs)
    θ0 = cu(collect(T, pinnrep.flat_init_params))
    terms = CUDA.zeros(T, n_pde + n_bc); total = CUDA.zeros(T, 1)
    adaloss = pinnrep.adaloss
    reweight! = NeuralPDE.generate_adaptive_loss_function(pinnrep, adaloss, pinnrep.loss_functions.pde_loss_functions,
                                                          pinnrep.loss_functions.bc_loss_functions)
    weights() = Float64[adaloss.pde_loss_weights; adaloss.bc_loss_weights]            # src/discretize.jl:553-559
    first_call = Ref(true)

    function evaluate!(G, θ)
        resample!(h[], pinnrep, lowered, sets, first_call)
        st = CUDA.stream().handle
        gptr = G === nothing ? CU_NULL : pointer(G)
        call!(g) = check(@ccall lib.pinn_loss_grad(h[]::Ptr{Cvoid}, pointer(θ)::CuPtr{Cvoid}, weights()::Ptr{Cdouble},
                                                   g::CuPtr{Cvoid}, pointer(terms)::CuPtr{Cvoid}, pointer(total)::CuPtr{Cvoid},
                                                   st::Ptr{Cvoid})::Cint)
        it_next = pinnrep.iteration isa Ref ? pinnrep.iteration[] + 1 : 0
        reweights = hasproperty(adaloss, :reweight_every) && it_next % adaloss.reweight_every == 0
        if reweights
            # :567-598 forms the weighted sum AFTER the reweighting: term losses first (loss-only launch), then the step
            call!(CU_NULL)
            tl = Array(terms)
            side_effects!(pinnrep, reweight!, tl[1:n_pde], tl[(n_pde + 1):end], θ)
            call!(gptr)
        else
            call!(gptr)
            tl = Array(terms)
            side_effects!(pinnrep, reweight!, tl[1:n_pde], tl[(n_pde + 1):end], θ)
        end
        L = Array(total)[1]
        pinnrep.iteration isa Ref && log_terms(pinnrep, tl[1:n_pde], tl[(n_pde + 1):end], L)
        return L
    end
    f(θ, p) = evaluate!(nothing, θ)
    g!(G, θ, p) = (evaluate!(G, θ); G)
    finalizer(_ -> (@ccall lib.pinn_destroy(h[]::Ptr{Cvoid})::Cint; nothing), h)
    return OptimizationProblem(OptimizationFunction(f; grad = g!), θ0)
end

end # module
