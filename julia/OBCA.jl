# julia/OBCA.jl -- drop-in replacements for the reference's NLP drivers, Julia >= 1.6.
#
# UNTESTED IN THIS REPOSITORY'S CI: the build image has no Julia.  The file documents the binding a maintainer of
# XiaojingGeorgeZhang/OBCA adds to switch `main.jl` to libobca.so: `include("OBCA.jl")` INSTEAD OF
# include("ParkingSignedDist.jl"), include("ParkingDist.jl"), include("DualMultWS.jl"), include("ParkingConstraints.jl")
# (AutonomousParking/setup.jl:44-47).  Names, argument order and return tuples are those of
#   ParkingSignedDist.jl:29/:313, ParkingDist.jl:29/:313, DualMultWS.jl:29/:86, ParkingConstraints.jl:29/:143-147.
# `using JuMP, Ipopt` is no longer needed for these four functions.

const LIBOBCA = get(ENV, "LIBOBCA", joinpath(@__DIR__, "..", "obca_b200", "libobca.so"))

# mirror of `struct obca_opts` (include/obca.h)
mutable struct ObcaOpts
    tol::Cdouble; max_iter::Cint; mu_init::Cdouble; mu_min::Cdouble
    kappa_eps::Cdouble; kappa_mu::Cdouble; theta_mu::Cdouble; tau_min::Cdouble
    kappa1::Cdouble; kappa2::Cdouble; kappa_sigma::Cdouble; s_max::Cdouble
    dual_inf_tol::Cdouble; constr_viol_tol::Cdouble; compl_inf_tol::Cdouble
    dw_min::Cdouble; dw_first::Cdouble; dw_max::Cdouble; kw_minus::Cdouble; kw_plus::Cdouble; kw_plus_first::Cdouble
    gamma_theta::Cdouble; gamma_phi::Cdouble; delta::Cdouble; s_theta::Cdouble; s_phi::Cdouble; eta_phi::Cdouble
    gamma_alpha::Cdouble; max_backtrack::Cint; dc::Cdouble; max_kick::Cint; quad_dual_ws::Cint
    device::Cint; retry::Cint; q4::Cint
    ObcaOpts() = new()
end

function obca_default_opts()
    o = ObcaOpts()
    ccall((:obca_default_opts, LIBOBCA), Cvoid, (Ref{ObcaOpts},), o)
    return o
end

_f64(a) = Array{Float64}(a)

function _parking(signed_dist::Int, x0, xF, N, Ts, L, ego, XYbounds, nOb, vOb, A, b, rx, ry, ryaw, fixTime, xWS, uWS)
    N = Int(N); nOb = Int(nOb)
    v = Cint.(vec(collect(vOb))); V = Int(sum(v))
    Aj = _f64(A); bj = vec(_f64(b))                      # A: sum(vOb) x 2 column-major, b: sum(vOb)   (obstHrep.jl:39-40)
    xw = _f64(xWS)[1:N+1, 1:4]                           # setvalue(x, xWS')        ParkingSignedDist.jl:216
    uw = _f64(uWS)[1:N, 1:2]                             # setvalue(u, uWS[1:N,:]') ParkingSignedDist.jl:217
    xp = Matrix{Float64}(undef, 4, N + 1); up = Matrix{Float64}(undef, 2, N); ts = Vector{Float64}(undef, N + 1)
    lp = Matrix{Float64}(undef, V, N + 1); np = Matrix{Float64}(undef, 4nOb, N + 1); sl = Matrix{Float64}(undef, nOb, N + 1)
    exitflag = Ref{Cint}(0); iters = Ref{Cint}(0); kkt = Ref{Cdouble}(0.0); secs = Ref{Cdouble}(0.0)
    o = obca_default_opts()
    rc = ccall((:obca_parking_solve_batch, LIBOBCA), Cint,
               (Cint, Cint, Cint, Ptr{Cint}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Cdouble, Cdouble,
                Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble},
                Ptr{Cdouble}, Ptr{Cdouble}, Cint, Cint, Ref{ObcaOpts},
                Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble},
                Ref{Cint}, Ref{Cint}, Ref{Cdouble}, Ref{Cdouble}),
               1, N, nOb, v, Aj, bj, vec(_f64(x0)), vec(_f64(xF)), Float64(Ts), Float64(L),
               vec(_f64(ego)), vec(_f64(XYbounds)), vec(_f64(rx)), vec(_f64(ry)), vec(_f64(ryaw)), xw, uw,
               C_NULL, C_NULL,                            # library runs DualMultWS itself (ParkingSignedDist.jl:219)
               Int(fixTime), signed_dist, o, xp, up, ts, lp, np, sl, exitflag, iters, kkt, secs)
    if rc != 0                                            # the reference never throws: failure == exitflag 0
        println("libobca error ", rc, ": ", unsafe_string(ccall((:obca_last_error, LIBOBCA), Cstring, ())))
        return xp, up, ones(1, N + 1), 0, 0.0, lp, np
    end
    timeScalep = fixTime == 1 ? ones(1, N + 1) : ts       # ParkingSignedDist.jl:304-308
    return xp, up, timeScalep, Int(exitflag[]), secs[], lp, np
end

ParkingSignedDist(x0, xF, N, Ts, L, ego, XYbounds, nOb, vOb, A, b, rx, ry, ryaw, fixTime, xWS, uWS) =
    _parking(1, x0, xF, N, Ts, L, ego, XYbounds, nOb, vOb, A, b, rx, ry, ryaw, fixTime, xWS, uWS)

ParkingDist(x0, xF, N, Ts, L, ego, XYbounds, nOb, vOb, A, b, rx, ry, ryaw, fixTime, xWS, uWS) =
    _parking(0, x0, xF, N, Ts, L, ego, XYbounds, nOb, vOb, A, b, rx, ry, ryaw, fixTime, xWS, uWS)

# DualMultWS.jl:29 -- reads the GLOBAL `ego` like the reference does (DualMultWS.jl:39)
function DualMultWS(N, nOb, vOb, A, b, rx, ry, ryaw)
    N = Int(N); nOb = Int(nOb)
    v = Cint.(vec(collect(vOb))); V = Int(sum(v))
    lp = Matrix{Float64}(undef, N + 1, V); np = Matrix{Float64}(undef, N + 1, 4nOb)   # already transposed (:81-84)
    o = obca_default_opts()
    rc = ccall((:obca_dualmultws_batch, LIBOBCA), Cint,
               (Cint, Cint, Cint, Ptr{Cint}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble},
                Ptr{Cdouble}, Ref{ObcaOpts}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}),
               1, N, nOb, v, _f64(A), vec(_f64(b)), vec(_f64(ego)), vec(_f64(rx)), vec(_f64(ry)), vec(_f64(ryaw)),
               o, lp, np, C_NULL)
    rc != 0 && println("libobca error ", rc)
    return lp, np
end

function ParkingConstraints(x0, xF, N, Ts, L, ego, XYbounds, nOb, vOb, A, b, x, u, l, n, timeScale, fixTime, sd)
    N = Int(N); nOb = Int(nOb)
    v = Cint.(vec(collect(vOb)))
    feas = Ref{Cint}(0)
    o = obca_default_opts()
    rc = ccall((:obca_check_parking, LIBOBCA), Cint,
               (Cint, Cint, Cint, Ptr{Cint}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Cdouble, Cdouble,
                Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble},
                Ptr{Cdouble}, Cint, Cint, Ref{ObcaOpts}, Ref{Cint}, Ptr{Cint}, Ptr{Cint}),
               1, N, nOb, v, _f64(A), vec(_f64(b)), vec(_f64(x0)), vec(_f64(xF)), Float64(Ts), Float64(L),
               vec(_f64(ego)), vec(_f64(XYbounds)), _f64(x), _f64(u), _f64(l), _f64(n), vec(_f64(timeScale)), C_NULL,
               Int(fixTime), Int(sd), o, feas, C_NULL, C_NULL)
    return rc == 0 ? Int(feas[]) : 0
end

# ---- quadcopter (QuadcopterNavigation/setupQuadcopter.jl:33-34 includes QuadcopterSignedDist.jl / QuadcopterDist.jl /
#      constrSatisfaction.jl; include this file instead) ----
function _quadcopter(signed_dist::Int, x0, xF, N, Ts, R, ob1, ob2, ob3, ob4, ob5, xWS, uWS, timeWS)
    N = Int(N)
    ob = hcat(vec(_f64(ob1)), vec(_f64(ob2)), vec(_f64(ob3)), vec(_f64(ob4)), vec(_f64(ob5)))     # 6 x 5
    xw = _f64(xWS)[1:12, 1:N+1]                          # setvalue(x, xWS)   QuadcopterSignedDist.jl:201 (uWS unused, :202)
    xp = Matrix{Float64}(undef, 12, N + 1); up = Matrix{Float64}(undef, 4, N); ts = Vector{Float64}(undef, N + 1)
    lp = Matrix{Float64}(undef, 30, N + 1); sl = Matrix{Float64}(undef, 5, N + 1)
    exitflag = Ref{Cint}(0); iters = Ref{Cint}(0); kkt = Ref{Cdouble}(0.0); secs = Ref{Cdouble}(0.0)
    rc = ccall((:obca_quadcopter_solve_batch, LIBOBCA), Cint,
               (Cint, Cint, Ptr{Cdouble}, Ptr{Cdouble}, Cdouble, Cdouble, Ptr{Cdouble}, Ptr{Cdouble}, Cdouble, Cint, Ptr{Cvoid},
                Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Ref{Cint}, Ref{Cint}, Ref{Cdouble}, Ref{Cdouble}),
               1, N, vec(_f64(x0)), vec(_f64(xF)), Float64(Ts), Float64(R), ob, xw, Float64(timeWS), signed_dist, C_NULL,
               xp, up, ts, lp, sl, exitflag, iters, kkt, secs)
    ef = rc == 0 ? Int(exitflag[]) : 0
    return xp, up, ts, ef, secs[], lp, (ef >= 1 ? "Optimal" : "Error")          # :298
end
QuadcopterSignedDist(x0, xF, N, Ts, R, ob1, ob2, ob3, ob4, ob5, xWS, uWS, timeWS) =
    _quadcopter(1, x0, xF, N, Ts, R, ob1, ob2, ob3, ob4, ob5, xWS, uWS, timeWS)
QuadcopterDist(x0, xF, N, Ts, R, ob1, ob2, ob3, ob4, ob5, xWS, uWS, timeWS) =
    _quadcopter(0, x0, xF, N, Ts, R, ob1, ob2, ob3, ob4, ob5, xWS, uWS, timeWS)

function constrSatisfaction(x, u, timeScale, x0, xF, Ts, lambda, ob1, ob2, ob3, ob4, ob5, R)
    N = size(x, 2) - 1
    ob = hcat(vec(_f64(ob1)), vec(_f64(ob2)), vec(_f64(ob3)), vec(_f64(ob4)), vec(_f64(ob5)))
    feas = Ref{Cint}(0)
    rc = ccall((:obca_check_quadcopter, LIBOBCA), Cint,
               (Cint, Cint, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Cdouble, Ptr{Cdouble}, Ptr{Cdouble},
                Cdouble, Ptr{Cvoid}, Ref{Cint}, Ptr{Cdouble}),
               1, N, _f64(x), _f64(u), vec(_f64(timeScale)), vec(_f64(x0)), vec(_f64(xF)), Float64(Ts), _f64(lambda), ob, Float64(R),
               C_NULL, feas, C_NULL)
    return rc == 0 && feas[] == 1
end


# ---- warm-start producer (include/obca_planner.h -> libobca_planner.so: Hybrid A* + veloSmooth + main.jl:215-248) ------------------
# Replaces hybrid_a_star.calc_hybrid_astar_path (main.jl:217) and the warm-start extraction (main.jl:222-248) for a Julia that can
# no longer run the reference's 0.5/0.6 planner files.  scenario: 0 = "backwards", 1 = "parallel" (main.jl:36).
const LIBOBCA_PLANNER = get(ENV, "LIBOBCA_PLANNER", joinpath(@__DIR__, "..", "obca_b200", "planner", "libobca_planner.so"))

function plan_warm_start(x0::AbstractVector, xF::AbstractVector, scenario::Int; Ts::Float64 = 0.0, L::Float64 = 2.7, sampleN::Int = 3)
    cap = 1024
    rx = zeros(cap); ry = zeros(cap); ryaw = zeros(cap); xWS = zeros(4 * cap); uWS = zeros(2 * cap); N = Ref{Cint}(0)
    rc = ccall((:obca_plan_warmstart, LIBOBCA_PLANNER), Cint,
               (Ptr{Cdouble}, Ptr{Cdouble}, Cint, Cdouble, Cdouble, Cint, Cint, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble},
                Ptr{Cdouble}, Ref{Cint}),
               Float64.(x0[1:3]), Float64.(xF[1:3]), scenario, Ts, L, sampleN, cap, rx, ry, ryaw, xWS, uWS, N)
    rc == 1 && return nothing                                   # no path (the reference prints "Error: Cannot find path")
    rc == 0 || error("obca_plan_warmstart: ", rc)
    n = Int(N[])
    return (rx = rx[1:n+1], ry = ry[1:n+1], ryaw = ryaw[1:n+1], xWS = reshape(xWS[1:4*(n+1)], n + 1, 4), uWS = reshape(uWS[1:2*n], n, 2), N = n)
end

# ---- plan -> solve -> check for a batch of start poses in one call (include/obca.h: obca_parking_plan_solve_goals) -------------------
# main.jl:215-269 for B start poses at once, nothing leaving the GPU between the stages.  x0s, xFs: B x 4 matrices (row i = pose i's
# x0 / xF as main.jl holds them); ox, oy: the planner's obstacle points; the NLP scene as for ParkingSignedDist.  Returns per-pose
# vectors in main.jl's shapes (xp[i] 4 x (N[i]+1), up[i] 2 x N[i], timeScale[i], lp[i], np[i]) with `nothing` where the pose was not
# solved, and status (0 solved, 1 no path, 2 horizon over Ncap, 4 planner scratch full), N, exitflag, iters, feasible.
# Like every stub in this file it is not executed in this repository (no Julia in the build image); the tested twin is
# obca_b200.planner.device.plan_solve_goals (tests/test_gpu_plan_solve.py).
function plan_solve_goals(x0s::AbstractMatrix, xFs::AbstractMatrix, ox::AbstractVector, oy::AbstractVector, Ts, L, nOb, vOb, A, b,
                          ego, XYbounds; sampleN::Int = 3, Ncap::Int = 319, fixTime::Int = 0, signed_dist::Int = 1,
                          max_nodes::Int = 0, max_expansions::Int = 0)
    B = size(x0s, 1); V = Int(sum(vOb)); NS = Ncap + 1
    xp = zeros(4, NS, B); up = zeros(2, Ncap, B); ts = zeros(NS, B); lp = zeros(V, NS, B); np = zeros(4 * nOb, NS, B)
    sl = zeros(nOb, NS, B); kkt = zeros(B); ps = Ref{Cdouble}(0.0); ss = Ref{Cdouble}(0.0)
    N = fill(Cint(-1), B); status = fill(Cint(-1), B); expansions = zeros(Cint, B); flag = zeros(Cint, B); iters = zeros(Cint, B)
    feasible = zeros(Cint, B); strict = zeros(Cint, B)
    rc = ccall((:obca_parking_plan_solve_goals, LIBOBCA), Cint,
               (Cint, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Cint, Cdouble, Cdouble, Cint, Cint, Cint, Cint, Ptr{Cint},
                Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Cint, Cint, Ref{ObcaOpts}, Cint, Ptr{Cdouble}, Ptr{Cdouble},
                Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cint}, Ptr{Cint}, Ptr{Cint}, Ptr{Cint}, Ptr{Cint},
                Ptr{Cdouble}, Ptr{Cint}, Ptr{Cint}, Ref{Cdouble}, Ref{Cdouble}),
               B, _f64(permutedims(x0s[:, 1:4])), _f64(permutedims(xFs[:, 1:4])), _f64(ox), _f64(oy), length(ox), Ts, L, sampleN,
               max_expansions, max_nodes, nOb, Cint.(vec(vOb)), _f64(A), _f64(vec(b)), _f64(vec(ego)), _f64(vec(XYbounds)), fixTime,
               signed_dist, obca_default_opts(), Ncap, xp, up, ts, lp, np, sl, N, status, expansions, flag, iters, kkt, feasible, strict,
               ps, ss)
    rc == 0 || error("obca_parking_plan_solve_goals: ", rc, " ", unsafe_string(ccall((:obca_last_error, LIBOBCA), Cstring, ())))
    ok = status .== 0
    cut(a, i, n) = ok[i] ? a[:, 1:n, i] : nothing
    return (xp = [cut(xp, i, N[i] + 1) for i in 1:B], up = [cut(up, i, N[i]) for i in 1:B],
            timeScale = [ok[i] ? ts[1:N[i]+1, i] : nothing for i in 1:B], lp = [cut(lp, i, N[i] + 1) for i in 1:B],
            np = [cut(np, i, N[i] + 1) for i in 1:B], status = status, N = N, exitflag = flag, iters = iters, feasible = feasible,
            plan_time = ps[], solve_time = ss[])
end

# ---- plan -> warm start -> solve -> check for a batch of quadcopter pairs in one call (include/obca.h: obca_quadcopter_plan_solve) ---
# mainQuadcopter.jl:114-154 for B start / goal pairs at once, nothing leaving the GPU between the stages.  x0s, xFs: B x 12 matrices
# (row i = pair i's x0 / xF in the solve's units); ox, oy, oz, lo, hi, reso: the 3-D A*'s obstacle points and bounds on its 10x grid
# (mainQuadcopter.jl:46-112); R, ob1..ob5 as for QuadcopterSignedDist.  Returns per-pair vectors in mainQuadcopter.jl's shapes (xp[i]
# 12 x (N[i]+1), up[i] 4 x N[i], timeScale[i], lp[i] 30 x (N[i]+1)) with `nothing` where the pair was not solved, and status (0 solved,
# 1 no path, 2 horizon outside [2, Ncap], 4 planner scratch full), N, Ts (each pair's sampling time), exitflag, iters, feasible.
# Like every stub in this file it is not executed in this repository (no Julia in the build image); the tested twin is
# obca_b200.planner.device.plan_solve_quadcopter (tests/test_gpu_quad_plan_solve.py).
function plan_solve_quadcopter(x0s::AbstractMatrix, xFs::AbstractMatrix, ox::AbstractVector, oy::AbstractVector, oz::AbstractVector,
                               lo::AbstractVector, hi::AbstractVector, R, ob1, ob2, ob3, ob4, ob5; Ts::Float64 = 0.25,
                               reso::Float64 = 1.0, Ncap::Int = 511, signed_dist::Int = 1, max_nodes::Int = 0, timeWS::Float64 = 1.0)
    B = size(x0s, 1); NS = Ncap + 1
    ob = hcat(vec(_f64(ob1)), vec(_f64(ob2)), vec(_f64(ob3)), vec(_f64(ob4)), vec(_f64(ob5)))     # 6 x 5
    xp = zeros(12, NS, B); up = zeros(4, Ncap, B); ts = zeros(NS, B); lp = zeros(30, NS, B); sl = zeros(5, NS, B)
    N = fill(Cint(-1), B); Tsb = zeros(B); status = fill(Cint(-1), B); expansions = zeros(Cint, B); flag = zeros(Cint, B)
    iters = zeros(Cint, B); kkt = zeros(B); feasible = zeros(Cint, B); worst = zeros(B); ps = Ref{Cdouble}(0.0); ss = Ref{Cdouble}(0.0)
    rc = ccall((:obca_quadcopter_plan_solve, LIBOBCA), Cint,
               (Cint, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Cint, Ptr{Cdouble}, Ptr{Cdouble}, Cdouble, Cint,
                Cdouble, Cdouble, Ptr{Cdouble}, Cdouble, Cint, Ref{ObcaOpts}, Cint, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble},
                Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cint}, Ptr{Cdouble}, Ptr{Cint}, Ptr{Cint}, Ptr{Cint}, Ptr{Cint}, Ptr{Cdouble},
                Ptr{Cint}, Ptr{Cdouble}, Ref{Cdouble}, Ref{Cdouble}),
               B, _f64(permutedims(x0s[:, 1:12])), _f64(permutedims(xFs[:, 1:12])), _f64(ox), _f64(oy), _f64(oz), length(ox),
               _f64(lo), _f64(hi), reso, max_nodes, Ts, Float64(R), ob, timeWS, signed_dist,
               (o = obca_default_opts(); o.max_iter = 3000; o), Ncap, xp, up, ts, lp, sl, N, Tsb, status, expansions, flag, iters,
               kkt, feasible, worst, ps, ss)
    rc == 0 || error("obca_quadcopter_plan_solve: ", rc, " ", unsafe_string(ccall((:obca_last_error, LIBOBCA), Cstring, ())))
    ok = status .== 0
    cut(a, i, n) = ok[i] ? a[:, 1:n, i] : nothing
    return (xp = [cut(xp, i, N[i] + 1) for i in 1:B], up = [cut(up, i, N[i]) for i in 1:B],
            timeScale = [ok[i] ? ts[1:N[i]+1, i] : nothing for i in 1:B], lp = [cut(lp, i, N[i] + 1) for i in 1:B],
            status = status, N = N, Ts = Tsb, exitflag = flag, iters = iters, feasible = feasible, plan_time = ps[], solve_time = ss[])
end

# ---- one plan, both formulations (include/obca.h: obca_parking_plan_solve_both, obca_quadcopter_plan_solve_both) ----------------------
# main.jl:215-269 and mainQuadcopter.jl:114-154 as the reference runs them: every problem planned once, then solved and checked with the
# Distance and then the Signed Distance formulation in the same call.  Each formulation's outputs go through one struct of pointers
# (obca_parking_flow_out / obca_quadcopter_flow_out), passed by Ref.  Like every stub in this file they are not executed in this
# repository (no Julia in the build image); the tested twins are obca_b200.planner.device.plan_solve_goals_both and
# plan_solve_quadcopter_both (tests/test_gpu_plan_solve_both.py).
struct ParkingFlowOut
    xp::Ptr{Cdouble}; up::Ptr{Cdouble}; ts::Ptr{Cdouble}; lp::Ptr{Cdouble}; np::Ptr{Cdouble}; sl::Ptr{Cdouble}
    exitflag::Ptr{Cint}; iters::Ptr{Cint}; kkt_err::Ptr{Cdouble}; feasible::Ptr{Cint}; strict::Ptr{Cint}; solve_seconds::Ptr{Cdouble}
end

struct QuadcopterFlowOut
    xp::Ptr{Cdouble}; up::Ptr{Cdouble}; ts::Ptr{Cdouble}; lp::Ptr{Cdouble}; slack::Ptr{Cdouble}
    exitflag::Ptr{Cint}; iters::Ptr{Cint}; kkt_err::Ptr{Cdouble}; feasible::Ptr{Cint}; worst::Ptr{Cdouble}; solve_seconds::Ptr{Cdouble}
end

# Returns (status, N, plan_time, dist, sd): dist and sd hold the per-pose vectors and values plan_solve_goals returns for one formulation.
function plan_solve_goals_both(x0s::AbstractMatrix, xFs::AbstractMatrix, ox::AbstractVector, oy::AbstractVector, Ts, L, nOb, vOb, A,
                               b, ego, XYbounds; sampleN::Int = 3, Ncap::Int = 319, fixTime::Int = 0, max_nodes::Int = 0,
                               max_expansions::Int = 0)
    B = size(x0s, 1); V = Int(sum(vOb)); NS = Ncap + 1
    mk() = (xp = zeros(4, NS, B), up = zeros(2, Ncap, B), ts = zeros(NS, B), lp = zeros(V, NS, B), np = zeros(4 * nOb, NS, B),
            sl = zeros(nOb, NS, B), flag = zeros(Cint, B), iters = zeros(Cint, B), kkt = zeros(B), feasible = zeros(Cint, B),
            strict = zeros(Cint, B), ss = zeros(1))
    sets = (mk(), mk())
    N = fill(Cint(-1), B); status = fill(Cint(-1), B); expansions = zeros(Cint, B); ps = Ref{Cdouble}(0.0)
    rc = GC.@preserve sets begin
        outs = [Ref(ParkingFlowOut(pointer(s.xp), pointer(s.up), pointer(s.ts), pointer(s.lp), pointer(s.np), pointer(s.sl), pointer(s.flag),
                                   pointer(s.iters), pointer(s.kkt), pointer(s.feasible), pointer(s.strict), pointer(s.ss))) for s in sets]
        ccall((:obca_parking_plan_solve_both, LIBOBCA), Cint,
              (Cint, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Cint, Cdouble, Cdouble, Cint, Cint, Cint, Cint, Ptr{Cint},
               Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Cint, Ref{ObcaOpts}, Cint, Ptr{Cint}, Ptr{Cint}, Ptr{Cint},
               Ref{Cdouble}, Ref{ParkingFlowOut}, Ref{ParkingFlowOut}),
              B, _f64(permutedims(x0s[:, 1:4])), _f64(permutedims(xFs[:, 1:4])), _f64(ox), _f64(oy), length(ox), Ts, L, sampleN,
              max_expansions, max_nodes, nOb, Cint.(vec(vOb)), _f64(A), _f64(vec(b)), _f64(vec(ego)), _f64(vec(XYbounds)), fixTime,
              obca_default_opts(), Ncap, N, status, expansions, ps, outs[1], outs[2])
    end
    rc == 0 || error("obca_parking_plan_solve_both: ", rc, " ", unsafe_string(ccall((:obca_last_error, LIBOBCA), Cstring, ())))
    ok = status .== 0
    cut(a, i, n) = ok[i] ? a[:, 1:n, i] : nothing
    one(s) = (xp = [cut(s.xp, i, N[i] + 1) for i in 1:B], up = [cut(s.up, i, N[i]) for i in 1:B],
              timeScale = [ok[i] ? s.ts[1:N[i]+1, i] : nothing for i in 1:B], lp = [cut(s.lp, i, N[i] + 1) for i in 1:B],
              np = [cut(s.np, i, N[i] + 1) for i in 1:B], exitflag = s.flag, iters = s.iters, feasible = s.feasible, solve_time = s.ss[1])
    return (status = status, N = N, plan_time = ps[], dist = one(sets[1]), sd = one(sets[2]))
end

# Returns (status, N, Ts, plan_time, dist, sd): dist and sd hold the per-pair vectors and values plan_solve_quadcopter returns for one
# formulation.
function plan_solve_quadcopter_both(x0s::AbstractMatrix, xFs::AbstractMatrix, ox::AbstractVector, oy::AbstractVector,
                                    oz::AbstractVector, lo::AbstractVector, hi::AbstractVector, R, ob1, ob2, ob3, ob4, ob5;
                                    Ts::Float64 = 0.25, reso::Float64 = 1.0, Ncap::Int = 511, max_nodes::Int = 0, timeWS::Float64 = 1.0)
    B = size(x0s, 1); NS = Ncap + 1
    ob = hcat(vec(_f64(ob1)), vec(_f64(ob2)), vec(_f64(ob3)), vec(_f64(ob4)), vec(_f64(ob5)))     # 6 x 5
    mk() = (xp = zeros(12, NS, B), up = zeros(4, Ncap, B), ts = zeros(NS, B), lp = zeros(30, NS, B), sl = zeros(5, NS, B),
            flag = zeros(Cint, B), iters = zeros(Cint, B), kkt = zeros(B), feasible = zeros(Cint, B), worst = zeros(B), ss = zeros(1))
    sets = (mk(), mk())
    N = fill(Cint(-1), B); Tsb = zeros(B); status = fill(Cint(-1), B); expansions = zeros(Cint, B); ps = Ref{Cdouble}(0.0)
    rc = GC.@preserve sets begin
        outs = [Ref(QuadcopterFlowOut(pointer(s.xp), pointer(s.up), pointer(s.ts), pointer(s.lp), pointer(s.sl), pointer(s.flag),
                                      pointer(s.iters), pointer(s.kkt), pointer(s.feasible), pointer(s.worst), pointer(s.ss))) for s in sets]
        ccall((:obca_quadcopter_plan_solve_both, LIBOBCA), Cint,
              (Cint, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Ptr{Cdouble}, Cint, Ptr{Cdouble}, Ptr{Cdouble}, Cdouble,
               Cint, Cdouble, Cdouble, Ptr{Cdouble}, Cdouble, Ref{ObcaOpts}, Cint, Ptr{Cint}, Ptr{Cdouble}, Ptr{Cint}, Ptr{Cint},
               Ref{Cdouble}, Ref{QuadcopterFlowOut}, Ref{QuadcopterFlowOut}),
              B, _f64(permutedims(x0s[:, 1:12])), _f64(permutedims(xFs[:, 1:12])), _f64(ox), _f64(oy), _f64(oz), length(ox),
              _f64(lo), _f64(hi), reso, max_nodes, Ts, Float64(R), ob, timeWS, (o = obca_default_opts(); o.max_iter = 3000; o), Ncap,
              N, Tsb, status, expansions, ps, outs[1], outs[2])
    end
    rc == 0 || error("obca_quadcopter_plan_solve_both: ", rc, " ", unsafe_string(ccall((:obca_last_error, LIBOBCA), Cstring, ())))
    ok = status .== 0
    cut(a, i, n) = ok[i] ? a[:, 1:n, i] : nothing
    one(s) = (xp = [cut(s.xp, i, N[i] + 1) for i in 1:B], up = [cut(s.up, i, N[i]) for i in 1:B],
              timeScale = [ok[i] ? s.ts[1:N[i]+1, i] : nothing for i in 1:B], lp = [cut(s.lp, i, N[i] + 1) for i in 1:B],
              exitflag = s.flag, iters = s.iters, feasible = s.feasible, solve_time = s.ss[1])
    return (status = status, N = N, Ts = Tsb, plan_time = ps[], dist = one(sets[1]), sd = one(sets[2]))
end
