"""Float64 NumPy restatement of the reference physics models (TEST INFRASTRUCTURE ONLY).

Every function is vectorised over an arbitrary batch shape but performs, element
by element, exactly the float64 operations of the reference in the reference's
order; the reference lines are cited next to each block (paths relative to
a checkout of the reference).  Ranges that the reference stores as ``None`` (no
constraint) are passed here as ``(-inf, +inf)``: ``np.clip`` with infinite
bounds is the identity, which is what the reference's ``if range is not None``
guard does.

Pinned against the unmodified reference by ``oracle/make_golden.py`` ->
``tests/golden/physics_*.npz`` -> ``tests/test_oracle_golden.py``.
"""

from __future__ import annotations

import numpy as np

G = 9.81  # tactics2d/physics/physics_model_base.py:25
DELTA_T = 5  # physics_model_base.py:23
MIN_DELTA_T = 1  # physics_model_base.py:24

INF = float("inf")


# --------------------------------------------------------------------------- ranges
def normalize_range_bicycle(r):
    """Constructor rule shared by the three bicycles.

    tactics2d/physics/single_track_kinematics.py:87-115: a Python ``float`` r>=0
    -> [-r, r]; a negative float -> None; a 2-sequence with lo<hi is kept, lo>=hi
    -> None; anything else (``None``, or an ``int``!) -> None.
    Returns ``(lo, hi)`` with infinities standing for None.
    """
    if isinstance(r, float):
        return (-INF, INF) if r < 0 else (-r, r)
    if hasattr(r, "__len__") and len(r) == 2:
        if r[0] >= r[1]:
            return (-INF, INF)
        return (float(r[0]), float(r[1]))
    return (-INF, INF)


def normalize_range_pointmass(r):
    """tactics2d/physics/point_mass.py:50-66: float r>=0 -> [0, r]; tuple ->
    [max(0,lo), max(0,hi)], None when that is empty; else None."""
    if isinstance(r, float):
        return (-INF, INF) if r < 0 else (0.0, r)
    if hasattr(r, "__len__") and len(r) == 2:
        lo, hi = max(0, r[0]), max(0, r[1])
        if lo >= hi:
            return (-INF, INF)
        return (float(lo), float(hi))
    return (-INF, INF)


def effective_delta_t(delta_t, interval):
    """physics constructors (single_track_kinematics.py:119-124)."""
    if delta_t is None:
        return DELTA_T
    d = max(delta_t, MIN_DELTA_T)
    if interval is not None:
        d = min(d, interval)
    return d


def _f64(*arrs):
    return [np.asarray(a, dtype=np.float64) for a in arrs]


# --------------------------------------------------------------------------- kinematics
def step_kinematics(x, y, phi, v, accel, delta, lf, lr, steer_rng, speed_rng, accel_rng,
                    interval=100, delta_t=DELTA_T):
    """SingleTrackKinematics.step/_step, single_track_kinematics.py:178-198,126-176.

    Returns dict(x, y, heading, speed, vx, vy, accel, delta) - ``accel``/``delta``
    are the clipped actions the reference returns next to the State.
    """
    x, y, phi, v, accel, delta, lf, lr = _f64(x, y, phi, v, accel, delta, lf, lr)
    s_lo, s_hi = _f64(*steer_rng)
    v_lo, v_hi = _f64(*speed_rng)
    a_lo, a_hi = _f64(*accel_rng)
    accel = np.clip(accel, a_lo, a_hi)  # :192
    delta = np.clip(delta, s_lo, s_hi)  # :193
    wheel_base = lf + lr  # :85
    beta = np.arctan(lr / wheel_base * np.tan(delta))  # :127
    dt = float(delta_t) / 1000  # :128
    n_steps = interval // delta_t  # :129
    remainder = interval % delta_t  # :130
    x, y, phi, v = (np.array(np.broadcast_to(a, np.broadcast(x, y, phi, v, accel, delta, lf).shape),
                             dtype=np.float64) for a in (x, y, phi, v))

    def sub(x, y, phi, v, h):  # :138-148 / :152-163
        dx = v * np.cos(phi + beta)
        dy = v * np.sin(phi + beta)
        dv = accel
        dphi = v / wheel_base * np.tan(delta) * np.cos(beta)
        x = x + dx * h
        y = y + dy * h
        phi = phi + dphi * h
        v = v + dv * h
        v = np.clip(v, v_lo, v_hi)
        return x, y, phi, v

    for _ in range(n_steps):
        x, y, phi, v = sub(x, y, phi, v, dt)
    if remainder > 0:
        x, y, phi, v = sub(x, y, phi, v, float(remainder) / 1000)
    return dict(x=x, y=y, heading=np.mod(phi, 2 * np.pi),  # :169
                vx=v * np.cos(phi), vy=v * np.sin(phi),  # :170-171 (unwrapped phi, no beta)
                speed=v, accel=accel + 0 * x, delta=delta + 0 * x)


# --------------------------------------------------------------------------- dynamics
def step_dynamics(x, y, phi, v, accel, delta, lf, lr, mass, mass_height, mu, I_z, cf, cr,
                  steer_rng, speed_rng, accel_rng, interval=100, delta_t=DELTA_T):
    """SingleTrackDynamics.step/_step, single_track_dynamics.py:231-251,140-229.

    No remainder sub-step (``remainder`` is computed at :143 and never used).  The
    reference State carries ``vx = vy = None``; ``vx, vy`` returned here are what
    ``State.velocity`` derives (state.py:160-165): speed*(cos, sin)(wrapped heading).
    """
    x, y, phi, v, accel, delta, lf, lr = _f64(x, y, phi, v, accel, delta, lf, lr)
    mass, mass_height, mu, I_z, cf, cr = _f64(mass, mass_height, mu, I_z, cf, cr)
    s_lo, s_hi = _f64(*steer_rng)
    v_lo, v_hi = _f64(*speed_rng)
    a_lo, a_hi = _f64(*accel_rng)
    accel = np.clip(accel, a_lo, a_hi)  # :245
    delta = np.clip(delta, s_lo, s_hi)  # :246
    wheel_base = lf + lr
    dt = float(delta_t) / 1000  # :141
    n_steps = interval // delta_t  # :142

    factor_f = (G * lr - accel * mass_height) / wheel_base  # :145
    factor_r = (G * lf + accel * mass_height) / wheel_base  # :146
    lf_cf_factor_f = lf * cf * factor_f  # :149-154
    lr_cr_factor_r = lr * cr * factor_r
    lf2_cf_factor_f = lf**2 * cf * factor_f
    lr2_cr_factor_r = lr**2 * cr * factor_r
    cf_factor_f = cf * factor_f
    cr_factor_r = cr * factor_r

    shape = np.broadcast(x, y, phi, v, accel, delta, lf).shape
    x, y, phi, v = (np.array(np.broadcast_to(a, shape), dtype=np.float64) for a in (x, y, phi, v))
    d_phi = v / wheel_base * np.tan(delta)  # :159
    beta = np.arctan(lr / lf * np.tan(delta)) + 0 * x  # :160  (lr/lf, not lr/L)

    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        for _ in range(n_steps):  # :163-218
            dx = v * np.cos(phi + beta)
            dy = v * np.sin(phi + beta)
            dv = accel
            v_safe = np.where(np.abs(v) > 1e-6, v, np.where(v >= 0, 1e-6, -1e-6))  # :169
            fast = np.abs(v) >= 0.1  # :171
            dd_phi = (mu * mass / I_z * (lf_cf_factor_f * delta
                                         + (lr_cr_factor_r - lf_cf_factor_f) * beta
                                         - (lf2_cf_factor_f + lr2_cr_factor_r) * d_phi / v_safe))  # :172-181
            d_beta_fast = (mu / v_safe * (cf_factor_f * delta - (cr_factor_r + cf_factor_f) * beta
                                          + (lr_cr_factor_r - lf_cf_factor_f) * d_phi / v_safe)
                           - d_phi)  # :182-191 (uses d_phi *before* its update)
            d_phi_fast = d_phi + dd_phi * dt  # :192
            d_beta_slow = (lr / (1 + np.tan(delta) * lr / wheel_base) ** 2 / wheel_base
                           / np.cos(delta) ** 2 * delta)  # :194-200
            d_phi_slow = d_phi + v * np.cos(beta) / wheel_base * np.tan(delta) * dt  # :210
            d_beta = np.where(fast, d_beta_fast, d_beta_slow)
            d_phi = np.where(fast, d_phi_fast, d_phi_slow)
            x = x + dx * dt  # :212-216
            y = y + dy * dt
            v = v + dv * dt
            phi = phi + d_phi * dt
            beta = beta + d_beta * dt
            v = np.clip(v, v_lo, v_hi)  # :218
    heading = np.mod(phi, 2 * np.pi)  # :224
    return dict(x=x, y=y, heading=heading, speed=v, vx=v * np.cos(heading), vy=v * np.sin(heading),
                accel=accel + 0 * x, delta=delta + 0 * x)


# --------------------------------------------------------------------------- drift bicycle
# Built-in tyre (class Tire, single_track_drift.py:14-49): Pacejka magic-formula coefficients of the CommonRoad
# single-track-drift model.  The reference evaluates every force with camber gamma = 0.
TIRE = dict(p_cx1=1.6411, p_dx1=1.1739, p_dx3=0.0, p_ex1=0.4640, p_kx1=22.303, p_hx1=1.2297e-3, p_vx1=-8.8098e-6,
            r_bx1=13.276, r_bx2=-13.778, r_ex1=1.2568, r_cx1=0.6522, r_hx1=5.0722e-3,
            p_cy1=1.3507, p_dy1=1.0489, p_dy3=-2.8821, p_ey1=-7.4722e-3, p_ky1=-21.920, p_hy1=2.6747e-3, p_hy3=3.1415e-2,
            p_vy1=3.7318e-2, p_vy3=-0.3293, r_by1=7.1433, r_by2=9.1917, r_by3=-2.7856e-2, r_cy1=1.0719, r_ey1=-0.2757,
            r_hy1=5.7448e-6, r_vy1=-2.7825e-2, r_vy3=-0.2756, r_vy4=12.120, r_vy5=1.9, r_vy6=-10.704)


def _safe(u):
    """``u if |u| > 1e-6 else (1e-6 if u >= 0 else -1e-6)`` (single_track_drift.py:287,289,308-309,345)."""
    return np.where(np.abs(u) > 1e-6, u, np.where(u >= 0, 1e-6, -1e-6))


def _magic(B, C, E, arg):
    return C * np.arctan(B * arg - E * (B * arg - np.arctan(B * arg)))


def _drift_tire_forces(v, delta, d_phi, beta, omega_wf, omega_wr, lf, lr, mass, radius):
    """``SingleTrackDrift._tire_forces`` (single_track_drift.py:282-338) with the four Pacejka helpers
    (:185-280) at gamma = 0."""
    T = TIRE
    v_safe = _safe(v)                                                                        # :287
    cos_beta_safe = _safe(np.cos(beta))                                                      # :288-289
    alpha_f = np.arctan((v_safe * np.sin(beta) + d_phi * lf) / (v_safe * cos_beta_safe)) - delta   # :292-294
    alpha_r = np.arctan((v_safe * np.sin(beta) - d_phi * lr) / (v_safe * cos_beta_safe))           # :295
    wheel_base = lf + lr
    F_zf = (mass * G * lr) / wheel_base                                                      # :298
    F_zr = (mass * G * lf) / wheel_base                                                      # :299
    u_wf = v_safe * cos_beta_safe * np.cos(delta) + (v_safe * np.sin(beta) + lf * d_phi) * np.sin(delta)   # :302-304
    u_wr = v_safe * cos_beta_safe                                                            # :305
    s_f = 1 - radius * omega_wf / _safe(u_wf)                                                # :308-313
    s_r = 1 - radius * omega_wr / _safe(u_wr)

    def pure_long(kappa, F_z):                                                               # :185-203
        kappa_x = -kappa + T["p_hx1"]
        D_x = T["p_dx1"] * (1 - T["p_dx3"] * 0.0) * F_z
        B_x = (T["p_kx1"] * F_z) / (T["p_cx1"] * D_x + 1e-6)
        return D_x * np.sin(_magic(B_x, T["p_cx1"], T["p_ex1"], kappa_x) + T["p_vx1"] * F_z)

    def pure_lat(alpha, F_z):                                                                # :205-224
        S_hy = np.sign(0.0) * (T["p_hy1"] + T["p_hy3"] * 0.0)
        mu_y = T["p_dy1"] * (1 - T["p_dy3"] * 0.0)
        D_y = mu_y * F_z
        B_y = (T["p_ky1"] * F_z) / (T["p_cy1"] * D_y + 1e-6)
        return D_y * np.sin(_magic(B_y, T["p_cy1"], T["p_ey1"], alpha + S_hy) + S_hy * F_z), mu_y

    def comb_long(kappa, alpha, F0_x):                                                       # :226-250
        B = T["r_bx1"] * np.cos(np.arctan(T["r_bx2"] * kappa))
        D = F0_x / np.cos(_magic(B, T["r_cx1"], T["r_ex1"], T["r_hx1"]))
        return D * np.cos(_magic(B, T["r_cx1"], T["r_ex1"], alpha + T["r_hx1"]))

    def comb_lat(kappa, alpha, mu_y, F_z, F0_y):                                             # :252-280
        B = T["r_by1"] * np.cos(np.arctan(T["r_by2"] * (alpha - T["r_by3"])))
        D = F0_y / np.cos(_magic(B, T["r_cy1"], T["r_ey1"], T["r_hy1"]))
        D_vy = mu_y * F_z * (T["r_vy1"] + T["r_vy3"] * 0.0) * np.cos(np.arctan(T["r_vy4"] * alpha))
        S_vy = D_vy * np.sin(T["r_vy5"] * np.arctan(T["r_vy6"] * kappa))
        return D * np.cos(_magic(B, T["r_cy1"], T["r_ey1"], kappa + T["r_hy1"])) + S_vy

    F0_xf, F0_xr = pure_long(s_f, F_zf), pure_long(s_r, F_zr)                                 # :317-318
    (F0_yf, mu_yf), (F0_yr, mu_yr) = pure_lat(alpha_f, F_zf), pure_lat(alpha_r, F_zr)        # :321-322
    F_xf, F_xr = comb_long(s_f, alpha_f, F0_xf), comb_long(s_r, alpha_r, F0_xr)               # :325-326
    F_yf = comb_lat(s_f, alpha_f, mu_yf, F_zf, F0_yf)                                        # :329-330
    F_yr = comb_lat(s_r, alpha_r, mu_yr, F_zr, F0_yr)
    return F_xf, F_xr, F_yf, F_yr


def step_drift(x, y, phi, v, omega_wf, omega_wr, accel, delta, lf, lr, mass, radius, T_sb, T_se, I_z, I_yw,
               steer_rng, speed_rng, accel_rng, interval=100, delta_t=DELTA_T):
    """SingleTrackDrift.step/_step, single_track_drift.py:467-499,340-465.  Unlike the dynamic bicycle this model
    DOES take the remainder sub-step (:352-355).  ``vx, vy`` as ``State.velocity`` derives them (state.py:160-165)."""
    x, y, phi, v, omega_wf, omega_wr, accel, delta = _f64(x, y, phi, v, omega_wf, omega_wr, accel, delta)
    lf, lr, mass, radius, T_sb, T_se, I_z, I_yw = _f64(lf, lr, mass, radius, T_sb, T_se, I_z, I_yw)
    s_lo, s_hi = _f64(*steer_rng)
    v_lo, v_hi = _f64(*speed_rng)
    a_lo, a_hi = _f64(*accel_rng)
    accel = np.clip(accel, a_lo, a_hi)                                                       # :490
    delta = np.clip(delta, s_lo, s_hi)                                                       # :491
    dts = [float(delta_t) / 1000] * (interval // delta_t)                                    # :352
    if interval % delta_t > 0:
        dts.append(float(interval % delta_t) / 1000)                                         # :353-355
    wheel_base = lf + lr
    shape = np.broadcast(x, y, phi, v, accel, delta, lf, omega_wf).shape
    x, y, phi, v, omega_wf, omega_wr = (np.array(np.broadcast_to(a, shape), dtype=np.float64)
                                        for a in (x, y, phi, v, omega_wf, omega_wr))
    d_phi = v / wheel_base * np.tan(delta)                                                   # :360
    beta = np.arctan(lr / lf * np.tan(delta)) + 0 * x                                        # :361
    T_B = np.where(accel > 0, 0.0, mass * radius * accel)                                    # :363-368
    T_E = np.where(accel > 0, mass * radius * accel, 0.0)
    with np.errstate(all="ignore"):
        for dt in dts:                                                                       # :370-447
            v_safe = _safe(v)
            F_lf, F_lr, F_sf, F_sr = _drift_tire_forces(v_safe, delta, d_phi, beta, omega_wf, omega_wr, lf, lr, mass, radius)
            dx = v * np.cos(phi + beta)
            dy = v * np.sin(phi + beta)
            fast = np.abs(v) >= 0.1                                                          # :381
            dv_f = 1 / mass * (-F_sf * np.sin(delta - beta) + F_sr * np.sin(beta) + F_lr * np.cos(beta)
                               + F_lf * np.cos(delta - beta))                                # :382-391
            d_beta_f = -d_phi + 1 / (mass * v_safe) * (F_sf * np.cos(delta - beta) + F_sr * np.cos(beta)
                                                       - F_lr * np.sin(beta) + F_lf * np.sin(delta - beta))   # :392-397
            dd_phi = 1 / I_z * (F_sf * np.cos(delta) * lf - F_sr * lr + F_lf * np.sin(delta) * lf)   # :398-406
            d_phi_f = d_phi + dd_phi * dt                                                    # :407
            d_om_f_f = 1 / I_yw * (-radius * F_lf + T_sb * T_B + T_se * T_E)                 # :408-410
            d_om_r_f = 1 / I_yw * (-radius * F_lr + (1 - T_sb) * T_B + (1 - T_se) * T_E)     # :411-415
            d_beta_s = lr / (1 + np.tan(delta) * lr / wheel_base) ** 2 / wheel_base / np.cos(delta) ** 2 * delta   # :418-424
            d_phi_s = d_phi + v * np.cos(beta) / wheel_base * np.tan(delta) * dt             # :434
            d_om_f_s = 1 / (np.cos(delta) * radius) * (accel * np.cos(beta) - v * np.sin(beta) * d_beta_s
                                                       + v * np.cos(beta) * np.tan(delta) * delta)   # :435-443
            d_om_r_s = 1 / radius * (accel * np.cos(beta) - v * np.sin(beta) * d_beta_s)     # :444
            dv = np.where(fast, dv_f, accel)                                                 # :417
            d_beta = np.where(fast, d_beta_f, d_beta_s)
            d_phi = np.where(fast, d_phi_f, d_phi_s)
            x = x + dx * dt                                                                  # :446-453
            y = y + dy * dt
            v = v + dv * dt
            phi = phi + d_phi * dt
            beta = beta + d_beta * dt
            omega_wf = omega_wf + np.where(fast, d_om_f_f, d_om_f_s) * dt
            omega_wr = omega_wr + np.where(fast, d_om_r_f, d_om_r_s) * dt
            v = np.clip(v, v_lo, v_hi)                                                       # :455
    heading = np.mod(phi, 2 * np.pi)                                                         # :461
    return dict(x=x, y=y, heading=heading, speed=v, vx=v * np.cos(heading), vy=v * np.sin(heading),
                omega_wf=omega_wf, omega_wr=omega_wr, accel=accel + 0 * x, delta=delta + 0 * x)


# --------------------------------------------------------------------------- point mass
def _newton_t1(ax, ay, vx, vy, limit, sign, dt):
    """point_mass.py:106-127 (sign=-1, lower limit) / :141-162 (sign=+1, upper limit)."""
    a_ = ax**2 + ay**2
    b_ = 2 * (ax * vx + ay * vy)
    c_ = vx**2 + vy**2 - limit**2
    with np.errstate(divide="ignore", invalid="ignore"):
        t_lin = np.where(np.abs(b_) < 1e-12, 0.0, -c_ / b_)
        disc = np.maximum(0.0, b_**2 - 4 * a_ * c_)
        t_quad = (-b_ + sign * np.sqrt(disc)) / (2 * a_)
    t1 = np.where(np.abs(a_) < 1e-12, t_lin, t_quad)
    return np.clip(t1, 0.0, dt)


def step_pointmass_newton(x, y, vx, vy, ax, ay, speed_rng, interval=100):
    """PointMass.step (newton backend), point_mass.py:209-232,83-175.

    ``step`` computes a clipped acceleration magnitude (:222-225) and never uses it:
    the acceleration is NOT clipped.  Heading = atan2 of the new velocity.
    """
    x, y, vx, vy, ax, ay = _f64(x, y, vx, vy, ax, ay)
    s_lo, s_hi = _f64(*speed_rng)
    dt = float(interval) / 1000  # :86
    next_vx = vx + ax * dt  # :88-90
    next_vy = vy + ay * dt
    next_speed = np.sqrt(next_vx**2 + next_vy**2)
    ok = (s_lo <= next_speed) & (next_speed <= s_hi)  # :93
    low = ~ok & (next_speed < s_lo)  # :105
    # branch 1  :94-101
    x1 = x + vx * dt + 0.5 * ax * dt**2
    y1 = y + vy * dt + 0.5 * ay * dt**2
    # branch 2 / 3
    lim = np.where(low, s_lo, s_hi)
    lim = np.where(np.isfinite(lim), lim, 0.0)
    sign = np.where(low, -1.0, 1.0)
    t1 = _newton_t1(ax, ay, vx, vy, lim, sign, dt)
    t2 = dt - t1
    vxl = vx + ax * t1
    vyl = vy + ay * t1
    x2 = x + vx * t1 + 0.5 * ax * t1**2 + vxl * t2
    y2 = y + vy * t1 + 0.5 * ay * t1**2 + vyl * t2
    nx = np.where(ok, x1, x2)
    ny = np.where(ok, y1, y2)
    nvx = np.where(ok, next_vx, vxl)
    nvy = np.where(ok, next_vy, vyl)
    return dict(x=nx, y=ny, heading=np.arctan2(nvy, nvx), vx=nvx, vy=nvy,
                speed=np.sqrt(nvx**2 + nvy**2))


def step_pointmass_euler(x, y, heading, vx, vy, ax, ay, speed_rng, interval=100, delta_t=DELTA_T):
    """PointMass._step_euler, point_mass.py:177-207."""
    x, y, heading, vx, vy, ax, ay = _f64(x, y, heading, vx, vy, ax, ay)
    s_lo, s_hi = _f64(*speed_rng)
    shape = np.broadcast(x, y, heading, vx, vy, ax, ay).shape
    x, y, heading, vx, vy = (np.array(np.broadcast_to(a, shape), dtype=np.float64)
                             for a in (x, y, heading, vx, vy))
    dts = [float(delta_t) / 1000] * (interval // delta_t)
    if interval % delta_t > 0:
        dts.append(float(interval % delta_t) / 1000)
    for dt in dts:
        vx = vx + ax * dt
        vy = vy + ay * dt
        speed = np.sqrt(vx**2 + vy**2)
        clipped = np.clip(speed, s_lo, s_hi)
        resc = np.abs(speed - clipped) > 1e-12  # :195
        vx = np.where(resc, clipped * np.cos(heading), vx)
        vy = np.where(resc, clipped * np.sin(heading), vy)
        x = x + vx * dt
        y = y + vy * dt
        heading = np.arctan2(vy, vx)
    return dict(x=x, y=y, heading=heading, vx=vx, vy=vy, speed=np.sqrt(vx**2 + vy**2))


# --------------------------------------------------------------------------- verify_state
def verify_state_bicycle(state, last_state, lr, wheel_base, steer_rng, speed_rng, accel_rng,
                         interval):
    """SingleTrackKinematics.verify_state, single_track_kinematics.py:200-250 (scalar).

    ``state``/``last_state`` are (x, y, heading, speed) tuples; ranges use infinities
    for None (-> True, :216-217)."""
    if interval == 0:
        return True
    dt = float(interval) / 1000
    if not all(np.isfinite(r).all() for r in (steer_rng, speed_rng, accel_rng)):
        return True
    lx, ly, lh, lv = last_state
    sx, sy, sh, sv = state
    steer = np.array(steer_rng, dtype=np.float64)
    beta_range = np.arctan(lr / wheel_base * steer)  # :220
    heading_range = np.mod(lh + lv / wheel_base * np.sin(beta_range) * dt, 2 * np.pi)
    if heading_range[0] < heading_range[1] and not heading_range[0] <= sh <= heading_range[1]:
        return False
    if heading_range[0] > heading_range[1] and not (heading_range[0] <= sh or sh <= heading_range[1]):
        return False
    sp = np.clip(lv + np.array(accel_rng, dtype=np.float64) * dt, *speed_rng)  # :238
    if not sp[0] <= sv <= sp[1]:
        return False
    x_range = lx + sp * np.cos(lh + beta_range) * dt
    y_range = ly + sp * np.sin(lh + beta_range) * dt
    if not x_range[0] < sx < x_range[1] or not y_range[0] < sy < y_range[1]:
        return False
    return True
