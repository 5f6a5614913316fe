"""Per-pixel fp64 reference of the 2DGS raster forward and backward (numpy, vectorised over every pixel of every tile, stepping over list
positions), following the per-pixel algebra of oracle/splat_oracle_impl.inc (oracle_raster2dgs_fwd / _bwd), backgrounds included.

The aggregated gradients are the C oracle's; this module adds what it cannot give:

* error scales. For the backward, A[s, k] = sum_p |t_{p,s,k}| (n_{p,s} + 4 + K_{p,s}): t is pixel p's contribution to component k of
  splat s's 16-float gradient record (rgb[3] normal[3] M_u[3] M_v[3] M_w[3] opacity) evaluated with absolute values at every sum, so a
  cancellation inside the record does not shrink it; n_{p,s} counts the splats p composites from s up to its last contributor (the
  fp32 backward carries T and the colour / normal / depth sums over that many steps); K_{p,s} is the fp32 rounding of h_u = px M_w - M_u
  and h_v (the cancellation of two terms of size px |M_w|) carried through zeta and (u, v) into sigma, plus the error of __expf (in
  units of 2^-24). A_state uses N_p, the pixel's whole composited count, in place of n_{p,s}: the bound for a backward that starts from
  an fp32 forward state. The forward gets the same kind of scale per output pixel and per visibility;
* absgrad under the kernel's definition: per (camera, tile, 8x8 block, splat) |sum over the block of dL/dM_u.z| * M_w.z (resp. M_v.z),
  summed over blocks; and the per-8x4-block sum the kernel used before, to show that the two differ;
* the fp64 margins of the discrete decisions (alpha vs 1/255, opacity * vis vs 0.999, T (1 - alpha) vs 1e-4, depth vs 0.05; T vs 0.5,
  which picks the median, per pixel)."""
import numpy as np

TILE = 16
U = 2.0 ** -24
ALPHA_T = float(np.float32(1.0 / 255.0))
CLIP = float(np.float32(0.999))
NEAR = float(np.float32(0.05))
T_STOP = 1e-4
NUDGE = 2e-3  # decisions closer than this (relative) to their threshold are reported, so the builder's result clears 1e-3


def lists_of(off, flat):
    """offsets [C, th, tw], flatten_ids -> (start [nb], length [nb], ids [nb, Lmax] with -1 padding, list index [nb, Lmax])."""
    start = np.asarray(off, np.int64).ravel()
    flat = np.asarray(flat, np.int64)
    L = np.append(start[1:], len(flat)) - start
    Lmax = max(int(L.max()), 1)
    k = np.arange(Lmax)[None]
    idx = start[:, None] + k
    g = np.where(k < L[:, None], flat[np.minimum(idx, max(len(flat) - 1, 0))] if len(flat) else -1, -1)
    return start, L, g, idx


def _pixels(sc):
    C, W, H = sc["C"], sc["W"], sc["H"]
    tw, th = -(-W // TILE), -(-H // TILE)
    nt = tw * th
    b = np.arange(C * nt)
    cam, t = b // nt, b % nt
    ly, lx = np.divmod(np.arange(TILE * TILE), TILE)
    x = (t % tw)[:, None] * TILE + lx[None]
    y = (t // tw)[:, None] * TILE + ly[None]
    inside = (x < W) & (y < H)
    pix = np.where(inside, (cam[:, None] * H + np.minimum(y, H - 1)) * W + np.minimum(x, W - 1), 0)
    return dict(cam=cam, x=x, y=y, px=x + 0.5, py=y + 0.5, inside=inside, pix=pix, lx=lx, ly=ly)


def _abscross(a, b):
    return np.stack([a[..., 1] * b[..., 2] + a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] + a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] + a[..., 1] * b[..., 0]], -1)


def _geom(M, P):
    """per (bin, pixel): h_u, h_v, zeta, (u, v), sigma, depth, vis and the conditioning term K."""
    Mu, Mv, Mw = M[:, None, 0:3], M[:, None, 3:6], M[:, None, 6:9]
    px, py = P["px"][..., None], P["py"][..., None]
    hu, hv = px * Mw - Mu, py * Mw - Mv
    z = np.cross(hu, hv)
    zz = z[..., 2]
    with np.errstate(divide="ignore", invalid="ignore"):
        sx, sy = z[..., 0] / zz, z[..., 1] / zz
        sigma = 0.5 * (sx * sx + sy * sy)
        depth = sx * Mw[..., 0] + sy * Mw[..., 1] + Mw[..., 2]
        vis = np.exp(-sigma)
        dhu, dhv = U * (np.abs(px * Mw) + np.abs(Mu)), U * (np.abs(py * Mw) + np.abs(Mv))
        dz = _abscross(dhu, np.abs(hv)) + _abscross(np.abs(hu), dhv)
        dsx = (dz[..., 0] + np.abs(sx) * dz[..., 2]) / np.abs(zz)
        dsy = (dz[..., 1] + np.abs(sy) * dz[..., 2]) / np.abs(zz)
        K = (np.abs(sx) * dsx + np.abs(sy) * dsy + dsx + dsy) / U + 2.0 + 1.2 * sigma
    return dict(hu=hu, hv=hv, zz=zz, sx=sx, sy=sy, sigma=sigma, depth=depth, vis=vis, K=K, Mw=M[:, 6:9])


def _rel(v, t):
    return np.abs(v / t - 1.0)


def forward(sc, off, flat):
    """fp64 forward: images [C, H, W, .], last_ids, median_ids, visibilities [nnz], the error scales img_scale / vis_scale, the composited
    count N [nb, 256], the minimum margin of each decision, and (splat, log opacity step) pairs that move every decision closer than NUDGE to its
    threshold away from it."""
    C, W, H = sc["C"], sc["W"], sc["H"]
    P = _pixels(sc)
    start, L, G, IDX = lists_of(off, flat)
    nb = len(start)
    Mall = np.asarray(sc["ray_transforms"], np.float64).reshape(-1, 9)
    opac = np.asarray(sc["opacities"], np.float64)
    col, nrm = np.asarray(sc["colors"], np.float64), np.asarray(sc["normals"], np.float64)
    nnz = len(opac)
    shp = (nb, TILE * TILE)
    T = np.ones(shp)
    done = ~P["inside"]
    pc, pn = np.zeros(shp + (3,)), np.zeros(shp + (3,))
    dout, med_d = np.zeros(shp), np.zeros(shp)
    cur, med = np.zeros(shp, np.int64), np.zeros(shp, np.int64)
    N, sumK = np.zeros(shp), np.zeros(shp)
    s_col, s_nrm, s_dep, s_alp, s_med = np.zeros(shp + (3,)), np.zeros(shp + (3,)), np.zeros(shp), np.zeros(shp), np.zeros(shp)
    med_m = np.full(shp, np.inf)
    vis_acc, vis_scale = np.zeros(nnz), np.zeros(nnz)
    mins = dict(alpha=np.inf, clip=np.inf, stop=np.inf, depth=np.inf)
    nudges = []
    for k in range(G.shape[1]):
        gb = G[:, k]
        live = gb >= 0
        if not live.any():
            break
        gg = np.maximum(gb, 0)
        g = _geom(Mall[gg], P)
        cand = live[:, None] & ~done
        a0 = opac[gg][:, None] * g["vis"]
        alpha = np.minimum(CLIP, a0)
        ok = cand & (g["zz"] != 0) & ~(g["depth"] < NEAR) & ~(g["sigma"] < 0) & ~(alpha < ALPHA_T)
        m_a, m_d = _rel(alpha, ALPHA_T), _rel(g["depth"], NEAR)
        next_T = T * (1.0 - alpha)
        stop = ok & (next_T <= T_STOP)
        m_s = _rel(next_T, T_STOP)
        comp = ok & ~stop
        m_c, m_m = _rel(a0, CLIP), _rel(T, 0.5)
        # nudges: a log-factor for the opacity of the splat that moves the decision away from its threshold by about 2 NUDGE
        up = lambda v, t: np.where(v >= t, 1.0, -1.0)
        lev = alpha / np.maximum(1.0 - alpha, 1e-6)  # -d ln T' / d ln opacity
        for name, m, where, step in (("alpha", m_a, cand, up(alpha, ALPHA_T) * 2 * NUDGE), ("depth", m_d, cand, 0.0 * m_a),
                                     ("stop", m_s, ok, -up(next_T, T_STOP) * 2 * NUDGE / np.maximum(lev, 1e-3)),
                                     ("clip", m_c, comp, -up(a0, CLIP) * 2 * NUDGE)):
            if where.any():
                mins[name] = min(mins[name], float(m[where].min()))
                hit = where & (m < NUDGE)
                nudges.extend(zip(np.broadcast_to(gb[:, None], shp)[hit].tolist(), np.broadcast_to(step, shp)[hit].tolist()))
        # T vs 0.5 picks render_median / median_ids only: not nudged (the tests give render_median a zero cotangent and compare the
        # median outputs where this margin clears 1e-3), recorded per pixel
        med_m = np.where(comp, np.minimum(med_m, m_m), med_m)
        done |= stop
        vis = np.where(comp, alpha * T, 0.0)
        N += comp
        f = N + 4.0 + np.where(comp, g["K"], 0.0)
        c3, n3 = col[gg][:, None], nrm[gg][:, None]
        pc += c3 * vis[..., None]
        pn += n3 * vis[..., None]
        dout += np.where(comp, g["depth"], 0.0) * vis
        s_col += np.abs(c3) * (vis * f)[..., None]
        s_nrm += np.abs(n3) * (vis * f)[..., None]
        s_dep += np.abs(np.where(comp, g["depth"], 0.0)) * vis * f
        s_alp += vis * f
        sumK += np.where(comp, g["K"], 0.0)
        mc = comp & (T > 0.5)
        med_d = np.where(mc, g["depth"], med_d)
        s_med = np.where(mc, np.abs(g["depth"]) * (4.0 + g["K"]), s_med)
        med = np.where(mc, IDX[:, k][:, None], med)
        cur = np.where(comp, IDX[:, k][:, None], cur)
        T = np.where(comp, next_T, T)
        np.add.at(vis_acc, gg[live], vis.sum(1)[live])
        np.add.at(vis_scale, gg[live], (vis * f).sum(1)[live])
    ins = P["inside"]
    bg = np.zeros((C, 3)) if sc.get("backgrounds") is None else np.asarray(sc["backgrounds"], np.float64)
    bgp = bg[P["cam"]][:, None]
    Tf = T
    img = dict(render_colors=pc + Tf[..., None] * bgp, render_depths=dout, render_alphas=1.0 - Tf, render_normals=pn,
               render_median=med_d, last_ids=cur, median_ids=med, median_margin=med_m)
    tscale = Tf * (N + 4.0 + sumK)
    scl = dict(render_colors=s_col + (tscale[..., None] * np.abs(bgp)), render_depths=s_dep, render_alphas=s_alp + tscale,
               render_normals=s_nrm, render_median=s_med)
    shape = dict(render_colors=(C, H, W, 3), render_normals=(C, H, W, 3), last_ids=(C, H, W), median_ids=(C, H, W))

    def scatter(v, name):
        out = np.zeros((C * H * W,) + v.shape[2:], v.dtype)
        out[P["pix"][ins]] = v[ins]
        return out.reshape(shape.get(name, (C, H, W, 1)))

    out = {k: scatter(v, k) for k, v in img.items()}
    out["last_ids"] = out["last_ids"].astype(np.int32)
    out["median_ids"] = out["median_ids"].astype(np.int32)
    out["img_scale"] = {k: scatter(v, k) for k, v in scl.items()}
    out.update(visibilities=vis_acc, vis_scale=vis_scale, N=N, margins=mins, nudges=nudges)
    return out


def backward(sc, off, flat, state, ct, N=None):
    """fp64 backward from a forward state (render_alphas, last_ids, median_ids) and cotangents. Returns rec [nnz, 16] (the kernel's record
    layout), the scales A and (with N, the composited count per pixel from `forward`) A_state, absgrad [nnz, 2] per 8x8 block with its
    scales, and absgrad_8x4 [nnz, 2] (the same per 8x4 block)."""
    C, W, H = sc["C"], sc["W"], sc["H"]
    P = _pixels(sc)
    start, L, G, IDX = lists_of(off, flat)
    nb = len(start)
    Mall = np.asarray(sc["ray_transforms"], np.float64).reshape(-1, 9)
    opac = np.asarray(sc["opacities"], np.float64)
    col, nrm = np.asarray(sc["colors"], np.float64), np.asarray(sc["normals"], np.float64)
    nnz = len(opac)
    ins, pix = P["inside"], P["pix"]
    gp = lambda a, d: np.asarray(a, np.float64).reshape(-1, d)[pix]
    Tf = np.where(ins, 1.0 - gp(state["render_alphas"], 1)[..., 0], 1.0)
    bin_final = np.where(ins, np.asarray(state["last_ids"]).reshape(-1)[pix], -1)
    med_idx = np.where(ins, np.asarray(state["median_ids"]).reshape(-1)[pix], -1)
    z = lambda a, d: np.where(ins[..., None], gp(a, d), 0.0)
    vc, vn = z(ct["v_render_colors"], 3), z(ct["v_render_normals"], 3)
    vd, va, vmed = z(ct["v_render_depths"], 1)[..., 0], z(ct["v_render_alphas"], 1)[..., 0], z(ct["v_render_median"], 1)[..., 0]
    bg = np.zeros((C, 3)) if sc.get("backgrounds") is None else np.asarray(sc["backgrounds"], np.float64)
    bgp = bg[P["cam"]][:, None]
    va_eff = Tf * (va - (bgp * vc).sum(-1))
    va_abs = Tf * (np.abs(va) + (np.abs(bgp) * np.abs(vc)).sum(-1))
    shp = (nb, TILE * TILE)
    T = Tf.copy()
    buf, bufn, bufn_abs = np.zeros(shp + (3,)), np.zeros(shp + (3,)), np.zeros(shp + (3,))
    bufd = np.zeros(shp)
    n = np.zeros(shp)
    rec, A, A_state = np.zeros((nnz, 16)), np.zeros((nnz, 16)), np.zeros((nnz, 16))
    absg, absg84, A_abs, A_abs_state = np.zeros((nnz, 2)), np.zeros((nnz, 2)), np.zeros((nnz, 2)), np.zeros((nnz, 2))
    blk8 = (P["lx"] >= 8).astype(int) + 2 * (P["ly"] >= 8)
    blk4 = (P["lx"] >= 8).astype(int) + 2 * (P["ly"] // 4)
    oh8, oh4 = np.eye(4)[blk8], np.eye(8)[blk4]  # [256, blocks]
    for k in reversed(range(G.shape[1])):
        gb = G[:, k]
        live = gb >= 0
        if not live.any():
            continue
        gg = np.maximum(gb, 0)
        g = _geom(Mall[gg], P)
        idx = IDX[:, k][:, None]
        o = opac[gg][:, None]
        a0 = o * g["vis"]
        alpha = np.minimum(CLIP, a0)
        valid = live[:, None] & ins & (idx <= bin_final) & (g["zz"] != 0) & ~(g["depth"] < NEAR) & ~(g["sigma"] < 0) & ~(alpha < ALPHA_T)
        alpha = np.where(valid, alpha, 0.0)
        ra = 1.0 / (1.0 - alpha)
        T = np.where(valid, T * ra, T)
        fac = alpha * T
        c3, n3 = col[gg][:, None], nrm[gg][:, None]
        depth = np.where(valid, g["depth"], 0.0)
        t = np.zeros(shp + (16,))
        ta = np.zeros(shp + (16,))
        t[..., 0:3], ta[..., 0:3] = fac[..., None] * vc, fac[..., None] * np.abs(vc)
        t[..., 3:6], ta[..., 3:6] = fac[..., None] * vn, fac[..., None] * np.abs(vn)
        v_alpha = (((c3 * T[..., None] - buf * ra[..., None]) * vc).sum(-1) + ((n3 * T[..., None] - bufn * ra[..., None]) * vn).sum(-1)
                   + ra * va_eff + (depth * T - bufd * ra) * vd)
        v_alpha_abs = (((np.abs(c3) * T[..., None] + buf * ra[..., None]) * np.abs(vc)).sum(-1)
                       + ((np.abs(n3) * T[..., None] + bufn_abs * ra[..., None]) * np.abs(vn)).sum(-1)
                       + ra * va_abs + (np.abs(depth) * T + bufd * ra) * np.abs(vd))
        unclip = valid & (a0 <= CLIP)
        v_depth = np.where(idx == med_idx, vmed, 0.0) + fac * vd
        v_depth_abs = np.where(idx == med_idx, np.abs(vmed), 0.0) + fac * np.abs(vd)
        v_G, v_G_abs = o * v_alpha, o * v_alpha_abs
        sx, sy, vis, Mw = g["sx"], g["sy"], g["vis"], g["Mw"][:, None]
        with np.errstate(divide="ignore", invalid="ignore"):
            izz = np.where(valid, 1.0 / g["zz"], 0.0)
        vsxz = (-v_G * vis * sx + v_depth * Mw[..., 0]) * izz
        vsyz = (-v_G * vis * sy + v_depth * Mw[..., 1]) * izz
        vsxz_a = (v_G_abs * vis * np.abs(sx) + v_depth_abs * np.abs(Mw[..., 0])) * np.abs(izz)
        vsyz_a = (v_G_abs * vis * np.abs(sy) + v_depth_abs * np.abs(Mw[..., 1])) * np.abs(izz)
        vrc = np.stack([vsxz, vsyz, -(vsxz * sx + vsyz * sy)], -1)
        vrc_a = np.stack([vsxz_a, vsyz_a, vsxz_a * np.abs(sx) + vsyz_a * np.abs(sy)], -1)
        vhu, vhv = np.cross(g["hv"], vrc), np.cross(vrc, g["hu"])
        vhu_a, vhv_a = _abscross(np.abs(g["hv"]), vrc_a), _abscross(vrc_a, np.abs(g["hu"]))
        px, py = P["px"][..., None], P["py"][..., None]
        zw = np.stack([sx, sy, np.ones_like(sx)], -1)
        t[..., 6:9], ta[..., 6:9] = -vhu, vhu_a
        t[..., 9:12], ta[..., 9:12] = -vhv, vhv_a
        t[..., 12:15] = px * vhu + py * vhv + v_depth[..., None] * zw
        ta[..., 12:15] = px * vhu_a + py * vhv_a + v_depth_abs[..., None] * np.abs(zw)
        t[..., 15], ta[..., 15] = vis * v_alpha, vis * v_alpha_abs
        t[..., 6:] *= unclip[..., None]
        ta[..., 6:] *= unclip[..., None]
        t *= valid[..., None]
        ta *= valid[..., None]
        n += valid
        Kv = np.where(valid, g["K"], 0.0)
        f = n + 4.0 + Kv
        fs = (N if N is not None else n) + 4.0 + Kv
        np.add.at(rec, gg[live], t.sum(1)[live])
        np.add.at(A, gg[live], (ta * f[..., None]).sum(1)[live])
        np.add.at(A_state, gg[live], (ta * fs[..., None]).sum(1)[live])
        mz = np.abs(Mw[:, 0, 2])[:, None]
        uv = t[..., [8, 11]]
        absg_t = (np.abs(np.einsum("bpk,pq->bqk", uv, oh8)).sum(1)) * mz
        absg84_t = (np.abs(np.einsum("bpk,pq->bqk", uv, oh4)).sum(1)) * mz
        np.add.at(absg, gg[live], absg_t[live])
        np.add.at(absg84, gg[live], absg84_t[live])
        np.add.at(A_abs, gg[live], ((ta[..., [8, 11]] * f[..., None]).sum(1) * mz)[live])
        np.add.at(A_abs_state, gg[live], ((ta[..., [8, 11]] * fs[..., None]).sum(1) * mz)[live])
        buf += c3 * fac[..., None]
        bufn += n3 * fac[..., None]
        bufn_abs += np.abs(n3) * fac[..., None]
        bufd += depth * fac
    return dict(rec=rec, A=A, A_state=A_state, absgrad=absg, absgrad_8x4=absg84, A_absgrad=A_abs, A_absgrad_state=A_abs_state)


def split_record(rec, ray_transforms):
    """[nnz, 16] record -> the raster backward's outputs (v_densify from the record's M_u.z, M_v.z times M_w.z, as the kernel's
    finalize pass)."""
    mz = np.asarray(ray_transforms, np.float64).reshape(-1, 9)[:, 8:9]
    return dict(v_colors=rec[:, 0:3], v_normals=rec[:, 3:6], v_ray_transforms=rec[:, 6:15].reshape(-1, 3, 3), v_opacities=rec[:, 15],
                v_densify=rec[:, [8, 11]] * mz)
