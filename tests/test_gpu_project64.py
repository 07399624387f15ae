"""The projection kernels (csrc/gh_project.cu, gh_strands.cu) per Gaussian against the float64 replay of
tests/_project64.py: every output and gradient element within the replay's error bound, every decided branch taken
as the replay takes it, culled rows exactly zero, the 29 camera gradients within their summed bounds.  The bounds
are rehearsed on the host build of the same header by tests/test_project64_cpu.py.

Through the product's wrappers (projection.project_forward / project_backward, strand_midpoints, strand_backward,
the capturable and the hair-segment / hair-strand entry points) at CTA tails (P = 1, 127, 128, 129, 255, 2^20), an
f_rest view that is 4- but not 16-byte aligned (the scalar staging branch), the hand-built decision edges, the strand
form's degenerate segments and every activation code."""
import numpy as np
import pytest
import torch

import _project64 as p64

pytestmark = pytest.mark.gpu
UNRESOLVED_CAP = 0.05            # as in test_project64_cpu.py


def _t(a, dev, *shape):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(np.asarray(a, np.float32).reshape(*shape))).to(dev)


def pack(sc, dev, misalign_rest=False):
    from gaussianhaircut_b200 import projection
    P, c, cfg = sc["P"], sc["cam"], sc["cfg"]
    strand = bool(cfg.get("strands"))
    f_rest = _t(sc["f_rest"], dev, P, 15, 3)
    if misalign_rest:
        buf = torch.zeros(P * 45 + 1, device=dev)
        buf[1:] = f_rest.reshape(-1)
        f_rest = buf[1:].view(P, 15, 3)
        assert f_rest.data_ptr() % 16 == 4
    return projection.pack_inputs(
        _t(sc["xyz"], dev, P, 3), _t(sc["scaling"], dev, 1) if strand else _t(sc["scaling"], dev, P, 3),
        None if strand else _t(sc["rotation"], dev, P, 4), _t(sc["dirs"], dev, P, 3), _t(sc["f_dc"], dev, P, 1, 3), f_rest,
        _t(sc["opacity"], dev, P, 1), _t(sc["label"], dev, P, 1), _t(sc["conf"], dev, P, 1), _t(c["V"], dev, 4, 4),
        _t(c["Pm"], dev, 4, 4), _t(c["campos"], dev, 3), c["tanx"], c["tany"], c["W"], c["H"], sc["deg"], sc["mod"], cfg)


def incoming(gi, dev):
    P = gi["m2x"].shape[0]
    m2 = torch.zeros(P, 3, device=dev)
    m2[:, 0] = torch.from_numpy(gi["m2x"]).to(dev); m2[:, 1] = torch.from_numpy(gi["m2y"]).to(dev)
    con = torch.from_numpy(gi["con"]).to(dev)
    conic4 = torch.zeros(P, 2, 2, device=dev)
    conic4[:, 0, 0] = con[:, 0]; conic4[:, 0, 1] = 0.5 * con[:, 1]; conic4[:, 1, 1] = con[:, 2]
    return dict(dL_dmeans2D=m2, dL_dconic4=conic4, dL_dcolors=torch.from_numpy(gi["color"]).to(dev),
                dL_dopacity=torch.from_numpy(gi["opacity"]).to(dev).reshape(P, 1))


def _np(t):
    return None if t is None else t.detach().cpu().numpy()


def forward_dict(out):
    return {"means2D": _np(out["means2D"]), "conic": _np(out["conic"]), "colors": _np(out["colors"]),
            "opacity": _np(out["opacity"]).reshape(-1), "visible": _np(out["visible"]).astype(bool), "cov3D": _np(out.get("cov3D"))}


def backward_dict(d):
    return {k: _np(d.get(src)) for k, src in (("xyz", "xyz"), ("scaling", "scaling"), ("rotation", "rotation"), ("dirs", "dirs"),
                                              ("f_dc", "f_dc"), ("rest", "f_rest"), ("opacity", "opacity"), ("label", "label"),
                                              ("conf", "conf"))}


def camera37(d):
    return torch.cat([d["viewmatrix"].reshape(16), d["projmatrix"].reshape(16), d["campos"].reshape(3), d["tanfov"].reshape(2)])


CASES = {
    **{f"gaussian_model_P{P}": (lambda P=P: p64.random_scene(P, P, "gaussian_model", deg=3), False) for P in (1, 127, 128, 129, 255)},
    "gaussian_model_P1M": (lambda: p64.random_scene(1 << 20, 12, "gaussian_model", deg=3, W=1920, H=1080), False),
    "gaussian_model_misaligned_rest": (lambda: p64.random_scene(255, 13, "gaussian_model", deg=3), True),
    "gaussian_model_deg1_mod": (lambda: p64.random_scene(5000, 2, "gaussian_model", deg=1, mod=0.7), False),
    "hair_P129": (lambda: p64.random_scene(129, 3, "hair", deg=3), False),
    "hair_P100k": (lambda: p64.random_scene(100000, 3, "hair", deg=3), False),
    "head_P255": (lambda: p64.random_scene(255, 4, "head", deg=0), False),
    "identity_P129": (lambda: p64.random_scene(129, 5, "identity", deg=2), False),
    "strands_P255": (lambda: p64.random_scene(255, 6, "strands", deg=3), False),
    "strands_P100k_misaligned_rest": (lambda: p64.random_scene(100000, 6, "strands", deg=3), True),
    "strand_edges": (p64.strand_edge_scene, False),
    "edges": (lambda: p64.edge_scene()[0], False),
}


@pytest.mark.parametrize("case", list(CASES))
def test_kernels_lie_within_the_bound(cuda_device, case):
    from gaussianhaircut_b200 import projection
    build, misalign = CASES[case]
    sc = build()
    P = sc["P"]
    pi = pack(sc, cuda_device, misalign)
    out = projection.project_forward(pi, want_cov3D=True)
    A = p64.inputs(sc)
    rp = p64.Replay(P)
    o, g = p64.forward(rp, A)
    gi = p64.neutralize(rp, p64.random_grads(P, 17))
    d = projection.project_backward(pi, out["visible"], camera_grads=True, **incoming(gi, cuda_device))
    torch.cuda.synchronize()
    got_f = forward_dict(out)
    stats = p64.Stats()
    p64.check_forward(rp, o, got_f, stats, P)
    go, cam = p64.backward(rp, A, gi, got_f["visible"], g)
    p64.check_backward(rp, go, cam, backward_dict(d), stats, P, _np(camera37(d)))
    amb = {k: int(v.sum()) for k, v in rp.amb.items() if v.any()}
    print(f"\n[{case}] ambiguous {amb or 0}, unresolved rows {int(rp.unres.sum())}, "
          f"unresolved elements {stats.unresolved_fraction():.2e}\n  {stats}")
    assert stats.unresolved_fraction() <= UNRESOLVED_CAP

    # the capturable backward, given the same tan(fov / 2), is its non-capturable twin bit for bit
    tan = torch.tensor([sc["cam"]["tanx"], sc["cam"]["tany"]], dtype=torch.float32, device=cuda_device)
    d2 = projection.project_backward(pi, out["visible"], camera_grads=True, tan_fov=tan, **incoming(gi, cuda_device))
    for k in ("xyz", "scaling", "rotation", "dirs", "f_dc", "f_rest", "opacity", "label", "conf"):
        if d[k] is not None:
            assert torch.equal(d[k], d2[k]), k
    assert torch.equal(camera37(d), camera37(d2))


def test_colour_clamp_keeps_its_gradient_at_exactly_zero(cuda_device):
    from gaussianhaircut_b200 import projection
    from test_project64_cpu import check_colour_tie
    sc, accs, kk, B = p64.colour_tie_scene()
    pi = pack(sc, cuda_device)
    out = projection.project_forward(pi)
    gi = p64.random_grads(sc["P"], 3)
    gi["color"][:] = 1.0
    d = projection.project_backward(pi, out["visible"], camera_grads=False, **incoming(gi, cuda_device))
    torch.cuda.synchronize()
    colors = _np(out["colors"])
    assert colors[0, 0] == 0.0 and colors[1, 1] > 0.0 and colors[2, 2] == 0.0
    check_colour_tie(forward_dict(out), backward_dict(d), kk, B)


def _acc16(geom, P):
    a = lambda n: (n + 255) // 256 * 256  # noqa: E731
    off = a(P * 32) + a(P * 4)
    return geom[off:off + 64 * P].view(torch.float32).view(P, 16).clone()


@pytest.mark.parametrize("cfg_name", ["gaussian_model", "strands"])
def test_geom_buffer_backward_equals_the_explicit_gradient_path(cuda_device, cfg_name):
    """project_backward(geom_buffer=...) fed a real blend backward's records == the explicit-tensor path fed the
    same gradients, bit for bit; and the capturable first phases equal their non-capturable twins"""
    from gaussianhaircut_b200 import projection, _C
    sc = p64.random_scene(20000, 31, cfg_name, deg=3)
    P, W, H = sc["P"], sc["cam"]["W"], sc["cam"]["H"]
    dev = cuda_device
    pi = pack(sc, dev)
    bg = torch.zeros(10, device=dev)
    b, radii, geom, img, R, max_len = projection.project_forward_binned(pi)
    _color, binning = _C.forward_render(bg, b["colors"], radii, geom, img, R, max_len, H, W)
    dL = torch.from_numpy(np.random.default_rng(2).normal(size=(10, H, W)).astype(np.float32)).to(dev)
    _C.rasterize_gaussians_backward_records(bg, pi.xyz, radii, b["colors"], b["conic"], pi.V, pi.Pm, pi.tanx, pi.tany, dL,
                                            pi.campos, geom, R, binning, img, False)
    rec = _acc16(geom, P)
    d_rec = projection.project_backward(pi, b["visible"], geom_buffer=geom, camera_grads=True)
    m2 = torch.zeros(P, 3, device=dev)
    m2[:, :2] = rec[:, 10:12]
    conic4 = torch.stack([rec[:, 12], rec[:, 13], torch.zeros_like(rec[:, 12]), rec[:, 14]], dim=-1).contiguous()
    d_exp = projection.project_backward(pi, b["visible"], dL_dmeans2D=m2, dL_dconic4=conic4, dL_dcolors=rec[:, :10].contiguous(),
                                        dL_dopacity=rec[:, 15:16].contiguous(), camera_grads=True)
    torch.cuda.synchronize()
    assert int(b["visible"].sum()) > 0 and float(rec.abs().sum()) > 0
    for k in ("xyz", "scaling", "rotation", "dirs", "f_dc", "f_rest", "opacity", "label", "conf"):
        if d_rec[k] is not None:
            assert torch.equal(d_rec[k], d_exp[k]), k
    assert torch.equal(camera37(d_rec), camera37(d_exp))

    # capturable first phases, given the same tan(fov / 2)
    tan = torch.tensor([sc["cam"]["tanx"], sc["cam"]["tany"]], dtype=torch.float32, device=dev)
    cap = max(4 * R, 1024)
    binning_c = _C.binning_workspace(cap, dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    if cfg_name == "gaussian_model":
        c_out, c_radii, _g, _i = projection.project_forward_binned_capturable(pi, tan, binning_c, cap, status)
    else:
        sp = projection.pack_segment_inputs(None, pi.xyz, pi.dirs, pi.scaling, pi.f_dc, pi.f_rest, pi.conf, pi.V, pi.Pm, pi.campos,
                                            tan, W, H, sc["deg"], sc["mod"])
        c_out, c_radii, _g, _i = projection.hair_segments_forward_binned_capturable(sp, binning_c, cap, status)
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    for k in ("means2D", "colors", "opacity", "conic", "visible"):
        assert torch.equal(c_out[k], b[k]), k
    assert torch.equal(c_radii, radii)


@pytest.mark.parametrize("L", [1, 31, 32, 33, 100])
def test_strand_kernels_lie_within_the_bound(cuda_device, L):
    """strand_midpoints and the suffix-sum strand_backward, and the capturable strand first phase's midpoints and
    segment rows against the two eager kernels"""
    from gaussianhaircut_b200 import projection, _C
    dev = cuda_device
    rng = np.random.default_rng(L)
    S = 300
    origins = rng.normal(0, 0.2, (S, 1, 3)).astype(np.float32)
    dirs = (rng.normal(0, 1, (S, L, 3)) * 4e-3).astype(np.float32)
    dirs[0, 0] = 0.0                                                    # a zero-length segment
    xyz = torch.empty(S * L, 3, device=dev)
    projection.strand_midpoints(torch.from_numpy(origins).to(dev), torch.from_numpy(dirs).to(dev), out=xyz)
    gx = rng.normal(size=(S, L, 3)).astype(np.float32)
    direct = rng.normal(size=(S, L, 3)).astype(np.float32)
    dd = torch.from_numpy(direct.reshape(S * L, 3)).to(dev)
    out = projection.strand_backward(S, L, torch.from_numpy(gx.reshape(S * L, 3)).to(dev), dd)
    torch.cuda.synchronize()
    stats = p64.Stats()
    v, e = p64.strand_midpoints(origins[:, 0], dirs)
    p64.within(stats, "midpoints", _np(xyz).reshape(S, L, 3), p64.E(v, e))
    v, e = p64.strand_backward(gx, direct)
    p64.within(stats, "strand_backward", _np(out), p64.E(v, e))
    print(f"\n[L={L}] {stats}")

    # the capturable strand first phase: its midpoints and segment rows equal the eager kernels'
    sc = p64.random_scene(S * L, L, "strands", deg=3)
    cam = sc["cam"]
    tan = torch.tensor([cam["tanx"], cam["tany"]], dtype=torch.float32, device=dev)
    t = lambda a, *shape: _t(a, dev, *shape)  # noqa: E731
    sp = projection.pack_strand_inputs(None, t(origins, S, 1, 3), t(dirs, S, L, 3), t(sc["scaling"], 1), t(sc["f_dc"], S * L, 1, 3),
                                       t(sc["f_rest"], S * L, 15, 3), t(sc["conf"], S * L, 1), t(cam["V"], 4, 4), t(cam["Pm"], 4, 4),
                                       t(cam["campos"], 3), tan, cam["W"], cam["H"], 3, 1.0)
    cap = 1 << 20
    c_out, c_radii, _g, _i, mid = projection.hair_strands_forward_binned_capturable(sp, _C.binning_workspace(cap, dev), cap,
                                                                                    torch.zeros(1, dtype=torch.int32, device=dev))
    sc.update(xyz=_np(xyz), dirs=dirs.reshape(S * L, 3), mod=1.0)
    b, radii, *_ = projection.project_forward_binned(pack(sc, dev))
    torch.cuda.synchronize()
    assert torch.equal(mid, xyz)
    for k in ("means2D", "colors", "opacity", "conic", "visible"):
        assert torch.equal(c_out[k], b[k]), k
    assert torch.equal(c_radii, radii)
