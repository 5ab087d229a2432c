"""Bring-up diagnostics for the CUDA ops (run on an H100).  Prints one line per check and never stops at the
first failure, so that a single GPU call yields a complete picture.  Usage: python tests/gpu_diag.py [section ...]"""
import math
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from micro_sam_b200 import _lib  # noqa: E402

torch.backends.cuda.matmul.allow_tf32 = False
torch.backends.cudnn.allow_tf32 = False
DEV = "cuda" if torch.cuda.is_available() else "cpu"
RESULTS = []


def report(name, got, ref, tol):
    got, ref = got.float(), ref.float()
    err = (got - ref).abs()
    rel = (got - ref).norm() / (ref.norm() + 1e-12)
    ok = bool(rel < tol) and bool(torch.isfinite(got).all())
    RESULTS.append(ok)
    print(f"[{'OK ' if ok else 'BAD'}] {name}: rel_l2={rel:.3e} max_abs={err.max():.3e} ref_absmax={ref.abs().max():.3e} "
          f"finite={bool(torch.isfinite(got).all())}", flush=True)
    if not ok:
        bad = (err > 10 * tol * ref.abs().max()).nonzero()
        print(f"      n_bad={len(bad)} of {got.numel()}  first bad idx: {bad[:8].tolist()}", flush=True)
        if got.ndim == 2:
            rows = torch.unique(bad[:, 0])[:16].tolist()
            cols = torch.unique(bad[:, 1])[:16].tolist()
            print(f"      bad rows(first16)={rows} bad cols(first16)={cols}", flush=True)
            print(f"      got[0,:8]={got[0,:8].tolist()}\n      ref[0,:8]={ref[0,:8].tolist()}", flush=True)
    return ok


def gemm(A, W, bias=None, residual=None, res_rows=0, out_fp32=False, act=0):
    M, K = A.shape
    N = W.shape[0]
    out = torch.empty(M, N, device=DEV, dtype=torch.float32 if out_fp32 else torch.bfloat16)
    L = _lib.lib()
    _lib.check(L.msam_op_gemm(_lib.ptr(A), _lib.ptr(W), M, N, K, _lib.ptr(bias), _lib.ptr(residual), res_rows,
                              _lib.ptr(out), int(out_fp32), act, _lib.cur_stream()))
    torch.cuda.synchronize()
    return out


def sec_gemm():
    g = torch.Generator(device="cpu").manual_seed(0)
    cases = [
        # M, N, K, bias, act, residual(res_rows), out_fp32
        (128, 256, 64, False, 0, 0, True),
        (128, 256, 128, False, 0, 0, True),
        (256, 256, 256, True, 0, 0, True),
        (4096, 768, 768, True, 1, 0, False),
        (1000, 2304, 768, True, 0, 0, False),
        (4096, 768, 3072, True, 0, 4096, True),
        (8192, 768, 768, True, 0, 4096, True),
        (300, 128, 256, True, 2, 0, False),
        (300, 96, 128, True, 0, 0, True),
        (4096, 256, 2304, False, 0, 0, True),
        (2 * 4900, 480, 160, True, 0, 0, False),
        (4096 * 4, 3072, 768, True, 1, 0, False),
    ]
    for (M, N, K, hb, act, rr, f32) in cases:
        A = (torch.randn(M, K, generator=g) * 0.5).to(DEV).bfloat16()
        W = (torch.randn(N, K, generator=g) / math.sqrt(K)).to(DEV).bfloat16()
        bias = torch.randn(N, generator=g).to(DEV) if hb else None
        res = torch.randn(rr, N, generator=g).to(DEV) if rr else None
        try:
            out = gemm(A, W, bias, res, rr, f32, act)
        except Exception as e:  # noqa: BLE001
            RESULTS.append(False)
            print(f"[BAD] gemm M={M} N={N} K={K}: EXCEPTION {e}", flush=True)
            continue
        ref = A.float() @ W.float().t()
        if hb:
            ref = ref + bias
        if act == 1:
            ref = torch.nn.functional.gelu(ref)
        elif act == 2:
            ref = torch.relu(ref)
        if rr:
            ref = ref + res.repeat(M // rr, 1)
        report(f"gemm M={M} N={N} K={K} bias={hb} act={act} res={rr} f32={f32}", out, ref, 1e-5 if f32 else 5e-3)
    # timing of a big one
    M, N, K = 16 * 4096, 3072, 768
    A = torch.randn(M, K, device=DEV).bfloat16()
    W = torch.randn(N, K, device=DEV).bfloat16()
    bias = torch.randn(N, device=DEV)
    for name, kw in (("fc1+gelu bf16out", dict(act=1)), ("plain bf16out", dict())):
        gemm(A, W, bias, **kw)
        t0 = torch.cuda.Event(enable_timing=True)
        t1 = torch.cuda.Event(enable_timing=True)
        out = torch.empty(M, N, device=DEV, dtype=torch.bfloat16)
        L = _lib.lib()
        t0.record()
        for _ in range(5):
            L.msam_op_gemm(_lib.ptr(A), _lib.ptr(W), M, N, K, _lib.ptr(bias), None, 0, _lib.ptr(out), 0, kw.get("act", 0),
                           _lib.cur_stream())
        t1.record()
        torch.cuda.synchronize()
        ms = t0.elapsed_time(t1) / 5
        print(f"[perf] gemm {name} M={M} N={N} K={K}: {ms:.3f} ms  {2*M*N*K/ms/1e9:.1f} TFLOP/s", flush=True)
    t0 = torch.cuda.Event(enable_timing=True); t1 = torch.cuda.Event(enable_timing=True)
    (A @ W.t())
    t0.record()
    for _ in range(5):
        (A @ W.t())
    t1.record(); torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / 5
    print(f"[perf] cublas same shape: {ms:.3f} ms  {2*M*N*K/ms/1e9:.1f} TFLOP/s", flush=True)


def sec_wgrad():
    """First backward piece (cfg 5): dW = dY^T X through msam_op_gemm_tn (MN-major operands) against torch AUTOGRAD of
    nn.Linear on the same bf16 inputs (fp32 accumulation both sides)."""
    g = torch.Generator(device="cpu").manual_seed(1)
    for (T, O, I) in ((256, 128, 128), (4096, 768, 768), (4096 * 2, 2304, 768), (1000, 256, 200), (4096, 3072, 768)):
        x = (torch.randn(T, I, generator=g) * 0.5).to(DEV).bfloat16()
        dy = (torch.randn(T, O, generator=g) * 0.5).to(DEV).bfloat16()
        lin = torch.nn.Linear(I, O, bias=False).to(DEV)
        y = lin(x.float())
        y.backward(dy.float())
        out = torch.empty(O, I, device=DEV, dtype=torch.float32)
        try:
            _lib.check(_lib.lib().msam_op_gemm_tn(_lib.ptr(dy), _lib.ptr(x), O, I, T, _lib.ptr(out), _lib.cur_stream()))
            torch.cuda.synchronize()
        except Exception as e:  # noqa: BLE001
            RESULTS.append(False)
            print(f"[BAD] wgrad T={T} O={O} I={I}: EXCEPTION {e}", flush=True)
            continue
        report(f"wgrad dW = dY^T X  T={T} O={O} I={I} (vs autograd)", out, lin.weight.grad, 1e-5)
        # dgrad through the same kernel family: dX = dY W with W = the forward weight [O, I] (bf16), vs autograd
        xg = x.float().requires_grad_(True)
        wb = lin.weight.detach().bfloat16()
        (xg @ wb.float().t()).backward(dy.float())
        dx = torch.empty(T, I, device=DEV, dtype=torch.float32)
        try:
            _lib.check(_lib.lib().msam_op_gemm_nn(_lib.ptr(dy), _lib.ptr(wb.contiguous()), T, I, O, _lib.ptr(dx), _lib.cur_stream()))
            torch.cuda.synchronize()
            report(f"dgrad dX = dY W    T={T} O={O} I={I} (vs autograd)", dx, xg.grad, 1e-5)
        except Exception as e:  # noqa: BLE001
            RESULTS.append(False)
            print(f"[BAD] dgrad T={T} O={O} I={I}: EXCEPTION {e}", flush=True)
    T, O, I = 16 * 4096, 3072, 768
    x, dy = torch.randn(T, I, device=DEV).bfloat16(), torch.randn(T, O, device=DEV).bfloat16()
    out = torch.empty(O, I, device=DEV, dtype=torch.float32)
    f = lambda: _lib.check(_lib.lib().msam_op_gemm_tn(_lib.ptr(dy), _lib.ptr(x), O, I, T, _lib.ptr(out), _lib.cur_stream()))  # noqa: E731
    ms = _time(f)
    print(f"wgrad {O}x{I} over {T} tokens: {ms:.3f} ms = {2.0 * T * O * I / ms / 1e9:.0f} TFLOP/s", flush=True)


def sec_gemmperf():
    """Event-timed throughput of the encoder GEMM shapes (batch of 4 tiles), next to cuBLAS for the bare product."""
    L = _lib.lib()
    for model, D in (("vit_b", 768), ("vit_h", 1280)):
        shapes = [("qkv (windowed rows)", 19600, 3 * D, D, 0, 0, False), ("proj +res f32", 16384, D, D, 0, 16384, True),
                  ("fc1 +gelu", 16384, 4 * D, D, 1, 0, False), ("fc2 +res f32", 16384, D, 4 * D, 0, 16384, True)]
        for name, M, N, K, act, rr, f32 in shapes:
            A = torch.randn(M, K, device=DEV).bfloat16()
            W = (torch.randn(N, K, device=DEV) / math.sqrt(K)).bfloat16()
            bias = torch.randn(N, device=DEV)
            res = torch.randn(rr, N, device=DEV) if rr else None
            out = torch.empty(M, N, device=DEV, dtype=torch.float32 if f32 else torch.bfloat16)

            def run():
                L.msam_op_gemm(_lib.ptr(A), _lib.ptr(W), M, N, K, _lib.ptr(bias), _lib.ptr(res), rr, _lib.ptr(out), int(f32),
                               act, _lib.cur_stream())
            ms = _time(run)
            ms_cb = _time(lambda: A @ W.t())
            print(f"[perf] {model} {name} M={M} N={N} K={K}: {ms*1e3:.1f} us {2*M*N*K/ms/1e9:.0f} TF/s | cublas bare "
                  f"{ms_cb*1e3:.1f} us {2*M*N*K/ms_cb/1e9:.0f} TF/s", flush=True)


def _time(fn, n=10):
    fn(); fn()
    t0 = torch.cuda.Event(enable_timing=True); t1 = torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(n):
        fn()
    t1.record(); torch.cuda.synchronize()
    return t0.elapsed_time(t1) / n


def sec_ln():
    L = _lib.lib()
    for D in (768, 1280, 256, 160):
        x = torch.randn(2 * 4096, D, device=DEV) * 2 + 0.5
        gam = torch.randn(D, device=DEV)
        bet = torch.randn(D, device=DEV)
        out = torch.empty(2 * 4096, D, device=DEV, dtype=torch.bfloat16)
        _lib.check(L.msam_op_layernorm(_lib.ptr(x), x.shape[0], D, _lib.ptr(gam), _lib.ptr(bet), 1e-6, _lib.ptr(out), 0,
                                       _lib.cur_stream()))
        torch.cuda.synchronize()
        ref = torch.nn.functional.layer_norm(x, (D,), gam, bet, 1e-6)
        report(f"layernorm D={D}", out, ref, 5e-3)
    D = 768
    x = torch.randn(2 * 4096, D, device=DEV)
    gam = torch.randn(D, device=DEV); bet = torch.randn(D, device=DEV)
    out = torch.zeros(2 * 25 * 196, D, device=DEV, dtype=torch.bfloat16)
    _lib.check(L.msam_op_layernorm(_lib.ptr(x), x.shape[0], D, _lib.ptr(gam), _lib.ptr(bet), 1e-6, _lib.ptr(out), 1,
                                   _lib.cur_stream()))
    torch.cuda.synchronize()
    ref = torch.nn.functional.layer_norm(x, (D,), gam, bet, 1e-6).view(2, 64, 64, D)
    ref = torch.nn.functional.pad(ref, (0, 0, 0, 6, 0, 6)).view(2, 5, 14, 5, 14, D).permute(0, 1, 3, 2, 4, 5).reshape(-1, D)
    report("layernorm window-partition", out, ref, 5e-3)


def attn_ref(qkv, rel_h, rel_w, B, heads, hd, S, groups_tokens):
    """qkv: [groups*G, 3*D] (bf16 values as float).  Returns [groups, G, D] fp32 following sam_ref.Attention."""
    D = heads * hd
    G = S * S
    x = qkv.view(-1, G, 3, heads, hd).permute(2, 0, 3, 1, 4)  # 3, groups, heads, G, hd
    q, k, v = x[0], x[1], x[2]
    attn = (q * hd ** -0.5) @ k.transpose(-2, -1)
    idx = torch.arange(S, device=qkv.device)
    rel = idx[:, None] - idx[None, :] + (S - 1)
    Rh, Rw = rel_h[rel], rel_w[rel]  # S,S,hd
    rq = q.reshape(q.shape[0], heads, S, S, hd)
    bh = torch.einsum("ghywc,ykc->ghywk", rq, Rh)
    bw = torch.einsum("ghywc,wkc->ghywk", rq, Rw)
    attn = (attn.view(-1, heads, S, S, S, S) + bh[..., :, None] + bw[..., None, :]).view(-1, heads, G, G)
    attn = attn.softmax(-1)
    return (attn @ v).permute(0, 2, 1, 3).reshape(-1, G, D)


def sec_attn(which=("w64", "g64", "w80", "g80")):
    L = _lib.lib()
    for tag in which:
        window = tag[0] == "w"
        hd = int(tag[1:])
        heads, B = 2, 1
        D = heads * hd
        S = 14 if window else 64
        groups = B * 25 if window else B
        G = S * S
        g = torch.Generator().manual_seed(1)
        qkv = (torch.randn(groups * G, 3 * D, generator=g) * 1.0).to(DEV).bfloat16()
        rel_h = (torch.randn(2 * S - 1, hd, generator=g) * 0.3).to(DEV).bfloat16()
        rel_w = (torch.randn(2 * S - 1, hd, generator=g) * 0.3).to(DEV).bfloat16()
        NT, WOFF = (64, 32) if window else (256, 128)
        cols = ((hd + 63) // 64) * 64
        tab = torch.zeros(NT, cols, device=DEV, dtype=torch.bfloat16)
        tab[: 2 * S - 1, :hd] = rel_h
        tab[WOFF: WOFF + 2 * S - 1, :hd] = rel_w
        out = torch.zeros(B * 4096, D, device=DEV, dtype=torch.bfloat16)
        try:
            _lib.check(L.msam_op_attention(_lib.ptr(qkv), _lib.ptr(tab), _lib.ptr(out), B, heads, hd, 14 if window else 0,
                                           hd ** -0.5, _lib.cur_stream()))
            torch.cuda.synchronize()
        except Exception as e:  # noqa: BLE001
            RESULTS.append(False)
            print(f"[BAD] attention {tag}: EXCEPTION {e}", flush=True)
            continue
        ref = attn_ref(qkv.float(), rel_h.float(), rel_w.float(), B, heads, hd, S, None)
        if window:
            ref = ref.view(B, 5, 5, 14, 14, D).permute(0, 1, 3, 2, 4, 5).reshape(B, 70, 70, D)[:, :64, :64].reshape(-1, D)
        else:
            ref = ref.reshape(-1, D)
        report(f"attention {tag} (heads={heads}, hd={hd})", out, ref, 1.5e-2)
        for h in range(heads):
            report(f"   head {h}", out[:, h * hd:(h + 1) * hd], ref[:, h * hd:(h + 1) * hd], 1.5e-2)


def build_engine(model_type, sd, max_batch=1):
    from oracle import sam_ref
    a = sam_ref.ARCH[model_type]
    L = _lib.lib()
    import ctypes
    ga = list(a["global_attn_indexes"]) + [-1] * (8 - len(a["global_attn_indexes"]))
    cfg = _lib.MsamConfig(a["embed_dim"], a["depth"], a["num_heads"], (ctypes.c_int32 * 8)(*ga), 14, 1024, 16, 256,
                          max_batch, 64)
    h = ctypes.c_void_p()
    _lib.check(L.msam_create(ctypes.byref(cfg), 0, ctypes.byref(h)))
    for k, v in sd.items():
        v = v.detach().float().contiguous().cpu()
        shape = (ctypes.c_int64 * v.ndim)(*v.shape)
        _lib.check(L.msam_load_weight(h, k.encode(), ctypes.c_void_p(v.data_ptr()), shape, v.ndim))
    _lib.check(L.msam_finalize_weights(h))
    return h


def sec_encoder(types=("vit_test", "vit_test80")):
    from oracle import sam_ref
    L = _lib.lib()
    for mt in types:
        sd = sam_ref.seeded_state_dict(mt, seed=1)
        sam = sam_ref.build_sam(mt)
        sam.load_state_dict(sd)
        try:
            h = build_engine(mt, sd, max_batch=2)
            torch.manual_seed(0)
            x = torch.rand(2, 3, 1024, 1024) * 255
            xin = sam.preprocess(x)
            t = time.time()
            with torch.no_grad():
                ref = sam.image_encoder(xin)
            tcpu = time.time() - t
            out = torch.empty(2, 256, 64, 64, device=DEV)
            xd = xin.to(DEV).contiguous()
            _lib.check(L.msam_encode_f32(h, _lib.ptr(xd), 2, _lib.ptr(out), _lib.cur_stream()))
            torch.cuda.synchronize()
        except Exception as e:  # noqa: BLE001
            RESULTS.append(False)
            print(f"[BAD] encoder {mt}: EXCEPTION {e}", flush=True)
            continue
        report(f"encoder {mt} vs fp32 oracle (cpu {tcpu:.1f}s)", out.cpu(), ref, 2e-2)
        L.msam_destroy(h)




# ------------------------------------------------------------------------------------------------ decoder & post
def _predictors(mt, seed=1):
    from oracle import sam_ref
    from micro_sam_b200.sam import B200Sam, B200SamPredictor
    sd = sam_ref.seeded_state_dict(mt, seed=seed)
    osam = sam_ref.build_sam(mt)
    osam.load_state_dict(sd)
    bsam = B200Sam(mt, sd, max_batch=2, max_prompts=64)
    return sam_ref.SamPredictor(osam), B200SamPredictor(bsam)


def sec_decoder(types=("vit_test",)):
    for mt in types:
        op, bp = _predictors(mt)
        torch.manual_seed(0)
        feat = torch.randn(1, 256, 64, 64)
        for pr in (op, bp):
            pr.features = feat.clone() if pr is op else feat.to(DEV)
            pr.is_image_set = True
            pr.original_size = pr.input_size = (1024, 1024)
        g = torch.Generator().manual_seed(3)
        pts = torch.rand(70, 1, 2, generator=g) * 1024
        lbl = torch.ones(70, 1, dtype=torch.int)
        _, iou_r, low_r = op.predict_torch(pts, lbl, multimask_output=True, return_logits=True)
        low, iou = bp.decode_low_res(pts, lbl, None, True)
        torch.cuda.synchronize()
        report(f"decoder {mt} points multimask: low_res", low.cpu(), low_r, 3e-2)
        report(f"decoder {mt} points multimask: iou", iou.cpu(), iou_r, 3e-2)
        agree = ((low.cpu() > 0) == (low_r > 0)).float().mean()
        print(f"      mask sign agreement {agree:.5f}", flush=True)
        boxes = torch.tensor([[100.0, 120.0, 300.0, 400.0], [10.0, 20.0, 1000.0, 900.0], [500, 500, 600, 640.0]])
        _, iou_r, low_r = op.predict_torch(None, None, boxes=boxes, multimask_output=False, return_logits=True)
        low, iou = bp.decode_low_res(None, None, boxes, False)
        report(f"decoder {mt} boxes single: low_res", low.cpu(), low_r, 3e-2)
        report(f"decoder {mt} boxes single: iou", iou.cpu(), iou_r, 3e-2)
        # box + 2 points
        pts2 = torch.rand(3, 2, 2, generator=g) * 1024
        lbl2 = torch.tensor([[1, 0], [1, 1], [0, 1]], dtype=torch.int)
        _, iou_r, low_r = op.predict_torch(pts2, lbl2, boxes=boxes, multimask_output=True, return_logits=True)
        low, iou = bp.decode_low_res(pts2, lbl2, boxes, True)
        report(f"decoder {mt} box+2pts multimask: low_res", low.cpu(), low_r, 3e-2)
        report(f"decoder {mt} box+2pts multimask: iou", iou.cpu(), iou_r, 3e-2)
        # mask prompts (PromptEncoder._embed_masks): mask + point, mask + box + 2 points (unfused path), mask only
        mk = torch.nn.functional.interpolate(torch.randn(3, 1, 16, 16, generator=g), (256, 256), mode="bicubic") * 4
        _, iou_r, low_r = op.predict_torch(pts[:3], lbl[:3], mask_input=mk, multimask_output=True, return_logits=True)
        low, iou = bp.decode_low_res(pts[:3], lbl[:3], None, True, mk)
        report(f"decoder {mt} mask+point multimask: low_res", low.cpu(), low_r, 3e-2)
        report(f"decoder {mt} mask+point multimask: iou", iou.cpu(), iou_r, 3e-2)
        _, iou_r, low_r = op.predict_torch(pts2, lbl2, boxes=boxes, mask_input=mk, multimask_output=False, return_logits=True)
        low, iou = bp.decode_low_res(pts2, lbl2, boxes, False, mk)
        report(f"decoder {mt} mask+box+2pts single: low_res", low.cpu(), low_r, 3e-2)
        report(f"decoder {mt} mask+box+2pts single: iou", iou.cpu(), iou_r, 3e-2)
        _, iou_r, low_r = op.predict_torch(None, None, mask_input=mk, multimask_output=False, return_logits=True)
        low, iou = bp.decode_low_res(None, None, None, False, mk)
        report(f"decoder {mt} mask only single: low_res", low.cpu(), low_r, 3e-2)
        report(f"decoder {mt} mask only single: iou", iou.cpu(), iou_r, 3e-2)


def sec_post():
    from oracle import sam_ref, amg_ref
    from micro_sam_b200 import sam as bsam
    L = _lib.lib()
    osam = sam_ref.build_sam("vit_test")
    g = torch.Generator().manual_seed(5)
    # mask_threshold="auto": local Otsu thresholds, bit-exact vs the CPU restatement (smooth, noisy, constant masks)
    lo = torch.nn.functional.interpolate(torch.randn(4, 1, 12, 12, generator=g), (256, 256), mode="bicubic")[:, 0] * 4
    lo[1] += torch.randn(256, 256, generator=g) * 0.5
    lo[2] = lo[2] - 6.0
    lo[3] = 1.5
    thr = bsam.local_otsu_threshold(lo.to(DEV)).cpu()
    thr_ref = amg_ref.local_otsu_threshold(lo[:, None]).view(-1)
    same = bool(torch.equal(thr, thr_ref))
    RESULTS.append(same)
    print(f"[{'OK ' if same else 'BAD'}] local Otsu thresholds {thr.tolist()} vs oracle {thr_ref.tolist()}", flush=True)
    b1, s1, a1 = bsam.mask_stats(lo.to(DEV), (1024, 1024), (1024, 1024), thr.to(DEV), 1.0)
    ok = True
    for k in range(4):
        b0, s0, a0 = bsam.mask_stats(lo[k:k + 1].to(DEV), (1024, 1024), (1024, 1024), float(thr[k]), 1.0)
        ok &= bool((b0[0] == b1[k]).all()) and int(a0[0]) == int(a1[k]) and bool(torch.equal(s0.nan_to_num(-1), s1[k:k + 1].nan_to_num(-1)))
    RESULTS.append(ok)
    print(f"[{'OK ' if ok else 'BAD'}] mask_stats with per-mask thresholds == scalar-threshold calls", flush=True)
    # remove_small_regions (8-connected components) + mask boxes vs the oracle
    rng = np.random.default_rng(3)
    mk = (torch.nn.functional.interpolate(torch.randn(6, 1, 10, 14, generator=g), (96, 130), mode="bicubic")[:, 0] > 0.3).numpy()
    mk |= rng.random(mk.shape) > 0.995                      # specks (islands)
    mk &= ~(rng.random(mk.shape) > 0.99)                   # pin holes
    mk[4] = False; mk[4, 10:12, 20:22] = True; mk[4, 50, 60] = True   # every island below the threshold -> keep the largest
    mk[5] = False                                          # empty mask
    dm = torch.from_numpy(mk).to(DEV).to(torch.uint8).contiguous()
    ws = torch.empty(6 * (2 * 96 * 130 + 4), dtype=torch.int32, device=DEV)
    ch = torch.zeros(2, 6, dtype=torch.int32, device=DEV)
    ok = True
    ref = mk.copy(); ref_ch = np.zeros((2, 6), dtype=bool)
    for q, (holes, mode) in enumerate(((1, "holes"), (0, "islands"))):
        _lib.check(L.msam_remove_small_regions(_lib.ptr(dm), 6, 96, 130, 12, holes, _lib.ptr(ch[q]), _lib.ptr(ws), _lib.cur_stream()))
        for k in range(6):
            ref[k], ref_ch[q, k] = amg_ref.remove_small_regions(ref[k], 12, mode)
        ok &= bool(np.array_equal(dm.cpu().numpy().astype(bool), ref)) and bool(np.array_equal(ch[q].cpu().numpy() != 0, ref_ch[q]))
    bx = torch.empty(6, 4, dtype=torch.int32, device=DEV); ar = torch.empty(6, dtype=torch.int32, device=DEV)
    _lib.check(L.msam_mask_boxes(_lib.ptr(dm), 6, 96, 130, _lib.ptr(bx), _lib.ptr(ar), _lib.cur_stream()))
    ok &= bool(np.array_equal(bx.cpu().numpy(), amg_ref.batched_mask_to_box(torch.from_numpy(ref)).numpy()))
    ok &= bool(np.array_equal(ar.cpu().numpy(), ref.reshape(6, -1).sum(1)))
    RESULTS.append(ok)
    print(f"[{'OK ' if ok else 'BAD'}] remove_small_regions (holes, islands; changed {ref_ch.tolist()}) + mask boxes == oracle", flush=True)
    # smooth random low-res logits with both signs
    low = torch.nn.functional.interpolate(torch.randn(12, 1, 16, 16, generator=g), (256, 256), mode="bicubic")[:, 0] * 3
    low[3] = -5.0  # empty mask
    low[4] = 5.0   # full mask
    for (inp, orig) in (((1024, 1024), (1024, 1024)), ((1024, 683), (768, 512)), ((640, 1024), (500, 800))):
        ref_full = osam.postprocess_masks(low[:, None], inp, orig)[:, 0]
        boxes, stab, area = bsam.mask_stats(low.to(DEV), inp, orig, 0.0, 1.0)
        if inp == (1024, 1024) and orig == (1024, 1024):  # 4x fast path vs the generic kernel (negative offset selects it)
            b2, s2, a2 = bsam.mask_stats(low.to(DEV), inp, orig, 0.0, -1.0)
            same = bool((b2 == boxes).all()) and bool((a2 == area).all()) and bool(torch.equal(s2.nan_to_num(-1), stab.nan_to_num(-1)))
            RESULTS.append(same)
            print(f"[{'OK ' if same else 'BAD'}] mask_stats 4x fast path == generic path", flush=True)
        full = torch.empty(12, orig[0], orig[1], device=DEV)
        binm = torch.empty(12, orig[0], orig[1], device=DEV, dtype=torch.uint8)
        dlow = low.to(DEV).contiguous()
        _lib.check(L.msam_upsample_masks(_lib.ptr(dlow), None, 12, inp[0], inp[1], orig[0], orig[1], 0.0,
                                         _lib.ptr(full), _lib.ptr(binm), _lib.cur_stream()))
        torch.cuda.synchronize()
        report(f"postprocess_masks {inp}->{orig}", full.cpu(), ref_full, 1e-5)
        rb = ref_full > 0
        mism = (binm.cpu().bool() != rb).sum().item()
        inter = (ref_full > 1.0).flatten(1).sum(1).float()
        union = (ref_full > -1.0).flatten(1).sum(1).float()
        ok_area = bool((area.cpu() == rb.flatten(1).sum(1)).all()) or mism > 0
        print(f"      binary mismatches={mism} area_equal={bool((area.cpu() == rb.flatten(1).sum(1)).all())} "
              f"stab max diff={(stab.cpu() - inter / union).nan_to_num(0).abs().max():.2e}", flush=True)
        # integer stages bit-exact GIVEN the GPU masks: boxes / area recomputed by the oracle from the GPU binary masks
        from oracle import amg_ref
        ref_boxes = amg_ref.batched_mask_to_box(binm.cpu().bool())
        okb = bool((ref_boxes.to(torch.int32) == boxes.cpu()).all()) and bool((area.cpu() == binm.cpu().flatten(1).sum(1)).all())
        RESULTS.append(okb)
        print(f"[{'OK ' if okb else 'BAD'}] mask_stats boxes/area bit-exact vs oracle on GPU masks {inp}->{orig}", flush=True)


def sec_nms():
    import torchvision
    L = _lib.lib()
    g = torch.Generator().manual_seed(7)
    for n in (1, 5, 300, 3072):
        xy = torch.randint(0, 900, (n, 2), generator=g)
        wh = torch.randint(1, 200, (n, 2), generator=g)
        boxes = torch.cat([xy, torch.minimum(xy + wh, torch.tensor(1023))], 1).to(torch.int32)
        boxes[: n // 3] = boxes[n // 3: 2 * (n // 3)]  # many duplicates / heavy overlaps
        boxes[: n // 3, 2:] += torch.randint(0, 4, (n // 3, 2), generator=g).to(torch.int32)
        scores = torch.rand(n, generator=g)
        stab = torch.rand(n, generator=g) * 0.2 + 0.85
        keep = torch.empty(n, dtype=torch.int32, device=DEV)
        nk = torch.zeros(1, dtype=torch.int32, device=DEV)
        import ctypes
        crop = (ctypes.c_int32 * 4)(0, 0, 1024, 1024)
        dboxes, dscores, dstab = boxes.to(DEV), scores.to(DEV), stab.to(DEV)
        for use_f in (0, 1):
            _lib.check(L.msam_amg_filter_nms(_lib.ptr(dboxes), _lib.ptr(dscores), _lib.ptr(dstab), n, use_f,
                                             0.5, 0.9, 0.7, crop, crop, _lib.ptr(keep), _lib.ptr(nk), _lib.cur_stream()))
            torch.cuda.synchronize()
            got = keep[: int(nk.item())].cpu().long()
            if use_f:
                from oracle import amg_ref
                m = (scores > 0.5) & (stab >= 0.9) & ~amg_ref.is_box_near_crop_edge(boxes, [0, 0, 1024, 1024], [0, 0, 1024, 1024])
                idx = m.nonzero()[:, 0]
            else:
                idx = torch.arange(n)
            ref = idx[torchvision.ops.nms(boxes[idx].float(), scores[idx], 0.7)]
            ok = got.tolist() == ref.tolist()
            RESULTS.append(ok)
            print(f"[{'OK ' if ok else 'BAD'}] filter_nms n={n} filters={use_f}: kept {len(got)} (ref {len(ref)})", flush=True)


SECTIONS = {"gemm": sec_gemm, "wgrad": sec_wgrad, "gemmperf": sec_gemmperf, "ln": sec_ln, "attn": sec_attn, "encoder": sec_encoder, "decoder": sec_decoder,
            "post": sec_post, "nms": sec_nms}

if __name__ == "__main__":
    names = sys.argv[1:] or list(SECTIONS)
    print("device:", torch.cuda.get_device_name(0), flush=True)
    for n in names:
        print(f"==== {n}", flush=True)
        n, _, sub = n.partition(":")
        try:
            SECTIONS[n](tuple(sub.split(","))) if sub else SECTIONS[n]()
        except Exception as e:  # noqa: BLE001
            RESULTS.append(False)
            print(f"[BAD] section {n}: EXCEPTION {type(e).__name__}: {e}", flush=True)
    print(f"==== {sum(RESULTS)}/{len(RESULTS)} checks ok", flush=True)
