#!/usr/bin/env python
"""Small ragged invocations of every kernel family, for compute-sanitizer (memcheck / racecheck /
synccheck) runs:  compute-sanitizer --tool memcheck python scripts/sanitize_small.py"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import gemm_hls_b200 as G  # noqa: E402
import oracle as O  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tests"))
import bf16_naive  # noqa: E402  (bfloat16 has no reference Naive<>: the test suite's restatement)

# (name, dtype, map, reduce, flags, (n, k, m)[, tuning])
CASES = [
    ("wgmma_tf32", G.FLOAT, G.MULTIPLY, G.ADD, 0, (257, 48, 272)),
    ("wgmma_tf32 multi-tile", G.FLOAT, G.MULTIPLY, G.ADD, 0, (600, 80, 528)),
    ("wgmma_tf32 direct stores", G.FLOAT, G.MULTIPLY, G.ADD, 0, (257, 48, 272), dict(tma_store=0)),
    ("wgmma_tf32 b_overlap=1 (no effect)", G.FLOAT, G.MULTIPLY, G.ADD, 0, (257, 48, 528), dict(b_overlap=1)),
    ("wgmma_tf32 K-major B, 1 CTA, 128 cols", G.FLOAT, G.MULTIPLY, G.ADD, 0, (257, 48, 272), dict(b_mn=0, cta_group=1, block_n=128)),
    ("wgmma_i8", G.UINT8, G.MULTIPLY, G.ADD, 0, (257, 192, 320)),
    ("wgmma_i8 TA, 1 CTA", G.UINT8, G.MULTIPLY, G.ADD, G.FLAG_TRANSPOSED_A, (130, 64, 192), dict(cta_group=1)),
    ("wgmma_tf32 TA", G.FLOAT, G.MULTIPLY, G.ADD, G.FLAG_TRANSPOSED_A, (130, 64, 192)),
    ("wgmma_tf32x3", G.FLOAT, G.MULTIPLY, G.ADD, G.FLAG_TF32X3, (129, 48, 272)),
    ("wgmma_f16", G.HALF, G.MULTIPLY, G.ADD, 0, (257, 96, 288)),
    ("dmma_f64", G.DOUBLE, G.MULTIPLY, G.ADD, 0, (130, 24, 136)),
    ("dmma_f64 TA", G.DOUBLE, G.MULTIPLY, G.ADD, G.FLAG_TRANSPOSED_A, (130, 24, 136)),
    ("dmma_f64 3 stages wrap", G.DOUBLE, G.MULTIPLY, G.ADD, 0, (70, 200, 264)),
    ("semiring f32 addmin", G.FLOAT, G.ADD, G.MIN, 0, (129, 48, 144)),
    ("semiring f32 exact", G.FLOAT, G.MULTIPLY, G.ADD, G.FLAG_EXACT, (129, 48, 144)),
    ("semiring i32", G.INT32, G.MULTIPLY, G.ADD, 0, (65, 32, 48)),
    ("semiring f32 addmin staged kernel", G.FLOAT, G.ADD, G.MIN, 0, (129, 48, 144), dict(semiring_ring=0)),
    ("semiring u8 exact", G.UINT8, G.MULTIPLY, G.ADD, G.FLAG_EXACT, (65, 128, 192)),
    ("semiring f16 exact", G.HALF, G.MULTIPLY, G.ADD, G.FLAG_EXACT, (65, 64, 96)),
    ("semiring f64 addmax TA", G.DOUBLE, G.ADD, G.MAX, G.FLAG_TRANSPOSED_A, (67, 16, 24)),
    ("wgmma_bf16", G.BFLOAT16, G.MULTIPLY, G.ADD, 0, (257, 96, 288)),
    ("wgmma_bf16 TA, 1 CTA, direct stores", G.BFLOAT16, G.MULTIPLY, G.ADD, G.FLAG_TRANSPOSED_A, (130, 64, 192),
     dict(cta_group=1, tma_store=0)),
    ("semiring bf16 exact", G.BFLOAT16, G.MULTIPLY, G.ADD, G.FLAG_EXACT, (65, 64, 96)),
    ("semiring bf16 addmin", G.BFLOAT16, G.ADD, G.MIN, 0, (65, 64, 96)),
    ("semiring bf16 addmax TA", G.BFLOAT16, G.ADD, G.MAX, G.FLAG_TRANSPOSED_A, (67, 32, 64)),
]


def bf16_within_one_ulp(c, a, b, n, k, m, transposed):
    """bf16 tensor path: every element within 1 ulp of an FP64 evaluation of the same inputs."""
    def f(x):
        return (np.asarray(x, dtype=np.uint16).astype(np.uint32) << 16).view(np.float32).astype(np.float64)
    av = f(a).reshape((k, n) if transposed else (n, k))
    ref = (av.T if transposed else av) @ f(b).reshape(k, m)
    ulp = 2.0 ** (np.floor(np.log2(np.maximum(np.abs(ref), 2.0 ** -126))) - 7)
    return bool(np.all(np.abs(f(c).reshape(n, m) - ref) <= ulp))


only = os.environ.get("SANITIZE_ONLY")  # substring filter on the case name, e.g. SANITIZE_ONLY=dmma
bad = 0
for case in CASES:
    name, dt, mp, rd, flags, (n, k, m) = case[:6]
    tuning = case[6] if len(case) > 6 else {}
    if only and only not in name:
        continue
    a, b = bf16_naive.fill(O, n, k, m, 3) if dt == G.BFLOAT16 else O.fill(dt, n, k, m, 3)
    if dt == G.HALF:
        a = (a.astype(np.float32) * np.float32(0.25)).astype(np.float16)
    with G.Context(0) as ctx:
        ctx.set_tuning(**tuning)
        c = ctx.gemm_host(dt, mp, rd, a, b, n, k, m, flags=flags)[0]
    if dt == G.BFLOAT16:
        ta = bool(flags & G.FLAG_TRANSPOSED_A)
        if G.kernel_path(dt, mp, rd, flags) == "semiring_simt":
            ok = bf16_naive.same_nan_free(c, bf16_naive.naive(mp, rd, a, b, n, k, m, transposed_a=ta))
        else:
            ok = bf16_within_one_ulp(c, a, b, n, k, m, ta)
    else:
        ref = O.naive(dt, mp, rd, a, b, n, k, m, transposed_a=bool(flags & G.FLAG_TRANSPOSED_A), threads=4)
        ok = O.verify(dt, c, ref) == -1 if G.kernel_path(dt, mp, rd, flags) == "semiring_simt" or dt != G.HALF else True
    print("%-42s %s" % (name, "ok" if ok else "MISMATCH"), flush=True)
    bad += 0 if ok else 1
# batched calls (3 ragged problems, packed or shared operands): every problem equals its single call
BATCHED = [
    ("batched wgmma_tf32", G.FLOAT, G.MULTIPLY, G.ADD, 0, (257, 48, 272)),
    ("batched wgmma_tf32 direct stores, shared B", G.FLOAT, G.MULTIPLY, G.ADD, G.FLAG_BATCH_SHARED_B, (129, 48, 272),
     dict(tma_store=0)),
    ("batched wgmma_f16 shared A", G.HALF, G.MULTIPLY, G.ADD, G.FLAG_BATCH_SHARED_A, (129, 96, 288)),
    ("batched wgmma_i8 TA, 1 CTA", G.UINT8, G.MULTIPLY, G.ADD, G.FLAG_TRANSPOSED_A, (130, 64, 192), dict(cta_group=1)),
    ("batched wgmma_tf32x3 TA", G.FLOAT, G.MULTIPLY, G.ADD, G.FLAG_TF32X3 | G.FLAG_TRANSPOSED_A, (130, 48, 144)),
    ("batched dmma_f64", G.DOUBLE, G.MULTIPLY, G.ADD, 0, (130, 40, 136)),
    ("batched dmma_f64 TA, shared B", G.DOUBLE, G.MULTIPLY, G.ADD, G.FLAG_TRANSPOSED_A | G.FLAG_BATCH_SHARED_B,
     (130, 24, 136)),
    ("batched semiring f32 addmin shared B", G.FLOAT, G.ADD, G.MIN, G.FLAG_BATCH_SHARED_B, (129, 48, 144)),
    ("batched semiring i32 staged kernel", G.INT32, G.MULTIPLY, G.ADD, 0, (65, 32, 48), dict(semiring_ring=0)),
    ("batched semiring f64 addmax TA", G.DOUBLE, G.ADD, G.MAX, G.FLAG_TRANSPOSED_A, (67, 16, 24)),
    ("batched wgmma_bf16 shared A", G.BFLOAT16, G.MULTIPLY, G.ADD, G.FLAG_BATCH_SHARED_A, (129, 96, 288)),
    ("batched wgmma_bf16 TA, shared B", G.BFLOAT16, G.MULTIPLY, G.ADD, G.FLAG_TRANSPOSED_A | G.FLAG_BATCH_SHARED_B,
     (130, 64, 192)),
    ("batched semiring bf16 addmin", G.BFLOAT16, G.ADD, G.MIN, 0, (65, 64, 96)),
]
shared_flags = G.FLAG_BATCH_SHARED_A | G.FLAG_BATCH_SHARED_B
for case in BATCHED:
    name, dt, mp, rd, flags, (n, k, m) = case[:6]
    tuning = case[6] if len(case) > 6 else {}
    if only and only not in name:
        continue
    batch = 3
    na = 1 if flags & G.FLAG_BATCH_SHARED_A else batch
    nb = 1 if flags & G.FLAG_BATCH_SHARED_B else batch
    data = [bf16_naive.fill(O, n, k, m, 40 + i) if dt == G.BFLOAT16 else O.fill(dt, n, k, m, 40 + i) for i in range(batch)]
    a = np.concatenate([d[0].reshape(-1) for d in data[:na]])
    b = np.concatenate([d[1].reshape(-1) for d in data[:nb]])
    if dt == G.HALF:
        a = (a.astype(np.float32) * np.float32(0.25)).astype(np.float16)
    with G.Context(0) as ctx:
        ctx.set_tuning(**tuning)
        da, db, dc = ctx.alloc(a.nbytes), ctx.alloc(b.nbytes), ctx.alloc(batch * n * m * a.itemsize)
        ctx.copy_to_device(da, a)
        ctx.copy_to_device(db, b)
        ctx.enqueue_batched(dt, mp, rd, da, db, dc, n, k, m, batch, flags=flags)
        c = np.empty((batch, n * m), dtype=a.dtype)
        ctx.copy_to_host(c, dc)   # ordered after the enqueue on the context's stream
        ok = True
        for i in range(batch):
            ai = a.reshape(na, -1)[0 if na == 1 else i]
            bi = b.reshape(nb, -1)[0 if nb == 1 else i]
            single = ctx.gemm_host(dt, mp, rd, ai, bi, n, k, m, flags=flags & ~shared_flags)[0]
            ok = ok and single.tobytes() == c[i].tobytes()
        for p in (da, db, dc):
            ctx.free(p)
    print("%-42s %s" % (name, "ok" if ok else "MISMATCH"), flush=True)
    bad += 0 if ok else 1
# witnesses (mm_kernel_enqueue_witness): ragged shapes on both witness kernels, a batch with a shared operand; C must
# equal the plain batched call and W the test suite's restatement (tests/witness_naive.py).  These cases have run on
# an H100 without compute-sanitizer so far; no memcheck / racecheck / synccheck pass over them has been made yet.
import witness_naive  # noqa: E402

WITNESS = [
    ("witness ring f32 addmin", G.FLOAT, G.ADD, G.MIN, 0, (129, 48, 144), 1),
    ("witness ring i32 addmax shared B", G.INT32, G.ADD, G.MAX, G.FLAG_BATCH_SHARED_B, (65, 32, 48), 3),
    ("witness staged f32 exact addmin", G.FLOAT, G.ADD, G.MIN, G.FLAG_EXACT, (129, 48, 144), 1, dict(semiring_ring=0)),
    ("witness staged f64 addmax TA", G.DOUBLE, G.ADD, G.MAX, G.FLAG_TRANSPOSED_A, (67, 16, 72), 2),
    ("witness staged u8 maxmin", G.UINT8, G.MAX, G.MIN, 0, (65, 128, 192), 1),
    ("witness staged bf16 addmax", G.BFLOAT16, G.ADD, G.MAX, 0, (65, 64, 96), 1),
]
for case in WITNESS:
    name, dt, mp, rd, flags, (n, k, m), batch = case[:7]
    tuning = case[7] if len(case) > 7 else {}
    if only and only not in name:
        continue
    shared_b = bool(flags & G.FLAG_BATCH_SHARED_B)
    data = [bf16_naive.fill(O, n, k, m, 50 + i) if dt == G.BFLOAT16 else O.fill(dt, n, k, m, 50 + i) for i in range(batch)]
    ta = bool(flags & G.FLAG_TRANSPOSED_A)
    a = np.concatenate([(np.ascontiguousarray(d[0].reshape(n, k).T) if ta else d[0]).reshape(-1) for d in data])
    b = np.concatenate([d[1].reshape(-1) for d in data[:1 if shared_b else batch]])
    with G.Context(0) as ctx:
        ctx.set_tuning(**tuning)
        da, db = ctx.alloc(a.nbytes), ctx.alloc(b.nbytes)
        dc, dp, dw = (ctx.alloc(batch * n * m * x) for x in (a.itemsize, a.itemsize, 4))
        ctx.copy_to_device(da, a)
        ctx.copy_to_device(db, b)
        ctx.enqueue_batched(dt, mp, rd, da, db, dp, n, k, m, batch, flags=flags)
        ctx.enqueue_witness(dt, mp, rd, da, db, dc, dw, n, k, m, batch=batch, flags=flags)
        c, p = np.empty(batch * n * m, dtype=a.dtype), np.empty(batch * n * m, dtype=a.dtype)
        w = np.empty((batch, n, m), dtype=np.uint32)
        for host, dev in ((c, dc), (p, dp), (w, dw)):
            ctx.copy_to_host(host, dev)
        for x in (da, db, dc, dp, dw):
            ctx.free(x)
    ok = c.tobytes() == p.tobytes()
    fm = dt == G.FLOAT and not flags & G.FLAG_EXACT
    for i in range(batch):
        want = witness_naive.witness(dt, mp, rd, data[i][0].reshape(n, k), data[0 if shared_b else i][1].reshape(k, m),
                                     fmnmx=fm)[1]
        ok = ok and np.array_equal(w[i], want)
    print("%-42s %s" % (name, "ok" if ok else "MISMATCH"), flush=True)
    bad += 0 if ok else 1
# accumulation (mm_kernel_enqueue_accumulate): ragged shapes on every family, one batch with a shared operand; C must
# equal R(C_old, P) with P the plain batched call (tests/accumulate_naive.py).  These cases have run on an H100 without
# compute-sanitizer so far.
import accumulate_naive  # noqa: E402

ACCUMULATE = [
    ("accumulate wgmma f32", G.FLOAT, G.MULTIPLY, G.ADD, 0, (129, 48, 144), 1),
    ("accumulate wgmma f32 direct stores", G.FLOAT, G.MULTIPLY, G.ADD, 0, (129, 48, 144), 1, dict(tma_store=0)),
    ("accumulate wgmma f16 shared B", G.HALF, G.MULTIPLY, G.ADD, G.FLAG_BATCH_SHARED_B, (65, 64, 96), 3),
    ("accumulate wgmma u8", G.UINT8, G.MULTIPLY, G.ADD, 0, (67, 128, 192), 1),
    ("accumulate dmma f64 TA", G.DOUBLE, G.MULTIPLY, G.ADD, G.FLAG_TRANSPOSED_A, (66, 16, 72), 1),
    ("accumulate ring f32 addmin", G.FLOAT, G.ADD, G.MIN, 0, (129, 48, 144), 1),
    ("accumulate tile bf16 exact", G.BFLOAT16, G.MULTIPLY, G.ADD, G.FLAG_EXACT, (65, 64, 96), 2),
]
for case in ACCUMULATE:
    name, dt, mp, rd, flags, (n, k, m), batch = case[:7]
    tuning = case[7] if len(case) > 7 else {}
    if only and only not in name:
        continue
    shared_b = bool(flags & G.FLAG_BATCH_SHARED_B)
    data = [bf16_naive.fill(O, n, k, m, 60 + i) if dt == G.BFLOAT16 else O.fill(dt, n, k, m, 60 + i) for i in range(batch)]
    ta = bool(flags & G.FLAG_TRANSPOSED_A)
    a = np.concatenate([(np.ascontiguousarray(d[0].reshape(n, k).T) if ta else d[0]).reshape(-1) for d in data])
    b = np.concatenate([d[1].reshape(-1) for d in data[:1 if shared_b else batch]])
    if dt == G.HALF:
        a = (a.astype(np.float32) * np.float32(0.25)).astype(np.float16)
    with G.Context(0) as ctx:
        ctx.set_tuning(**tuning)
        da, db = ctx.alloc(a.nbytes), ctx.alloc(b.nbytes)
        dc, dp = (ctx.alloc(batch * n * m * a.itemsize) for _ in range(2))
        ctx.copy_to_device(da, a)
        ctx.copy_to_device(db, b)
        ctx.enqueue_batched(dt, mp, rd, da, db, dp, n, k, m, batch, flags=flags)
        p = np.empty(batch * n * m, dtype=a.dtype)
        ctx.copy_to_host(p, dp)
        c0 = accumulate_naive.c_old(dt, rd, p, 7)
        ctx.copy_to_device(dc, c0)
        ctx.enqueue_accumulate(dt, mp, rd, da, db, dc, n, k, m, batch=batch, flags=flags)
        c = np.empty_like(p)
        ctx.copy_to_host(c, dc)
        for x in (da, db, dc, dp):
            ctx.free(x)
    fm = dt == G.FLOAT and rd in (G.MIN, G.MAX) and not flags & G.FLAG_EXACT
    ok = accumulate_naive.same(dt, c, accumulate_naive.reduce_once(dt, rd, c0, p, fm), rd)
    print("%-42s %s" % (name, "ok" if ok else "MISMATCH"), flush=True)
    bad += 0 if ok else 1
# closures (mm_kernel_enqueue_closure): a ragged last block on the ring and the tile remainder kernels, one partial
# block, and a batch; D must equal the test suite's restatement (tests/closure_naive.py).  These cases have run on an
# H100 without compute-sanitizer so far.
import closure_data  # noqa: E402
import closure_naive  # noqa: E402

CLOSURE = [
    ("closure ring f32 addmin", G.FLOAT, G.ADD, G.MIN, 0, 2 * 128 + 16, 1),
    ("closure ring i32 addmax batch", G.INT32, G.ADD, G.MAX, 0, 128 + 16, 2),
    ("closure tile f64 exact minmax", G.DOUBLE, G.MIN, G.MAX, G.FLAG_EXACT, 2 * 128 + 8, 1),
    ("closure tile u8 andmax", G.UINT8, G.AND, G.MAX, 0, 128 + 64, 1),
    ("closure pivot only bf16 addmin", G.BFLOAT16, G.ADD, G.MIN, 0, 96, 1),
]
for name, dt, mp, rd, flags, n, batch in CLOSURE:
    if only and only not in name:
        continue
    d = closure_data.case(dt, mp, rd, n, 3, exact=bool(flags & G.FLAG_EXACT), batch=batch)
    with G.Context(0) as ctx:
        dd = ctx.alloc(d.nbytes)
        ctx.copy_to_device(dd, d)
        ctx.enqueue_closure(dt, mp, rd, dd, n, batch, flags=flags)
        c = np.empty_like(d)
        ctx.copy_to_host(c, dd)
        ctx.free(dd)
    fm = dt == G.FLOAT and not flags & G.FLAG_EXACT
    ok = closure_naive.sd.same(c, closure_naive.closure(dt, mp, rd, d, fmnmx=fm))
    print("%-42s %s" % (name, "ok" if ok else "MISMATCH"), flush=True)
    bad += 0 if ok else 1
# bit-packed Boolean products and closures (mm_kernel_enqueue_bool / _closure) at ragged shapes: partial row tiles, a
# partial last column tile, a batch, and a closure whose last block of indices is half full; against tests/bool_naive.py.
import bool_naive  # noqa: E402

BOOL = [("bool product 129x384x384", 129, 384, 384, 1), ("bool product 1x1152x640 batch", 1, 1152, 640, 2),
        ("bool closure 384", 384, 384, 384, 1), ("bool closure 640 batch", 640, 640, 640, 2)]
for name, n, k, m, batch in BOOL:
    if only and only not in name:
        continue
    with G.Context(0) as ctx:
        if "closure" in name:
            d = np.stack([bool_naive.hamiltonian_cycle(n, p) | bool_naive.random_bits((n, n), 0.002, p)
                          for p in range(batch)])
            dd = ctx.alloc(d.size // 8)
            ctx.copy_to_device(dd, bool_naive.pack(d))
            ctx.enqueue_bool_closure(dd, n, batch)
            want = np.stack([bool_naive.closure(x) for x in d])
        else:
            a = bool_naive.random_bits((batch, n, k), 0.01, 1)
            b = bool_naive.random_bits((batch, k, m), 0.01, 2)
            da, db, dd = ctx.alloc(a.size // 8), ctx.alloc(b.size // 8), ctx.alloc(batch * n * m // 8)
            ctx.copy_to_device(da, bool_naive.pack(a))
            ctx.copy_to_device(db, bool_naive.pack(b))
            ctx.enqueue_bool(da, db, dd, n, k, m, batch)
            want = bool_naive.product(a, b)
            ctx.free(da)
            ctx.free(db)
        c = np.empty((batch, n, m // 8), np.uint8)
        ctx.copy_to_host(c, dd)
        ctx.free(dd)
    ok = np.array_equal(bool_naive.unpack(c, m), want)
    print("%-42s %s" % (name, "ok" if ok else "MISMATCH"), flush=True)
    bad += 0 if ok else 1
# the row-block split on one device listed twice: sliced upload of B, the gather kernel, host barriers
if not only or "multi" in only:
    for dt, shape in ((G.FLOAT, (300, 128, 272)), (G.HALF, (257, 128, 288)), (G.DOUBLE, (130, 128, 136)),
                      (G.BFLOAT16, (257, 128, 288))):
        n, k, m = shape
        a, b = bf16_naive.fill(O, n, k, m, 5) if dt == G.BFLOAT16 else O.fill(dt, n, k, m, 5)
        if dt == G.HALF:
            a = (a.astype(np.float32) * np.float32(0.25)).astype(np.float16)
        single = G.matrix_multiplication_kernel(a, b, n, k, m, dtype=dt)
        with G.Multi(2, devices=[0, 0]) as multi:
            c = multi.gemm_host(dt, G.MULTIPLY, G.ADD, a, b, n, k, m)[0]
        ok = c.tobytes() == single.tobytes()
        print("%-42s %s" % ("multi x2 dtype %d" % dt, "ok" if ok else "MISMATCH"), flush=True)
        bad += 0 if ok else 1
sys.exit(1 if bad else 0)
