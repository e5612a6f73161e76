"""A/B timing of two builds of the grouped 3xTF32 GEMM (phc_gemm_group) on the bench's launches, in one process.

    python tools/time_gemm_ab.py [A.so] [B.so] [--turns 5] [--iters 20]

A defaults to phc_b200/lib/alt_parent/libphc_b200.so, B to the working tree's phc_b200/lib/libphc_b200.so.  Both are
loaded with their own ctypes handle, so each keeps its own device module and scheduler state.  To make A the parent
commit's build (from the repository root; phc_b200/lib/ is ignored by git, so the copy travels with the tree):

    rm -rf /tmp/parent && mkdir /tmp/parent && git archive HEAD~1 | tar -x -C /tmp/parent   # or the commit to compare against
    (cd /tmp/parent && python -m phc_b200.build)
    mkdir -p phc_b200/lib/alt_parent && cp /tmp/parent/phc_b200/lib/libphc_b200.so phc_b200/lib/alt_parent/

The launch groups are those of bench.py:gemm_roofline, from an AMPAgent at the bench configuration (4096 envs, im.yaml
networks): the three forward launches of one 16384-row minibatch (actor, critic, discriminator advance together) and the
backward launches by layer index (dW split-K into the gradient bucket + dX), then the rollout forward at 4096 rows, then the
minibatch launches again with 128 x 256 tiles (phc_gemm_tc5s_set_tile(256)).  Each backward launch is also timed split into
its weight-gradient problems alone ("dW L-k") and its input-gradient problems alone ("dX L-k").  Each group alternates A and B
`--turns` times; a turn is `--iters` launches between two CUDA events after a warm-up.  A build that takes activation images
(PhcGemmDesc.A_img) gets them the way MLPEngine.run_group does: one phc_gemm_make_images launch before every launch that reads
them, inside the timed window.  A build that also takes output images (PhcGemmDesc.C_img) runs the hidden layers' forward and dX
from the images the launch before wrote, as MLPEngine does; a build without them, and any build with 128 x 256 tiles, runs those
problems from the fp32 activations.  Printed per group: median [min, max] us per launch
and the TFLOP/s of tensor work (3 tensor-core products per fp32 product) for A and B, and B / A.

Before any timing, the whole chain (forward, then backward) runs once per build from the same seeded workspaces, and every
tensor it writes -- activations, ReLU bit masks, dX, and the split-K sums in the gradient bucket -- must be torch.equal.
"""
import argparse
import ctypes as C
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import bench  # noqa: E402
from phc_b200 import _lib  # noqa: E402


class GemmDescNoImage(C.Structure):
    """PhcGemmDesc of a build from before the weight images (no B_img field)."""
    _fields_ = [f for f in _lib.PhcGemmDesc._fields_ if f[0] not in ("B_img", "A_img")]


class GemmDescNoActImage(C.Structure):
    """PhcGemmDesc of a build from before the activation images (no A_img field)."""
    _fields_ = [f for f in _lib.PhcGemmDesc._fields_ if f[0] not in ("A_img", "C_img")]


class GemmDescNoOutImage(C.Structure):
    """PhcGemmDesc of a build from before the epilogue's output images (no C_img field)."""
    _fields_ = [f for f in _lib.PhcGemmDesc._fields_ if f[0] != "C_img"]


def open_lib(path):
    lib = C.CDLL(os.path.abspath(path))
    for name in ("phc_gemm_group", "phc_gemm_make_images", "phc_gemm_image_floats", "phc_gemm_set_precision", "phc_gemm_tc5s_set_tile", "phc_gemm_tc5s_set_sched", "phc_last_error"):
        if hasattr(lib, name):
            res, args = _lib.SIGNATURES[name]
            getattr(lib, name).restype, getattr(lib, name).argtypes = res, args
    # each build gets descriptors in its own layout; one without images computes the same problems from the staged operands
    # (a build that knows A_img names it in its validation message)
    with open(path, "rb") as f:
        blob = f.read()
    lib.desc_type = (GemmDescNoImage if not hasattr(lib, "phc_gemm_make_images") else GemmDescNoActImage if b"A_img" not in blob
                     else GemmDescNoOutImage if b"C_img" not in blob else _lib.PhcGemmDesc)
    lib.phc_gemm_group.argtypes = [C.POINTER(lib.desc_type), C.c_int32, C.c_void_p]
    return lib


def is_dw(d):
    return d.accumulate and not d.a_kmajor


def desc_array(lib, descs, out_images=True):
    """out_images False: the problems as a build without C_img runs them (forward and dX read A from fp32 on the image loop)"""
    T = lib.desc_type
    names = [f for f, _ in T._fields_]
    plain = "C_img" not in names or not out_images
    # without A_img a build stages the weight gradient from the fp32 operands (it refuses B_img with mn-major A)
    drop_b = lambda d: "A_img" not in names and bool(d.A_img)  # noqa: E731
    drop = lambda d, f: (f == "B_img" and drop_b(d)) or (plain and (f == "C_img" or (f == "A_img" and not is_dw(d))))  # noqa: E731
    return (T * len(descs))(*[T(*[None if drop(d, f) else getattr(d, f) for f in names]) for d in descs])


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("a", nargs="?", default=os.path.join(ROOT, "phc_b200", "lib", "alt_parent", "libphc_b200.so"))
    ap.add_argument("b", nargs="?", default=os.path.join(ROOT, "phc_b200", "lib", "libphc_b200.so"))
    ap.add_argument("--turns", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    libs = {"A": open_lib(args.a), "B": open_lib(args.b)}
    print(f"A = {args.a}\nB = {args.b}")
    print(f"gpu: {torch.cuda.get_device_name(0)} | {gpu_info()}  (name, power limit, SM clock, max SM clock)")

    dev = torch.device("cuda:0")
    agent, _ = bench.build_agent(bench.NUM_ENVS, dev, 0, 1, host_bank=False)
    eng, net = agent.engine, agent.model
    assert eng.backend == "tc5s" and eng.precision == "fp32"
    x, xa = agent._x_mb, agent._amp_mb
    stacks = [(net.actor, x, agent._ws_actor), (net.critic, x, agent._ws_critic), (net.disc, xa, agent._ws_disc)]
    n_roll = agent._ws_actor_roll["out"].shape[0]
    x_roll = torch.zeros(n_roll, x.shape[1], device=dev)
    roll = [(net.actor, x_roll, agent._ws_actor_roll), (net.critic, x_roll, agent._ws_critic_roll)]

    # seeded operands: inputs, every workspace tensor a launch reads, the gradient bucket
    gen = torch.Generator(device=dev).manual_seed(0)
    state = [x, xa, x_roll, net.grads]
    for _, _, ws in stacks + roll:
        for v in ws.values():
            state += v if isinstance(v, list) else [v]
    for t in state:
        if t.dtype == torch.float32:
            t.copy_(torch.randn(t.shape, generator=gen, device=dev))
        else:
            t.copy_(torch.randint(-2**31, 2**31 - 1, t.shape, generator=gen, device=dev, dtype=torch.int64).to(t.dtype))
    saved = [t.clone() for t in state]

    depth = max(len(st.layers) for st, _, _ in stacks)
    fwd = [[eng.fwd_desc(st, li, xin, ws) for st, xin, ws in stacks if li < len(st.layers)] for li in range(depth)]
    bwd = []
    for k in range(depth):
        descs = []
        for st, xin, ws in stacks:
            li = len(st.layers) - 1 - k
            if li >= 0:
                descs += [d for d in eng.bwd_descs(st, li, xin, ws) if d is not None]
        bwd.append(descs)
    fwd_roll = [[eng.fwd_desc(st, li, xin, ws) for st, xin, ws in roll if li < len(st.layers)] for li in range(depth)]
    groups = [(f"fwd L{li}", g) for li, g in enumerate(fwd)] + [(f"bwd L-{k + 1}", g) for k, g in enumerate(bwd)]
    groups += [(f"rollout fwd L{li} ({n_roll} rows)", g) for li, g in enumerate(fwd_roll)]
    split = [(f"{part} L-{k + 1}", [d for d in g if is_dw(d) == (part == "dW")]) for k, g in enumerate(bwd) for part in ("dW", "dX")]
    split = [(name, g) for name, g in split if g]                  # the first layer has no dX
    # activation images made before a launch: requested by eng.bwd_descs / eng.fwd_desc, made by eng.make_images (it also points
    # the descriptors at them).  A build without C_img (and any build with 128 x 256 tiles, which refuse it) runs the forward and
    # dX problems from the fp32 operands and only makes the weight gradient's images.
    jobs = {(name, True): eng.make_images(g) for name, g in groups + split}
    jobs.update({(name, False): eng.make_images([d for d in g if is_dw(d)]) for name, g in groups + split})
    arrays = {(key, o): {name: (desc_array(lib, g, o), len(g)) for name, g in groups + split} for key, lib in libs.items() for o in (True, False)}
    for name, g in groups:
        assert len(g) <= _lib.PHC_GEMM_GROUP_MAX, name

    tile = [128]

    def launch(lib, name):
        o = lib.desc_type is _lib.PhcGemmDesc and tile[0] == 128
        arr, n = arrays[("A" if lib is libs["A"] else "B", o)][name]
        stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        if lib.desc_type in (_lib.PhcGemmDesc, GemmDescNoOutImage) and jobs[(name, o)][1]:
            rc = lib.phc_gemm_make_images(jobs[(name, o)][0], jobs[(name, o)][1], stream)
            if rc:
                raise RuntimeError(f"phc_gemm_make_images({name}) = {rc}: {lib.phc_last_error().decode()}")
        rc = lib.phc_gemm_group(arr, n, stream)
        if rc:
            raise RuntimeError(f"phc_gemm_group({name}) = {rc}: {lib.phc_last_error().decode()}")

    def set_tile(w):
        tile[0] = w
        for lib in libs.values():
            assert lib.phc_gemm_set_precision(_lib.PHC_GEMM_FP32_3XTF32) == 0 and lib.phc_gemm_tc5s_set_tile(w) == 0
            assert lib.phc_gemm_tc5s_set_sched(-1) == 0

    # ---- bit identity: the whole chain once per build from the same state
    ok_all = True
    for w in (128, 256):
        set_tile(w)
        outs = {}
        for key, lib in libs.items():
            for t, s in zip(state, saved):
                t.copy_(s)
            for name, _ in groups:
                launch(lib, name)
            torch.cuda.synchronize()
            outs[key] = [t.clone() for t in state]
        bad = [i for i, (a, b) in enumerate(zip(outs["A"], outs["B"])) if not torch.equal(a, b)]
        ok_all &= not bad
        print(f"tile 128x{w}: outputs of A and B torch.equal over {len(state)} tensors: {'yes' if not bad else 'NO, differ at %s' % bad}")
    for t, s in zip(state, saved):
        t.copy_(s)

    # ---- timing
    def turn(lib, name):
        launch(lib, name)
        launch(lib, name)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.iters):
            launch(lib, name)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e3 / args.iters

    tot = {}
    for w in (128, 256):
        set_tile(w)
        print(f"\n128 x {w} tiles: us per launch, median [min, max] of {args.turns} alternating turns of {args.iters} launches")
        print(f"{'group':28s} {'TFLOP':>7s} | {'A us':>24s} {'A TF/s':>7s} | {'B us':>24s} {'B TF/s':>7s} | B/A")
        for name, g in groups + split:
            if w == 256 and name.startswith("rollout"):
                continue
            flop = 3.0 * sum(2.0 * d.M * d.N * d.K for d in g)
            ts = {"A": [], "B": []}
            for _ in range(args.turns):
                for key, lib in libs.items():
                    ts[key].append(turn(lib, name))
            med = {k: statistics.median(v) for k, v in ts.items()}
            for k in ts:
                tot[(w, k, name.split()[0])] = tot.get((w, k, name.split()[0]), 0.0) + med[k]
            cell = lambda k: f"{med[k]:8.1f} [{min(ts[k]):6.1f}, {max(ts[k]):6.1f}] {flop / med[k] / 1e6:7.1f}"  # noqa: E731
            print(f"{name:28s} {flop / 1e12:7.3f} | {cell('A')} | {cell('B')} | {med['B'] / med['A']:.3f}")
        for part in ("fwd", "bwd", "dW", "dX", "rollout"):
            if (w, "A", part) in tot:
                a, b = tot[(w, "A", part)], tot[(w, "B", part)]
                print(f"sum of medians, {part:8s}: A {a:9.1f} us   B {b:9.1f} us   B/A {b / a:.3f}")

    # ---- the activation images alone (part of B's backward times above): bytes read (the operands) and written (the images)
    if libs["B"].desc_type is _lib.PhcGemmDesc:
        set_tile(128)
        print("\nactivation images made before the launches (B's phc_gemm_make_images alone)")
        stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        for name, _ in groups:
            arr, n = jobs[(name, True)]
            if not n:
                continue
            rd = sum(4.0 * arr[i].N * arr[i].K for i in range(n))
            wr = sum(4.0 * libs["B"].phc_gemm_image_floats(arr[i].N, arr[i].K) for i in range(n))
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            libs["B"].phc_gemm_make_images(arr, n, stream)
            e0.record()
            for _ in range(args.iters):
                libs["B"].phc_gemm_make_images(arr, n, stream)
            e1.record()
            torch.cuda.synchronize()
            us = e0.elapsed_time(e1) * 1e3 / args.iters
            print(f"{name:28s} {n} images: {us:8.1f} us, read {rd / 1e9:.3f} GB + write {wr / 1e9:.3f} GB = {(rd + wr) / us / 1e3:7.1f} GB/s")
    net.grads.zero_()
    print(f"gpu after: {gpu_info()}")
    if not ok_all:
        print("FAIL: outputs differ")
        sys.exit(1)


if __name__ == "__main__":
    main()
