"""dfgpu_hash_partition_device with bit-packed columns on 100M rows, against the same shape without them, for one or more builds.

  python scripts/partition_bits_timing.py --lib A/datafusion_b200/libdfgpu.so [--lib B/...] [--rows N] [--parts 8 32] [--rounds 2] [--out f.json]

Each --lib is measured in a subprocess that imports the datafusion_b200 package next to that library, so two builds (say a parent
commit's tree and this one) alternate in one run.  Shapes, all with an Int64 key:
  bits : key, nullable Int64, nullable Decimal128(38, 4), Boolean   (validity ~50% NULL, random bits)
  floor: key, Int64, Decimal128(38, 4)                               (no bit-packed data: the fixed-width traffic alone)
Time = median of 5 calls between CUDA events, after 2 warm-up calls.  Bytes = the least traffic the pass needs: the histogram reads the
key, the scatter reads and writes every column once (bit-packed columns at 1 bit per row); "of_peak" is that over the H100 SXM
data sheet's 3.35 TB/s HBM3 bandwidth.  The outputs of every build are fingerprinted on the device (offsets, values, validity bits up to
the row count) and must agree across builds."""
import argparse
import json
import os
import subprocess
import sys


def worker(lib, rows, parts):
    root = os.path.dirname(os.path.dirname(os.path.abspath(lib)))
    sys.path.insert(0, root)
    import numpy as np
    import torch
    from datafusion_b200 import capi as D
    assert os.path.abspath(D.LIB_PATH) == os.path.abspath(lib), (D.LIB_PATH, lib)
    ctx = D.Context(0)
    n = rows
    dec = D.decimal128(38, 4)
    words = (n + 63) // 64
    gen = lambda seed, k: ctx.generate_i64(D.GEN_SPLITMIX, seed, 0, 0, 0, k)
    key, v64, vdec = gen(42, n), gen(8, n), gen(9, 2 * n)
    m64, mdec, bvals = gen(11, words), gen(12, words), gen(13, words)

    def col(t, buf, valid=None):
        c = D.Column()
        c.type, c.flags, c.length, c.offset, c.null_count = t, 0, n, 0, (-1 if valid is not None else 0)
        c.values, c.validity = buf.ptr, (valid.ptr if valid is not None else None)
        return c

    shapes = {"bits": [col(D.INT64, key), col(D.INT64, v64, m64), col(dec, vdec, mdec), col(D.BOOL, bvals)],
              "floor": [col(D.INT64, key), col(D.INT64, v64), col(dec, vdec)]}
    dev = torch.device("cuda", 0)

    def dev_bytes(ptr, nbytes):
        from datafusion_b200.exchange import _CudaView
        return torch.as_tensor(_CudaView(ptr, nbytes, "|u1", None), device=dev)

    def fingerprint(t):
        # position-weighted wrapping sum of the bytes as int64 words (the tail bytes added one by one)
        full = t[: t.numel() // 8 * 8].view(torch.int64)
        w = torch.arange(full.numel(), device=dev, dtype=torch.int64) * 2 + 1
        s = int((full * w).sum().item()) if full.numel() else 0
        return s ^ int(t[full.numel() * 8:].to(torch.int64).sum().item()) if t.numel() % 8 else s

    res = []
    for shape, cols in shapes.items():
        bits_per_row = sum(1 for c in cols if c.type == D.BOOL) + sum(1 for c in cols if c.validity)
        fixed = sum(D.WIDTH[c.type] for c in cols if c.type != D.BOOL)
        need = n * (8 + 2 * fixed) + 2 * (n * bits_per_row) / 8
        for P in parts:
            ms = []
            for it in range(7):
                e0, e1 = ctx.event(), ctx.event()
                ctx.record(e0)
                b, offs = D.hash_partition_device(ctx, cols, [0], P)
                ctx.record(e1)
                ctx.sync()
                if it >= 2:
                    ms.append(ctx.elapsed_ms(e0, e1))
                if it < 6:
                    b.release()
            fp = [list(offs)]
            for i in range(b.num_columns):
                c = b.column(i)
                nb = (n + 7) // 8 if c.type == D.BOOL else n * D.WIDTH[c.type]
                f = [fingerprint(dev_bytes(c.values, nb))]
                if c.validity:
                    f.append(fingerprint(dev_bytes(c.validity, (n + 7) // 8)))
                fp.append(f)
            b.release()
            med = float(np.median(ms))
            res.append({"shape": shape, "parts": P, "rows": n, "ms": round(med, 3), "ms_all": [round(x, 3) for x in ms], "bytes": int(need),
                        "TBps": round(need / med / 1e9, 3), "of_peak": round(need / med / 1e9 / 3.35, 3), "fingerprint": fp})
    ctx.close()
    print("RESULT " + json.dumps(res), flush=True)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", required=True, help="path of a libdfgpu.so inside a datafusion_b200 package directory")
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--parts", type=int, nargs="+", default=[8, 32])
    ap.add_argument("--rounds", type=int, default=2, help="times every build is measured, alternating")
    ap.add_argument("--out", default=None)
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        worker(a.lib[0], a.rows, a.parts)
        return
    info = gpu_info()
    print("gpu (name, power limit, max SM clock, SM clock):", info, flush=True)
    runs = []
    for rnd in range(a.rounds):
        for lib in a.lib:
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", "--lib", lib, "--rows", str(a.rows), "--parts", *map(str, a.parts)],
                               capture_output=True, text=True)
            line = [x for x in r.stdout.splitlines() if x.startswith("RESULT ")]
            if r.returncode != 0 or not line:
                print(r.stdout[-2000:], r.stderr[-4000:], flush=True)
                raise SystemExit(f"worker failed for {lib}")
            for x in json.loads(line[0][7:]):
                x.update(lib=lib, round=rnd)
                runs.append(x)
                print(f"round {rnd} {lib}: {x['shape']:5s} P={x['parts']:2d} {x['ms']:8.3f} ms  {x['TBps']:.3f} TB/s  {x['of_peak']:.3f} of 3.35 TB/s", flush=True)
    same = True
    for shape in ("bits", "floor"):
        for P in a.parts:
            fps = {json.dumps(x["fingerprint"]) for x in runs if x["shape"] == shape and x["parts"] == P}
            same &= len(fps) == 1
            print(f"{shape} P={P}: outputs identical across builds and rounds: {len(fps) == 1}", flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump({"gpu": info, "runs": runs, "outputs_identical": same}, f, indent=1)
    if not same:
        raise SystemExit("outputs differ between builds")


if __name__ == "__main__":
    main()
