"""k1_budget.py -- static instruction budget of K1 (pyr_fast_kernel) per phase, CPU only.

Compiles pyr_fast_kernel.cu for sm_90a with the Makefile's flags, disassembles it with line info (nvdisasm -g) and attributes
every SASS instruction to a phase of the kernel by the source line it comes from (the phase comments "---- ..." of the kernel;
the FAST helpers count to FAST, CUDA's intrinsic headers take the phase of the line before them).  The warp instructions a phase issues per tile
are then estimated from the thread mapping of its loop: a rolled loop body (a backward branch) counts once per warp iteration,
unrolled copies count in proportion to the iterations each warp runs.  Multiplied by the config-2 tile counts per level (bench.py:
754x480, 8 levels x1.2, 3 cameras x 128 frames, the cameras' mirror masks), with tiles of flag 0 (no pixel inside the mask)
left out of FAST and NMS, this gives the warp instructions per step.  It is a static estimate: branches inside a phase
(border tests, the mask look-up of the NMS, the corner appends) are counted as if taken by every warp, and the
source staging is counted for the TMA path (its fall-back loops are left out).  Compare numbers from the same tool only.

python tools/k1_budget.py [--src path/to/pyr_fast_kernel.cu] [--sass-out FILE]"""
import argparse
import math
import pathlib
import re
import subprocess
import sys
import tempfile

import numpy as np

ROOT = pathlib.Path(__file__).resolve().parents[1]
CSRC = ROOT / "multicol_slam_b200" / "csrc"
NVCC = "/usr/local/cuda/bin/nvcc"
NVDISASM = "/usr/local/cuda/bin/nvdisasm"
THREADS, TW, TH = 256, 64, 32

# phase comment (substring of the kernel source) -> phase; the first phase starts at the kernel's signature
MARKERS = [("per-tile slices", "set-up"), ("stage the source rows", "staging"), ("every pixel of the score tile", "set-up"),
           ("identity resize of a tile", "level-0 copy"), ("bilinear resize", "resize"), ("same-cell masks", "set-up"),
           ("(a) store the unblurred", "stores"), ("(b) packed horizontal", "h-sums"), ("(c) FAST", "FAST"),
           ("(d) blurred tile", "blur"), ("(e) per-cell", "NMS")]
HELPERS = {"fast_margin2": "FAST", "fast_pair_margin": "FAST", "fast_pair_score": "FAST"}
# lines of the two arms of the resize's level test, counted only on the levels that take them
ARMS = [(re.compile(r"v0 = r0\[xs00\]"), "resize, level-0 arm"),
        (re.compile(r"const int h[01][01] = |v[01] = \(\(\(b0|v0 = min\(max"), "resize, bilinear arm")]


def makefile_flags():
    mk = (CSRC / "Makefile").read_text()
    arch = re.search(r"^ARCH := (.*)$", mk, re.M).group(1)
    flags = re.search(r"^NVFLAGS := (.*)$", mk, re.M).group(1).replace("$(ARCH)", arch)
    return flags.split()


def compile_sass(src, tmp):
    cubin = pathlib.Path(tmp) / "k1.cubin"
    # -I: the kernel's includes resolve against the package's csrc even when --src points at another copy of the file
    r = subprocess.run([NVCC, *makefile_flags(), "-I", str(CSRC), "-cubin", "-o", str(cubin), str(src)],
                       capture_output=True, text=True, check=True)
    m = re.search(r"pyr_fast_kernel.*?\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n"
                  r".*?Used (\d+) registers.*?(\d+) bytes smem", r.stderr, re.S)
    info = dict(zip(("stack", "spill_st", "spill_ld", "regs", "smem"), map(int, m.groups())))
    sass = subprocess.run([NVDISASM, "-g", "-c", str(cubin)], capture_output=True, text=True, check=True).stdout
    return sass, info


def phase_of_lines(src_lines):
    """source line (1-based) -> phase for the kernel body; None outside it"""
    first = next(i for i, l in enumerate(src_lines) if re.search(r"^pyr_fast_kernel\(", l))
    last = next(i for i in range(first, len(src_lines)) if src_lines[i].startswith("}"))
    out, cur = {}, "set-up"
    for name, ph in HELPERS.items():               # inlined helpers of one phase
        for i, l in enumerate(src_lines):
            if re.search(r"__device__.*\b" + name + r"\(", l):
                j = next(k for k in range(i, len(src_lines)) if src_lines[k].startswith("}"))
                out.update({k + 1: ph for k in range(i, j + 1)})
    for i in range(first, last + 1):
        for key, ph in MARKERS:
            if key in src_lines[i] and "//" in src_lines[i]:
                cur = ph
        ph = cur
        for pat, arm in ARMS:
            if pat.search(src_lines[i]):
                ph = arm
        out[i + 1] = ph
    return out


def parse(sass, src_name, lines):
    """-> [(address, phase, text)] of pyr_fast_kernel, and {label: address}"""
    body = sass[re.search(r"^\.text\._ZN3mcs15pyr_fast_kernel\S*:$", sass, re.M).end():]
    end = re.search(r"^\s*\.section\s", body, re.M)
    body = body[:end.start()] if end else body
    instrs, labels, phase, pending = [], {}, "set-up", []
    for raw in body.splitlines():
        m = re.match(r'\s*//## File "([^"]+)", line (\d+)', raw)
        if m:
            if m.group(1).endswith(src_name) and int(m.group(2)) in lines:
                phase = lines[int(m.group(2))]
            continue
        m = re.match(r"^(\.L_x_\d+):", raw)
        if m:
            pending.append(m.group(1))
            continue
        m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(.*?);", raw)
        if m:
            addr = int(m.group(1), 16)
            for p in pending:
                labels[p] = addr
            pending = []
            instrs.append((addr, phase, m.group(2)))
    return instrs, labels


def loop_bodies(instrs, labels):
    """addresses inside rolled loops: from the target of a conditional backward branch to the branch (an unconditional one
    returns from a block the compiler placed out of line)"""
    inside = set()
    for addr, ph, text in instrs:
        m = re.search(r"^@!?U?P\d BRA `\((\.L_x_\d+)\)", text)
        if m and labels.get(m.group(1), addr + 1) <= addr:
            inside.update(a for a, _, _ in instrs if labels[m.group(1)] <= a <= addr)
    return inside


def warp_iters(per_thread):
    """per-thread iteration counts -> per-warp counts (a warp runs an iteration if any lane does)"""
    t = np.asarray(per_thread).reshape(THREADS // 32, 32)
    return t.max(1)


def mappings(src_text):
    """phase -> per-warp iteration counts of its loop over one full tile"""
    tid = np.arange(THREADS)
    strided = lambda n: np.array([len(range(t, n, THREADS)) for t in tid])                 # noqa: E731
    m = {"stores": strided(TH * TW // 4), "h-sums": strided((TH + 4) * TW // 2), "blur": strided(TH * TW // 4),
         "NMS": strided(TH * TW // 2),
         "resize": np.array([len(range(t // 36, 40, 7)) if t < 252 else 0 for t in tid]),
         "level-0 copy": np.array([len(range(t // 18, 40, 14)) if t < 252 else 0 for t in tid])}
    if "one lane per pair column" in src_text:
        m["FAST"] = np.array([4 + (t < 2 * 32 + TH + 2) for t in tid])
    else:
        m["FAST"] = strided((TH + 2) * (TW + 2) // 2)
    m["resize, level-0 arm"] = m["resize, bilinear arm"] = m["resize"]
    return {k: warp_iters(v) for k, v in m.items()}


def config2_tiles():
    """per level: (tiles, tiles with flag != 0, level-0 tiles whose columns need no reflection) for one config-2 step"""
    sys.path.insert(0, str(ROOT))
    sys.path.insert(0, str(ROOT / "oracle"))
    import bench
    import pyref
    from multicol_slam_b200 import synth
    cfg = bench.CONFIGS[2]
    cams = bench.rig_cams(cfg)
    frames = cfg["frames"]
    out = []
    per_cam = []
    for c in cams:
        ex = pyref.Extractor(nlevels=bench.NLEVELS)
        ex.compute_pyramid(np.zeros((cfg["h"], cfg["w"]), np.uint8), synth.mirror_mask(c))
        per_cam.append([(ex.roi[l], ex.mpyr[l][pyref.EDGE:pyref.EDGE + ex.roi[l][1], pyref.EDGE:pyref.EDGE + ex.roi[l][0]])
                        for l in range(bench.NLEVELS)])
    for l in range(bench.NLEVELS):
        (w, h), _ = per_cam[0][l]
        tx, ty = math.ceil(w / TW), math.ceil(h / TH)
        on = 0
        for c in range(len(cams)):
            m = per_cam[c][l][1]
            for y in range(ty):
                for x in range(tx):
                    on += bool(m[y * TH:(y + 1) * TH, x * TW:(x + 1) * TW].any())
        interior_cols = sum(1 for x in range(tx) if x * TW >= 4 and x * TW + TW + 4 <= w) if l == 0 else 0
        out.append(dict(w=w, h=h, tiles=tx * ty * len(cams) * frames, fast_tiles=on * frames,
                        copy_tiles=interior_cols * ty * len(cams) * frames))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--src", default=str(CSRC / "pyr_fast_kernel.cu"))
    ap.add_argument("--sass-out", help="write the annotated SASS (phase per instruction) here")
    args = ap.parse_args()
    src = pathlib.Path(args.src).resolve()
    text = src.read_text()
    with tempfile.TemporaryDirectory() as tmp:
        sass, info = compile_sass(src, tmp)
    instrs, labels = parse(sass, src.name, phase_of_lines(text.splitlines()))
    loops = loop_bodies(instrs, labels)
    maps = mappings(text)
    has_copy = "identity resize of a tile" in text
    per_tile = {}                                   # phase -> warp instructions per tile that runs it
    static = {}
    for addr, ph, _ in instrs:
        static[ph] = static.get(ph, 0) + 1
        it = maps.get(ph)
        if ph == "staging" and addr in loops:       # fall-back staging loops: not taken with TMA
            w = 0.0
        elif it is None:                            # straight code: once per warp
            w = THREADS // 32
        elif addr in loops:                         # rolled loop body: once per warp iteration
            w = float(it.sum())
        else:                                       # unrolled copies: the share of them each warp runs
            w = float((it / max(it.max(), 1)).sum())
        per_tile[ph] = per_tile.get(ph, 0.0) + w
    tiles = config2_tiles()
    total = {}
    for l, t in enumerate(tiles):
        copy = t["copy_tiles"] if has_copy else 0
        n = {"set-up": t["tiles"], "staging": t["tiles"], "stores": t["tiles"], "h-sums": t["tiles"], "blur": t["tiles"],
             "level-0 copy": copy, "resize": t["tiles"] - copy,
             "resize, level-0 arm": (t["tiles"] - copy) if l == 0 else 0, "resize, bilinear arm": t["tiles"] if l else 0,
             "FAST": t["fast_tiles"], "NMS": t["fast_tiles"]}
        for ph, v in per_tile.items():
            total[ph] = total.get(ph, 0.0) + v * n[ph]
    print(f"{src}: {info['regs']} registers, {info['spill_st']} B spill stores, {info['spill_ld']} B spill loads, "
          f"{info['smem']} B static shared memory")
    print("config 2 per step: " + ", ".join(f"level {l} {t['w']}x{t['h']}: {t['tiles']} tiles ({t['fast_tiles']} with FAST)"
                                            for l, t in enumerate(tiles)))
    print(f"{'phase':24s} {'SASS':>6s} {'warp instr / tile':>18s} {'M warp instr / step':>20s}")
    for ph in sorted(per_tile, key=lambda p: -total[p]):
        print(f"{ph:24s} {static[ph]:6d} {per_tile[ph]:18.0f} {total[ph] / 1e6:20.1f}")
    print(f"{'total':24s} {len(instrs):6d} {'':18s} {sum(total.values()) / 1e6:20.1f}")
    if args.sass_out:
        pathlib.Path(args.sass_out).write_text("\n".join(f"{a:06x} {p:22s} {t}" for a, p, t in instrs) + "\n")


if __name__ == "__main__":
    main()
