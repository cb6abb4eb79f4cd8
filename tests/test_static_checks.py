"""Static checks of the CUDA sources for hazards the CPU emulation cannot see."""
import pathlib, re
CSRC = pathlib.Path(__file__).resolve().parents[1] / "dedalus_b200" / "csrc"


def _launches(text):
    for m in re.finditer(r"DB_LAUNCH\(\s*([A-Za-z_0-9]+)(<[^()]*?>)?\s*,", text):
        i = m.end(); depth = 0; args = []; cur = ""           # split the macro arguments at top-level commas
        while True:
            ch = text[i]
            if ch in "([{":
                depth += 1
            if ch in ")]}":
                if depth == 0:
                    args.append(cur.strip()); break
                depth -= 1
            if ch == "," and depth == 0:
                args.append(cur.strip()); cur = ""
            else:
                cur += ch
            i += 1
        yield m.group(1), args[2], m.start()          # kernel name, dynamic shared memory expression (after grid, block), position


def _constant(expr, defines):
    """Value of a compile-time size expression, or None if it depends on run-time values."""
    e = expr
    for _ in range(6):
        for name, val in defines.items():
            e = re.sub(rf"\b{name}\b", f"({val})", e)
    e = re.sub(r"sizeof\((double|int64_t|size_t)\)", "8", e)
    e = re.sub(r"sizeof\((int|int32_t|float|unsigned)\)", "4", e)
    e = re.sub(r"\((size_t|int|int64_t)\)", "", e)
    if not re.fullmatch(r"[0-9+\-*/() ]+", e):
        return None
    try:
        return int(eval(e.replace("/", "//")))
    except Exception:
        return None


def test_every_runtime_sized_launch_above_48k_opts_in():
    """A launch asking for more than 48 KB of dynamic shared memory fails on the GPU with 'invalid argument' unless the kernel was
    given cudaFuncAttributeMaxDynamicSharedMemorySize first; the emulation accepts anything up to the 227 KB hardware limit.  Every
    DB_LAUNCH whose size is not a compile-time constant <= 48 KB must have the attribute set for the same kernel in the same file."""
    common = (CSRC / "db_common.cuh").read_text()
    checked = set()
    for f in sorted(CSRC.glob("*.cu")):
        text = f.read_text()
        defines = dict(re.findall(r"#define\s+([A-Z_0-9]+)\s+([0-9][0-9 *+()]*)\s*(?://.*)?$", common + "\n" + text, flags=re.M))
        opted = set(re.findall(r"(?:cudaFuncSetAttribute|DB_SET_SMEM_ATTR)\(\s*([A-Za-z_0-9]+)", text))
        for kern, smem, pos in _launches(text):
            if re.fullmatch(r"[A-Za-z_]+", smem):                       # a named size: take its definition closest above the launch
                defs = [m for m in re.finditer(rf"\b{smem}\s*=\s*([^;]+);", text[:pos])]
                smem_expr = defs[-1].group(1) if defs else smem
            else:
                smem_expr = smem
            val = _constant(smem_expr, defines)
            if val is not None and val <= 48 * 1024:
                continue
            checked.add(kern)
            assert kern in opted, f"{f.name}: {kern} is launched with dynamic shared memory '{smem_expr}' but never opts in above 48 KB"
    # the launches with a run-time size (the parse must find every one of them)
    assert checked >= {"k_banded_solve", "k_dense_solve", "k_band_lines", "k_batches_matvec", "k_pointwise", "k_pointwise_v3",
                       "k_pointwise_pairs"}, checked
