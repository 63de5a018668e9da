"""The YDSCHED_DEBUG solve lines (DESIGN.md §7c) as the tests read them."""


def solves(err: str) -> list[dict]:
    """The `key value` pairs of every YDSCHED_DEBUG solve line."""
    out = []
    for line in err.splitlines():
        if line.startswith("ydsched: solve n "):
            t = line[len("ydsched: solve "):].split()
            out.append({k: float(v) if "." in v else int(v) for k, v in zip(t[::2], t[1::2])})
    return out
