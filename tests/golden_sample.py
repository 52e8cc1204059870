"""Golden arrays too large to keep whole store every step-th index along one axis, recorded in the file as
`<key>_sample` = [axis, step] (oracle/make_golden.py: strided_sample); tests take the same sample of what they compute."""


def as_stored(t, g, key):
    """`t` sampled the way g[key] was stored (unchanged when the golden keeps the whole array)."""
    names = g.files if hasattr(g, "files") else g
    if key + "_sample" not in names:
        return t
    axis, step = (int(v) for v in g[key + "_sample"])
    sl = [slice(None)] * t.ndim
    sl[axis] = slice(None, None, step)
    return t[tuple(sl)]
