"""A seeded generator of MNIST-like digits for the dimensionality-reduction template's tests and benchmark: 28 x 28
integer intensities 0-255, mostly zeros, drawn from per-class strokes with a random shift and noise; labels 0-9."""
import numpy as np

SIDE = 28


def _strokes(seed=1234):
    """Ten fixed stroke templates: each class is a few thick line segments in the centre 20 x 20."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(10):
        img = np.zeros((SIDE, SIDE))
        for _ in range(int(rng.integers(2, 5))):
            (r0, c0), (r1, c1) = rng.integers(4, 24, size=(2, 2))
            for t in np.linspace(0.0, 1.0, 40):
                r, c = int(round(r0 + t * (r1 - r0))), int(round(c0 + t * (c1 - c0)))
                img[max(r - 1, 0):r + 2, max(c - 1, 0):c + 2] = 1.0
        out.append(img)
    return out


def digits(n, seed=0, labels=10):
    """(pixels int [n, 784], labels float [n]) with labels 0 .. labels - 1."""
    rng = np.random.default_rng(seed)
    base = _strokes()
    y = rng.integers(0, labels, size=n)
    x = np.zeros((n, SIDE * SIDE), np.int64)
    for i in range(n):
        img = np.roll(base[int(y[i])], (int(rng.integers(-2, 3)), int(rng.integers(-2, 3))), axis=(0, 1))
        v = img * rng.uniform(150, 255) + (rng.random((SIDE, SIDE)) < 0.02) * rng.uniform(0, 255, (SIDE, SIDE))
        x[i] = np.clip(np.rint(v), 0, 255).astype(np.int64).reshape(-1)
    return x, y.astype(np.float64)


def feature_string(row) -> str:
    """The doc's feature string: the values joined by ", "."""
    return ", ".join(str(int(v)) if float(v).is_integer() and abs(v) < 2 ** 53 else repr(float(v)) for v in row)


def events(x, y):
    """digitData events of rows x with labels y."""
    return [dict(event="digitData", entityType="digit", entityId=str(i),
                 properties={"label": float(lab), "features": feature_string(row)}) for i, (row, lab) in
            enumerate(zip(x, y))]
