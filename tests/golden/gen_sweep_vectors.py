"""Generator of tests/golden/sweep_vectors.npz: the 8-bit conversion of GenerateCameraOverlaps' and GenerateEquirect's
slices pinned to cv2 4.13.

Both apps write imwrite(filename, 255.0f * image) of a float B, G, R, A image.  The fp32 product is formed first (here
in numpy, as float32 * float32); imwrite then converts the CV_32F matrix to CV_8U (convertTo: cvRound, round half to
even, saturate; NaN and +-inf become 0) and encodes it.  cv2.imencode runs that conversion and the PNG encoder;
cv2.imdecode gives back the stored bytes.  The inputs mix ordinary values, NaN, +-inf, negative numbers, values that
scale past 255 and past the int range, and values whose product with 255 is exactly k + 0.5 (rounding ties)."""
import os

import cv2
import numpy as np

rng = np.random.default_rng(17)
special = np.float32([np.nan, np.inf, -np.inf, -0.0, 0.0, -1e-9, -0.3, 1.0, 1.0 + 1e-6, 1.5, 3e6, 1e10, -1e10,
                      8421504.0, 8421505.0])
k = np.arange(0, 255, dtype=np.float64)
cand = ((k + 0.5) / 255).astype(np.float32)
ties = cand[cand * np.float32(255) == (k + 0.5).astype(np.float32)]
assert len(ties) > 20
v = np.concatenate([rng.random(600, dtype=np.float32), rng.normal(0.5, 1.0, 200).astype(np.float32), special, ties])
v = np.concatenate([v, np.zeros((-len(v)) % 4, np.float32)]).reshape(1, -1, 4)
assert cv2.__version__.startswith("4.13")
scaled = (np.float32(255.0) * v).astype(np.float32)
ok, buf = cv2.imencode(".png", scaled)
assert ok
png = cv2.imdecode(buf, cv2.IMREAD_UNCHANGED)
assert png.dtype == np.uint8 and png.shape == v.shape
np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "sweep_vectors.npz"), img=v, png=png,
                    ties=ties)
