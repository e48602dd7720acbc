"""Generator of tests/golden/smr_vectors.npz: SimpleMeshRenderer's png conversion pinned to cv2 4.13.

save() writes cv_util::convertImage<cv::Vec3w>(result): Mat::convertTo(CV_16U, 65535) of the float B, G, R, A image,
then BGRA -> BGR.  cv2 has no convertTo binding; cv2.multiply with dtype CV_16U runs the same fp32 product and the same
saturate_cast (cvRound, round half to even; NaN -> 0).  The image mixes ordinary values, NaN, values below 0 and above
1, +-inf and values whose fp32 product with 65535 is exactly k + 0.5 (rounding ties)."""
import os

import cv2
import numpy as np

rng = np.random.default_rng(13)
vals = [rng.random(500, dtype=np.float32), np.float32([np.nan, -0.25, -1e-9, 0.0, 1.0, 1.0 + 1e-6, 3.5, np.inf, -np.inf])]
k = np.arange(0, 65535, 97, dtype=np.float64)
cand = ((k + 0.5) / 65535).astype(np.float32)
ties = cand[cand * np.float32(65535) == (k + 0.5).astype(np.float32)]
assert len(ties) > 20
vals.append(ties)
v = np.concatenate(vals)
v = np.concatenate([v, np.zeros((-len(v)) % 4, np.float32)]).reshape(-1, 1, 4)
assert cv2.__version__.startswith("4.13")
png = cv2.cvtColor(cv2.multiply(v, np.ones_like(v), scale=65535.0, dtype=cv2.CV_16U), cv2.COLOR_BGRA2BGR)
np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "smr_vectors.npz"), img=v, png=png,
                    ties=ties)
