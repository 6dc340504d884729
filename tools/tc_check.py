import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import lance_b200 as lb
from lance_b200 import synth
os.environ["LB2_TC_STATS"] = "1"
lb.set_device(0)
data = synth.sift_like(200000, 128, seed=5)
cent = data[np.random.default_rng(0).choice(200000, 256, replace=False)].copy()
# a few Lloyd iterations to get realistic centroids
km = lb.train_kmeans(data[:65536], 128, 256, max_iters=5, centroids=cent)
cent = km.centroids
dd = lb.DeviceArray.from_numpy(data)
lb.profile.reset(); lb.profile.enable(True)
p1, d1, v1 = lb.compute_partitions(cent, dd)
lb.profile.enable(False)
for name in ("tc_filter", "tc_rerank", "assign_exact_fallback", "tc_row_norms", "tc_prep_centroids", "assign_exact"):
    print(name, lb.profile.get(name))
os.environ["LB2_DISABLE_TC"] = "1"
lb.profile.reset(); lb.profile.enable(True)
p2, d2, v2 = lb.compute_partitions(cent, dd)
lb.profile.enable(False)
print("exact", lb.profile.get("assign_exact"))
print("equal:", np.array_equal(p1, p2), np.array_equal(d1, d2))
