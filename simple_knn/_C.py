"""`distCUDA2(points)`: per point, the mean of the squared distances to its three nearest neighbours
(gaussianhaircut_b200/knn.py)."""
from gaussianhaircut_b200.knn import mean_dist3 as distCUDA2  # noqa: F401
