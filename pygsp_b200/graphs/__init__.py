"""Graph object and the generators the BASELINE configurations use."""
from .csr import DeviceCSR  # noqa: F401
from .graph import Graph, symmetrize_device  # noqa: F401
from .generators import (Grid2d, Grid2dImgPatches, ImgPatches, KnnSlabs, Logo,  # noqa: F401
                         NNGraph, Ring, Sensor, SensorStrips, StochasticBlockModel,
                         grid2d_adjacency_device, image_patches_device, knn_adjacency_device,
                         knn_device, laplacian_rows, morton_order, morton_order_device,
                         radius_device, sbm_adjacency)
from .random_graphs import BarabasiAlbert, ErdosRenyi, RandomRegular  # noqa: F401
from .sampled import (Community, Cube, Sphere, SwissRoll, TwoMoons,  # noqa: F401
                      knn_segments_device, radius_segments_device, subset_device)
from .structured import (Comet, FullConnected, LineGraph, LowStretchTree, Path,  # noqa: F401
                         RandomRing, Star, Torus)
