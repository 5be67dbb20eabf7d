"""Graph object and the generators the BASELINE configurations use."""
from .csr import DeviceCSR  # noqa: F401
from .graph import Graph, symmetrize_device  # noqa: F401
from .generators import (Grid2d, Grid2dImgPatches, ImgPatches, KnnSlabs, Logo,  # noqa: F401
                         NNGraph, Ring, Sensor, SensorStrips, StochasticBlockModel,
                         grid2d_adjacency_device, image_patches_device, knn_adjacency_device,
                         knn_device, laplacian_rows, morton_order, morton_order_device,
                         radius_device, sbm_adjacency)
from .random_graphs import BarabasiAlbert, ErdosRenyi  # noqa: F401
