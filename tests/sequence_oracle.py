"""numpy restatements of demon_b200.sequence and csrc/fusion.cu for the tests: the chaining of consecutive pairs, the TSDF
integration in the kernel's float32 order, and marching cubes with this file's own transcription of the standard
Lorensen-Cline triangle table.  Every float32 operation is a separate numpy operation on float32 operands, which is the
kernels' round-to-nearest order without FMA contraction."""
import numpy as np

from oracle.dataset_tools import depth_ratios_numpy

f32 = np.float32
NETWORK_INTRINSICS = (0.89115971, 1.18821287, 0.5, 0.5)

# corner q of a cube is voxel (i, j, k) + CORNERS[q]; bit q of the case is set when its tsdf is < 0
CORNERS = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0], [0, 0, 1], [1, 0, 1], [1, 1, 1], [0, 1, 1]])
# the corners of the 12 edges, lower grid coordinate first (a vertex is interpolated from that corner)
EDGES = np.array([[0, 1], [1, 2], [3, 2], [0, 3], [4, 5], [5, 6], [7, 6], [4, 7], [0, 4], [1, 5], [2, 6], [3, 7]])
# the edges of each case's triangles, three per triangle
TRIANGLES = (
    (),
    (0, 8, 3),
    (0, 1, 9),
    (1, 8, 3, 9, 8, 1),
    (1, 2, 10),
    (0, 8, 3, 1, 2, 10),
    (9, 2, 10, 0, 2, 9),
    (2, 8, 3, 2, 10, 8, 10, 9, 8),
    (3, 11, 2),
    (0, 11, 2, 8, 11, 0),
    (1, 9, 0, 2, 3, 11),
    (1, 11, 2, 1, 9, 11, 9, 8, 11),
    (3, 10, 1, 11, 10, 3),
    (0, 10, 1, 0, 8, 10, 8, 11, 10),
    (3, 9, 0, 3, 11, 9, 11, 10, 9),
    (9, 8, 10, 10, 8, 11),
    (4, 7, 8),
    (4, 3, 0, 7, 3, 4),
    (0, 1, 9, 8, 4, 7),
    (4, 1, 9, 4, 7, 1, 7, 3, 1),
    (1, 2, 10, 8, 4, 7),
    (3, 4, 7, 3, 0, 4, 1, 2, 10),
    (9, 2, 10, 9, 0, 2, 8, 4, 7),
    (2, 10, 9, 2, 9, 7, 2, 7, 3, 7, 9, 4),
    (8, 4, 7, 3, 11, 2),
    (11, 4, 7, 11, 2, 4, 2, 0, 4),
    (9, 0, 1, 8, 4, 7, 2, 3, 11),
    (4, 7, 11, 9, 4, 11, 9, 11, 2, 9, 2, 1),
    (3, 10, 1, 3, 11, 10, 7, 8, 4),
    (1, 11, 10, 1, 4, 11, 1, 0, 4, 7, 11, 4),
    (4, 7, 8, 9, 0, 11, 9, 11, 10, 11, 0, 3),
    (4, 7, 11, 4, 11, 9, 9, 11, 10),
    (9, 5, 4),
    (9, 5, 4, 0, 8, 3),
    (0, 5, 4, 1, 5, 0),
    (8, 5, 4, 8, 3, 5, 3, 1, 5),
    (1, 2, 10, 9, 5, 4),
    (3, 0, 8, 1, 2, 10, 4, 9, 5),
    (5, 2, 10, 5, 4, 2, 4, 0, 2),
    (2, 10, 5, 3, 2, 5, 3, 5, 4, 3, 4, 8),
    (9, 5, 4, 2, 3, 11),
    (0, 11, 2, 0, 8, 11, 4, 9, 5),
    (0, 5, 4, 0, 1, 5, 2, 3, 11),
    (2, 1, 5, 2, 5, 8, 2, 8, 11, 4, 8, 5),
    (10, 3, 11, 10, 1, 3, 9, 5, 4),
    (4, 9, 5, 0, 8, 1, 8, 10, 1, 8, 11, 10),
    (5, 4, 0, 5, 0, 11, 5, 11, 10, 11, 0, 3),
    (5, 4, 8, 5, 8, 10, 10, 8, 11),
    (9, 7, 8, 5, 7, 9),
    (9, 3, 0, 9, 5, 3, 5, 7, 3),
    (0, 7, 8, 0, 1, 7, 1, 5, 7),
    (1, 5, 3, 3, 5, 7),
    (9, 7, 8, 9, 5, 7, 10, 1, 2),
    (10, 1, 2, 9, 5, 0, 5, 3, 0, 5, 7, 3),
    (8, 0, 2, 8, 2, 5, 8, 5, 7, 10, 5, 2),
    (2, 10, 5, 2, 5, 3, 3, 5, 7),
    (7, 9, 5, 7, 8, 9, 3, 11, 2),
    (9, 5, 7, 9, 7, 2, 9, 2, 0, 2, 7, 11),
    (2, 3, 11, 0, 1, 8, 1, 7, 8, 1, 5, 7),
    (11, 2, 1, 11, 1, 7, 7, 1, 5),
    (9, 5, 8, 8, 5, 7, 10, 1, 3, 10, 3, 11),
    (5, 7, 0, 5, 0, 9, 7, 11, 0, 1, 0, 10, 11, 10, 0),
    (11, 10, 0, 11, 0, 3, 10, 5, 0, 8, 0, 7, 5, 7, 0),
    (11, 10, 5, 7, 11, 5),
    (10, 6, 5),
    (0, 8, 3, 5, 10, 6),
    (9, 0, 1, 5, 10, 6),
    (1, 8, 3, 1, 9, 8, 5, 10, 6),
    (1, 6, 5, 2, 6, 1),
    (1, 6, 5, 1, 2, 6, 3, 0, 8),
    (9, 6, 5, 9, 0, 6, 0, 2, 6),
    (5, 9, 8, 5, 8, 2, 5, 2, 6, 3, 2, 8),
    (2, 3, 11, 10, 6, 5),
    (11, 0, 8, 11, 2, 0, 10, 6, 5),
    (0, 1, 9, 2, 3, 11, 5, 10, 6),
    (5, 10, 6, 1, 9, 2, 9, 11, 2, 9, 8, 11),
    (6, 3, 11, 6, 5, 3, 5, 1, 3),
    (0, 8, 11, 0, 11, 5, 0, 5, 1, 5, 11, 6),
    (3, 11, 6, 0, 3, 6, 0, 6, 5, 0, 5, 9),
    (6, 5, 9, 6, 9, 11, 11, 9, 8),
    (5, 10, 6, 4, 7, 8),
    (4, 3, 0, 4, 7, 3, 6, 5, 10),
    (1, 9, 0, 5, 10, 6, 8, 4, 7),
    (10, 6, 5, 1, 9, 7, 1, 7, 3, 7, 9, 4),
    (6, 1, 2, 6, 5, 1, 4, 7, 8),
    (1, 2, 5, 5, 2, 6, 3, 0, 4, 3, 4, 7),
    (8, 4, 7, 9, 0, 5, 0, 6, 5, 0, 2, 6),
    (7, 3, 9, 7, 9, 4, 3, 2, 9, 5, 9, 6, 2, 6, 9),
    (3, 11, 2, 7, 8, 4, 10, 6, 5),
    (5, 10, 6, 4, 7, 2, 4, 2, 0, 2, 7, 11),
    (0, 1, 9, 4, 7, 8, 2, 3, 11, 5, 10, 6),
    (9, 2, 1, 9, 11, 2, 9, 4, 11, 7, 11, 4, 5, 10, 6),
    (8, 4, 7, 3, 11, 5, 3, 5, 1, 5, 11, 6),
    (5, 1, 11, 5, 11, 6, 1, 0, 11, 7, 11, 4, 0, 4, 11),
    (0, 5, 9, 0, 6, 5, 0, 3, 6, 11, 6, 3, 8, 4, 7),
    (6, 5, 9, 6, 9, 11, 4, 7, 9, 7, 11, 9),
    (10, 4, 9, 6, 4, 10),
    (4, 10, 6, 4, 9, 10, 0, 8, 3),
    (10, 0, 1, 10, 6, 0, 6, 4, 0),
    (8, 3, 1, 8, 1, 6, 8, 6, 4, 6, 1, 10),
    (1, 4, 9, 1, 2, 4, 2, 6, 4),
    (3, 0, 8, 1, 2, 9, 2, 4, 9, 2, 6, 4),
    (0, 2, 4, 4, 2, 6),
    (8, 3, 2, 8, 2, 4, 4, 2, 6),
    (10, 4, 9, 10, 6, 4, 11, 2, 3),
    (0, 8, 2, 2, 8, 11, 4, 9, 10, 4, 10, 6),
    (3, 11, 2, 0, 1, 6, 0, 6, 4, 6, 1, 10),
    (6, 4, 1, 6, 1, 10, 4, 8, 1, 2, 1, 11, 8, 11, 1),
    (9, 6, 4, 9, 3, 6, 9, 1, 3, 11, 6, 3),
    (8, 11, 1, 8, 1, 0, 11, 6, 1, 9, 1, 4, 6, 4, 1),
    (3, 11, 6, 3, 6, 0, 0, 6, 4),
    (6, 4, 8, 11, 6, 8),
    (7, 10, 6, 7, 8, 10, 8, 9, 10),
    (0, 7, 3, 0, 10, 7, 0, 9, 10, 6, 7, 10),
    (10, 6, 7, 1, 10, 7, 1, 7, 8, 1, 8, 0),
    (10, 6, 7, 10, 7, 1, 1, 7, 3),
    (1, 2, 6, 1, 6, 8, 1, 8, 9, 8, 6, 7),
    (2, 6, 9, 2, 9, 1, 6, 7, 9, 0, 9, 3, 7, 3, 9),
    (7, 8, 0, 7, 0, 6, 6, 0, 2),
    (7, 3, 2, 6, 7, 2),
    (2, 3, 11, 10, 6, 8, 10, 8, 9, 8, 6, 7),
    (2, 0, 7, 2, 7, 11, 0, 9, 7, 6, 7, 10, 9, 10, 7),
    (1, 8, 0, 1, 7, 8, 1, 10, 7, 6, 7, 10, 2, 3, 11),
    (11, 2, 1, 11, 1, 7, 10, 6, 1, 6, 7, 1),
    (8, 9, 6, 8, 6, 7, 9, 1, 6, 11, 6, 3, 1, 3, 6),
    (0, 9, 1, 11, 6, 7),
    (7, 8, 0, 7, 0, 6, 3, 11, 0, 11, 6, 0),
    (7, 11, 6),
    (7, 6, 11),
    (3, 0, 8, 11, 7, 6),
    (0, 1, 9, 11, 7, 6),
    (8, 1, 9, 8, 3, 1, 11, 7, 6),
    (10, 1, 2, 6, 11, 7),
    (1, 2, 10, 3, 0, 8, 6, 11, 7),
    (2, 9, 0, 2, 10, 9, 6, 11, 7),
    (6, 11, 7, 2, 10, 3, 10, 8, 3, 10, 9, 8),
    (7, 2, 3, 6, 2, 7),
    (7, 0, 8, 7, 6, 0, 6, 2, 0),
    (2, 7, 6, 2, 3, 7, 0, 1, 9),
    (1, 6, 2, 1, 8, 6, 1, 9, 8, 8, 7, 6),
    (10, 7, 6, 10, 1, 7, 1, 3, 7),
    (10, 7, 6, 1, 7, 10, 1, 8, 7, 1, 0, 8),
    (0, 3, 7, 0, 7, 10, 0, 10, 9, 6, 10, 7),
    (7, 6, 10, 7, 10, 8, 8, 10, 9),
    (6, 8, 4, 11, 8, 6),
    (3, 6, 11, 3, 0, 6, 0, 4, 6),
    (8, 6, 11, 8, 4, 6, 9, 0, 1),
    (9, 4, 6, 9, 6, 3, 9, 3, 1, 11, 3, 6),
    (6, 8, 4, 6, 11, 8, 2, 10, 1),
    (1, 2, 10, 3, 0, 11, 0, 6, 11, 0, 4, 6),
    (4, 11, 8, 4, 6, 11, 0, 2, 9, 2, 10, 9),
    (10, 9, 3, 10, 3, 2, 9, 4, 3, 11, 3, 6, 4, 6, 3),
    (8, 2, 3, 8, 4, 2, 4, 6, 2),
    (0, 4, 2, 4, 6, 2),
    (1, 9, 0, 2, 3, 4, 2, 4, 6, 4, 3, 8),
    (1, 9, 4, 1, 4, 2, 2, 4, 6),
    (8, 1, 3, 8, 6, 1, 8, 4, 6, 6, 10, 1),
    (10, 1, 0, 10, 0, 6, 6, 0, 4),
    (4, 6, 3, 4, 3, 8, 6, 10, 3, 0, 3, 9, 10, 9, 3),
    (10, 9, 4, 6, 10, 4),
    (4, 9, 5, 7, 6, 11),
    (0, 8, 3, 4, 9, 5, 11, 7, 6),
    (5, 0, 1, 5, 4, 0, 7, 6, 11),
    (11, 7, 6, 8, 3, 4, 3, 5, 4, 3, 1, 5),
    (9, 5, 4, 10, 1, 2, 7, 6, 11),
    (6, 11, 7, 1, 2, 10, 0, 8, 3, 4, 9, 5),
    (7, 6, 11, 5, 4, 10, 4, 2, 10, 4, 0, 2),
    (3, 4, 8, 3, 5, 4, 3, 2, 5, 10, 5, 2, 11, 7, 6),
    (7, 2, 3, 7, 6, 2, 5, 4, 9),
    (9, 5, 4, 0, 8, 6, 0, 6, 2, 6, 8, 7),
    (3, 6, 2, 3, 7, 6, 1, 5, 0, 5, 4, 0),
    (6, 2, 8, 6, 8, 7, 2, 1, 8, 4, 8, 5, 1, 5, 8),
    (9, 5, 4, 10, 1, 6, 1, 7, 6, 1, 3, 7),
    (1, 6, 10, 1, 7, 6, 1, 0, 7, 8, 7, 0, 9, 5, 4),
    (4, 0, 10, 4, 10, 5, 0, 3, 10, 6, 10, 7, 3, 7, 10),
    (7, 6, 10, 7, 10, 8, 5, 4, 10, 4, 8, 10),
    (6, 9, 5, 6, 11, 9, 11, 8, 9),
    (3, 6, 11, 0, 6, 3, 0, 5, 6, 0, 9, 5),
    (0, 11, 8, 0, 5, 11, 0, 1, 5, 5, 6, 11),
    (6, 11, 3, 6, 3, 5, 5, 3, 1),
    (1, 2, 10, 9, 5, 11, 9, 11, 8, 11, 5, 6),
    (0, 11, 3, 0, 6, 11, 0, 9, 6, 5, 6, 9, 1, 2, 10),
    (11, 8, 5, 11, 5, 6, 8, 0, 5, 10, 5, 2, 0, 2, 5),
    (6, 11, 3, 6, 3, 5, 2, 10, 3, 10, 5, 3),
    (5, 8, 9, 5, 2, 8, 5, 6, 2, 3, 8, 2),
    (9, 5, 6, 9, 6, 0, 0, 6, 2),
    (1, 5, 8, 1, 8, 0, 5, 6, 8, 3, 8, 2, 6, 2, 8),
    (1, 5, 6, 2, 1, 6),
    (1, 3, 6, 1, 6, 10, 3, 8, 6, 5, 6, 9, 8, 9, 6),
    (10, 1, 0, 10, 0, 6, 9, 5, 0, 5, 6, 0),
    (0, 3, 8, 5, 6, 10),
    (10, 5, 6),
    (11, 5, 10, 7, 5, 11),
    (11, 5, 10, 11, 7, 5, 8, 3, 0),
    (5, 11, 7, 5, 10, 11, 1, 9, 0),
    (10, 7, 5, 10, 11, 7, 9, 8, 1, 8, 3, 1),
    (11, 1, 2, 11, 7, 1, 7, 5, 1),
    (0, 8, 3, 1, 2, 7, 1, 7, 5, 7, 2, 11),
    (9, 7, 5, 9, 2, 7, 9, 0, 2, 2, 11, 7),
    (7, 5, 2, 7, 2, 11, 5, 9, 2, 3, 2, 8, 9, 8, 2),
    (2, 5, 10, 2, 3, 5, 3, 7, 5),
    (8, 2, 0, 8, 5, 2, 8, 7, 5, 10, 2, 5),
    (9, 0, 1, 5, 10, 3, 5, 3, 7, 3, 10, 2),
    (9, 8, 2, 9, 2, 1, 8, 7, 2, 10, 2, 5, 7, 5, 2),
    (1, 3, 5, 3, 7, 5),
    (0, 8, 7, 0, 7, 1, 1, 7, 5),
    (9, 0, 3, 9, 3, 5, 5, 3, 7),
    (9, 8, 7, 5, 9, 7),
    (5, 8, 4, 5, 10, 8, 10, 11, 8),
    (5, 0, 4, 5, 11, 0, 5, 10, 11, 11, 3, 0),
    (0, 1, 9, 8, 4, 10, 8, 10, 11, 10, 4, 5),
    (10, 11, 4, 10, 4, 5, 11, 3, 4, 9, 4, 1, 3, 1, 4),
    (2, 5, 1, 2, 8, 5, 2, 11, 8, 4, 5, 8),
    (0, 4, 11, 0, 11, 3, 4, 5, 11, 2, 11, 1, 5, 1, 11),
    (0, 2, 5, 0, 5, 9, 2, 11, 5, 4, 5, 8, 11, 8, 5),
    (9, 4, 5, 2, 11, 3),
    (2, 5, 10, 3, 5, 2, 3, 4, 5, 3, 8, 4),
    (5, 10, 2, 5, 2, 4, 4, 2, 0),
    (3, 10, 2, 3, 5, 10, 3, 8, 5, 4, 5, 8, 0, 1, 9),
    (5, 10, 2, 5, 2, 4, 1, 9, 2, 9, 4, 2),
    (8, 4, 5, 8, 5, 3, 3, 5, 1),
    (0, 4, 5, 1, 0, 5),
    (8, 4, 5, 8, 5, 3, 9, 0, 5, 0, 3, 5),
    (9, 4, 5),
    (4, 11, 7, 4, 9, 11, 9, 10, 11),
    (0, 8, 3, 4, 9, 7, 9, 11, 7, 9, 10, 11),
    (1, 10, 11, 1, 11, 4, 1, 4, 0, 7, 4, 11),
    (3, 1, 4, 3, 4, 8, 1, 10, 4, 7, 4, 11, 10, 11, 4),
    (4, 11, 7, 9, 11, 4, 9, 2, 11, 9, 1, 2),
    (9, 7, 4, 9, 11, 7, 9, 1, 11, 2, 11, 1, 0, 8, 3),
    (11, 7, 4, 11, 4, 2, 2, 4, 0),
    (11, 7, 4, 11, 4, 2, 8, 3, 4, 3, 2, 4),
    (2, 9, 10, 2, 7, 9, 2, 3, 7, 7, 4, 9),
    (9, 10, 7, 9, 7, 4, 10, 2, 7, 8, 7, 0, 2, 0, 7),
    (3, 7, 10, 3, 10, 2, 7, 4, 10, 1, 10, 0, 4, 0, 10),
    (1, 10, 2, 8, 7, 4),
    (4, 9, 1, 4, 1, 7, 7, 1, 3),
    (4, 9, 1, 4, 1, 7, 0, 8, 1, 8, 7, 1),
    (4, 0, 3, 7, 4, 3),
    (4, 8, 7),
    (9, 10, 8, 10, 11, 8),
    (3, 0, 9, 3, 9, 11, 11, 9, 10),
    (0, 1, 10, 0, 10, 8, 8, 10, 11),
    (3, 1, 10, 11, 3, 10),
    (1, 2, 11, 1, 11, 9, 9, 11, 8),
    (3, 0, 9, 3, 9, 11, 1, 2, 9, 2, 11, 9),
    (0, 2, 11, 8, 0, 11),
    (3, 2, 11),
    (2, 3, 8, 2, 8, 10, 10, 8, 9),
    (9, 10, 2, 0, 9, 2),
    (2, 3, 8, 2, 8, 10, 0, 1, 8, 1, 10, 8),
    (1, 10, 2),
    (1, 3, 8, 9, 1, 8),
    (0, 9, 1),
    (0, 3, 8),
    (),
)


def rodrigues(aa):
    """float64 R of a float64 angle-axis: c I + (1-c) u u^T + s [u]x for |aa| > 1e-6, else I (depthmotionnet/helpers.py)."""
    aa = np.asarray(aa, dtype=np.float64)
    angle = np.sqrt(aa.dot(aa))
    if not angle > 1e-6:
        return np.eye(3)
    c, s = np.cos(angle), np.sin(angle)
    u = np.array([aa[0] / angle, aa[1] / angle, aa[2] / angle])
    cross = np.array([[0, -u[2], u[1]], [u[2], 0, -u[0]], [-u[1], u[0], 0]], dtype=u.dtype)
    R = np.empty((3, 3))
    R[...] = np.outer(u, u) * (1 - c) + c * np.eye(3, dtype=u.dtype) + cross * s
    return R


def K_pixels(intrinsics, w, h):
    fx, fy, cx, cy = np.asarray(intrinsics, dtype=np.float64)
    return np.array([[fx * w, 0, cx * w], [0, fy * h, cy * h], [0, 0, 1]], dtype=np.float64)


def projection(K64, R, t):
    """K [R|t] with [R|t] stored as float32 first and the float64 product cast to float32."""
    Rt = np.empty((3, 4), dtype=f32)
    Rt[:, :3] = R
    Rt[:, 3] = np.asarray(t).reshape(3)
    return K64.dot(Rt).astype(f32)


def lower_median(x):
    v = np.sort(x[np.isfinite(x)])
    return v[(v.size - 1) // 2], v.size


def pair_ratios(inverse_depth, rotation, translation, intrinsics=NETWORK_INTRINSICS):
    """[P-1,h,w]: the ratios of depth map k against depth map k+1 through pair k's motion."""
    inv = np.asarray(inverse_depth, dtype=f32).reshape(len(rotation), *np.shape(inverse_depth)[-2:])
    h, w = inv.shape[1:]
    depth = f32(1) / inv
    K64 = K_pixels(intrinsics, w, h)
    out = []
    for k in range(len(rotation) - 1):
        P = projection(K64, rodrigues(rotation[k]), np.asarray(translation[k], dtype=np.float64))
        out.append(depth_ratios_numpy(depth[k], depth[k + 1], K64.astype(f32), np.eye(3, dtype=f32), np.zeros(3, f32), P)[0])
    return np.array(out, dtype=f32).reshape(-1, h, w)


def chain_poses(rotation, translation, scales):
    """sigma [P], R [P+1,3,3], t [P+1,3] (float64) of the pair motions and the relative scales s_k."""
    p = len(rotation)
    sigma = np.empty(p)
    sigma[0] = 1.0
    for k in range(p - 1):
        sigma[k + 1] = sigma[k] * scales[k]
    R, t = [np.eye(3)], [np.zeros(3)]
    for k in range(p):
        Rk = rodrigues(np.asarray(rotation[k], dtype=np.float64))
        R.append(Rk.dot(R[k]))
        t.append(Rk.dot(t[k]) + sigma[k] * np.asarray(translation[k], dtype=np.float64))
    return sigma, np.array(R), np.array(t)


def chain(inverse_depth, rotation, translation, intrinsics=NETWORK_INTRINSICS):
    """The whole chain: scales [P-1], counts [P-1] of finite ratios, sigma, R, t, and depth [P,h,w] = sigma_k / inverse_depth_k."""
    ratios = pair_ratios(inverse_depth, rotation, translation, intrinsics)
    med = [lower_median(r) for r in ratios]
    scales = np.array([m[0] for m in med], dtype=np.float64)
    sigma, R, t = chain_poses(rotation, translation, scales)
    inv = np.asarray(inverse_depth, dtype=f32).reshape((len(rotation),) + np.shape(inverse_depth)[-2:])
    return {"scales": scales, "counts": np.array([m[1] for m in med]), "sigma": sigma, "R": R, "t": t,
            "depth": sigma.astype(f32)[:, None, None] / inv}


def voxel_points(dims, origin, voxel_size):
    """float32 X0, X1, X2 of every voxel, x fastest: origin + voxel_size * (i, j, k)."""
    nx, ny, nz = dims
    k, j, i = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    o, vs = np.asarray(origin, dtype=f32), f32(voxel_size)
    return [o[a] + vs * g.reshape(-1).astype(f32) for a, g in enumerate((i, j, k))]


def integrate(tsdf, weight, color, origin, voxel_size, trunc, depth, K, R, t, image=None):
    """demon_tsdf_integrate_f32 on numpy float32 state (tsdf, weight [nz,ny,nx], color [nz,ny,nx,3] or None), in place."""
    nz, ny, nx = tsdf.shape
    X0, X1, X2 = voxel_points((nx, ny, nz), origin, voxel_size)
    s, W = tsdf.reshape(-1), weight.reshape(-1)
    col = None if color is None else color.reshape(-1, 3)
    tr = f32(trunc)
    depth = np.asarray(depth, dtype=f32)
    n, h, w = depth.shape
    for fr in range(n):
        Kf, Rf, tf = np.asarray(K[fr], dtype=f32), np.asarray(R[fr], dtype=f32), np.asarray(t[fr], dtype=f32)
        with np.errstate(all="ignore"):
            cam = [((Rf[r, 0] * X0 + Rf[r, 1] * X1) + Rf[r, 2] * X2) + tf[r] for r in range(3)]
            z = cam[2]
            u = (Kf[0, 0] * cam[0]) / z + Kf[0, 2]
            v = (Kf[1, 1] * cam[1]) / z + Kf[1, 2]
            ok = (z > 0) & (u >= 0) & (u < f32(w)) & (v >= 0) & (v < f32(h))
            px = np.where(ok, np.floor(u), 0).astype(np.int64)
            py = np.where(ok, np.floor(v), 0).astype(np.int64)
            d = depth[fr][py, px]
            ok &= np.isfinite(d) & (d > 0)
            sdf = d - z
            ok &= ~(sdf < -tr)
            fv = np.minimum(f32(1), sdf / tr)
            W1 = W + f32(1)
            s[...] = np.where(ok, (s * W + fv) / W1, s)
            if col is not None:
                pix = image[fr][py, px].astype(f32)
                for c in range(3):
                    col[:, c] = np.where(ok, (col[:, c] * W + pix[:, c]) / W1, col[:, c])
            W[...] = np.where(ok, W1, W)
    return tsdf, weight, color


def marching_cubes(tsdf, weight, color, origin, voxel_size):
    """demon_marching_cubes_f32: vertices [3T,3] float32, colors [3T,3] uint8 (None without color), faces [T,3] int32."""
    nz, ny, nx = tsdf.shape
    k, j, i = (g.reshape(-1) for g in np.meshgrid(np.arange(nz - 1), np.arange(ny - 1), np.arange(nx - 1), indexing="ij"))
    vals, valid = [], np.ones(k.shape, dtype=bool)
    for q in range(8):
        dx, dy, dz = CORNERS[q]
        valid &= weight[k + dz, j + dy, i + dx] > 0
        vals.append(tsdf[k + dz, j + dy, i + dx])
    case = np.zeros(k.shape, dtype=np.int64)
    for q in range(8):
        case |= (vals[q] < 0).astype(np.int64) << q
    table = np.full((256, 15), -1, dtype=np.int64)
    for c, row in enumerate(TRIANGLES):
        table[c, :len(row)] = row
    count = np.where(valid, (table[case] >= 0).sum(axis=1) // 3, 0)
    cube = np.repeat(np.arange(k.size), count)
    m = np.arange(cube.size) - np.repeat(np.cumsum(count) - count, count)   # triangle number within its cube
    o, vs = np.asarray(origin, dtype=f32), f32(voxel_size)
    g = np.stack([i[cube], j[cube], k[cube]], axis=1)
    verts, cols = [], []
    for e3 in range(3):
        edge = table[case[cube], 3 * m + e3]
        ga, gb = g + CORNERS[EDGES[edge, 0]], g + CORNERS[EDGES[edge, 1]]
        pa, pb = o + vs * ga.astype(f32), o + vs * gb.astype(f32)
        fa, fb = tsdf[ga[:, 2], ga[:, 1], ga[:, 0]], tsdf[gb[:, 2], gb[:, 1], gb[:, 0]]
        mu = (fa / (fa - fb))[:, None]
        verts.append(pa + mu * (pb - pa))
        if color is not None:
            ca, cb = color[ga[:, 2], ga[:, 1], ga[:, 0]], color[gb[:, 2], gb[:, 1], gb[:, 0]]
            cols.append(np.clip(np.rint(ca + mu * (cb - ca)), 0, 255).astype(np.uint8))
    vertices = np.stack(verts, axis=1).reshape(-1, 3).astype(f32)
    colors = None if color is None else np.stack(cols, axis=1).reshape(-1, 3)
    faces = np.arange(vertices.shape[0], dtype=np.int32).reshape(-1, 3)
    return vertices, colors, faces


def welded_edges(vertices, faces):
    """Counts of every undirected edge after welding vertices with equal coordinates: a closed mesh has every count 2."""
    _, idx = np.unique(np.asarray(vertices).reshape(-1, 3), axis=0, return_inverse=True)
    fw = idx.reshape(-1)[np.asarray(faces)]
    e = np.concatenate([fw[:, [0, 1]], fw[:, [1, 2]], fw[:, [2, 0]]])
    e = np.sort(e, axis=1)
    _, counts = np.unique(e, axis=0, return_counts=True)
    return counts


# ---- synthetic scenes with analytic depth -----------------------------------------------------------------------------
def render_depth(R, t, K, h, w, sphere=None, box=None):
    """float64 camera z [h,w] of pixel centres (x+0.5, y+0.5) for a world-to-camera (R, t): the nearest hit of the sphere
    (centre, radius) and of the inside of the axis-aligned box ((lo), (hi)); inf where the ray hits nothing."""
    R, t, K = (np.asarray(a, dtype=np.float64) for a in (R, t, K))
    x, y = np.meshgrid(np.arange(w) + 0.5, np.arange(h) + 0.5)
    dc = np.stack([(x - K[0, 2]) / K[0, 0], (y - K[1, 2]) / K[1, 1], np.ones_like(x)], axis=-1)   # camera z = 1
    d = dc.dot(R)                     # world directions R^T dc
    o = -R.T.dot(t)                   # camera centre
    lam = np.full((h, w), np.inf)
    if sphere is not None:
        c, r = np.asarray(sphere[0], dtype=np.float64), float(sphere[1])
        oc = o - c
        a, b, cc = (d * d).sum(-1), 2 * d.dot(oc), oc.dot(oc) - r * r
        disc = b * b - 4 * a * cc
        with np.errstate(invalid="ignore"):
            hit = (-b - np.sqrt(disc)) / (2 * a)
        lam = np.where((disc >= 0) & (hit > 0), np.minimum(lam, hit), lam)
    if box is not None:
        for axis in range(3):
            for bound in box:
                with np.errstate(divide="ignore", invalid="ignore"):
                    hit = (bound[axis] - o[axis]) / d[..., axis]
                lam = np.where(hit > 0, np.minimum(lam, hit), lam)
    return lam


def rot_z(phi):
    c, s = np.cos(phi), np.sin(phi)
    return np.array([[c, -s, 0], [s, c, 0], [0, 0, 1.0]])


def look_at(centre, target, up=(0, 0, 1)):
    """world-to-camera (R, t) of a camera at `centre` looking at `target` (camera z forward, y down)."""
    centre, target, up = (np.asarray(a, dtype=np.float64) for a in (centre, target, up))
    z = target - centre
    z /= np.linalg.norm(z)
    if abs(z.dot(up)) > 0.99:
        up = np.array([0.0, 1.0, 0.0])
    x = np.cross(z, up)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    R = np.stack([x, y, z])
    return R, -R.dot(centre)


def orbit_pairs(frames=6, seed=0, h=192, w=256, intrinsics=NETWORK_INTRINSICS):
    """A camera orbiting a circle inside a box with a sphere in it, looking at the box's back wall and rolling about its
    axis, with random steps.  Returns the pairs as a DeMoN pipeline would give them, each normalised to |t| = 1 with its
    depth scaled to match: inverse_depth float32 [P,1,h,w], rotation / translation float32 [P,3]; and the truth: scales
    s_k = L_{k+1} / L_k of the baselines L_k, the true camera z [T,h,w], and the world-to-camera poses of frames 0..P (frame 0 the world) in pair 0's
    units.  The back wall is fronto-parallel in every frame and covers most of each image, so most depth ratios are exact."""
    rng = np.random.RandomState(seed)
    K = K_pixels(intrinsics, w, h)
    theta = np.cumsum(rng.uniform(0.15, 0.6, frames))
    centres = np.stack([0.4 * np.cos(theta), 0.4 * np.sin(theta), rng.uniform(-0.2, 0.2, frames)], axis=1)
    phi = np.cumsum(rng.uniform(-0.08, 0.08, frames))
    Rw = [rot_z(p) for p in phi]
    tw = [-R.dot(c) for R, c in zip(Rw, centres)]
    scene = dict(sphere=((0.3, -0.2, 3.5), 0.8), box=((-6, -6, -2), (6, 6, 6)))
    depth = [render_depth(R, t, K, h, w, **scene) for R, t in zip(Rw, tw)]
    R0, t0 = Rw[0], tw[0]
    Rr = [R.dot(R0.T) for R in Rw]
    tr = [t - R.dot(t0) for R, t in zip(Rr, tw)]
    inv, rot, trans, L = [], [], [], []
    for k in range(frames - 1):
        Rrel = Rw[k + 1].dot(Rw[k].T)
        trel = tw[k + 1] - Rrel.dot(tw[k])
        L.append(np.linalg.norm(trel))
        rot.append([0.0, 0.0, phi[k + 1] - phi[k]])   # the roll about the common z axis
        trans.append(trel / L[-1])
        inv.append(L[-1] / depth[k])
    L = np.array(L)
    return {"inverse_depth": np.array(inv, dtype=f32)[:, None], "rotation": np.array(rot, dtype=f32),
            "translation": np.array(trans, dtype=f32), "baselines": L, "scales": L[1:] / L[:-1], "R": np.array(Rr), "t": np.array(tr) / L[0],
            "depth": np.array(depth), "K": K}


def sphere_views(n=24, h=48, w=64, radius=0.6, distance=3.0, seed=1):
    """Depth maps float32 [n,h,w] of a sphere of `radius` at the origin seen from n cameras spread over a sphere of
    `distance` (a Fibonacci lattice), each looking at the centre: (depth, K [n,3,3], R [n,3,3], t [n,3]) float32, and
    images uint8 [n,h,w,3] of random colours."""
    K = np.array([[60.0, 0, w / 2], [0, 60.0, h / 2], [0, 0, 1]])
    i = np.arange(n) + 0.5
    zc = 1 - 2 * i / n
    ang = np.pi * (1 + 5 ** 0.5) * i
    dirs = np.stack([np.sqrt(1 - zc * zc) * np.cos(ang), np.sqrt(1 - zc * zc) * np.sin(ang), zc], axis=1)
    Rs, ts, ds = [], [], []
    for d in dirs:
        R, t = look_at(distance * d, np.zeros(3))
        Rs.append(R)
        ts.append(t)
        ds.append(render_depth(R, t, K, h, w, sphere=((0, 0, 0), radius)))
    img = np.random.RandomState(seed).randint(0, 256, (n, h, w, 3)).astype(np.uint8)
    return (np.array(ds, dtype=f32), np.broadcast_to(K.astype(f32), (n, 3, 3)).copy(), np.array(Rs, dtype=f32),
            np.array(ts, dtype=f32), img)
