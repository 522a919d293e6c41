from .geom2d import ray_angles, dist_to_coord, polygons_to_label, polygons_to_label_coord, star_dist, relabel_image_stardist
from .geom3d import polyhedron_to_label, dist_to_coord3D, star_dist3D, relabel_image_stardist3D
from .distances import star_dist_device, star_dist3D_device
