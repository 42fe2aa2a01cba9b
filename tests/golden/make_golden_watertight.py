"""Writes tests/golden/wand_mesh.npz (vertices fp32 [V, 3], faces int32 [F, 3]) from the reference's example mesh
examples/wand.obj, read with mesh_to_pc.SimpleMesh.load_obj.  Data only: the watertight tests read the npz.

    python tests/golden/make_golden_watertight.py /path/to/MeshAnything/examples/wand.obj
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from mesh_to_pc import SimpleMesh  # noqa: E402


def main(obj_path):
    m = SimpleMesh.load_obj(obj_path)
    out = os.path.join(HERE, "wand_mesh.npz")
    np.savez_compressed(out, vertices=m.vertices.astype(np.float32), faces=m.faces.astype(np.int32))
    print(out, m.vertices.shape, m.faces.shape)


if __name__ == "__main__":
    main(sys.argv[1])
