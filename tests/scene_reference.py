"""Drives the UNMODIFIED reference viewer (fast3r/viz/viser_visualizer.py) without a browser, for the scene goldens
(tools/make_golden_scene.py) and the CPU tests.

``import_reference_viewer()`` loads the module with stand-ins for its display-only imports (viser, viser.transforms,
imageio.v3, matplotlib.cm) and for the Lightning module it only takes ``estimate_camera_poses`` from (the poses feed
the camera frustums, which are not part of the scene).  Its playback thread never starts: ``threading`` in the module
is replaced by a stand-in whose threads do not run.  ``run_viewer(output, actions)`` calls ``start_visualization`` with
a fake server, records the frame data and the launch state, then replays each action's slider / checkbox callbacks
followed by the "Download PLY" callback, and returns what the viewer sent."""
import os
import sys
import types

import numpy as np

from tests.conftest import ROOT

VIEWER = os.path.join("fast3r", "viz", "viser_visualizer.py")


def reference_viewer_path():
    sys.path.insert(0, ROOT)
    from oracle import ref_harness as RH
    return os.path.join(RH.REFERENCE_ROOT, VIEWER)


class _Widget:
    def __init__(self, value=None):
        self.value, self.disabled, self.callbacks = value, False, []

    def on_update(self, fn):
        self.callbacks.append(fn)
        return fn

    on_click = on_update

    def fire(self, value=None, event=None):
        if value is not None:
            self.value = value
        for cb in list(self.callbacks):
            cb(event)


class _Node:
    def __init__(self, **kw):
        self.__dict__.update(kw)


class _Ctx:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


class _Gui:
    def __init__(self):
        self.widgets = {}

    def _add(self, label, value=None):
        w = self.widgets[label] = _Widget(value)
        return w

    def set_panel_label(self, *a, **k):
        pass

    def configure_theme(self, *a, **k):
        pass

    def add_folder(self, *a, **k):
        return _Ctx()

    def add_slider(self, label, min, max, step, initial_value):
        return self._add(label, initial_value)

    def add_checkbox(self, label, initial_value):
        return self._add(label, initial_value)

    def add_button(self, label):
        return self._add(label)

    def add_button_group(self, label, options):
        return self._add(label, options[0])


class _Scene:
    def __init__(self):
        self.world_axes = _Node(visible=True)
        self.nodes = {}

    def set_up_direction(self, *a):
        pass

    def add_frame(self, name, **kw):
        self.nodes[name] = _Node(name=name, visible=True, **kw)
        return self.nodes[name]

    def add_point_cloud(self, name, **kw):
        self.nodes[name] = _Node(name=name, initial=dict(kw), **kw)
        return self.nodes[name]

    def add_camera_frustum(self, name, **kw):
        self.nodes[name] = _Node(name=name, initial=dict(kw), **kw)
        return self.nodes[name]


class FakeServer:
    def __init__(self, *a, **k):
        self.gui, self.scene, self.downloads = _Gui(), _Scene(), []
        self.client = _Node(send_file_download=lambda name, data: self.downloads.append(bytes(data)))

    def on_client_connect(self, fn):
        return fn

    def atomic(self):
        return _Ctx()

    def flush(self):
        pass

    def request_share_url(self):
        return None


def import_reference_viewer():
    """The reference viewer module's namespace (a dict), loaded from its unmodified source."""
    path = reference_viewer_path()
    if not os.path.exists(path):
        raise FileNotFoundError(path)
    names = ("viser", "viser.transforms", "imageio", "imageio.v3", "matplotlib", "matplotlib.cm",
             "fast3r.models.multiview_dust3r_module")
    saved = {k: sys.modules.get(k) for k in names}
    viser = types.ModuleType("viser")
    viser.transforms = types.ModuleType("viser.transforms")
    viser.transforms.SO3 = types.SimpleNamespace(from_matrix=lambda m: _Node(wxyz=np.array([1.0, 0.0, 0.0, 0.0])))
    viser.ViserServer, viser.ClientHandle, viser.GuiEvent = FakeServer, object, object
    imageio = types.ModuleType("imageio")
    imageio.v3 = types.ModuleType("imageio.v3")
    mpl = types.ModuleType("matplotlib")
    mpl.cm = types.ModuleType("matplotlib.cm")
    mpl.cm.turbo = lambda x: np.zeros((len(x), 4))  # the confidence colours are not part of the scene
    mdm = types.ModuleType("fast3r.models.multiview_dust3r_module")

    class Lit:
        @staticmethod
        def estimate_camera_poses(preds, **kw):  # feeds the frustums only
            return [np.stack([np.eye(4, dtype=np.float32)] * len(preds))], [[500.0] * len(preds)]

    mdm.MultiViewDUSt3RLitModule = Lit
    sys.modules.update({"viser": viser, "viser.transforms": viser.transforms, "imageio": imageio,
                        "imageio.v3": imageio.v3, "matplotlib": mpl, "matplotlib.cm": mpl.cm,
                        "fast3r.models.multiview_dust3r_module": mdm})
    from oracle import ref_harness as RH
    if RH.REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, RH.REFERENCE_ROOT)
    try:
        ns = {"__name__": "reference_viser_visualizer", "__file__": path}
        with open(path) as f:
            exec(compile(f.read(), path, "exec"), ns)
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
    # the playback loop never ends: its thread must not run
    ns["threading"] = types.SimpleNamespace(Thread=lambda target=None, **k: _Node(start=lambda: None))
    return ns


# Replayed actions: (what, widget label, value).  The expected visible_points arguments after each action are
# maintained by tests/test_scene_cpu.py / test_scene_gpu.py from the same list.
ACTIONS = [
    ("p", "Per-View Conf Percentile", 10), ("p", "Per-View Conf Percentile", 65),
    ("p", "Per-View Conf Percentile", 99.99), ("p", "Per-View Conf Percentile", 100),
    ("p", "Per-View Conf Percentile", 0), ("sky", "Mask Sky", "toggle"),
    ("global", "Global", True), ("timestep", "Timestep", "middle"), ("timestep", "Timestep", 0),
    ("timestep", "Timestep", "last"), ("color", "Color by View", True), ("sky", "Mask Sky", "toggle"),
    ("local", "Local", False), ("local", "Local", True), ("drop_low", "Show High-Conf Views", True),
    ("p", "Per-View Conf Percentile", 10),
]


def states(n, is_outdoor):
    """visible_points keyword arguments of the launch state and after each action of ACTIONS."""
    st = dict(timestep=None, min_conf_thr_percentile=None, mask_sky=None, show_global=False, show_local=True,
              drop_low_conf_views=False, color="rgb")
    out = [dict(st)]
    sky = is_outdoor
    for what, _, value in ACTIONS:
        if what == "p":
            st["min_conf_thr_percentile"] = value
        elif what == "sky":
            sky = not sky
            st["mask_sky"] = sky
        elif what == "global":
            st["show_global"] = value
        elif what == "local":
            st["show_local"] = value
        elif what == "timestep":
            st["timestep"] = {"middle": n // 2, "last": n - 1}.get(value, value)
        elif what == "color":
            st["color"] = "view"
        elif what == "drop_low":
            st["drop_low_conf_views"] = True
        out.append(dict(st))
    return out


def run_viewer(ns, output):
    """Runs start_visualization on `output` and replays ACTIONS.  Returns (frames, is_outdoor, max_extent, PLY bytes
    (None where the viewer found no points) of the launch state and after each action).  Each frame is the data the
    viewer built: its sorted points and float colours of both heads, is_high_confidence (the local node's visibility
    at creation) and its rainbow colour (the frustum's)."""
    server = ns["start_visualization"](output)
    w = server.gui.widgets
    n = len(output["preds"])
    frames = []
    for i in range(n):
        gl = server.scene.nodes[f"/pts3d_global/t{i}"].initial
        lo = server.scene.nodes[f"/pts3d_local/t{i}"].initial
        fr = server.scene.nodes[f"/cams/t{i}/frustum"].initial
        frames.append(dict(pts_global=gl["points"], colors_global=gl["colors"], pts_local=lo["points"],
                           colors_local=lo["colors"], is_high_confidence=bool(lo["visible"]),
                           rainbow=np.asarray(fr["color"], np.float64)))
    is_outdoor = bool(w["Mask Sky"].value)
    w["Camera Size (%)"].fire(100.0)  # frustum scale = max_extent * (100 / 100): the extent itself
    max_extent = server.scene.nodes["/cams/t0/frustum"].scale
    event = _Node(client=server.client)

    def download():
        before = len(server.downloads)
        w["Download PLY"].fire(event=event)
        return server.downloads[-1] if len(server.downloads) > before else None

    plys = [download()]
    for what, label, value in ACTIONS:
        if value == "toggle":
            value = not w[label].value
        elif value == "middle":
            value = n // 2
        elif value == "last":
            value = n - 1
        w[label].fire(value)
        plys.append(download())
    return frames, is_outdoor, max_extent, plys
