"""``matplotlib.colors.ListedColormap`` as a name only (used by ``binary_cmap``, never called here)."""


class ListedColormap(object):
    def __init__(self, colors, name="from_list", N=None):
        self.colors, self.name, self.N = colors, name, N
