"""The PolygonBox methods (surya/common/polygon.py) that the layout slice join and the table geometry use, over a `polygon`
attribute of four [x, y] corners.  One implementation for layout_pages.LayoutBox and the table_rec result types."""
from __future__ import annotations

from typing import List


class PolygonMethods:
    polygon: List[List[float]]

    @property
    def bbox(self) -> List[float]:
        xs = [p[0] for p in self.polygon]
        ys = [p[1] for p in self.polygon]
        return [min(xs), min(ys), max(xs), max(ys)]

    @property
    def width(self):
        b = self.bbox
        return b[2] - b[0]

    @property
    def height(self):
        b = self.bbox
        return b[3] - b[1]

    @property
    def area(self):
        return self.width * self.height

    def shift(self, x_shift=None, y_shift=None):
        if x_shift is not None:
            for p in self.polygon:
                p[0] += x_shift
        if y_shift is not None:
            for p in self.polygon:
                p[1] += y_shift

    def merge(self, other: "PolygonMethods"):
        a, b = self.bbox, other.bbox
        x1, y1, x2, y2 = min(a[0], b[0]), min(a[1], b[1]), max(a[2], b[2]), max(a[3], b[3])
        self.polygon = [[x1, y1], [x2, y1], [x2, y2], [x1, y2]]

    def x_overlap(self, other: "PolygonMethods", x_margin=0):
        a, b = self.bbox, other.bbox
        return max(0, min(a[2] + x_margin, b[2] + x_margin) - max(a[0] - x_margin, b[0] - x_margin))

    def y_overlap(self, other: "PolygonMethods", y_margin=0):
        a, b = self.bbox, other.bbox
        return max(0, min(a[3] + y_margin, b[3] + y_margin) - max(a[1] - y_margin, b[1] - y_margin))

    def intersection_pct(self, other: "PolygonMethods", x_margin=0, y_margin=0):
        if self.area == 0:
            return 0
        if x_margin:
            x_margin = int(min(self.width, other.width) * x_margin)
        if y_margin:
            y_margin = int(min(self.height, other.height) * y_margin)
        return self.x_overlap(other, x_margin) * self.y_overlap(other, y_margin) / self.area

    def intersection_polygon(self, other: "PolygonMethods") -> List[List[float]]:
        """Corner by corner: the inner edges of two axis-ordered quadrilaterals (corners top-left, top-right, bottom-right,
        bottom-left)."""
        a, b = self.polygon, other.polygon
        return [[max(a[0][0], b[0][0]), max(a[0][1], b[0][1])], [min(a[1][0], b[1][0]), max(a[1][1], b[1][1])],
                [min(a[2][0], b[2][0]), min(a[2][1], b[2][1])], [max(a[3][0], b[3][0]), min(a[3][1], b[3][1])]]
