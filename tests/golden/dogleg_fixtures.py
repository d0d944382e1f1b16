"""The fixtures of Ceres' internal/ceres/dogleg_strategy_test.cc:45-127, as data.

ELLIPSE: J = sqrt(diag(DDIAG)) BASIS, so J'J = BASIS' diag(DDIAG) BASIS; r = -J ELLIPSE_MINIMUM.
VALLEY:  J = diag(DDIAG), r = -J VALLEY_MINIMUM; the gradient at the origin points at the minimum.
Both set min_lm_diagonal = max_lm_diagonal = 1.  The expected values are those of the six tests (:131-272)."""

# dogleg_strategy_test.cc:64-71, a random orthonormal basis of R^6 (rows as written there)
BASIS = [
    [-0.1046920933796121, -0.7449367449921986, -0.4190744502875876, -0.4480450716142566, 0.2375351607929440, -0.0363053418882862],
    [0.4064975684355914, 0.2681113508511354, -0.7463625494601520, -0.0803264850508117, -0.4463149623021321, 0.0130224954867195],
    [-0.5514387729089798, 0.1026621026168657, -0.5008316122125011, 0.5738122212666414, 0.2974664724007106, 0.1296020877535158],
    [0.5037835370947156, 0.2668479925183712, -0.1051754618492798, -0.0272739396578799, 0.7947481647088278, -0.1776623363955670],
    [-0.4005458426625444, 0.2939330589634109, -0.0682629380550051, -0.2895448882503687, -0.0457239396341685, -0.8139899477847840],
    [-0.3247764582762654, 0.4528151365941945, -0.0276683863102816, -0.6155994592510784, 0.1489240599972848, 0.5362574892189350],
]
DDIAG = [1.0, 2.0, 4.0, 8.0, 16.0, 32.0]
ELLIPSE_MINIMUM = [1.0, 1.0, 1.0, 1.0, 1.0, 1.0]
VALLEY_MINIMUM = [0.0, 0.0, 1.0, 0.0, 0.0, 0.0]
MIN_LM_DIAGONAL = MAX_LM_DIAGONAL = 1.0

K_TOLERANCE = 1e-14        # :125
K_TOLERANCE_LOOSE = 1e-5   # :126

# (test, fixture, dogleg type, radius, expected): the radius bound is |x| <= radius (1 + 4 eps); the steps are expected
# to within K_TOLERANCE_LOOSE per entry
CASES = [
    ("TrustRegionObeyedTraditional", "ellipse", "traditional", 2.0, "obeyed"),
    ("TrustRegionObeyedSubspace", "ellipse", "subspace", 2.0, "obeyed"),
    ("CorrectGaussNewtonStep", "ellipse", "subspace", 10.0, [1.0, 1.0, 1.0, 1.0, 1.0, 1.0]),
    ("ValidSubspaceBasis", "ellipse", "subspace", 2.0, "basis"),
    ("CorrectStepLocalOptimumAlongGradient", "valley", "subspace", 0.25, [0.0, 0.0, 0.25, 0.0, 0.0, 0.0]),
    ("CorrectStepGlobalOptimumAlongGradient", "valley", "subspace", 2.0, [0.0, 0.0, 1.0, 0.0, 0.0, 0.0]),
]
