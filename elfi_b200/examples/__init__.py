"""Benchmark models of the hot path (MA2, Gaussian noise, univariate and bivariate g-and-k, Ricker,
Lorenz, toad movement, Lotka-Volterra, day care, ARCH(1), M/G/1 queue, alpha-stable stochastic
volatility, scratch assay, birth-death-mutation) on the elfi_b200 node API."""
