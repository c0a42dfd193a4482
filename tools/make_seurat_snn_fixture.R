#!/usr/bin/env Rscript
## make_seurat_snn_fixture.R - run Seurat 5 the way .leiden_seurat_preprocess_routine does
## (R/inferCNV_tumor_subclusters.R:699-723) on a planted-clone matrix this script draws itself, and write what K18
## (icnv_snn.cu) is pinned against: the variable features and the SNN graph of FindNeighbors(nn.method = "rann"), whose
## kNN is exact as the device's is.  It also records how many uniform draws RunPCA(seed.use = 42) leaves behind on R's
## RNG, by finding n with set.seed(42); runif(n) reproducing .Random.seed after RunPCA.
##
##   Rscript tools/make_seurat_snn_fixture.R fixture_dir           # on a box with R, Seurat >= 5 and RANN
##   ICNV_SEURAT_FIXTURE_DIR=fixture_dir python -m pytest tests/test_seurat_snn_r_fixture.py
##
## Writes fixture_dir/x.bin (G x C doubles, column-major, little-endian), meta.txt, features.txt (1-based gene indices in
## VariableFeatures order), snn_i.bin / snn_j.bin (int32, 0-based) / snn_x.bin (double), rng_draws.txt.
## Not executed yet: written against Seurat 5 semantics; the first run should be watched.
suppressPackageStartupMessages({ library(Seurat); library(Matrix) })
args <- commandArgs(trailingOnly = TRUE)
if (length(args) < 1) stop("usage: Rscript make_seurat_snn_fixture.R <fixture dir>")
dir <- args[1]
dir.create(dir, showWarnings = FALSE, recursive = TRUE)

set.seed(1)
G <- 3000L; C <- 2000L; clones <- 4L
base <- rgamma(G, 3) + 0.5
lab <- sample.int(clones, C, replace = TRUE)
cnv <- matrix(1, clones, G)
for (cl in seq_len(clones)) for (s in 1:4) {
    a <- sample.int(G - G %/% 10, 1)
    cnv[cl, a:(a + G %/% 10 - 1)] <- sample(c(0.5, 1.5, 2), 1)
}
x <- base * t(cnv[lab, ]) * exp(matrix(rnorm(G * C, sd = 0.3), G, C))
rownames(x) <- paste0("g", seq_len(G)); colnames(x) <- paste0("c", seq_len(C))

obj <- CreateSeuratObject(x, assay = "infercnv", project = "infercnv", names.field = 1)
obj <- FindVariableFeatures(obj)
obj <- ScaleData(obj, features = rownames(obj), layer = "counts")
obj <- RunPCA(obj, npcs = 10)
after_pca <- .Random.seed
draws <- NA
for (n in 0:100000) {
    set.seed(42)
    if (n > 0) runif(n)
    if (identical(.Random.seed, after_pca)) { draws <- n; break }
}
obj <- FindNeighbors(obj, k.param = 20, nn.method = "rann")
snn <- as(obj@graphs$infercnv_snn, "TsparseMatrix")

writeBin(as.double(x), file.path(dir, "x.bin"), size = 8, endian = "little")
writeLines(c(paste0("G=", G), paste0("C=", C), "k=20"), file.path(dir, "meta.txt"))
writeLines(as.character(match(VariableFeatures(obj), rownames(x))), file.path(dir, "features.txt"))
writeBin(as.integer(snn@i), file.path(dir, "snn_i.bin"), size = 4, endian = "little")
writeBin(as.integer(snn@j), file.path(dir, "snn_j.bin"), size = 4, endian = "little")
writeBin(as.double(snn@x), file.path(dir, "snn_x.bin"), size = 8, endian = "little")
writeLines(as.character(draws), file.path(dir, "rng_draws.txt"))
