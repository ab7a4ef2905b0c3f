// Importance-sampling tables of tpt_set_environment's lat-long map ("environment_sampling") and of
// tpt_set_emission_textures' layers ("emission_texture_sampling", at the end). Host-only, plain C++: the library builds
// them in those calls, and tests/host_sim/env_tables_check.cpp and emit_tables_check.cpp run the same code under g++.
//
// Weight of cell (i, j), the texel footprint [i, i+1) x [j, j+1) in the (u, v) of include/tpt_b200.h's mapping:
//   w(i, j) = sin(theta_j) * max over di, dj in {-1, 0, 1} of (R + G + B) / 3 at texel (i + di wrapped, j + dj clamped),
//   theta_j = (j + 1/2) * pi / H (the row centre).
// The 3 x 3 maximum covers every texel the bilinear filter blends into the cell, so the sampling density is non-zero
// wherever the filtered map is. Weights, marginals and alias tables are built in double and stored as float.
//
// Sampler (fast module, sample_env): six draws of the path's stream, in this order:
//   k1 = XorShift32 & 0xFFFFFF   row     j = (k1 * H) >> 24
//   u2 = RandomFloat01           row alias test: keep j when u2 < rows[j].prob, else j = rows[j].alias
//   k3 = XorShift32 & 0xFFFFFF   column  i = (k3 * W) >> 24
//   u4 = RandomFloat01           column alias test in row j's table: keep i when u4 < cols[j * W + i].prob, else its alias
//   u5, u6 = RandomFloat01       in-cell offsets: u = i + u5, v = j + u6
// and the direction is the inverse of the lookup's mapping at (u, v): phi = 2 pi u / W - pi, theta = pi v / H,
// d = (sin theta sin phi, cos theta, -sin theta cos phi). Its solid-angle density is
//   pdf_e = P(i, j) * W * H / (2 pi^2 sin theta),
// where P(i, j) is the probability the sampler realises for the cell: env_realised() counts, on the 2^-24 grid of the
// draws, exactly which draws select each entry with the stored float thresholds.
//
// Slot layout (one device allocation per environment slot, env_slot_bytes):
//   [W * H float4 texels: R, G, B, P(i, j)] [H EnvAlias: rows] [W * H EnvAlias: each row's columns, row-major]
// i.e. 24 W H + 8 H bytes, of which the tables are 8 W H + 8 H (and the texels' alpha channel).
#pragma once
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <vector>

struct EnvAlias
{
    float prob;       // keep the drawn entry when RandomFloat01 < prob
    int32_t alias;    // the entry taken otherwise
};

inline size_t env_slot_bytes(int W, int H) { return (size_t)W * H * 16 + (size_t)H * 8 + (size_t)W * H * 8; }

// Walker's alias table (Vose's construction) for n weights w (>= 0, sum > 0). A zero weight gets prob 0 and is never
// an alias: it can never be drawn.
inline void env_alias_build(const double* w, int n, EnvAlias* t)
{
    double sum = 0.0;
    for (int i = 0; i < n; ++i) sum += w[i];
    std::vector<double> q(n);
    std::vector<int> small, large;
    int anyPositive = 0;
    for (int i = 0; i < n; ++i)
    {
        q[i] = w[i] * n / sum;
        if (w[i] > 0.0) anyPositive = i;
        (q[i] < 1.0 ? small : large).push_back(i);
    }
    while (!small.empty() && !large.empty())
    {
        const int s = small.back(); small.pop_back();
        const int l = large.back(); large.pop_back();
        t[s].prob = (float)q[s];
        t[s].alias = l;
        q[l] = (q[l] + q[s]) - 1.0;
        (q[l] < 1.0 ? small : large).push_back(l);
    }
    // what rounding leaves over: full entries, except that a zero weight still never selects itself
    for (int i : large) { t[i].prob = 1.0f; t[i].alias = i; }
    for (int i : small)
    {
        t[i].prob = w[i] > 0.0 ? 1.0f : 0.0f;
        t[i].alias = w[i] > 0.0 ? i : anyPositive;
    }
}

// The probability with which the sampler draws each entry of table t: index k * n >> 24 over the 2^24 values of k,
// kept when the 24-bit test draw lies below prob, else replaced by its alias. Exact (every term is an integer over 2^48).
inline void env_realised(const EnvAlias* t, int n, double* p)
{
    const uint64_t one = 1ull << 24;
    for (int i = 0; i < n; ++i) p[i] = 0.0;
    for (int i = 0; i < n; ++i)
    {
        // the k in [0, 2^24) with (k * n) >> 24 == i: k in [ceil(i 2^24 / n), ceil((i + 1) 2^24 / n))
        const uint64_t lo = ((uint64_t)i * one + n - 1) / n, hi = ((uint64_t)(i + 1) * one + n - 1) / n;
        const double cnt = (double)(hi - lo);
        // the test draws u = m / 2^24 with u < prob: m < prob * 2^24
        double keep = std::ceil((double)t[i].prob * (double)one);
        keep = keep < 0.0 ? 0.0 : (keep > (double)one ? (double)one : keep);
        p[i] += cnt * keep;
        p[t[i].alias] += cnt * ((double)one - keep);
    }
    for (int i = 0; i < n; ++i) p[i] *= 1.0 / ((double)one * (double)one);
}

// The pinned weights, w[j * W + i], from texels at rgb + 4 * (j * W + i) (R, G, B of a float4 texel).
inline void env_weights(const float* rgb, int W, int H, std::vector<double>& w)
{
    const double kPi = 3.14159265358979323846;
    std::vector<double> mean((size_t)W * H), rowMax((size_t)W * H);
    for (size_t k = 0; k < (size_t)W * H; ++k)
        mean[k] = ((double)rgb[4 * k] + (double)rgb[4 * k + 1] + (double)rgb[4 * k + 2]) / 3.0;
    for (int j = 0; j < H; ++j)
        for (int i = 0; i < W; ++i)
        {
            const double* r = &mean[(size_t)j * W];
            const double a = r[i == 0 ? W - 1 : i - 1], b = r[i], c = r[i + 1 == W ? 0 : i + 1];
            rowMax[(size_t)j * W + i] = std::fmax(a, std::fmax(b, c));
        }
    w.resize((size_t)W * H);
    for (int j = 0; j < H; ++j)
    {
        const double s = std::sin((j + 0.5) * kPi / H);
        const double* up = &rowMax[(size_t)(j > 0 ? j - 1 : 0) * W];
        const double* mid = &rowMax[(size_t)j * W];
        const double* dn = &rowMax[(size_t)(j + 1 < H ? j + 1 : H - 1) * W];
        for (int i = 0; i < W; ++i) w[(size_t)j * W + i] = s * std::fmax(up[i], std::fmax(mid[i], dn[i]));
    }
}

// All tables of a W x H map: rows (H), cols (W * H), and each cell's realised probability into the texels' alpha
// (texels: W * H float4, R, G, B read, alpha written). Returns false, leaving the tables unwritten, when every weight
// is zero: such a map is not sampled.
inline bool env_build_tables(float* texels, int W, int H, EnvAlias* rows, EnvAlias* cols)
{
    std::vector<double> w;
    env_weights(texels, W, H, w);
    std::vector<double> rowW(H, 0.0);
    double total = 0.0;
    for (int j = 0; j < H; ++j)
    {
        for (int i = 0; i < W; ++i) rowW[j] += w[(size_t)j * W + i];
        total += rowW[j];
    }
    if (!(total > 0.0)) return false;
    env_alias_build(rowW.data(), H, rows);
    std::vector<double> pRow(H), pCol(W);
    env_realised(rows, H, pRow.data());
    for (int j = 0; j < H; ++j)
    {
        EnvAlias* c = cols + (size_t)j * W;
        if (rowW[j] > 0.0) env_alias_build(&w[(size_t)j * W], W, c);
        else for (int i = 0; i < W; ++i) { c[i].prob = 1.0f; c[i].alias = i; }      // never drawn: the row has P = 0
        env_realised(c, W, pCol.data());
        for (int i = 0; i < W; ++i) texels[4 * ((size_t)j * W + i) + 3] = (float)(pRow[j] * pCol[i]);
    }
    return true;
}

// ---- emission layers ("emission_texture_sampling") -----------------------------------------------------------------
// tpt_set_emission_textures builds the same tables for each of its L layers of W x H texels, each layer alone, with
// env_build_tables: the layers use the map's lat-long mapping, so a layer's sampler is sample_env's with the sphere's
// normal for the direction. Slot layout (one device allocation per emission-texture slot, emit_slot_bytes):
//   [L * W * H float4 texels: R, G, B, P] [S int32 sphere layers] [4 bytes of padding when S is odd]
//   [L blocks of (H + W * H) EnvAlias: layer k's rows, then its columns, row-major]
// i.e. 16 W H L + 4 S (+ 4) + 8 H L + 8 W H L bytes. The tables start emit_table_words(S) int32 words behind the sphere
// table (S rounded up to even, keeping them 8-byte aligned); TexSet::tabWords carries that count to the kernels.
// A layer whose weights are all zero has no tables: every entry of its block is the sentinel {prob 0, alias -1} (the
// kernels test rows[0].alias < 0) and its texels' alpha is 0. Albedo textures (tpt_set_textures) build no tables and
// keep their 16 W H L + 4 S byte slots.
constexpr int32_t kEmitNoTables = -1;

inline size_t emit_table_words(int S) { return ((size_t)S + 1) & ~(size_t)1; }
inline size_t emit_table_offset(int W, int H, int L, int S) { return (size_t)W * H * L * 16 + emit_table_words(S) * 4; }
inline size_t emit_slot_bytes(int W, int H, int L, int S)
{
    return emit_table_offset(W, H, L, S) + (size_t)L * ((size_t)H + (size_t)W * H) * 8;
}

// Tables of every layer into `tables` (L blocks of H + W * H entries) and the alpha of `texels` (L * W * H float4, R, G
// and B read). Returns true when some layer has a non-zero weight.
inline bool emit_build_tables(float* texels, int W, int H, int L, EnvAlias* tables)
{
    bool any = false;
    const size_t plane = (size_t)W * H, block = (size_t)H + plane;
    for (int k = 0; k < L; ++k)
    {
        float* t = texels + 4 * plane * k;
        EnvAlias* rows = tables + block * k;
        if (env_build_tables(t, W, H, rows, rows + H)) { any = true; continue; }
        for (size_t e = 0; e < block; ++e) { rows[e].prob = 0.0f; rows[e].alias = kEmitNoTables; }
        for (size_t i = 0; i < plane; ++i) t[4 * i + 3] = 0.0f;
    }
    return any;
}
