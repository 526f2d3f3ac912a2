// TEST INFRASTRUCTURE: a serial CPU restatement of the world generators (include/isdf.h, isdf_world_*): the reference's loops run one
// point at a time with libc's own rand(), std::shuffle and std::sort, no jump-ahead, no segments, no selection. Built by
// tests/world_oracle.py with -ffp-contract=off, so every FP64 operation rounds on its own as in the reference's g++ build (no -march).
// Each generator writes the first cap records (x, y, z, 1.0f) and returns the cloud's size; -1 where the library refuses the arguments
// for tpos out of range.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <numeric>
#include <random>
#include <vector>

namespace {

struct Out {
    float *p; long long cap, n = 0;
    void push(double x, double y, double z) {
        if (n < cap) { p[4 * n] = (float)x; p[4 * n + 1] = (float)y; p[4 * n + 2] = (float)z; p[4 * n + 3] = 1.0f; }
        n++;
    }
};

struct Globalmap {
    Out &o;
    double res, init[3];
    void wall(double ox, double oy, double l, double w, double h) { wall(ox, oy, 0.0, l, w, h); }
    void wall(double ox, double oy, double oz, double l, double w, double h) {
        for (double tz = oz; tz < h + oz; tz += res)
            for (double ty = oy; ty < oy + w; ty += res)
                for (double tx = ox; tx < ox + l; tx += res) {
                    const double x = tx + (rand() % 10) / 250.0;
                    const double y = ty + (rand() % 10) / 250.0;
                    const double z = tz + (rand() % 10) / 800.0;
                    o.push(x, y, z);
                }
    }
    void road(const double sp[3], const double ep[3], double width) {
        double dir[3], ex[3];
        for (int a = 0; a < 3; a++) dir[a] = ep[a] - sp[a];
        const double length = std::sqrt((dir[0] * dir[0] + dir[1] * dir[1]) + dir[2] * dir[2]);
        const double t_step = res / length, k_step = res / width;
        ex[0] = -dir[1]; ex[1] = dir[0]; ex[2] = 0;
        const double en = std::sqrt((ex[0] * ex[0] + ex[1] * ex[1]) + ex[2] * ex[2]);
        for (double &e : ex) { if (en > 0) e /= en; e *= width; }
        for (double t = 0; t <= 1; t += t_step) {
            double pv[3];
            for (int a = 0; a < 3; a++) pv[a] = sp[a] + t * dir[a];
            for (double k = -0.5; k <= 0.5; k += k_step) {
                double h[3];
                for (int a = 0; a < 3; a++) h[a] = pv[a] + k * ex[a];
                const double x = h[0] + (rand() % 10) / 250.0;
                const double y = h[1] + (rand() % 10) / 250.0;
                const double z = h[2] + (rand() % 10) / 800.0;
                o.push(x, y, z);
            }
        }
    }
    void cubes(int num, int lo, unsigned srand_seed) {
        srand(srand_seed);
        for (int i = 0; i < num; i++) {
            const double x = (rand() % 450 + lo) / 10;
            const double y = (rand() % 450 + lo) / 10;
            const double z = (rand() % 250 + 50) / 10;
            wall(x, y, z, 1.5 * res, 1.5 * res, 1.5 * res);
        }
    }
};

}  // namespace

extern "C" {

// glibc rand() after srand(seed), offset draws discarded
int32_t world_serial_rand_at(uint32_t seed, uint64_t offset) {
    srand(seed);
    for (uint64_t i = 0; i < offset; i++) rand();
    return rand();
}

long long world_serial_globalmap(int id, uint32_t rand_seed, uint32_t srand_seed, double res, const double *init, float *out, long long cap) {
    Out o{out, cap};
    Globalmap G{o, res, {init[0], init[1], init[2]}};
    srand(rand_seed);
    G.wall(0, 0, 0.2, 0.2, 3.0);
    switch (id) {
    case 1: G.wall(50, 20, 15.0, 0.2, 0.2, 3.0); G.wall(25.0, 0.0, 2.0, 10.0, 5.0); G.wall(25.0, 0.0, 7.0, 2.0, 10.0, 5.0); break;
    case 2: {
        G.wall(100, 100, 0.2, 0.2, 3.0);
        int trees = 20;
        while (trees--) {
            const double x = (rand() % 3000) / 50.0;
            const double y = (rand() % 3000) / 50.0;
            if (std::sqrt((x - init[0]) * (x - init[0]) + (y - init[1]) * (y - init[1])) < 0.09) { trees++; continue; }
            G.wall(x, y, 5, 5, 20);
        }
        break;
    }
    case 3:
        G.wall(50, 50, 15.0, 0.2, 0.2, 3.0);
        for (double x0 : {10.0, 20.0}) {
            const bool a = x0 == 10.0;
            G.wall(x0, 0.0, 2.0, 2.0, 14.0); G.wall(x0, 10.0, 2.0, 2.0, 14.0); G.wall(x0, 2.0, 2.0, 8.0, a ? 3.0 : 5.0);
            G.wall(x0, 2.0, a ? 12.0 : 14.0, 2.0, 8.0, a ? 2.0 : 0.0); G.wall(x0, 5.0, a ? 3.0 : 5.0, 2.0, 5.0, 5.5);
            G.wall(x0, 10.0, 2.0, 40.0, 15.0);
        }
        G.wall(10.0, 0.0, 13.0, 2.0, 50.0, 5.0); G.wall(20.0, 0.0, 13.0, 2.0, 50.0, 5.0);
        break;
    case 4: G.wall(60, 60, 35.0, 0.2, 0.2, 3.0); G.cubes(250, 50, srand_seed); break;
    case 11: G.wall(60, 60, 35.0, 0.2, 0.2, 3.0); G.cubes(300, 15, srand_seed); break;
    case 5: G.wall(60, 60, 35.0, 0.2, 0.2, 3.0); G.wall(30, 0, 2.0, 50, 15.0); G.wall(30, 0, 18.0, 2.0, 50, 16.0); break;
    case 6: G.wall(60, 60, 35.0, 0.2, 0.2, 3.0); break;
    case 7:
        G.wall(60, 60, 35.0, 0.2, 0.2, 3.0);
        G.wall(30, 0, 1.1, 60.0, 8.0); G.wall(30, 0, 5.0, 1.1, 25.0, 7.0); G.wall(30, 35.0, 5.0, 1.1, 25.0, 7.0);
        G.wall(30, 0.0, 12.0, 1.1, 21.0, 9.0); G.wall(30, 39.0, 12.0, 1.1, 21.0, 9.0);
        G.wall(30, 0.0, 21.0, 1.1, 60.0, 4.0); G.wall(30, 28.0, 14.0, 1.1, 4.0, 2.0);
        break;
    case 8: G.wall(60, 60, 35.0, 0.2, 0.2, 3.0); o.push(30, 30, 2.0); break;
    case 9:
        G.wall(60, 60, 35.0, 0.2, 0.2, 3.0);
        for (double h = -60; h < 30; h += 0.5) {
            if (h > 0.0 && h < 5.5) continue;
            double spt[3] = {0, 20, h};
            if (h < 0) { spt[0] -= h; spt[2] = 0; }
            const double ept[3] = {50, spt[1], spt[2] + 45};
            G.road(spt, ept, 0.5);
        }
        break;
    case 10:
        G.wall(50, 50, 15.0, 0.2, 0.2, 3.0);
        G.wall(10.0, 0.0, 2.0, 50.0, 35.0); G.wall(25.0, 0.0, 2.0, 50.0, 35.0); G.wall(40.0, 0.0, 2.0, 50.0, 35.0);
        G.wall(10.0, 49.0, 30.0, 1.0, 35.0); G.wall(0.0, 0.0, -1.0, 50.0, 50.0, 1.0);
        break;
    default: return -1;
    }
    return o.n;
}

namespace {
double fade(double t) { return t * t * t * (t * (t * 6 - 15) + 10); }
double lerp(double t, double a, double b) { return a + t * (b - a); }
double grad(int hash, double x, double y, double z) {
    const int h = hash & 15;
    const double u = h < 8 ? x : y, v = h < 4 ? y : h == 12 || h == 14 ? x : z;
    return ((h & 1) == 0 ? u : -u) + ((h & 2) == 0 ? v : -v);
}
double noise(const std::vector<int> &p, double x, double y, double z) {
    const int X = (int)std::floor(x) & 255, Y = (int)std::floor(y) & 255, Z = (int)std::floor(z) & 255;
    x -= std::floor(x); y -= std::floor(y); z -= std::floor(z);
    const double u = fade(x), v = fade(y), w = fade(z);
    const int A = p[X] + Y, AA = p[A] + Z, AB = p[A + 1] + Z, B = p[X + 1] + Y, BA = p[B] + Z, BB = p[B + 1] + Z;
    const double r = lerp(w, lerp(v, lerp(u, grad(p[AA], x, y, z), grad(p[BA], x - 1, y, z)),
                                     lerp(u, grad(p[AB], x, y - 1, z), grad(p[BB], x - 1, y - 1, z))),
                             lerp(v, lerp(u, grad(p[AA + 1], x, y, z - 1), grad(p[BA + 1], x - 1, y, z - 1)),
                                     lerp(u, grad(p[AB + 1], x, y - 1, z - 1), grad(p[BB + 1], x - 1, y - 1, z - 1))));
    return (r + 1.0) / 2.0;
}
}  // namespace

long long world_serial_perlin(uint32_t seed, int X, int Y, int Z, double scale, double complexity, double fill, double attenuation,
                              int fractal, float *out, long long cap) {
    std::vector<int> p(256);
    std::iota(p.begin(), p.end(), 0);
    std::default_random_engine engine(seed);
    std::shuffle(p.begin(), p.end(), engine);
    p.insert(p.end(), p.begin(), p.end());
    const long long n = (long long)X * Y * Z;
    std::vector<double> v;
    v.reserve(n);
    auto tn = [&](int i, int j, int k) {
        double t = 0;
        for (int it = 1; it <= fractal; ++it) {
            const int dfv = (int)std::pow(2, it);
            const double ta = attenuation / it;
            t += ta * noise(p, dfv * i * complexity, dfv * j * complexity, dfv * k * complexity);
        }
        return t;
    };
    for (int i = 0; i < X; ++i) for (int j = 0; j < Y; ++j) for (int k = 0; k < Z; ++k) v.push_back(tn(i, j, k));
    std::sort(v.begin(), v.end());
    const int tpos = (uint32_t)n * (1 - fill);
    if (tpos < 0 || tpos >= n) return -1;
    const double thr = v[tpos];
    Out o{out, cap};
    for (int i = 0; i < X; ++i) for (int j = 0; j < Y; ++j) for (int k = 0; k < Z; ++k)
        if (tn(i, j, k) > thr) o.push(i / scale - X / (2 * scale), j / scale - Y / (2 * scale), k / scale);
    return o.n;
}

long long world_serial_boxes(uint32_t seed, int X, int Y, int Z, double scale, int obstacles, double wmin, double wmax, float *out,
                             long long cap) {
    std::default_random_engine eng((int)seed);
    const double res = 1 / scale;
    std::uniform_real_distribution<double> rx(-X / (2 * scale), X / (2 * scale)), ry(-Y / (2 * scale), Y / (2 * scale)), rw(wmin, wmax),
        rh(0, Z / scale);
    Out o{out, cap};
    for (int i = 0; i < obstacles; i++) {
        const double x = rx(eng), y = ry(eng), w = rw(eng), h = rh(eng);
        const int widNum = (int)std::ceil(w / res), heiNum = (int)std::ceil(h / res);
        const int rl = -widNum / 2, rh_ = widNum / 2;
        for (int r = rl; r < rh_; r++)
            for (int s = rl; s < rh_; s++)
                for (int t = 0; t < heiNum; t++)
                    if ((long long)(r - rl) * (r - rh_ + 1) * (s - rl) * (s - rh_ + 1) * t * (t - heiNum + 1) == 0)
                        o.push(x + r * res, y + s * res, t * res);
    }
    return o.n;
}

}  // extern "C"
