// mt_scene_check.cu -- CPU check (test infrastructure): scene.cuh's MT19937 and scene generator compiled FOR THE HOST
// (MT and generate_scene are __host__ __device__) against the CPU oracle (oracle/crowdsim_oracle.c, exported by
// tests/native/stream_oracle.c), word for word and bit for bit:
//   W  MT against the oracle's mt_next over the first 4 x 624 + 8 words of many seeds, on one scratch column that every
//      seed reuses, prefilled with junk, as a scene_kernel lane does. Hand-over: after k words (k on and beside the
//      first-block edges 227, 397, 624 and 1248), store_seeded() on a junk-prefilled column, and a fresh generator resumed
//      at pos continues with the oracle's next 624 + 8 words.
//   S  generate_scene and the next 2 x 624 + 4 words of its stream, as scene_kernel runs it (scene, then continue) and as
//      the draws kernel leaves it (scene, store_seeded(), resume on the same column), for the long scenes of
//      tests/golden/reset_scenes_long (square N = 40 and 63 at both profiles, square N = 32 with random attributes, circle
//      N = 15). After every long scene the same column generates a short one (N = 5) and its stream. Circle scenes take
//      glibc's cos / sin here, like the oracle, so they too match bit for bit.
// Build (tests/test_native_cpu.py): gcc -c stream_oracle.c with the oracle's flags, then
//   nvcc -O2 --fmad=false -Xcompiler -ffp-contract=off -std=c++17 mt_scene_check.cu stream_oracle.o -lgomp
// Usage: mt_scene_check <seeds per config>; stdin: extra "<config> <seed>" lines (the fixture's seeds). Prints coverage
// counters; exit code 0 iff every comparison was identical.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cstdint>
#include <string>
#include <vector>
#include "../../crowdnav_b200/csrc/scene.cuh"

extern "C" {
void so_mt_words(uint32_t seed, int n, uint32_t *out);
void so_scene_stream(const crowdsim_reset_args *a, int N, uint32_t seed, double *hp, double *hg, double *ha, int n_after,
                     uint32_t *after);
long so_scene_words(const crowdsim_reset_args *a, int N, uint32_t seed);
}

namespace {

constexpr int kWords = 4 * 624 + 8;      // part W
constexpr int kAfter = 2 * 624 + 4;      // part S: words drawn after a scene
constexpr int kResume = 624 + 8;         // part W: words after a hand-over
constexpr int kStride = 3;               // columns of the scratch array; the generators use column 1
const int kHandover[] = {0, 1, 226, 227, 228, 396, 397, 398, 623, 624, 625, 1247, 1248, 1249};

struct Config { const char *name; int rule, N, randomize; bool env_config; };
const Config kConfigs[] = {
    {"square40", CROWDSIM_RULE_SQUARE, 40, 0, false},
    {"square40_envcfg", CROWDSIM_RULE_SQUARE, 40, 0, true},
    {"square63", CROWDSIM_RULE_SQUARE, 63, 0, false},
    {"square63_envcfg", CROWDSIM_RULE_SQUARE, 63, 0, true},
    {"square32_random_attr", CROWDSIM_RULE_SQUARE, 32, 1, false},
    {"circle15", CROWDSIM_RULE_CIRCLE, 15, 0, false},
};

crowdsim_reset_args make_args(int rule, int randomize, bool env_config)
{
    crowdsim_reset_args a;
    memset(&a, 0, sizeof(a));
    a.rule = rule; a.randomize_attributes = randomize;
    if (env_config) {       // tests/util.py PROFILES['env_config']
        a.circle_radius = 5.0; a.square_width = 12.0; a.human_radius = 0.25; a.human_v_pref = 1.2;
        a.robot_radius = 0.35; a.robot_v_pref = 0.8; a.discomfort_dist = 0.3;
    } else {
        a.circle_radius = 4.0; a.square_width = 10.0; a.human_radius = 0.3; a.human_v_pref = 1.0;
        a.robot_radius = 0.3; a.robot_v_pref = 1.0; a.discomfort_dist = 0.2;
    }
    return a;
}

std::vector<uint32_t> g_col(624 * kStride);     // the scratch column scene_kernel's generator keeps for every seed and scene

void fill_junk(std::vector<uint32_t> &v, uint32_t x)
{
    for (auto &w : v) { x ^= x << 13; x ^= x >> 17; x ^= x << 5; w = x; }
}

// Part W: seeding and the raw stream across three block edges, and the stored state after k words.
bool check_words(uint32_t seed, long *words, long *handovers)
{
    std::vector<uint32_t> want(kWords);
    so_mt_words(seed, kWords, want.data());
    cs::MT mt; mt.mt = g_col.data() + 1; mt.stride = kStride; mt.seed(seed);
    for (int i = 0; i < kWords; ++i) {
        const uint32_t w = mt.next();
        if (w != want[i]) { printf("W seed %u word %d: MT %08x oracle %08x\n", seed, i, w, want[i]); return false; }
    }
    *words += kWords;
    for (int k : kHandover) {
        std::vector<uint32_t> col(624 * kStride);
        fill_junk(col, seed ^ (uint32_t)k ^ 0x85ebca6bu);
        cs::MT src; src.mt = col.data() + 1; src.stride = kStride; src.seed(seed);
        for (int i = 0; i < k; ++i) src.next();
        src.store_seeded();
        cs::MT dst; dst.mt = col.data() + 1; dst.stride = kStride; dst.resume(src.pos);
        for (int i = 0; i < kResume; ++i) {
            const uint32_t w = dst.next();
            if (w != want[k + i]) {
                printf("W seed %u: resumed after %d words, word %d: MT %08x oracle %08x\n", seed, k, i, w, want[k + i]);
                return false;
            }
        }
        ++*handovers;
    }
    return true;
}

// One scene from `seed` on the generator's column, then kAfter words: straight on (scene_kernel), or after store_seeded()
// and a fresh generator resumed on the same column (the draws kernel).
bool same_scene(cs::MT &rng, bool hand_over, const crowdsim_reset_args &a, int N, uint32_t seed, const char *what,
                const double *ohp, const double *ohg, const double *oha, const uint32_t *oafter)
{
    double hp[2 * CROWDSIM_MAX_HUMANS], hg[2 * CROWDSIM_MAX_HUMANS], ha[2 * CROWDSIM_MAX_HUMANS];
    rng.seed(seed);
    cs::generate_scene(rng, a, N, hp, hg, ha);
    const size_t bytes = sizeof(double) * 2 * N;
    if (memcmp(hp, ohp, bytes) || memcmp(hg, ohg, bytes) || memcmp(ha, oha, bytes)) {
        printf("S %s N=%d seed %u: scene differs\n", what, N, seed);
        return false;
    }
    cs::MT fresh; fresh.mt = rng.mt; fresh.stride = rng.stride;
    if (hand_over) { rng.store_seeded(); fresh.resume(rng.pos); }
    cs::MT &g = hand_over ? fresh : rng;
    for (int i = 0; i < kAfter; ++i) {
        const uint32_t w = g.next();
        if (w != oafter[i]) { printf("S %s N=%d seed %u: word %d after the scene %08x vs %08x\n", what, N, seed, i, w, oafter[i]); return false; }
    }
    return true;
}

// Part S: one scene through both kernels' paths against the oracle's.
bool check_scene(const crowdsim_reset_args &a, int N, uint32_t seed, const char *what)
{
    double hp[2 * CROWDSIM_MAX_HUMANS], hg[2 * CROWDSIM_MAX_HUMANS], ha[2 * CROWDSIM_MAX_HUMANS];
    std::vector<uint32_t> after(kAfter);
    so_scene_stream(&a, N, seed, hp, hg, ha, kAfter, after.data());
    cs::MT scene; scene.mt = g_col.data() + 1; scene.stride = kStride;
    std::vector<uint32_t> own(624);
    fill_junk(own, seed | 1u);
    cs::MT draws; draws.mt = own.data(); draws.stride = 1;
    return same_scene(scene, false, a, N, seed, what, hp, hg, ha, after.data()) &&
           same_scene(draws, true, a, N, seed, what, hp, hg, ha, after.data());
}

}  // namespace

int main(int argc, char **argv)
{
    const int per_config = argc > 1 ? atoi(argv[1]) : 40;
    fill_junk(g_col, 0x2545f491u);
    // ---- W ----
    std::vector<uint32_t> seeds = {0u, 1u, 2u, 5489u, 2000u, 4294967294u, 4294967295u, 2147483648u};
    uint32_t x = 0x9e3779b9u;
    for (int i = 0; i < 200; ++i) { x ^= x << 13; x ^= x >> 17; x ^= x << 5; seeds.push_back(x); }
    long words = 0, handovers = 0;
    for (uint32_t s : seeds)
        if (!check_words(s, &words, &handovers)) return 1;
    // ---- S ----
    std::vector<std::vector<uint32_t>> scene_seeds(sizeof(kConfigs) / sizeof(kConfigs[0]));
    for (auto &v : scene_seeds) {
        for (int i = 0; i < per_config; ++i) v.push_back(2000u + (uint32_t)i);
        v.push_back(0u); v.push_back(4294967295u);
    }
    char name[64]; unsigned long long seed;
    while (scanf("%63s %llu", name, &seed) == 2) {
        bool found = false;
        for (size_t c = 0; c < scene_seeds.size(); ++c)
            if (!strcmp(name, kConfigs[c].name)) { scene_seeds[c].push_back((uint32_t)seed); found = true; }
        if (!found) { printf("unknown config %s\n", name); return 2; }
    }
    long scenes = 0, above624 = 0, above1248 = 0, edge624 = 0, edge1248 = 0, short_after_long = 0;
    for (size_t c = 0; c < scene_seeds.size(); ++c) {
        const Config &k = kConfigs[c];
        const crowdsim_reset_args a = make_args(k.rule, k.randomize, k.env_config);
        const crowdsim_reset_args small = make_args(k.rule, 0, k.env_config);
        for (uint32_t s : scene_seeds[c]) {
            if (!check_scene(a, k.N, s, k.name)) return 1;
            const long w = so_scene_words(&a, k.N, s);
            ++scenes; above624 += w > 624; above1248 += w > 1248; edge624 += w == 624; edge1248 += w == 1248;
            if (w > 624) {                                   // the column that held a long scene generates a short one
                if (!check_scene(small, 5, s ^ 0x5bd1e995u, k.name)) return 1;
                ++short_after_long;
            }
        }
    }
    printf("ok words=%ld handovers=%ld seeds=%zu scenes=%ld above624=%ld above1248=%ld edge624=%ld edge1248=%ld "
           "short_after_long=%ld\n", words, handovers, seeds.size(), scenes, above624, above1248, edge624, edge1248,
           short_after_long);
    return 0;
}
