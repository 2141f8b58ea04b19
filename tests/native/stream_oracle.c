/* Test-side export of the CPU oracle's MT19937 after a scene (tests/explore_oracle.py compiles it with the CPU oracle's
 * flags): oracle/crowdsim_oracle.c is included as it stands, seeded with `seed` and run through its own generate_scene, and
 * the generator's state is returned in numpy's representation (key[624], pos; pos 624 = a full twist comes next), or the
 * number of words the scene drew, or the words themselves (tests/native/mt_scene_check.cu). */
#include "../../oracle/crowdsim_oracle.c"

void so_post_generation(const crowdsim_reset_args *a, int N, uint32_t seed, uint32_t *key, int32_t *pos)
{
    double hp[2 * CROWDSIM_MAX_HUMANS], hg[2 * CROWDSIM_MAX_HUMANS], ha[2 * CROWDSIM_MAX_HUMANS];
    mt_state s;
    mt_seed(&s, seed);
    generate_scene(&s, a, N, hp, hg, ha);
    memcpy(key, s.mt, sizeof(s.mt));
    *pos = s.pos;
}

/* tests/native/mt_scene_check.cu (linked with this file): the first n words after seeding, and a scene followed by the
 * next n_after words of its stream. */
void so_mt_words(uint32_t seed, int n, uint32_t *out)
{
    mt_state s;
    mt_seed(&s, seed);
    for (int i = 0; i < n; ++i) out[i] = mt_next(&s);
}

void so_scene_stream(const crowdsim_reset_args *a, int N, uint32_t seed, double *hp, double *hg, double *ha, int n_after,
                     uint32_t *after)
{
    mt_state s;
    mt_seed(&s, seed);
    generate_scene(&s, a, N, hp, hg, ha);
    for (int i = 0; i < n_after; ++i) after[i] = mt_next(&s);
}

/* Words the scene of `seed` draws. The key changes only when a block is twisted, so the number of twists is found by
 * twisting a freshly seeded state until its key equals the key after the scene: after w > 0 words there were
 * t = ceil(w / 624) twists and pos = w - 624 (t - 1), in 1..624. */
long so_scene_words(const crowdsim_reset_args *a, int N, uint32_t seed)
{
    double hp[2 * CROWDSIM_MAX_HUMANS], hg[2 * CROWDSIM_MAX_HUMANS], ha[2 * CROWDSIM_MAX_HUMANS];
    mt_state s, f;
    mt_seed(&s, seed);
    generate_scene(&s, a, N, hp, hg, ha);
    mt_seed(&f, seed);
    long t = 0;
    while (memcmp(f.mt, s.mt, sizeof(s.mt)) != 0) { mt_twist(&f); ++t; }
    return t == 0 ? 0 : 624 * (t - 1) + s.pos;
}
