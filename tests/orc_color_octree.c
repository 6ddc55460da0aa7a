/* orc_color_octree -- oracle of gem_color_octree: the octomap::ColorOcTree that pointCloudtoOctomap builds
 * (ElevationMapping.cpp:1146-1174) from a cloud of 32-byte PointXYZRGBICT records, as a literal pointer octree, and the
 * stream ColorOcTree::writeData writes.  TEST INFRASTRUCTURE ONLY.  Compiled with -ffp-contract=off.
 *
 * PARITY UNPINNED (octomap): restated from octomap 1.9 OccupancyOcTreeBase / ColorOcTree with default parameters
 * (DESIGN.md f7, items O1-O6):
 *   O1 keys: s = floor((1.0 / resolution) * (double)c) per axis; the point is inserted iff every s is in
 *      [-32768, 32767] (non-finite coordinates DEFINED as skipped), key = (int)s + 32768; depth 16, child index at
 *      bit d = bit_d(kx) + 2 bit_d(ky) + 4 bit_d(kz), d = 15 below the root.
 *   O2 hit = (float)log(0.7 / 0.3), max = (float)log(0.971 / 0.029); p(v) = 1 - 1 / (1 + exp((double)v)).
 *   O3 updateNode(key, hit): early return if search(key) holds a value >= max; missing children are created (value 0,
 *      white), a childless not-just-created node is expanded; leaf v += hit clamped to max; on the way up every node is
 *      pruned when its 8 children exist, are childless and have equal values (colour ignored); a pruned node copies
 *      child 0 and, if that colour is set, takes the average colour of the children whose colour is set.
 *   O4 integrateNodeColor: n = search(key); colour unset (== 255,255,255): set; else per channel
 *      (uint8_t)((double)prev * p(n) + (double)new * (0.99 - p(n))).
 *   O5 updateInnerOccupancy: bottom-up, every node with children: max child value, truncating mean of the set child
 *      colours (white if none).
 *   O6 stream: preorder, children 0..7, per node float value, r, g, b, child bitset; an empty tree writes nothing. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define DEPTH 16

typedef struct Node {
    float v;
    uint8_t r, g, b;
    struct Node **ch; /* NULL: no children */
} Node;

typedef struct Tree {
    Node *root;
    float hit, max;
    long long nodes, leaves;
} Tree;

static Node *new_node(void)
{
    Node *n = (Node *)calloc(1, sizeof(Node));
    n->r = n->g = n->b = 255;
    return n;
}

static int has_children(const Node *n)
{
    if (!n->ch) return 0;
    for (int i = 0; i < 8; i++)
        if (n->ch[i]) return 1;
    return 0;
}

static void free_node(Node *n)
{
    if (!n) return;
    if (n->ch) {
        for (int i = 0; i < 8; i++) free_node(n->ch[i]);
        free(n->ch);
    }
    free(n);
}

static int colour_set(const Node *n) { return !(n->r == 255 && n->g == 255 && n->b == 255); }

/* ColorOcTreeNode::getAverageChildColor */
static void average_child_colour(const Node *n, uint8_t *r, uint8_t *g, uint8_t *b)
{
    int mr = 0, mg = 0, mb = 0, c = 0;
    for (int i = 0; n->ch && i < 8; i++) {
        const Node *k = n->ch[i];
        if (k && colour_set(k)) { mr += k->r; mg += k->g; mb += k->b; c++; }
    }
    if (c) { *r = (uint8_t)(mr / c); *g = (uint8_t)(mg / c); *b = (uint8_t)(mb / c); }
    else { *r = *g = *b = 255; }
}

/* O1 */
static int key_of(double rf, float c, int *key)
{
    const double s = floor(rf * (double)c);
    if (!(s >= -32768.0 && s <= 32767.0)) return 0; /* NaN fails both */
    *key = (int)s + 32768;
    return 1;
}

static int child_idx(const int k[3], int d) { return ((k[0] >> d) & 1) | (((k[1] >> d) & 1) << 1) | (((k[2] >> d) & 1) << 2); }

/* OcTreeBaseImpl::search at full depth: the leaf or the childless (pruned) node on the key's path, or NULL */
static Node *search(Node *root, const int k[3])
{
    Node *n = root;
    if (!n) return NULL;
    for (int d = DEPTH - 1; d >= 0; d--) {
        if (!has_children(n)) return n;
        n = n->ch[child_idx(k, d)];
        if (!n) return NULL;
    }
    return n;
}

/* ColorOcTree::isNodeCollapsible + pruneNode */
static int prune(Node *n)
{
    if (!n->ch || !n->ch[0] || has_children(n->ch[0])) return 0;
    for (int i = 1; i < 8; i++)
        if (!n->ch[i] || has_children(n->ch[i]) || !(n->ch[i]->v == n->ch[0]->v)) return 0;
    n->v = n->ch[0]->v;
    n->r = n->ch[0]->r; n->g = n->ch[0]->g; n->b = n->ch[0]->b;
    if (colour_set(n)) average_child_colour(n, &n->r, &n->g, &n->b);
    for (int i = 0; i < 8; i++) free(n->ch[i]);
    free(n->ch);
    n->ch = NULL;
    return 1;
}

/* O3, iteratively: the path is recorded on the way down and pruned bottom-up */
static void update_node(Tree *t, const int k[3])
{
    Node *hitn = search(t->root, k);
    if (hitn && hitn->v >= t->max) return;
    int just_created = 0;
    if (!t->root) { t->root = new_node(); just_created = 1; }
    Node *path[DEPTH + 1];
    Node *n = t->root;
    path[0] = n;
    for (int depth = 0; depth < DEPTH; depth++) {
        const int pos = child_idx(k, DEPTH - 1 - depth);
        int created = 0;
        if (!n->ch || !n->ch[pos]) {
            if (!has_children(n) && !just_created) { /* expandNode: 8 copies of the pruned node */
                if (!n->ch) n->ch = (Node **)calloc(8, sizeof(Node *));
                for (int i = 0; i < 8; i++) {
                    n->ch[i] = new_node();
                    n->ch[i]->v = n->v;
                    n->ch[i]->r = n->r; n->ch[i]->g = n->g; n->ch[i]->b = n->b;
                }
            } else {
                if (!n->ch) n->ch = (Node **)calloc(8, sizeof(Node *));
                n->ch[pos] = new_node();
                created = 1;
            }
        }
        n = n->ch[pos];
        just_created = created;
        path[depth + 1] = n;
    }
    float v = n->v + t->hit;
    if (v > t->max) v = t->max;
    n->v = v;
    for (int depth = DEPTH - 1; depth >= 0; depth--) prune(path[depth]);
}

/* O4 */
static void integrate_colour(Tree *t, const int k[3], uint8_t r, uint8_t g, uint8_t b)
{
    Node *n = search(t->root, k);
    if (!n) return;
    if (colour_set(n)) {
        const double p = 1.0 - 1.0 / (1.0 + exp((double)n->v));
        n->r = (uint8_t)((double)n->r * p + (double)r * (0.99 - p));
        n->g = (uint8_t)((double)n->g * p + (double)g * (0.99 - p));
        n->b = (uint8_t)((double)n->b * p + (double)b * (0.99 - p));
    } else {
        n->r = r; n->g = g; n->b = b;
    }
}

/* O5 */
static void inner_occupancy(Node *n)
{
    if (!has_children(n)) return;
    float mx = -INFINITY;
    for (int i = 0; i < 8; i++) {
        if (!n->ch[i]) continue;
        inner_occupancy(n->ch[i]);
        if (n->ch[i]->v > mx) mx = n->ch[i]->v;
    }
    n->v = mx;
    average_child_colour(n, &n->r, &n->g, &n->b);
}

static void count(Tree *t, const Node *n)
{
    t->nodes++;
    if (!has_children(n)) { t->leaves++; return; }
    for (int i = 0; i < 8; i++)
        if (n->ch[i]) count(t, n->ch[i]);
}

/* recs: n records of 8 floats ({x, y, z, pad, bgra, ...}).  info[4] = {nodes, leaves, inserted, skipped}; the stream is
 * 8 * nodes bytes, read with orc_octree_write */
void *orc_octree_build(int n, const float *recs, double resolution, long long info[4])
{
    Tree *t = (Tree *)calloc(1, sizeof(Tree));
    t->hit = (float)log(0.7 / 0.3);
    t->max = (float)log(0.971 / 0.029);
    const double rf = 1.0 / resolution;
    long long inserted = 0;
    for (int i = 0; i < n; i++) {
        const float *p = recs + (size_t)8 * i;
        int k[3];
        if (!key_of(rf, p[0], &k[0]) || !key_of(rf, p[1], &k[1]) || !key_of(rf, p[2], &k[2])) continue;
        uint32_t bgra;
        memcpy(&bgra, p + 4, 4);
        update_node(t, k);
        integrate_colour(t, k, (uint8_t)(bgra >> 16), (uint8_t)(bgra >> 8), (uint8_t)bgra);
        inserted++;
    }
    if (t->root) {
        inner_occupancy(t->root);
        count(t, t->root);
    }
    info[0] = t->nodes;
    info[1] = t->leaves;
    info[2] = inserted;
    info[3] = n - inserted;
    return t;
}

static uint8_t *write_rec(const Node *n, uint8_t *o)
{
    memcpy(o, &n->v, 4);
    o[4] = n->r; o[5] = n->g; o[6] = n->b;
    uint8_t bits = 0;
    for (int i = 0; n->ch && i < 8; i++)
        if (n->ch[i]) bits |= (uint8_t)(1u << i);
    o[7] = bits;
    o += 8;
    for (int i = 0; n->ch && i < 8; i++)
        if (n->ch[i]) o = write_rec(n->ch[i], o);
    return o;
}

void orc_octree_write(void *tree, uint8_t *out)
{
    Tree *t = (Tree *)tree;
    if (t->root) write_rec(t->root, out);
}

void orc_octree_free(void *tree)
{
    Tree *t = (Tree *)tree;
    free_node(t->root);
    free(t);
}
