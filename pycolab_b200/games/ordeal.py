"""Ordeal set-up (reference `pycolab/examples/ordeal.py:37-97`): three sub-games —
castle (player + dragonduck), cavern (player + sword drape), kansas (player on a
10x45 map seen through an 8x15 scrolling cropper) — chained by
`storytelling.Story`; the player carries `has_sword` and `last_position` from
game to game in the Plot.

Set-up only: per-step logic of the three classes is the fused kernel
csrc/ordeal.cu (one program, the chapter picks the rules); the plot entries the
reference keeps in Python dict slots travel in the device plot record and are
mirrored back after every step (programs/ordeal.py).
"""

from pycolab_b200 import ascii_art
from pycolab_b200 import cropping
from pycolab_b200 import storytelling
from pycolab_b200 import things as plab_things
from pycolab_b200.prefab_parts import sprites as prefab_sprites

GAME_ART_CASTLE = ['##  ##   ##  ##',
                   '###############',
                   '#             #',
                   '#      D      #',
                   '#             #',
                   '#             #',
                   '#             #',
                   '###### P ######']

GAME_ART_CAVERN = ['@@@@@@@@@@@@@@@',
                   '@@@@@@     @@@@',
                   '@@@@@      @@@@',
                   '@ @@    S    @@',
                   '            @@@',
                   'P @@@     @@@@@',
                   '@@@@@@  @@@@@@@',
                   '@@@@@@@@@@@@@@@']

GAME_ART_KANSAS = ['######%%%######wwwwwwwwwwwwwwwwwwwwww@wwwwwww',
                   'w~~~~~%%%~~~~~~~~~~~~~~~~@~~~wwwww~~~~~~~~~~@',
                   'ww~~~~%%%~~~~~~~~~@~~~~~~~~~~~~~~~~~~~~~~@@@@',
                   'ww~~~~~%%%%~~~~~~~~~~~~~~~~~~~~~~~~~~~~~@@@@@',
                   '@ww~~~~~~%%%%~~~~~~~~~~~~~@~~%%%%%%%%%%%%%%%%',
                   'ww~~~~~~~~~~%%%%%%%%%%%%%%%%%%%%%%%%%%%%%%%%%',
                   'w~~~~~~@~~~~~~~~%%%%%%%%%%%%%%~~~~~~~~~~~~@@@',
                   'ww~~~~~~~~~~P~~~~~~~~~~~~~~~~~~~~~~~~~@~~~@@@',
                   'wwww~@www~~~~~~~~~wwwwww~~~@~~~~wwwww~~~~~~ww',
                   'wwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwwww']

ARTS = {'castle': GAME_ART_CASTLE, 'cavern': GAME_ART_CAVERN, 'kansas': GAME_ART_KANSAS}


def make_castle():
  return ascii_art.ascii_art_to_game(
      GAME_ART_CASTLE, what_lies_beneath=' ',
      sprites=dict(P=PlayerSprite, D=DragonduckSprite),
      update_schedule=['P', 'D'], z_order=['D', 'P'])


def make_cavern():
  return ascii_art.ascii_art_to_game(
      GAME_ART_CAVERN, what_lies_beneath=' ',
      sprites=dict(P=PlayerSprite), drapes=dict(S=SwordDrape),
      update_schedule=['P', 'S'])


def make_kansas():
  return ascii_art.ascii_art_to_game(
      GAME_ART_KANSAS, what_lies_beneath='~', sprites=dict(P=PlayerSprite))


def make_game():
  """ordeal.py:74-97."""
  crop_kansas = cropping.ScrollingCropper(rows=8, cols=15, to_track='P', scroll_margins=(2, 3))
  return storytelling.Story(
      chapters=dict(castle=make_castle, cavern=make_cavern, kansas=make_kansas),
      croppers=dict(castle=None, cavern=None, kansas=crop_kansas),
      first_chapter='kansas')


class SwordDrape(plab_things.Drape):
  """Vanishes when the player steps on it; sets `has_sword`, pays 1.0 (:108-124)."""

  def update(self, actions, board, layers, backdrop, things, the_plot):
    raise NotImplementedError('runs on the device: csrc/ordeal.cu')


class DragonduckSprite(prefab_sprites.MazeWalker):
  """Shuffles toward the player, diagonals included; contact ends the game, the
  sword decides who wins and who is drawn on top (:127-185)."""

  def __init__(self, corner, position, character):
    super(DragonduckSprite, self).__init__(
        corner, position, character, impassable='#', confined_to_board=True)

  def update(self, actions, board, layers, backdrop, things, the_plot):
    raise NotImplementedError('runs on the device: csrc/ordeal.cu')


class PlayerSprite(prefab_sprites.MazeWalker):
  """Arrow-key walker; walking off the matching edge ends the sub-game and names the
  next one; the first frame lines the player up with where the last game was left
  (:188-266)."""

  def __init__(self, corner, position, character):
    super(PlayerSprite, self).__init__(
        corner, position, character, impassable='@#w', confined_to_board=True)
    self._limits = self.Position(corner.row - 1, corner.col - 1)

  def update(self, actions, board, layers, backdrop, things, the_plot):
    raise NotImplementedError('runs on the device: csrc/ordeal.cu')
